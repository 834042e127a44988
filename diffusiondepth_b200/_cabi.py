"""ctypes binding of libddengine.so (include/dd_engine.h).  There is no fallback: if the shared library
is missing or does not export the ABI, importing the engine raises."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


class EngineError(RuntimeError):
    """Raised for any non-zero status coming back across the C ABI."""


class DDConfig(C.Structure):
    _fields_ = [("abi_version", C.c_int32), ("variant", C.c_int32), ("batch", C.c_int32),
                ("latent_h", C.c_int32), ("latent_w", C.c_int32), ("cond_h", C.c_int32),
                ("cond_w", C.c_int32), ("num_inference_steps", C.c_int32), ("device", C.c_int32),
                ("flags", C.c_int32)]


class DDProducerConfig(C.Structure):
    _fields_ = [("num_levels", C.c_int32), ("channels", C.c_int32 * 4), ("heights", C.c_int32 * 4),
                ("widths", C.c_int32 * 4), ("has_neck", C.c_int32)]


class DDBackboneConfig(C.Structure):
    _fields_ = [("kind", C.c_int32), ("embed_dims", C.c_int32), ("depths", C.c_int32 * 4),
                ("num_heads", C.c_int32 * 4), ("window", C.c_int32), ("height", C.c_int32), ("width", C.c_int32),
                ("mp_dims", C.c_int32 * 4), ("mp_paths", C.c_int32 * 4), ("mlp_ratio", C.c_int32),
                ("mp_drop_path", C.c_int32 * 4)]


class DDGenLayerDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("taps", "stride", "transposed", "act", "add_first", "tokens", "batch",
                                         "height", "width", "src_h", "src_w", "c0", "c1", "cin", "cout", "ld_out",
                                         "ch_off", "n_tile", "alt_tile")]


class DDConvGnDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("batch", "cin", "cout", "height", "width", "mode", "cond_h", "cond_w",
                                         "up_qpb")] + [("c_x", C.c_float), ("c_eps", C.c_float)]


ABI_VERSION = 3
VARIANT_RES, VARIANT_SWIN = 0, 1
FLAG_CUDA_GRAPH, FLAG_SIMT_CONV, FLAG_CHECK_RANGE, FLAG_HALO_CONV, FLAG_SWAP_NARROW, FLAG_PAIR_WIDE = 1, 2, 4, 8, 16, 32
FLAG_STEP_DECODE, FLAG_FP8_CORR, FLAG_BACKWARD, FLAG_LOOP_BACKWARD = 64, 128, 256, 512
FLAG_CHAIN_PRED, FLAG_PRODUCER_TRAIN = 1024, 2048
CODEC_EVAL, CODEC_TRAIN = 0, 1
# dd_codec_kind, carried in the flags at FLAG_CODEC_SHIFT
CODEC_UP2, CODEC_UP2_1X1, CODEC_UP4, CODEC_FULL = 0, 1, 2, 3
FLAG_CODEC_SHIFT = 12
PRODUCER_EVAL, PRODUCER_TRAIN = 0, 1
STATUS = {0: "DD_OK", 1: "DD_ERR_INVALID", 2: "DD_ERR_CUDA", 3: "DD_ERR_UNSUPPORTED", 4: "DD_ERR_RANGE"}
# dd_allgather_fn: (in, out, count, cuda_stream, user) -> 0 on success
ALLGATHER_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p)

# name -> (restype, argtypes); every symbol include/dd_engine.h declares
SIGNATURES = {
    "dd_abi_version": (C.c_int, []),
    "dd_last_error": (C.c_char_p, []),
    "dd_create": (C.c_int, [C.POINTER(DDConfig), C.POINTER(C.c_void_p)]),
    "dd_destroy": (C.c_int, [C.c_void_p]),
    "dd_set_weight": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.POINTER(C.c_int64), C.c_int32]),
    "dd_finalize_weights": (C.c_int, [C.c_void_p, C.c_void_p]),
    "dd_update_weights": (C.c_int, [C.c_void_p, C.c_void_p]),
    "dd_graph_capture_count": (C.c_int64, [C.c_void_p]),
    "dd_set_schedule": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_double),
                                  C.POINTER(C.c_double), C.c_int32]),
    "dd_set_schedule_eta": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_double),
                                      C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int32]),
    "dd_set_step_io": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "dd_workspace_bytes": (C.c_size_t, [C.c_void_p]),
    "dd_enable_producers": (C.c_int, [C.c_void_p, C.POINTER(DDProducerConfig)]),
    "dd_enable_backbone": (C.c_int, [C.c_void_p, C.POINTER(DDBackboneConfig)]),
    "dd_run_backbone": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p, C.c_size_t, C.c_void_p]),
    "dd_build_condition": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p, C.c_size_t,
                                     C.c_void_p]),
    "dd_denoise_decode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_size_t, C.c_void_p]),
    "dd_denoise_decode_steps": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_size_t, C.c_void_p]),
    "dd_denoiser_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64), C.c_void_p,
                                      C.c_void_p, C.c_size_t, C.c_void_p]),
    "dd_denoiser_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64), C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p, C.c_size_t,
                                       C.c_void_p]),
    "dd_denoiser_relu_inputs": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64),
                                          C.POINTER(C.c_void_p), C.c_void_p, C.c_size_t, C.c_void_p]),
    "dd_denoise_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_void_p,
                                      C.c_void_p, C.c_size_t, C.c_void_p]),
    "dd_decode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dd_decode_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p),
                                     C.c_void_p, C.c_size_t, C.c_void_p]),
    "dd_encode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "dd_encode_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.POINTER(C.c_void_p),
                                     C.c_void_p, C.c_size_t, C.c_void_p]),
    "dd_set_codec_mode": (C.c_int, [C.c_void_p, C.c_int32]),
    "dd_codec_batch_stats": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.c_void_p]),
    "dd_set_producer_mode": (C.c_int, [C.c_void_p, C.c_int32]),
    "dd_set_drop_path": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "dd_producer_batch_stats": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int32), C.c_void_p]),
    "dd_producer_bn_info": (C.c_int, [C.c_void_p, C.c_int32, C.c_char_p, C.c_int32, C.POINTER(C.c_int32),
                                      C.POINTER(C.c_int64), C.POINTER(C.c_int32)]),
    "dd_set_bn_allgather": (C.c_int, [C.c_void_p, ALLGATHER_FN, C.c_void_p, C.c_int32]),
    "dd_last_launch_count": (C.c_int64, [C.c_void_p]),
    "dd_poll_status": (C.c_int, [C.c_void_p, C.c_void_p]),
    "dd_conv3x3": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                             C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dd_conv3x3_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "dd_conv3x3_wgrad": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                   C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dd_conv3x3_wgrad_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "dd_gen_layer": (C.c_int, [C.c_void_p, C.POINTER(DDGenLayerDesc), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.POINTER(C.c_int32), C.c_void_p]),
    "dd_window_attention": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                      C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int32),
                                      C.c_void_p]),
    "dd_factor_attention": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_void_p,
                                      C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int32), C.c_void_p]),
    "dd_depthwise_conv": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                    C.c_int32, C.c_int32, C.POINTER(C.c_int32), C.c_void_p]),
    "dd_layer_norm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                C.c_float, C.c_void_p]),
    "dd_swin_patch_embed": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "dd_swin_layer_norm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "dd_swin_patch_merge": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                      C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "dd_conv_groupnorm": (C.c_int, [C.c_void_p, C.POINTER(DDConvGnDesc), C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_void_p]),
    "dd_bench_gemm": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_float)]),
    "dd_bench_conv": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_float), C.c_void_p,
                                C.c_size_t, C.c_void_p]),
    "dd_bench_pred_fold": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_float), C.c_void_p, C.c_size_t,
                                     C.c_void_p]),
    "dd_bench_decoder": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(C.c_float), C.c_void_p, C.c_size_t,
                                   C.c_void_p]),
}


def lib_path() -> str:
    return os.environ.get("DD_ENGINE_LIB", os.path.join(_HERE, "libddengine.so"))


def load_library():
    """dlopen libddengine.so and type every entry point; raises EngineError if anything is missing."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = lib_path()
    if not os.path.exists(path):
        raise EngineError(
            f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc -gencode arch=compute_90a,code=sm_90a). There is no CPU/PyTorch fallback.")
    lib = C.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:  # pragma: no cover
            raise EngineError(f"{path} does not export {name}") from e
        fn.restype, fn.argtypes = res, args
    if lib.dd_abi_version() != ABI_VERSION:
        raise EngineError(f"ABI mismatch: library {lib.dd_abi_version()} vs binding {ABI_VERSION}")
    _LIB = lib
    return lib


def check(status: int):
    if status != 0:
        msg = load_library().dd_last_error().decode("utf-8", "replace")
        raise EngineError(f"{STATUS.get(status, status)}: {msg}")
