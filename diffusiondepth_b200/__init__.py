"""diffusiondepth_b200 — H100-native (sm_90a) engine for the DiffusionDepth hot path.

Hot path = the T-step DDIM denoising loop over the 16-channel depth latent + the depth-latent decoder
(reference: duanyiqun/DiffusionDepth src/model/head/ddim_depth_estimate_res_swin_addHAHI.py:254-303,
361-382; src/model/ops/depth_transform.py:33-35), hand-written CUDA behind the C ABI in include/dd_engine.h.

`diffusiondepth_b200.model` mirrors the reference's `src/model` plugin surface (same class names, ctor
arguments, state_dict keys, output dict) so `src/main.py` can use it unchanged; see INTEGRATION.md.
"""
from ._cabi import EngineError, lib_path, load_library  # noqa: F401
from .engine import DenoiseEngine, ddim_coefficients  # noqa: F401

__all__ = ["DenoiseEngine", "EngineError", "ddim_coefficients", "lib_path", "load_library"]
