#!/usr/bin/env python
"""Where the step-invariant producers' tensor-core time goes (convgen_wgmma_kernel), and A/B timing of the producer
chain between two builds of the engine library.

  python profiles/producer_ab.py --profile [--out DIR]   per-launch table of one C3 forward (torch.profiler)
  python profiles/producer_ab.py --lib base=diffusiondepth_b200/libddengine_base.so --lib new=diffusiondepth_b200/libddengine.so

C3 is Swin-L, B = 4, 352 x 1216.  The profile mode runs one forward without CUDA graphs, so that every kernel is
recorded, and attributes every convgen_wgmma_kernel launch to its layer by launch order.  That order is fixed by the
engine: run_swin (per block qkv, proj, fc1, fc2; the patch-merge reduction after stages 0-2), then the HAHI neck
(per level lateral, proj, fusion) and the FPN top-down (level 3 .. 0: lateral conv, then the transposed conv of the
level below), every layer split along K (parts > 1) launching once per part.  Per launch it prints M x N x K, taps,
the K iterations of one work item, the work items, grid and parts, the time and the algorithmic rate
(2 * M * N * K FLOPs; the 3-pass split issues 3x that).  It is a breakdown, not a timing.

The A/B mode times the producer chain, dd_run_backbone + dd_build_condition, as a forward runs it (CUDA graphs on)
with CUDA events over `--iters` back-to-back calls.  Each library runs in its own process (DD_ENGINE_LIB), the
libraries alternate for `--rounds` rounds, and each library's profile is summed per layer family once.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B, IH, IW = 4, 352, 1216
E, DEPTHS = 192, (2, 2, 18, 2)  # Swin-L
GEN_BK, SPLIT_ITERS = 64, 110   # csrc/convgen.cuh GEN_BK, csrc/engine.cu kGenSplitIters


def cdiv(a, b):
    return (a + b - 1) // b


def c3_launches():
    """Every convgen_wgmma_kernel launch of one C3 producer chain, in launch order:
    dict(layer, family, M, N, K, taps, conv = (H, W) or None, kc = 64-channel chunks of this launch)."""
    out = []
    hs, ws = [cdiv(IH, 4)], [cdiv(IW, 4)]
    for _ in range(3):
        hs.append(cdiv(hs[-1], 2))
        ws.append(cdiv(ws[-1], 2))

    def gemm(layer, fam, M, N, K):
        out.append(dict(layer=layer, family=fam, M=M, N=N, K=K, taps=1, conv=None, kc=cdiv(K, GEN_BK)))

    def conv(layer, fam, s, N, cin, taps):
        kc = cdiv(cin, GEN_BK)
        parts = cdiv(taps * kc, SPLIT_ITERS)
        per = cdiv(kc, parts)
        for p in range(parts):
            ka, kb = p * per, min(kc, p * per + per)
            if ka >= kc:
                break
            name = layer + (f" part {p + 1}/{parts}" if parts > 1 else "")
            out.append(dict(layer=name, family=fam, M=B * hs[s] * ws[s], N=N, K=taps * cin, taps=taps,
                            conv=(hs[s], ws[s]), kc=kb - ka))

    for s in range(4):
        C, M = E << s, B * hs[s] * ws[s]
        for k in range(DEPTHS[s]):
            gemm(f"s{s}.b{k}.qkv", f"swin s{s} qkv", M, 3 * C, C)
            gemm(f"s{s}.b{k}.proj", f"swin s{s} proj", M, C, C)
            gemm(f"s{s}.b{k}.fc1", f"swin s{s} fc1", M, 4 * C, C)
            gemm(f"s{s}.b{k}.fc2", f"swin s{s} fc2", M, C, 4 * C)
        if s < 3:
            gemm(f"s{s}.reduction", f"swin s{s} merge", B * hs[s + 1] * ws[s + 1], 2 * C, 4 * C)
    for i in range(4):
        C = E << i
        conv(f"neck.lat{i}", "neck lateral", i, C, C, 1)
        conv(f"neck.proj{i}", "neck proj", i, 512, C, 1)
        conv(f"neck.fus{i}", "neck fusion", i, C, C + 512, 9)
    for i in range(3, -1, -1):
        conv(f"fpn.lat{i}", "fpn lateral", i, 256, E << i, 9)
        if i > 0:
            conv(f"fpn.up{i - 1}", "fpn up", i, 1024, 256, 1)
    return out


def m_tiles(L):
    if L["conv"] is None:  # GEMM mode: tokens as a [ceil(M/16)][16] image, 8 x 16 tiles
        return cdiv(L["M"], 128)
    h, w = L["conv"]
    return B * cdiv(h, 8) * cdiv(w, 16)


def profile_rows(out_dir=None):
    """One un-graphed C3 forward under torch.profiler -> per-launch rows (see the module docstring)."""
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile
    import dd_helpers
    from oracle import configs, restate

    dev = torch.device("cuda:0")
    model = dd_helpers.build_mirror("swinl", 20).to(dev)
    model.depth_head.use_cuda_graph = False
    sample = {k: v.to(dev) for k, v in restate.synthetic_sample(B, IH, IW, configs.SEED_INPUTS).items()}
    with torch.no_grad():
        for _ in range(2):
            model(sample)
        torch.cuda.synchronize()
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            model(sample)
            torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    kern = sorted((e for e in trace["traceEvents"] if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    total_ms = sum(e["dur"] for e in kern) / 1e3
    gen = [e for e in kern if "convgen_wgmma_kernel" in e["name"]]
    layers = c3_launches()
    if len(gen) != len(layers):
        raise SystemExit(f"{len(gen)} convgen launches, expected {len(layers)}: the launch order changed")
    rows = []
    for L, ev in zip(layers, gen):
        nt = int(re.search(r"convgen_wgmma_kernel<(\d+)>", ev["name"]).group(1))
        work = m_tiles(L) * cdiv(L["N"], nt)
        ms = ev["dur"] / 1e3
        kc, kc_total = L["kc"], cdiv(L["K"] // L["taps"], GEN_BK)
        flops = 2.0 * L["M"] * L["N"] * L["K"] * kc / kc_total  # a split part does its share of K
        parts = cdiv(L["taps"] * kc_total, SPLIT_ITERS)
        rows.append(dict(layer=L["layer"], family=L["family"], M=L["M"], N=L["N"], K=L["K"], taps=L["taps"],
                         k_iters=L["taps"] * kc, nt=nt, work=work, grid=ev["args"]["grid"][0], parts=parts, ms=ms,
                         tflops=flops / (ms * 1e-3) / 1e12, flops=flops))
    res = {"gpu": torch.cuda.get_device_name(0), "forward_kernel_ms": total_ms, "rows": rows}
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "producer_profile.json"), "w") as f:
            json.dump(res, f, indent=1)
    return res


def families(rows):
    fam = {}
    for r in rows:
        f = fam.setdefault(r["family"], {"launches": 0, "ms": 0.0, "flops": 0.0})
        f["launches"] += 1
        f["ms"] += r["ms"]
        f["flops"] += r["flops"]
    return fam


def print_profile(res):
    rows = res["rows"]
    gen_ms = sum(r["ms"] for r in rows)
    gen_fl = sum(r["flops"] for r in rows)
    print(f"{res['gpu']}: one C3 forward, profiler on, no CUDA graph: {res['forward_kernel_ms']:.1f} ms of kernel time; "
          f"convgen_wgmma_kernel {gen_ms:.2f} ms in {len(rows)} launches, {gen_fl / 1e12:.3f} TFLOP, "
          f"{gen_fl / (gen_ms * 1e-3) / 1e12:.1f} TFLOP/s")
    print(f"{'layer':<24} {'M x N x K':>22} {'taps':>4} {'kit':>4} {'NT':>4} {'work':>6} {'grid':>5} {'parts':>5} "
          f"{'ms':>8} {'TF/s':>7}")
    for r in rows:
        print(f"{r['layer']:<24} {r['M']:>8} x {r['N']:>4} x {r['K']:>5} {r['taps']:>4} {r['k_iters']:>4} {r['nt']:>4} "
              f"{r['work']:>6} {r['grid']:>5} {r['parts']:>5} {r['ms']:8.3f} {r['tflops']:7.1f}")
    print(f"\n{'family':<18} {'launches':>8} {'ms':>8} {'TF/s':>7}")
    for name, f in families(rows).items():
        print(f"{name:<18} {f['launches']:>8} {f['ms']:8.3f} {f['flops'] / (f['ms'] * 1e-3) / 1e12:7.1f}")


def worker(iters, warmup):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import dd_helpers
    from diffusiondepth_b200 import lib_path
    from diffusiondepth_b200.engine import DenoiseEngine
    from oracle import configs, restate

    if not torch.cuda.is_available():
        raise SystemExit("producer_ab.py times kernels on an H100; there is no CPU path")
    dev = torch.device("cuda:0")
    model = dd_helpers.build_mirror("swinl", 20).to(dev)
    sample = {k: v.to(dev) for k, v in restate.synthetic_sample(B, IH, IW, configs.SEED_INPUTS).items()}
    seen = {}
    orig = DenoiseEngine.run_backbone

    def spy(self, rgb, want_feats=False):
        seen["eng"], seen["rgb"] = self, rgb
        return orig(self, rgb, want_feats)

    DenoiseEngine.run_backbone = spy
    with torch.no_grad():
        model(sample)  # builds the engine and captures its graphs
    DenoiseEngine.run_backbone = orig
    eng, rgb = seen["eng"], seen["rgb"]

    def chain():
        eng.run_backbone(rgb)
        eng.build_condition(None)

    for _ in range(warmup):
        chain()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        chain()
    t1.record()
    t1.synchronize()
    eng.poll_status()
    print(json.dumps({"lib": lib_path(), "gpu": torch.cuda.get_device_name(0), "ms": t0.elapsed_time(t1) / iters}),
          flush=True)


def ab(libs, rounds, iters, warmup):
    def run(path, *args):
        env = dict(os.environ, DD_ENGINE_LIB=os.path.abspath(path))
        out = subprocess.run([sys.executable, os.path.abspath(__file__), *args], env=env, cwd=ROOT, check=True,
                             stdout=subprocess.PIPE, text=True).stdout
        return json.loads(out.strip().splitlines()[-1])

    runs = {name: [] for name, _ in libs}
    for _ in range(rounds):
        for name, path in libs:
            runs[name].append(run(path, "--worker", "--iters", str(iters), "--warmup", str(warmup))["ms"])
    prof = {name: run(path, "--profile-json") for name, path in libs}
    base = libs[0][0]
    print(f"producer chain (dd_run_backbone + dd_build_condition, graphed), ms per call, {rounds} alternating rounds "
          f"of {iters}:")
    for name, _ in libs:
        ms = sorted(runs[name])
        med, bmed = ms[len(ms) // 2], sorted(runs[base])[len(ms) // 2]
        print(f"  {name:>8}: {' '.join(f'{m:.2f}' for m in runs[name])}  median {med:.2f} "
              f"({100 * (med / bmed - 1):+.1f} % vs {base})")
    print("\nconvgen_wgmma_kernel per layer family (profiled forward, ms):")
    fams = {name: families(prof[name]["rows"]) for name, _ in libs}
    print(f"{'family':<18} " + " ".join(f"{n:>10}" for n, _ in libs))
    for fam in fams[base]:
        print(f"{fam:<18} " + " ".join(f"{fams[n][fam]['ms']:10.3f}" for n, _ in libs))
    print(f"{'total':<18} " + " ".join(f"{sum(f['ms'] for f in fams[n].values()):10.3f}" for n, _ in libs))
    print(json.dumps({"gpu": prof[base]["gpu"], "chain_ms": runs,
                      "families": {n: {k: v["ms"] for k, v in fams[n].items()} for n, _ in libs}}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=PATH", help="library to time (repeatable)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None, help="profile mode: directory for producer_profile.json")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--profile-json", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args.iters, args.warmup)
    if args.profile_json:
        return print(json.dumps(profile_rows()))
    if args.profile:
        return print_profile(profile_rows(args.out))
    libs = [tuple(s.split("=", 1)) for s in args.lib] or [("current", os.path.join(ROOT, "diffusiondepth_b200",
                                                                                    "libddengine.so"))]
    ab(libs, args.rounds, args.iters, args.warmup)


if __name__ == "__main__":
    main()
