"""Time the fused-epilogue wgmma linear kernel (csrc/gemm_wgmma.cu) next to the library path it replaces (cuBLAS GEMM +
stand-alone GELU pass / transposing copy) on the shapes of the bench step (B images of 1024^2).
usage: B=4 python tools/bench_gemm.py"""
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from psalm_b200 import kernels  # noqa: E402


def timeit(fn, flush, iters=20):
    ts = []
    for i in range(iters + 3):
        flush.zero_()
        torch.cuda._sleep(1_000_000)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        if i >= 3:
            ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default=None, help="run one shape by name")
    ap.add_argument("--once", action="store_true", help="one fused call per shape (profiler runs)")
    args = ap.parse_args()
    B = int(os.environ.get("B", "4"))
    dt = torch.bfloat16
    hbm = 6650.0
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        hbm = json.load(open(p)).get("hbm_gbs", hbm)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    g = torch.Generator().manual_seed(0)
    shapes = [("swin_fc1_stage%d" % s, B * (256 >> s) ** 2, 512 << s, 128 << s, "gelu_erf", 0) for s in range(4)]
    shapes.append(("msda_value_proj", B * 21504, 256, 256, "head_major", 21504))
    for name, M, N, K, epi, S in shapes:
        if args.only and name != args.only:
            continue
        x = torch.randn(M, K, generator=g).to(dt).cuda()
        w = (torch.randn(N, K, generator=g) * K ** -0.5).to(dt).cuda()
        b = torch.randn(N, generator=g).to(dt).cuda()
        if epi == "gelu_erf":
            lib = lambda: F.gelu(F.linear(x, w, b))
        else:
            lib = lambda: F.linear(x, w, b).view(M // S, S, 8, 32).permute(0, 2, 1, 3).contiguous()
        ours = lambda: kernels.linear_fused(x, w, b, epi, S)
        if args.once:
            ours()
            ours()
            torch.cuda.synchronize()
            continue
        t_lib, t_ours = timeit(lib, flush), timeit(ours, flush)
        nbytes = 2 * (M * K + N * K + M * N)
        print(f"{name:18s} M={M:7d} N={N:5d} K={K:5d}  library {t_lib:7.1f} us   fused {t_ours:7.1f} us   "
              f"{nbytes / t_ours / 1e3:7.1f} GB/s = {nbytes / t_ours / 1e3 / hbm:.3f} of HBM peak   "
              f"{2.0 * M * N * K / t_ours / 1e6:7.1f} TFLOP/s")


if __name__ == "__main__":
    main()
