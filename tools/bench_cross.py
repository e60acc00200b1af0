"""Time masked cross-attention (100 queries x Lk keys, 8 heads x 32): the TMA-fed all-heads kernel (csrc/xattn_tma.cu)
next to the per-head kernel it replaces, against the HBM roofline (K + V + mask + q/out bytes, DESIGN.md section 4).
usage: B=4 python tools/bench_cross.py [--ncu]   (--ncu: one call per configuration, for a profiler run)"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from psalm_b200 import kernels  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ncu", action="store_true")
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--blocked", type=float, default=0.5, help="fraction of keys blocked per query row")
    a = ap.parse_args()
    dt = torch.bfloat16
    B = int(os.environ.get("B", "4"))
    Lq, nh, C = 100, 8, 256
    hbm = 6650.0
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        hbm = json.load(open(p)).get("hbm_gbs", hbm)
    g = torch.Generator().manual_seed(0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for Lk in (1024, 4096, 16384):
        q = torch.randn(B, Lq, C, generator=g).to(dt).cuda()
        kall, vall = (torch.randn(B, Lk, 768, generator=g).to(dt).cuda() for _ in range(2))
        k, v = kall[:, :, 256:512], vall[:, :, 256:512]
        kc, vc = k.contiguous(), v.contiguous()
        # spatially smooth random mask (what thresholded mask logits look like): blocked runs of ~64 keys
        coarse = torch.rand(B, Lq, (Lk + 63) // 64, generator=g) < a.blocked
        blocked = coarse.repeat_interleave(64, dim=2)[:, :, :Lk]
        w = torch.zeros(B, Lq, (Lk + 31) // 32 * 32, dtype=torch.int64)
        w[:, :, :Lk] = blocked.long()
        words = (w.view(B, Lq, -1, 32) << torch.arange(32)).sum(-1)
        bits = torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32).cuda()
        row_open = torch.zeros(B, Lq, dtype=torch.uint8).cuda()
        nbytes = B * (2 * Lk * C * 2 + Lq * Lk // 8 + 2 * Lq * C * 2)
        from psalm_b200 import _lib
        runs = (("tma_auto", 0, lambda: kernels.masked_cross_attention(q, k, v, bits, row_open, nh)),
                ("mma_tma", 1, lambda: kernels.masked_cross_attention(q, k, v, bits, row_open, nh)),
                ("per_head_mma", 0, lambda: kernels.cross_attention(q, kc, vc, bits, row_open, nh)))
        for name, impl, fn in runs:
            _lib.lib().psalm_set_cross_impl(impl)
            if a.ncu:
                fn()
                torch.cuda.synchronize()
                continue
            ts = []
            for i in range(a.iters + 3):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda._sleep(2_000_000)
                e0.record()
                fn()
                e1.record()
                torch.cuda.synchronize()
                if i >= 3:
                    ts.append(e0.elapsed_time(e1) * 1e3)
            ts.sort()
            med = ts[len(ts) // 2]
            print(f"B={B} Lk={Lk:6d} {name:14s} median {med:7.1f} us  min {ts[0]:7.1f} us   {nbytes / med / 1e3:7.1f} GB/s  "
                  f"frac {nbytes / med / 1e3 / hbm:.3f} of measured HBM peak")


if __name__ == "__main__":
    main()
