#!/usr/bin/env python
"""Store what the reference's own MSDeformAttn CUDA op (oracle/build_ref_msda.py -> oracle/_ref/) computes at the 1024^2
encoder geometry as tests/golden/msda_ref_cuda.npz, so that tests/test_msda_gpu.py compares our kernel with it
without the reference being present.  Needs a GPU:

    python oracle/gen_golden_msda_cuda.py

Inputs come from `ref_inputs` (seeded CPU generator, shared with the test); the fixture keeps a fixed, seeded sample of
the outputs (the full output is 11 M values per dtype).
"""
import glob
import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(32, 32), (64, 64), (128, 128)]
B, M, D, L, P = 2, 8, 32, 3, 4
N_SAMPLE = 16384
OUT = os.path.join(ROOT, "tests", "golden", "msda_ref_cuda.npz")


def ref_inputs(dtype, seed=7):
    """value [B,S,M,D], loc [B,S,M,L,P,2], aw [B,S,M,L,P] in `dtype` (CPU), from a seeded CPU generator."""
    g = torch.Generator().manual_seed(seed)
    S = sum(h * w for h, w in SHAPES)
    v = torch.randn(B, S, M, D, generator=g).to(dtype)
    loc = (torch.rand(B, S, M, L, P, 2, generator=g) * 1.2 - 0.1).to(dtype)
    aw = torch.softmax(torch.randn(B, S, M, L * P, generator=g), -1).view(B, S, M, L, P).to(dtype)
    return v, loc, aw


def sample_index(n, seed=11):
    return np.sort(np.random.default_rng(seed).choice(n, N_SAMPLE, replace=False)).astype(np.int64)


def main():
    so = glob.glob(os.path.join(ROOT, "oracle", "_ref", "MultiScaleDeformableAttention*.so"))
    if not so:
        print("oracle/_ref not built (oracle/build_ref_msda.py)")
        return 1
    spec = importlib.util.spec_from_file_location("MultiScaleDeformableAttention", so[0])
    refop = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(refop)
    starts = np.cumsum([0] + [h * w for h, w in SHAPES])[:-1]
    sh = torch.tensor(SHAPES, dtype=torch.long, device="cuda")
    st = torch.tensor(starts, dtype=torch.long, device="cuda")
    gold = {}
    for name, dt in (("f32", torch.float32), ("f16", torch.float16)):
        v, loc, aw = (t.cuda() for t in ref_inputs(dt))
        out = refop.ms_deform_attn_forward(v, sh, st, loc, aw, 128)
        torch.cuda.synchronize()
        flat = out.float().reshape(-1).cpu()
        idx = sample_index(flat.numel())
        gold["idx"] = idx
        gold["out_" + name] = flat[torch.from_numpy(idx)].numpy()
        gold["absmax_" + name] = np.float32(flat.abs().max())
    np.savez_compressed(OUT, **gold)
    print("wrote", OUT, os.path.getsize(OUT), "bytes;", torch.cuda.get_device_name(0))
    return 0


if __name__ == "__main__":
    sys.exit(main())
