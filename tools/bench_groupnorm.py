"""Time groupnorm_tokens (partial + finalize + apply) at the pixel-decoder shapes, with CUDA events.

Each --lib is a built libpsalm_b200.so (default: the package's own); with several, the libraries are timed in
alternating rounds on the same inputs, so that a comparison of two builds sees the same machine state, and their
outputs are compared.  Prints one line per (shape, library): median time of a call over the rounds.

    python tools/bench_groupnorm.py [--lib A.so --lib B.so] [--rounds 7] [--iters 50]
"""
import argparse
import ctypes
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from psalm_b200 import _lib  # noqa: E402

SHAPES = [  # (B, N, C, pre_bias): adapter / layer GroupNorm at stride 4, and the input projections at strides 8 / 16 / 32
    (4, 256 * 256, 256, True),
    (4, 128 * 128, 256, False),
    (4, 64 * 64, 256, False),
    (4, 32 * 32, 256, False),
]


def load(path):
    h = ctypes.CDLL(path)
    f = h.psalm_groupnorm_tokens
    f.argtypes = [ctypes.c_void_p] * 6 + [ctypes.c_int] * 4 + [ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    f.restype = ctypes.c_int
    return f


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=None)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    libs = args.lib or [_lib.LIB_PATH]
    fns = [load(p) for p in libs]
    assert torch.cuda.is_available(), "needs a GPU"
    props = torch.cuda.get_device_properties(0)
    print("device %s" % props.name)
    dt = torch.bfloat16
    g = torch.Generator(device="cuda").manual_seed(0)
    for B, N, C, pre in SHAPES:
        x = (torch.randn(B, N, C, device="cuda", generator=g) * 2 + 3).to(dt)
        w = torch.randn(C, device="cuda", generator=g).to(dt)
        b = torch.randn(C, device="cuda", generator=g).to(dt)
        pb = torch.randn(C, device="cuda", generator=g).to(dt) if pre else None
        ws = torch.empty(B * 32 * (2 + 4 * ((N + 63) // 64)) + 4, dtype=torch.float64, device="cuda")
        ys = [torch.empty_like(x) for _ in fns]
        stream = _lib.stream_ptr()

        def call(k):
            rc = fns[k](x.data_ptr(), pb.data_ptr() if pb is not None else None, w.data_ptr(), b.data_ptr(), ys[k].data_ptr(),
                        ws.data_ptr(), B, N, C, 32, 1e-5, 1, _lib.dtype_code(dt), stream)
            assert rc == 0, rc

        times = [[] for _ in fns]
        for k in range(len(fns)):                                  # warm-up
            for _ in range(5):
                call(k)
        for _ in range(args.rounds):
            for k in range(len(fns)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    call(k)
                e1.record()
                torch.cuda.synchronize()
                times[k].append(e0.elapsed_time(e1) * 1e3 / args.iters)
        for k, p in enumerate(libs):
            diff = float((ys[k].float() - ys[0].float()).abs().max())
            print("B %d N %6d C %d pre_bias %d  %-60s median %8.2f us  (min %8.2f)  max |y - y_lib0| %.3e"
                  % (B, N, C, pre, p[-60:], statistics.median(times[k]), min(times[k]), diff))


if __name__ == "__main__":
    main()
