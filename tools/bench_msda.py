"""Micro-benchmark of the MSDeformAttn kernels at the 1024^2 geometry (one encoder layer-image).
Prints per-variant CUDA-event times and achieved algorithmic GB/s against MEASURED_PEAKS.json."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from psalm_b200 import msda  # noqa: E402


def timeit(fn, iters=20, warmup=5, flush=None):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.add_(1.0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def load_reference_op():
    """The reference's own CUDA op built for sm_90a by oracle/build_ref_msda.py (None if it was not built)."""
    import importlib.util
    so = os.path.join(ROOT, "oracle", "_ref", "MultiScaleDeformableAttention.so")
    if not os.path.exists(so):
        return None
    spec = importlib.util.spec_from_file_location("MultiScaleDeformableAttention", so)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    refop = load_reference_op()
    peaks = {}
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        peaks = json.load(open(p))
    hbm = peaks.get("hbm_gbs", 6650.0)
    B = int(os.environ.get("B", "1"))
    shapes = [(32, 32), (64, 64), (128, 128)]
    st = [0, 1024, 5120]
    S, M, D, L, P = 21504, 8, 32, 3, 4
    dev = "cuda"
    torch.manual_seed(0)
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)  # 256 MB > L2
    ref = torch.cat([torch.stack(torch.meshgrid((torch.arange(h) + 0.5) / h, (torch.arange(w) + 0.5) / w, indexing="ij"), -1).flip(-1).reshape(-1, 2)
                     for h, w in shapes]).to(dev)  # [S,2] (x,y)
    norm = torch.tensor([[w, h] for h, w in shapes], device=dev, dtype=torch.float32)
    res = {}
    for spread in (2.0, 6.0):
        off = torch.randn(B, S, M, L, P, 2, device=dev) * spread
        loc = (ref[None, :, None, None, None, :] + off / norm[None, None, None, :, None, :]).contiguous()
        logits = torch.randn(B, S, M, L * P, device=dev)
        aw = torch.softmax(logits, -1).view(B, S, M, L, P).contiguous()
        for dt, name in ((torch.float32, "f32"), (torch.bfloat16, "bf16"), (torch.float16, "f16")):
            v = torch.randn(B, S, M, D, device=dev).to(dt)
            vh = v.permute(0, 2, 1, 3).contiguous()
            es = 4 if dt == torch.float32 else 2
            bytes_boundary = B * (es * S * M * D * 2 + 4 * S * M * L * P * 3)
            for lay, vv in ((0, v), (1, vh)):
                med, best = timeit(lambda: msda.ms_deform_attn_forward(vv, shapes, st, loc, aw, 128, value_layout=lay), flush=flush)
                key = "%s_layout%d_spread%g" % (name, lay, spread)
                res[key] = dict(us=med, best_us=best, gbs=bytes_boundary / med / 1e3, frac=bytes_boundary / med / 1e3 / hbm)
            sh_t = torch.tensor(shapes, dtype=torch.long, device=dev)
            st_t = torch.tensor(st, dtype=torch.long, device=dev)
            if refop is not None and dt != torch.bfloat16:   # the reference dispatches float / double / half only
                # the kernel to beat: ms_deformable_im2col_gpu_kernel at ITS boundary (loc / w in value's dtype)
                locr, awr = loc.to(dt), aw.to(dt)
                bytes_ref = B * (es * S * M * D * 2 + es * S * M * L * P * 3)
                med, best = timeit(lambda: refop.ms_deform_attn_forward(v, sh_t, st_t, locr, awr, 128), flush=flush)
                res["%s_REFERENCE_kernel_spread%g" % (name, spread)] = dict(us=med, best_us=best, gbs=bytes_ref / med / 1e3,
                                                                            frac=bytes_ref / med / 1e3 / hbm)
                ours = msda.ms_deform_attn_forward(v, sh_t, st_t, locr, awr, 128)
                theirs = refop.ms_deform_attn_forward(v, sh_t, st_t, locr, awr, 128)
                res["%s_REFERENCE_kernel_spread%g" % (name, spread)]["max_abs_diff_vs_ours"] = float((ours.float() - theirs.float()).abs().max())
            if lay == 1:
                med, best = timeit(lambda: msda.ms_deform_attn_forward(v, sh_t, st_t, loc, aw, 128), flush=flush)
                res["%s_devshapes_linear_spread%g" % (name, spread)] = dict(us=med, best_us=best, gbs=bytes_boundary / med / 1e3)
            # fused: ow in the value dtype and in fp32
            for odt, oname in ((dt, name), (torch.float32, "f32")):
                ow = torch.cat([off.reshape(B, S, -1), logits.reshape(B, S, -1)], -1).to(odt).contiguous()
                bytes_fused = B * (es * S * M * D * 2 + ow.element_size() * S * M * L * P * 3)
                med, best = timeit(lambda: msda.msda_encoder_fused(vh, ow, shapes, st, P), flush=flush)
                res["%s_fused_ow%s_spread%g" % (name, oname, spread)] = dict(us=med, best_us=best, gbs=bytes_fused / med / 1e3, frac=bytes_fused / med / 1e3 / hbm)
    for k, v in res.items():
        print("%-40s %8.1f us (best %7.1f)  %8.1f GB/s  frac %.3f" % (k, v["us"], v["best_us"], v["gbs"], v.get("frac", 0)))
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    json.dump(res, open(os.path.join(ROOT, "gpurun_out", "bench_msda.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
