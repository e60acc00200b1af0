"""Device COCO RLE encode (csrc/rle.cu) vs the host path it replaces.

Workload: 100 fp32 instance masks per image (the `Instances.pred_masks` of a COCO-instance step) at 1024^2 and 1333^2,
for 1 and 4 images encoded in one call.  Masks are random ellipses (instance-like: a few hundred to a few thousand runs
per mask).  Reports, with the GPU name and power limit read in the same run:
  * device encode time per image (CUDA events around `rle.encode_device`, which includes its two small device-to-host
    size copies), and GB/s against the dense bytes read;
  * the host path of detectron2's COCOEvaluator: device-to-host copy of the dense masks, then the encoder on the host
    (pycocotools when importable, else oracle/coco_rle.py), timed separately;
  * per-kernel device times from torch.profiler, in a separate pass.
Usage: python tools/bench_rle.py [--iters 20] [--json out.json]"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import coco_rle  # noqa: E402
from psalm_b200 import rle  # noqa: E402


def card():
    name = torch.cuda.get_device_name()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                                str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def ellipses(n, H, W, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda lo, hi: lo + (hi - lo) * torch.rand(n, 1, 1, device="cuda", generator=g)  # noqa: E731
    cy, cx, a, b = r(0, H), r(0, W), r(H / 40, H / 4), r(W / 40, W / 4)
    y = torch.arange(H, device="cuda", dtype=torch.float32).view(1, H, 1)
    x = torch.arange(W, device="cuda", dtype=torch.float32).view(1, 1, W)
    return ((((y - cy) / a) ** 2 + ((x - cx) / b) ** 2) < 1).float()


def host_encoder():
    try:
        from pycocotools import mask as mask_util
        return "pycocotools", lambda m: mask_util.encode(np.asfortranarray(m.transpose(1, 2, 0).astype(np.uint8)))
    except ImportError:
        return "oracle/coco_rle.py", coco_rle.encode_masks


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_rle needs a GPU"
    name, power = card()
    print("gpu: %s, power limit %s" % (name, power))
    hname, henc = host_encoder()
    rows = []
    for S in (1024, 1333):
        for images in (1, 4):
            masks = [ellipses(100, S, S, seed=i) for i in range(images)]
            dense = sum(m.numel() * m.element_size() for m in masks)
            for _ in range(3):                                   # warm-up (allocator, module load)
                rle.encode_device(masks)
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.iters):
                d = rle.encode_device(masks)
            b.record()
            torch.cuda.synchronize()
            ms = a.elapsed_time(b) / args.iters
            nbytes = int(d["offsets"][-1])
            row = dict(size=S, images=images, masks=100 * images, dense_MB=dense / 1e6, device_us_per_image=1e3 * ms / images,
                       device_GBps=dense / (ms * 1e-3) / 1e9, rle_bytes=nbytes)
            # host path for one image's masks: D2H of the dense fp32 masks, then the host encoder
            m0 = masks[0]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            host = m0.cpu()
            t1 = time.perf_counter()
            ref = henc(host.numpy())
            t2 = time.perf_counter()
            assert [r["counts"] for r in ref] == [r["counts"] for r in rle.to_dicts(rle.encode_device(m0))]
            row.update(host_d2h_ms_per_image=1e3 * (t1 - t0), host_encode_ms_per_image=1e3 * (t2 - t1), host_encoder=hname)
            rows.append(row)
            print("%4d^2 x %d img: device %8.1f us/img  %6.0f GB/s  (%d string bytes) | host: D2H %7.1f ms/img + %s %8.1f ms/img"
                  % (S, images, row["device_us_per_image"], row["device_GBps"], nbytes, row["host_d2h_ms_per_image"], hname,
                     row["host_encode_ms_per_image"]))
            del masks, d
    # per-kernel breakdown, separate pass (tracing slows the host)
    masks = [ellipses(100, 1024, 1024, seed=0)]
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            rle.encode_device(masks)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        k = re.search(r"rle_\w+_kernel(<\w+>)?", e.key)
        if k:
            kern[k.group(0)] = e.device_time
    print("per-kernel device us (100 x 1024^2 fp32, mean per call):", json.dumps({k: round(v, 1) for k, v in kern.items()}))
    out = dict(gpu=name, power_limit=power, rows=rows, kernels_us_1024_1img=kern)
    print(json.dumps(out))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
