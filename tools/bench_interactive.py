"""Interactive segmentation against one image (bf16, CUDA graphs, full-size synthetic weights): per interaction of K
visual prompts of one kind (K = 1 / 3 / 8; point, scribble, box, mask) on COCO-sized originals padded to 1024^2,
  (a) the reference flow: the mapper's host mask preparation (oracle/visual_prompt.py, the reference's per-seed disks,
      Pillow NEAREST, padding) then `eval_seg` with instances.region_masks,
  (b) `open_image` once, then `ImageSession.eval_seg` with `visual_prompts`: the first interaction (graph capture) and
      the median of the later ones,
  (c) the rasteriser kernel alone (psalm_visual_prompt_raster, CUDA events over many launches).
Host times are perf_counter around work that ends in a device synchronise.  Prints one JSON object with the GPU name,
power limit and maximum SM clock.  Usage: python tools/bench_interactive.py [--reps 5] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import visual_prompt as VP  # noqa: E402
from psalm_b200 import kernels, synth  # noqa: E402
from psalm_b200.image_processor import nearest_pad_tables, resize_shortest_edge_shape  # noqa: E402
from psalm_b200.layout import PsalmConfig  # noqa: E402
from psalm_b200.psalm import PSALM  # noqa: E402
from psalm_b200.region import _source_masks  # noqa: E402
from psalm_b200.structures import BitMasks, Instances  # noqa: E402

KINDS = ("point", "scribble", "box", "mask")
S = 1024


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = "nvidia-smi unavailable: %s" % e
    return dict(name=torch.cuda.get_device_name(), nvidia_smi=q)


def prompt_masks(rng, kind, H, W, K):
    """K prompts of `kind` as COCO-Interactive makes them: single clicks, 300-pixel scribbles, boxes, object masks."""
    out = []
    for _ in range(K):
        m = np.zeros((H, W), np.uint8)
        if kind == "point":
            m[rng.integers(H), rng.integers(W)] = 1
        elif kind == "scribble":
            y, x = int(rng.integers(H)), int(rng.integers(W))
            while m.sum() < 300:
                m[y, x] = 1
                y, x = int(np.clip(y + rng.integers(-1, 2), 0, H - 1)), int(np.clip(x + rng.integers(-1, 2), 0, W - 1))
        elif kind == "box":
            y0, x0 = int(rng.integers(H // 2)), int(rng.integers(W // 2))
            m = VP.paint_box(H, W, (y0, x0, y0 + H // 4, x0 + W // 4))
        else:
            yy, xx = np.ogrid[:H, :W]
            m[((yy - rng.integers(H)) / (H // 6)) ** 2 + ((xx - rng.integers(W)) / (W // 6)) ** 2 <= 1] = 1
        out.append(m)
    return out


def host_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--kernel-reps", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    cfg = PsalmConfig()
    sd = synth.synth_state_dict(cfg, seed=2)
    m = PSALM(sd, cfg, torch.bfloat16, "cuda", "region", use_cuda_graph=True)
    del sd
    rows = []
    for H0, W0 in ((480, 640), (427, 640)):
        oh, ow = resize_shortest_edge_shape(H0, W0, S, S)
        inp = synth.synth_inputs(batch=1, height=S, width=S, task="region", seed=3, n_regions=1)
        pad = torch.ones(S, S, dtype=torch.bool)
        pad[:oh, :ow] = False
        info = dict(padding_mask=pad, height=H0, width=W0)
        rng = np.random.default_rng(H0 * W0)
        for K in (1, 3, 8):
            p = synth.synth_inputs(batch=1, height=64, width=64, task="region", seed=3, n_regions=K)
            for kind in KINDS:
                masks = prompt_masks(rng, kind, H0, W0, K)
                vp = [(kind, torch.from_numpy(mk)) for mk in masks]
                prompt = dict(input_ids=p["input_ids"], attention_mask=p["attention_mask"], visual_prompts=vp)

                def reference():           # (a) host mask preparation, then eval_seg with the region masks
                    t0 = time.perf_counter()
                    rm = torch.from_numpy(np.stack([VP.region_mask(kind, mk, (oh, ow), (S, S), literal=True)
                                                    for mk in masks]))
                    inst = Instances((S, S))
                    inst.region_masks = BitMasks(rm)
                    prep = (time.perf_counter() - t0) * 1e3
                    ms, _ = host_ms(lambda: m.eval_seg(input_ids=p["input_ids"], attention_mask=p["attention_mask"],
                                                       images=inp["images"], seg_info=[dict(info, instances=inst)]))
                    return prep, ms
                reference()                # warm-up (eval_seg region prompts run eagerly)
                ref = [reference() for _ in range(2 if kind == "scribble" and K == 8 else args.reps)]
                sess = m.open_image(inp["images"], [info])
                first, _ = host_ms(lambda: sess.eval_seg([prompt]))
                later = sorted(host_ms(lambda: sess.eval_seg([prompt]))[0] for _ in range(args.reps))
                src, radius = _source_masks(vp, H0, W0, "cuda")
                tr, tc = (t.cuda() for t in nearest_pad_tables(H0, W0, (oh, ow), (S, S)))
                for _ in range(10):
                    kernels.visual_prompt_raster(src, radius, tr, tc)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.kernel_reps):
                    kernels.visual_prompt_raster(src, radius, tr, tc)
                b.record()
                torch.cuda.synchronize()
                prep = sorted(r[0] for r in ref)
                seg = sorted(r[1] for r in ref)
                row = dict(size="%dx%d" % (H0, W0), kind=kind, K=K,
                           ref_prep_ms=round(prep[len(prep) // 2], 2), ref_eval_seg_ms=round(seg[len(seg) // 2], 2),
                           ref_total_ms=round(prep[len(prep) // 2] + seg[len(seg) // 2], 2),
                           session_first_ms=round(first, 2), session_later_ms=round(later[len(later) // 2], 2),
                           raster_us=round(a.elapsed_time(b) * 1e3 / args.kernel_reps, 1))
                print(json.dumps(row), flush=True)
                rows.append(row)
    res = dict(gpu=gpu_info(), rows=rows)
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_interactive.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
