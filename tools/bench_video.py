"""DAVIS-style video clip on one GPU (bf16, CUDA graphs, synthetic weights of the full model): milliseconds per frame of
  (a) eval_video + the reference's per-frame loop on the host (oracle/davis_loop.py: pick, fuse, memory check, memory
      update with Pillow-NEAREST resized masks) - what a user writes today,
  (b) open_video + VideoSession.step,
at 1024^2 padded frames with 480x854 outputs, for K objects.  Also the session's per-frame device time (CUDA events
around one step, which ends in its small device-to-host copy), the launches of our kernels per eager prompt phase, and
the kernel times of vos_pick / vos_fuse / region_points_gather (CUDA events over many launches).  Prints one JSON object
with the GPU name and power limit.  Usage: python tools/bench_video.py [--ks 1,3,5,10] [--frames 12] [--warm 3] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import davis_loop as D  # noqa: E402
from psalm_b200 import kernels, synth  # noqa: E402
from psalm_b200.image_processor import nearest_pad_tables  # noqa: E402
from psalm_b200.layout import PsalmConfig  # noqa: E402
from psalm_b200.psalm import PSALMForDAVISEval  # noqa: E402
from psalm_b200.structures import BitMasks, Instances  # noqa: E402

S, OUT_HW, RESIZED = 1024, (480, 854), (576, 1024)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = "nvidia-smi unavailable: %s" % e
    return dict(name=torch.cuda.get_device_name(), nvidia_smi=q)


def clip(K, n):
    first = synth.synth_inputs(batch=1, height=S, width=S, task="region", seed=40, n_regions=K)
    pad = torch.ones(S, S, dtype=torch.bool)
    pad[:RESIZED[0], :RESIZED[1]] = False
    info = dict(padding_mask=pad, height=OUT_HW[0], width=OUT_HW[1])
    g = torch.Generator().manual_seed(3)
    frames = [torch.randn(1, 3, S, S, generator=g).pin_memory() for _ in range(n)]
    fills = torch.arange(1, K + 1, dtype=torch.int64)
    return first, first["seg_info"][0]["instances"].region_masks.tensor.clone(), fills, frames, info


def run_loop(m, first, vp_masks, fills, frames, info):
    loop = D.DavisLoop(first["images"], vp_masks.numpy(), fills.tolist(), True)
    for img in frames:
        vp_img, vp_m, vp_f = loop.inputs()
        inst = Instances(OUT_HW)
        inst.vp_region_masks = BitMasks(torch.as_tensor(vp_m))
        inst.vp_fill_number = torch.as_tensor(vp_f)
        inst.gt_masks = torch.zeros(len(vp_f), 1, 1)
        res = m.eval_video(input_ids=first["input_ids"], attention_mask=first["attention_mask"], images=img,
                           vp_images=vp_img, seg_info=[dict(info, instances=inst)])[0]
        loop.update(res, vp_f, img, RESIZED, (S, S))


def run_session(m, first, vp_masks, fills, frames, info):
    inst = Instances(OUT_HW)
    inst.vp_region_masks = BitMasks(vp_masks)
    inst.vp_fill_number = fills
    vid = m.open_video(first["images"], [dict(info, instances=inst)], first["input_ids"], first["attention_mask"])
    pend = [vid.step_async(img, [info]) for img in frames]     # each step resolves the previous frame
    return [p.result() for p in pend], vid


def host_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def kernel_ms(fn, reps=200):
    for _ in range(5):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return round(a.elapsed_time(b) * 1e3 / reps, 2)


def kernel_times(K):
    H, W = OUT_HW
    g = torch.Generator().manual_seed(K)
    logits = torch.randn(K, 100, generator=g).bfloat16().cuda()
    stats = torch.rand(100, 5, generator=g).cuda() * 1000
    masks = (torch.rand(K, H, W, generator=g) > 0.7).float().cuda()
    rows, cols = (t.cuda() for t in nearest_pad_tables(H, W, RESIZED, (S, S)))
    bits = torch.zeros(K, S, S // 32, dtype=torch.int32, device="cuda")
    rp = torch.zeros(K, S + 1, dtype=torch.int32, device="cuda")
    cnt = torch.zeros(K, dtype=torch.int32, device="cuda")
    fill = torch.arange(1, K + 1, dtype=torch.int32, device="cuda")
    labels = torch.zeros(H, W, dtype=torch.uint8, device="cuda")
    area = torch.zeros(K, dtype=torch.int32, device="cuda")
    inter = torch.zeros(K, K, dtype=torch.int32, device="cuda")
    kernels.vos_fuse(masks, rows, cols, bits, rp, cnt, fill, labels, area, inter)
    torch.cuda.synchronize()
    sel = torch.stack([torch.randint(0, max(1, int(c)), (256,)) for c in cnt.cpu()]).to(torch.int32).cuda()
    mor = torch.arange(K, dtype=torch.int32, device="cuda")
    return dict(vos_pick_us=kernel_ms(lambda: kernels.vos_pick(logits, stats)),
                vos_fuse_us=kernel_ms(lambda: kernels.vos_fuse(masks, rows, cols, bits, rp, cnt, fill, labels, area, inter)),
                region_points_gather_us=kernel_ms(lambda: kernels.region_points_gather(bits, rp, sel, mor, S, S)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,3,5,10")
    ap.add_argument("--frames", type=int, default=12)
    ap.add_argument("--warm", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_video.py needs a GPU"
    cfg = PsalmConfig()
    sd = synth.synth_state_dict(cfg, seed=0, dtype=torch.bfloat16, device="cuda")
    loop_m = PSALMForDAVISEval(sd, cfg, torch.bfloat16, "cuda", "region")
    sess_m = PSALMForDAVISEval(sd, cfg, torch.bfloat16, "cuda", "region", use_cuda_graph=True)
    eager_m = PSALMForDAVISEval(sd, cfg, torch.bfloat16, "cuda", "region")
    res = dict(gpu=gpu_info(), frames=a.frames, frame=[S, S], output=list(OUT_HW), dtype="bf16", per_k={})
    for K in [int(k) for k in a.ks.split(",")]:
        first, vp_masks, fills, frames, info = clip(K, a.warm + a.frames)
        warm, timed = frames[:a.warm], frames[a.warm:]
        run_loop(loop_m, first, vp_masks, fills, warm, info)
        run_session(sess_m, first, vp_masks, fills, warm, info)
        r = {}
        for rep in range(2):          # alternate (a) and (b)
            r.setdefault("loop_ms_per_frame", []).append(
                round(host_ms(lambda: run_loop(loop_m, first, vp_masks, fills, timed, info)) / len(timed), 2))
            r.setdefault("session_ms_per_frame", []).append(
                round(host_ms(lambda: run_session(sess_m, first, vp_masks, fills, timed, info)) / len(timed), 2))
        _, vid = run_session(sess_m, first, vp_masks, fills, warm, info)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        dev = []
        for img in timed:
            ev[0].record()
            vid.step(img, [info])
            ev[1].record()
            torch.cuda.synchronize()
            dev.append(ev[0].elapsed_time(ev[1]))
        r["session_step_device_ms_median"] = round(float(np.median(dev)), 2)
        _, evid = run_session(eager_m, first, vp_masks, fills, warm[:1], info)
        n0 = kernels.launches()
        evid.step(timed[0], [info])
        r["own_kernel_launches_per_eager_step"] = kernels.launches() - n0
        r["session_graph_replays_per_step"] = 2
        r["kernels"] = kernel_times(K)
        res["per_k"][K] = r
        print(json.dumps({K: r}), flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_video.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
