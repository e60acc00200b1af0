"""Several referring prompts against one 1024^2 image (bf16, CUDA graphs, synthetic weights): milliseconds per image for
  (a) K eval_seg calls at batch 1,
  (b) one eval_seg call with the image repeated K times,
  (c) open_image + ImageSession.eval_seg of the K prompts,
  (d) ImageSession.eval_seg alone (image already open),
each as device time (CUDA events) and host time (perf_counter around the work, ending in a synchronise); plus the
prefix-causal attention kernel beside causal_attention at T = 399 (the unsplit prompt).  Prints one JSON object with
the GPU name and power limit.  Usage: python tools/bench_prompts.py [--ks 1,2,4,8,16] [--reps 10] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import torch  # noqa: E402

from psalm_b200 import kernels, synth  # noqa: E402
from psalm_b200 import sequence as SEQ  # noqa: E402
from psalm_b200.layout import PsalmConfig  # noqa: E402
from psalm_b200.psalm import PSALM  # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = "nvidia-smi unavailable: %s" % e
    return dict(name=torch.cuda.get_device_name(), nvidia_smi=q)


def timed(fn, reps, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dev, host = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        host.append((time.perf_counter() - t0) * 1e3)
        dev.append(a.elapsed_time(b))
    dev.sort(), host.sort()
    return dict(device_ms=round(dev[len(dev) // 2], 3), host_ms=round(host[len(host) // 2], 3),
                host_ms_min=round(host[0], 3), host_ms_max=round(host[-1], 3))


def kernel_times(reps=50):
    """prefix_causal_attention (P = 276 shared rows, 123 own rows) beside causal_attention over all 399 rows, one prompt."""
    nh, hd, P, Ts = 32, 64, 276, 123
    qkv = torch.randn(1, P + Ts, 3, nh, hd, device="cuda").bfloat16()
    page = -(-P // 64) * 64
    pk = torch.zeros(nh, page, hd, device="cuda").bfloat16()
    pv = torch.zeros_like(pk)
    pk[:, :P] = qkv[0, :P, 1].transpose(0, 1)
    pv[:, :P] = qkv[0, :P, 2].transpose(0, 1)
    suf = qkv[:, P:].contiguous()
    out = {}
    for name, fn in (("causal_attention_T399", lambda: kernels.causal_attention(qkv, None, 1, P + Ts, nh, hd)),
                     ("prefix_causal_attention_P276_T123", lambda: kernels.prefix_causal_attention(suf, pk, pv, P, None, 1, Ts, nh, hd))):
        for _ in range(5):
            fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        out[name + "_us"] = round(a.elapsed_time(b) / reps * 1e3, 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,2,4,8,16")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_prompts: needs a CUDA device")
    info = gpu_info()
    cfg = PsalmConfig()
    sd = synth.synth_state_dict(cfg, seed=2)
    m = PSALM(sd, cfg, torch.bfloat16, "cuda", "referring", use_cuda_graph=True)
    del sd
    S = args.size
    rows = []
    for K in [int(k) for k in args.ks.split(",")]:
        # one template, K referred objects of 12 tokens each (one graph per path, no re-capture inside the timing)
        base = synth.synth_inputs(batch=1, height=S, width=S, task="referring", refer_len=12, seed=3)
        g = torch.Generator().manual_seed(K)
        ins = []
        for k in range(K):
            i = dict(base)
            r = base["token_refer_id"][0].clone()
            r[:-1] = torch.randint(5, 50000, (r.numel() - 1,), generator=g)
            i["token_refer_id"] = [r]
            ins.append(i)
        prompts = [{n: i[n] for n in SEQ.PROMPT_KEYS if i.get(n) is not None} for i in ins]
        img = ins[0]["images"].cuda()
        info0 = ins[0]["seg_info"]

        def per_prompt():
            for i in ins:
                m.eval_seg(input_ids=i["input_ids"], attention_mask=i["attention_mask"], images=img, seg_info=info0,
                           token_refer_id=i["token_refer_id"], refer_embedding_indices=i["refer_embedding_indices"])

        batch = synth.synth_inputs(batch=K, height=S, width=S, task="referring", refer_len=8, seed=3, ragged=K > 1)
        bimg = img.expand(K, -1, -1, -1).contiguous()

        def batched():
            m.eval_seg(input_ids=batch["input_ids"], attention_mask=batch["attention_mask"], images=bimg,
                       seg_info=batch["seg_info"], token_refer_id=batch["token_refer_id"],
                       refer_embedding_indices=batch["refer_embedding_indices"])

        def session():
            m.open_image(img, info0).eval_seg(prompts)

        opened = m.open_image(img, info0, lane=1)

        def prompts_only():
            opened.eval_seg(prompts)

        row = dict(K=K)
        for name, fn in (("a_eval_seg_x_K", per_prompt), ("b_eval_seg_batch_K", batched), ("c_open_image_plus_session", session),
                         ("d_session_eval_seg", prompts_only)):
            row[name] = timed(fn, args.reps)
        rows.append(row)
        print(json.dumps(row), flush=True)
    res = dict(gpu=info, size=S, dtype="bf16", graphs=True, rows=rows, kernels=kernel_times())
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_prompts.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
