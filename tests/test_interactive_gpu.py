"""Interactive segmentation on the GPU: the visual-prompt rasteriser (csrc/vos.cu) bit for bit against the region-mask
oracle (oracle/visual_prompt.py, pinned to the reference in tests/test_interactive_cpu.py), the sample points it feeds,
and ImageSession.eval_seg with `visual_prompts` against per-prompt eval_seg fed the oracle's region masks."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import visual_prompt as VP
from psalm_b200 import synth
from psalm_b200.image_processor import resize_shortest_edge_shape
from psalm_b200.layout import PhiConfig, PsalmConfig
from psalm_b200.region import draw_point_indices, rasterize_visual_prompts, sample_region_points
from psalm_b200.structures import BitMasks, Instances

pytestmark = pytest.mark.gpu
SMALL = PsalmConfig(phi=PhiConfig(hidden=256, layers=2, heads=4, inter=1024))
KINDS = ("point", "scribble", "box", "mask")


def _unpack(bits, Wp):
    b = ((bits.long().cpu() & 0xFFFFFFFF).unsqueeze(-1) >> torch.arange(32)) & 1
    return b.view(bits.shape[0], bits.shape[1], -1)[..., :Wp].bool()


def _src(rng, kind, H, W, j):
    """A prompt of `kind` as (source for the session, 0/1 uint8 mask at the original size).  Every fourth touches a
    border or a corner."""
    edge = j % 4 == 0
    if kind == "point":
        y, x = (0, W - 1) if edge else (int(rng.integers(H)), int(rng.integers(W)))
        m = np.zeros((H, W), np.uint8)
        m[y, x] = 1
        return (y, x), m
    if kind == "box":
        y0, x0 = (H - 30, 0) if edge else (int(rng.integers(H - 2)), int(rng.integers(W - 2)))
        box = (y0, x0, y0 + int(rng.integers(1, H // 3)), x0 + int(rng.integers(1, W // 3)))
        return box, VP.paint_box(H, W, box)
    m = np.zeros((H, W), np.uint8)
    if kind == "scribble":
        y, x = (H - 1, int(rng.integers(W))) if edge else (int(rng.integers(H)), int(rng.integers(W)))
        for _ in range(int(rng.integers(20, 300))):
            m[y, x] = 1
            y, x = int(np.clip(y + rng.integers(-1, 2), 0, H - 1)), int(np.clip(x + rng.integers(-1, 2), 0, W - 1))
    else:
        yy, xx = np.ogrid[:H, :W]
        cy, cx = (0, 0) if edge else (rng.integers(H), rng.integers(W))
        m[((yy - cy) / rng.integers(3, H // 4)) ** 2 + ((xx - cx) / rng.integers(3, W // 4)) ** 2 <= 1] = 1
    return torch.from_numpy(m), m


@pytest.mark.parametrize("H,W", [(480, 640), (640, 427), (333, 500), (1333, 1000)])
def test_raster_is_bit_identical_to_the_oracle(H, W):
    rng = np.random.default_rng(H * W)
    oh, ow = resize_shortest_edge_shape(H, W, 1024, 1024)
    prompts, want = [], []
    for j in range(40):
        kind = KINDS[j % 4]
        s, m = _src(rng, kind, H, W, j)
        prompts.append((kind, s))
        want.append(VP.region_mask(kind, m, (oh, ow), (1024, 1024)))
    want = np.stack(want)
    for K in (1, 7, 40):
        bits, rp, cnt = rasterize_visual_prompts(prompts[:K], H, W, (oh, ow), (1024, 1024), "cuda")
        torch.cuda.synchronize()
        assert np.array_equal(_unpack(bits, 1024).numpy(), want[:K]), K
        assert np.array_equal(cnt.cpu().numpy(), want[:K].sum((1, 2)))
        assert np.array_equal(rp[:, 0].cpu().numpy(), np.zeros(K)) and \
            np.array_equal(rp[:, 1:].cpu().numpy(), want[:K].sum(2).cumsum(1))


def test_rle_tensor_and_coordinate_sources_give_identical_bits():
    from psalm_b200 import rle
    H, W = 480, 640
    oh, ow = resize_shortest_edge_shape(H, W, 1024, 1024)
    rng = np.random.default_rng(5)
    forms = []
    for kind, j in (("point", 0), ("point", 1), ("box", 0), ("box", 1), ("scribble", 2), ("mask", 3)):
        s, m = _src(rng, kind, H, W, j)
        t = torch.from_numpy(m)
        enc = rle.encode(t.cuda()[None])[0]
        enc = {"size": enc["size"], "counts": enc["counts"].decode("ascii")}
        variants = [t, t.cuda(), enc] + ([s] if not isinstance(s, torch.Tensor) else [])
        forms.append([(kind, v) for v in variants])
    outs = [rasterize_visual_prompts([f[i] if i < len(f) else f[0] for f in forms], H, W, (oh, ow), (1024, 1024), "cuda")
            for i in range(4)]
    for o in outs[1:]:
        for a, b in zip(o, outs[0]):
            assert torch.equal(a, b)


def test_points_from_the_raster_equal_sample_region_points():
    from psalm_b200 import kernels
    H, W = 333, 500
    oh, ow = resize_shortest_edge_shape(H, W, 1024, 1024)
    rng = np.random.default_rng(9)
    prompts, masks = [], []
    for j in range(8):
        kind = KINDS[j % 4]
        s, m = _src(rng, kind, H, W, j)
        prompts.append((kind, s))
        masks.append(torch.from_numpy(VP.region_mask(kind, m, (oh, ow), (1024, 1024))))
    bits, rp, cnt = rasterize_visual_prompts(prompts, H, W, (oh, ow), (1024, 1024), "cuda")
    torch.manual_seed(3)
    sel = draw_point_indices(cnt.tolist())
    got = kernels.region_points_gather(bits, rp, sel.cuda(), torch.arange(8, dtype=torch.int32, device="cuda"), 1024, 1024)
    torch.manual_seed(3)
    assert torch.equal(got.cpu(), sample_region_points(torch.stack(masks)))


# ---- sessions against per-prompt eval_seg ---------------------------------------------------------------------------------
def _scene(S, H0, W0, Ks, seed):
    """An S x S input holding an (H0, W0) original resized into its top-left box, and one prompt per K in Ks with K
    regions of mixed kinds: (inputs, session prompts, per-prompt seg_info with the oracle's region masks)."""
    oh, ow = resize_shortest_edge_shape(H0, W0, S, S)
    inp = synth.synth_inputs(batch=1, height=S, width=S, task="region", seed=seed, n_regions=max(Ks))
    pad = torch.ones(S, S, dtype=torch.bool)
    pad[:oh, :ow] = False
    info = dict(padding_mask=pad, height=H0, width=W0)
    rng = np.random.default_rng(seed)
    prompts, infos = [], []
    for i, K in enumerate(Ks):
        p = synth.synth_inputs(batch=1, height=64, width=64, task="region", seed=seed, n_regions=K)
        vp, rm = [], []
        for j in range(K):
            kind = KINDS[(i + j) % 4]
            s, m = _src(rng, kind, H0, W0, j + 1)
            vp.append((kind, s))
            rm.append(torch.from_numpy(VP.region_mask(kind, m, (oh, ow), (S, S))))
        prompts.append(dict(input_ids=p["input_ids"], attention_mask=p["attention_mask"], visual_prompts=vp))
        inst = Instances((S, S))
        inst.region_masks = BitMasks(torch.stack(rm))
        inst.gt_masks = torch.stack(rm).float()
        infos.append([dict(info, instances=inst)])
    return inp, info, prompts, infos


def _per_prompt(m, inp, prompts, infos, seed, logits=False):
    """Per-prompt eval_seg in prompt order from `seed`: (scores, pred_masks[, region logits of the same forward])."""
    from psalm_b200.region import region_inputs
    torch.manual_seed(seed)
    out = []
    for p, si in zip(prompts, infos):
        pts, img, _ = region_inputs(si)                      # the draws eval_seg makes, in the same order
        r = m.eval_seg(input_ids=p["input_ids"], attention_mask=p["attention_mask"], images=inp["images"], seg_info=si,
                       region_points=[pts])
        row = (r[0]["instances"].scores.float().clone(), r[0]["instances"].pred_masks.clone())
        if logits:
            plan = m.make_plan(p["input_ids"], p["attention_mask"], inp["images"].shape[-2:])
            plan.region_points, plan.region_image = pts, img
            row += (m.forward_core(inp["images"].cuda(), plan.to("cuda"))["pred_region_logits"][0].float(),)
        out.append(row)
    return out


def _snap(res):
    return [(r["instances"].scores.float().clone(), r["instances"].pred_masks.clone()) for r in res]


@pytest.mark.parametrize("S,H0,W0", [(192, 150, 120), (1024, 480, 640)])
def test_fp32_session_matches_per_prompt_eval_seg(S, H0, W0):
    """Region logits within 2e-3 max-rel, scores within the fp32 bar of tests/test_region_gpu.py (l2-rel < 1e-3), the
    same top-1 query per region and its identical masks.  The masked decoder thresholds mask logits into attention
    masks, so a logit within rounding of 0 that the split prefill flips moves the region logits at the 1e-3 level
    (tests/test_region_gpu.py notes the same for the oracle across thread counts).  Measured on an H100 80GB HBM3
    (700 W): 3.0e-5 at 192^2; 1.15e-3 at 1024^2 for the K = 1 prompt, where one pixel of one of its 100 masks differs
    (score l2-rel 4.9e-4)."""
    from psalm_b200.psalm import PSALM
    sd = synth.synth_state_dict(SMALL, seed=9)
    m = PSALM(sd, SMALL, torch.float32, "cuda", "region")
    inp, info, prompts, infos = _scene(S, H0, W0, (1, 3, 2), seed=21)
    want = _per_prompt(m, inp, prompts, infos, 77, logits=True)
    torch.manual_seed(77)
    pend = m.open_image(inp["images"], infos[0]).eval_seg_async(prompts)
    logits = [part[0]["pred_region_logits"][0].float().clone() for part in pend.parts]
    res = pend.result()
    measured = []
    for k, (r, lg, (ws, wm, wl)) in enumerate(zip(res, logits, want)):
        s, pm = r["instances"].scores.float(), r["instances"].pred_masks
        assert s.shape == ws.shape and lg.shape == wl.shape
        lerr = float((lg - wl).abs().max() / wl.abs().max())
        smax = float((s - ws).abs().max() / ws.abs().max())
        sl2 = float((s - ws).norm() / ws.norm())
        measured.append(dict(logit_maxrel=lerr, score_maxrel=smax, score_l2rel=sl2,
                             mask_pixels_differ=float((pm != wm).float().mean())))
        assert lerr < 2e-3, (k, measured[-1])
        assert sl2 < 1e-3, (k, measured[-1])
        assert torch.equal(s.argmax(0), ws.argmax(0)), k                 # the same top-1 query per region
        top = ws.argmax(0)
        assert torch.equal(pm[top], wm[top]), k                           # its masks are identical
    print("fp32 session vs eval_seg at %d^2:" % S, measured)
    gt = m.eval_seg(input_ids=prompts[0]["input_ids"], attention_mask=prompts[0]["attention_mask"], images=inp["images"],
                    seg_info=infos[0])[0]["gt"]
    assert torch.equal(res[0]["gt"], gt)          # the opened image's gt_masks


def test_bf16_graph_sessions_replay_like_eager():
    """Region structures K = 1, 3, 7, two prompts of K = 3, and a repeat at 1024^2: graph replays equal eager launches."""
    from psalm_b200.psalm import PSALM
    sd = synth.synth_state_dict(SMALL, seed=9)
    eager = PSALM(sd, SMALL, torch.bfloat16, "cuda", "region")
    graphed = PSALM(sd, SMALL, torch.bfloat16, "cuda", "region", use_cuda_graph=True)
    inp, info, prompts, infos = _scene(1024, 480, 640, (1, 3, 7, 3), seed=23)
    calls = [[prompts[0]], [prompts[1]], [prompts[2]], [prompts[3], prompts[1]], [prompts[1]]]
    sess_e = eager.open_image(inp["images"], infos[0])
    sess_g = graphed.open_image(inp["images"], infos[0])
    for call in calls:
        torch.manual_seed(5)
        a = _snap(sess_e.eval_seg(call))
        torch.manual_seed(5)
        b = _snap(sess_g.eval_seg(call))
        for (sa, ma), (sb, mb) in zip(a, b):
            assert torch.allclose(sa, sb, rtol=1e-5, atol=1e-7) and torch.equal(ma, mb)
    assert len(graphed._prompt_graphs) == 4


def test_bf16_full_size_graph_session_tracks_per_prompt_eval_seg():
    """Full-size synthetic weights, K = 1, 3, 7 at 1024^2: per region, the IoU of the top-1 mask against per-prompt
    eval_seg is at least 0.95 (the bar of tests/test_prompts_gpu.py), for each side's own top-1 and for eval_seg's top-1
    query in both."""
    from psalm_b200.psalm import PSALM
    cfg = PsalmConfig()
    sd = synth.synth_state_dict(cfg, seed=2)
    m = PSALM(sd, cfg, torch.bfloat16, "cuda", "region", use_cuda_graph=True)
    del sd
    inp, info, prompts, infos = _scene(1024, 480, 640, (1, 3, 7), seed=23)
    want = _per_prompt(m, inp, prompts, infos, 8)
    torch.manual_seed(8)
    got = _snap(m.open_image(inp["images"], infos[0]).eval_seg(prompts))

    def iou(a, b):
        a, b = a > 0.5, b > 0.5
        return float((a & b).sum()) / max(float((a | b).sum()), 1.0)
    measured = []
    for (s, pm), (ws, wm) in zip(got, want):
        for j in range(s.shape[1]):
            top_s, top_r = int(s[:, j].argmax()), int(ws[:, j].argmax())
            measured.append(dict(same_top1=top_s == top_r, top1_iou=round(iou(pm[top_s], wm[top_r]), 4),
                                 same_query_iou=round(iou(pm[top_r], wm[top_r]), 4), area=int((wm[top_r] > 0.5).sum())))
    print("bf16 full-size session vs eval_seg per region:", measured)
    for d in measured:
        assert d["top1_iou"] >= 0.95 and d["same_query_iou"] >= 0.95, d


def test_graph_sessions_lanes_staleness_and_rle():
    from psalm_b200 import rle
    from psalm_b200.psalm import PSALM
    sd = synth.synth_state_dict(SMALL, seed=9)
    eager = PSALM(sd, SMALL, torch.bfloat16, "cuda", "region")
    graphed = PSALM(sd, SMALL, torch.bfloat16, "cuda", "region", use_cuda_graph=True)
    scenes = {s: _scene(192, 150, 120, (2, 3), seed=s) for s in (31, 32)}

    def run(m, s, lane=0, **kw):
        inp, _, prompts, infos = scenes[s]
        torch.manual_seed(s)
        return m.open_image(inp["images"], infos[0], lane=lane).eval_seg(prompts, **kw)
    want = {s: _snap(run(eager, s)) for s in scenes}
    for _ in range(2):
        sessions = {}
        for lane, s in enumerate(scenes):
            inp, _, prompts, infos = scenes[s]
            sessions[s] = graphed.open_image(inp["images"], infos[0], lane=lane)
        for s, sess in sessions.items():
            torch.manual_seed(s)
            for (a, am), (b, bm) in zip(_snap(sess.eval_seg(scenes[s][2])), want[s]):
                assert torch.allclose(a, b, rtol=1e-5, atol=1e-7) and torch.equal(am, bm)
    stale = sessions[31]
    inp, _, prompts, infos = scenes[31]
    graphed.open_image(inp["images"], infos[0], lane=0)
    with pytest.raises(RuntimeError, match="stale"):
        stale.eval_seg(prompts)
    res = run(graphed, 32, lane=0, mask_format="rle")
    for r, (ws, _) in zip(res, want[32]):
        inst = r["instances"]
        assert torch.allclose(inst.scores.float(), ws, rtol=1e-5, atol=1e-7)
        assert torch.equal(rle.decode(inst.pred_masks_rle).bool(), inst.pred_masks.bool())


def test_raster_kernel_has_no_spills():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not shutil.which(nvcc):
        pytest.skip("nvcc not found")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-I", os.path.join(root, "include"), "-c", os.path.join(root, "psalm_b200", "csrc", "vos.cu"),
                          "-o", os.devnull], capture_output=True, text=True, check=True).stderr
    lines = out.splitlines()
    for name in ("vp_pack_kernel", "vp_raster_kernel"):
        i = next(i for i, ln in enumerate(lines) if "Function properties" in ln and name in ln)
        assert "0 bytes spill stores, 0 bytes spill loads" in lines[i + 1], lines[i + 1]
