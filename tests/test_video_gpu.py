"""Video sessions on the GPU: the kernels of csrc/vos.cu against their torch / numpy restatements, and
PSALMForDAVISEval.open_video + VideoSession.step against eval_video + the reference's DAVIS loop (oracle/davis_loop.py)."""
import numpy as np
import pytest
import torch

from oracle import davis_loop as D
from psalm_b200 import synth
from psalm_b200.image_processor import nearest_pad_tables
from psalm_b200.layout import PhiConfig, PsalmConfig
from psalm_b200.structures import BitMasks, Instances
from test_video_cpu import pack_bits, region_points_gather, vos_fuse, vos_pick

pytestmark = pytest.mark.gpu
SMALL = PsalmConfig(phi=PhiConfig(hidden=256, layers=2, heads=4, inter=1024))


# ---- kernels -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("K", [1, 5, 32])
def test_vos_pick_kernel(dt, K):
    from psalm_b200 import kernels
    g = torch.Generator().manual_seed(K)
    Q = 100
    logits = (torch.randn(K, Q, generator=g) * 3).to(dt)
    logits[:, 40:50] = 4.0                      # exact ties, and (K > 10) objects whose top 10 are all taken
    stats = torch.zeros(Q, 5)
    stats[:, 0] = torch.randint(1, 5000, (Q,), generator=g).float()
    stats[:, 1] = stats[:, 0] * torch.rand(Q, generator=g)
    stats[40:50, 0], stats[40:50, 1] = 64.0, 48.0
    ref_p, ref_s = vos_pick(logits, stats)
    p, s = kernels.vos_pick(logits.cuda(), stats.cuda())
    assert torch.equal(p.cpu(), ref_p)
    assert torch.allclose(s.cpu(), ref_s, rtol=1e-6, atol=0)
    table = (torch.sigmoid(logits.float()) * (stats[:, 1] / (stats[:, 0] + 1e-6))[None]).t().numpy()
    assert np.array_equal(p.cpu().numpy(), D.pick_objects(table)[0])


@pytest.mark.parametrize("geom", [(480, 854, 576, 1024, 1024, 1024), (90, 120, 144, 192, 192, 192), (37, 53, 60, 61, 64, 96)])
@pytest.mark.parametrize("K", [1, 3, 32])
def test_vos_fuse_kernel(geom, K):
    from psalm_b200 import kernels
    H, W, oh, ow, Hp, Wp = geom
    g = torch.Generator().manual_seed(K + H)
    masks = torch.zeros(K, H, W)
    for k in range(K):                          # overlapping rectangles, one empty mask when K > 1
        if k == 1:
            continue
        y0, x0 = int(torch.randint(0, H // 2, (1,), generator=g)), int(torch.randint(0, W // 2, (1,), generator=g))
        masks[k, y0:y0 + H // 2, x0:x0 + W // 3] = 1.0
    masks[0] = (torch.rand(H, W, generator=g) > 0.5).float()
    rows, cols = nearest_pad_tables(H, W, (oh, ow), (Hp, Wp))
    fill = torch.randint(1, 256, (K,), generator=g).to(torch.int32)
    W32 = (Wp + 31) // 32
    ref = [torch.zeros(K, Hp, W32, dtype=torch.int32), torch.zeros(K, Hp + 1, dtype=torch.int32), torch.zeros(K, dtype=torch.int32),
           fill, torch.zeros(H, W, dtype=torch.uint8), torch.zeros(K, dtype=torch.int32), torch.zeros(K, K, dtype=torch.int32)]
    vos_fuse(masks, rows, cols, *ref[:3], fill=ref[3], labels=ref[4], area=ref[5], inter=ref[6])
    got = [t.cuda() for t in ref]
    for t in got[:3] + got[4:]:
        t.fill_(-1 if t.dtype == torch.int32 else 0)
    kernels.vos_fuse(masks.cuda(), rows.cuda(), cols.cuda(), *got[:3], fill=got[3], labels=got[4], area=got[5], inter=got[6])
    for a, b in zip(got, ref):
        assert torch.equal(a.cpu(), b)
    labels = D.fuse_davis_mask(list(masks.numpy().astype(np.uint8)), fill.tolist())
    assert np.array_equal(got[4].cpu().numpy(), labels)


def test_region_points_gather_kernel():
    from psalm_b200 import kernels
    from psalm_b200.region import draw_point_indices, sample_region_points
    Hp, Wp = 1024, 1000
    g = torch.Generator().manual_seed(3)
    m = torch.zeros(4, Hp, Wp, dtype=torch.bool)
    m[0, 500, 7] = True                                     # one pixel
    m[1, 100:116, 200:216] = True                           # 256
    m[2] = torch.rand(Hp, Wp, generator=g) > 0.7            # ~300k
    m[3, 900:1024, 990:1000] = True
    torch.manual_seed(11)
    ref = sample_region_points(m)
    torch.manual_seed(11)
    sel = draw_point_indices(m.flatten(1).sum(1).tolist())
    rp = torch.zeros(4, Hp + 1, dtype=torch.int32)
    rp[:, 1:] = m.sum(-1).cumsum(1)
    got = kernels.region_points_gather(pack_bits(m).cuda(), rp.cuda(), sel.cuda(), torch.arange(4, dtype=torch.int32).cuda(),
                                       Hp, Wp)
    assert torch.equal(got.cpu(), ref)
    assert torch.equal(region_points_gather(pack_bits(m), rp, sel, torch.arange(4, dtype=torch.int32), Hp, Wp), ref)


# ---- the session against eval_video + the reference loop -----------------------------------------------------------------
def _clip(K, n_frames, S, out_hw, resized):
    first = synth.synth_inputs(batch=1, height=S, width=S, task="region", seed=40, n_regions=K)
    pad = torch.ones(S, S, dtype=torch.bool)
    pad[:resized[0], :resized[1]] = False
    info = dict(padding_mask=pad, height=out_hw[0], width=out_hw[1])
    frames = [first["images"]] + [torch.randn(1, 3, S, S, generator=torch.Generator().manual_seed(50 + t))
                                  for t in range(1, n_frames)]
    return first, first["seg_info"][0]["instances"].region_masks.tensor.clone(), \
        torch.arange(1, K + 1, dtype=torch.int64) * 40, frames, info


def _loop(m, first, vp_masks, fills, frames, info, S, resized, with_memory):
    loop = D.DavisLoop(first["images"], vp_masks.numpy(), fills.tolist(), with_memory)
    out = []
    for img in frames:
        vp_img, vp_m, vp_f = loop.inputs()
        inst = Instances((info["height"], info["width"]))
        inst.vp_region_masks = BitMasks(torch.as_tensor(vp_m))
        inst.vp_fill_number = torch.as_tensor(vp_f)
        inst.gt_masks = torch.zeros(len(vp_f), S, S)
        res = m.eval_video(input_ids=first["input_ids"], attention_mask=first["attention_mask"], images=img,
                           vp_images=vp_img, seg_info=[dict(info, instances=inst)])[0]
        r = loop.update(res, vp_f, img, resized, (S, S))
        sc = np.sort(res["instances"].scores.float().cpu().numpy(), axis=0)
        r["margin"] = float((sc[-1] - sc[-2]).min())            # top-2 score margin, smallest over the objects
        out.append(r)
    return out


def _session(m, first, vp_masks, fills, frames, info, with_memory):
    inst = Instances((info["height"], info["width"]))
    inst.vp_region_masks = BitMasks(vp_masks)
    inst.vp_fill_number = fills
    vid = m.open_video(first["images"], [dict(info, instances=inst)], first["input_ids"], first["attention_mask"],
                       with_memory=with_memory)
    out = []
    for img in frames:
        f = vid.step(img, [info])
        out.append(dict(labels=f.labels.cpu().numpy(), pick=f.query_index.numpy(), memory_updated=f.memory_updated))
    return out


def _label_iou(a, b, fills):
    return [float(np.logical_and(a == f, b == f).sum()) / max(1, np.logical_or(a == f, b == f).sum()) for f in fills]


@pytest.mark.parametrize("S,out_hw,resized,K,n_frames", [(192, (90, 120), (144, 192), 3, 5),
                                                         (1024, (480, 854), (576, 1024), 3, 6)], ids=["192", "1024"])
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_session_fp32_equals_eval_video_loop(S, out_hw, resized, K, n_frames, graph):
    """fp32: the region heads of eval_video run the exact torch path, the session the fused kernel; a mask logit within
    rounding of 0 may threshold differently, so the labels are compared pixel for pixel with that slack reported."""
    from psalm_b200.psalm import PSALMForDAVISEval
    sd = synth.synth_state_dict(SMALL, seed=5)
    first, vp_masks, fills, frames, info = _clip(K, n_frames, S, out_hw, resized)
    ref_m = PSALMForDAVISEval(sd, SMALL, torch.float32, "cuda", "region")
    m = PSALMForDAVISEval(sd, SMALL, torch.float32, "cuda", "region", use_cuda_graph=graph)
    for with_memory in (True, False):
        torch.manual_seed(99)
        ref = _loop(ref_m, first, vp_masks, fills, frames, info, S, resized, with_memory)
        torch.manual_seed(99)
        got = _session(m, first, vp_masks, fills, frames, info, with_memory)
        for t, (a, r) in enumerate(zip(got, ref)):
            diff = int((a["labels"] != r["labels"]).sum())
            print("fp32 S=%d graph=%s memory=%s frame %d: picks %s / %s, memory %s / %s, %d label pixels differ, margin %.3e"
                  % (S, graph, with_memory, t, a["pick"], r["pick"], a["memory_updated"], r["memory_updated"], diff,
                     r["margin"]))
            assert np.array_equal(a["pick"], r["pick"]), t
            assert a["memory_updated"] == r["memory_updated"], t
            assert diff <= 1e-4 * a["labels"].size, t


def test_session_bf16_full_size_tracks_the_bf16_loop():
    """bf16 graphs at 1024^2 with 480x854 outputs: per-object IoU of the label maps >= 0.95 while both sides kept the same
    memory; picks compared where the loop's top-2 margin is clear of bf16 noise (margins printed)."""
    from psalm_b200.psalm import PSALMForDAVISEval
    S, out_hw, resized, K = 1024, (480, 854), (576, 1024), 3
    sd = synth.synth_state_dict(SMALL, seed=5)
    first, vp_masks, fills, frames, info = _clip(K, 6, S, out_hw, resized)
    ref_m = PSALMForDAVISEval(sd, SMALL, torch.bfloat16, "cuda", "region")
    m = PSALMForDAVISEval(sd, SMALL, torch.bfloat16, "cuda", "region", use_cuda_graph=True)
    torch.manual_seed(7)
    ref = _loop(ref_m, first, vp_masks, fills, frames, info, S, resized, True)
    torch.manual_seed(7)
    got = _session(m, first, vp_masks, fills, frames, info, True)
    for t, (a, r) in enumerate(zip(got, ref)):
        ious = _label_iou(a["labels"], r["labels"], fills.tolist())
        print("bf16 frame %d: picks %s / %s, memory %s / %s, label IoU %s, loop top-2 margin %.3e"
              % (t, a["pick"], r["pick"], a["memory_updated"], r["memory_updated"], ["%.4f" % v for v in ious], r["margin"]))
        if np.array_equal(a["pick"], r["pick"]):
            assert min(ious) >= 0.95, t
        else:
            assert r["margin"] < 1e-2, t          # a different pick only where the loop's own choice is a near tie
        if a["memory_updated"] != r["memory_updated"] or not np.array_equal(a["pick"], r["pick"]):
            break                                 # the two loops now pool from different memories
