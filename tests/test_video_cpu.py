"""Video sessions (PSALMForDAVISEval.open_video / VideoSession.step): the host side of the DAVIS loop on the device, with
the CUDA entry points emulated (tests/emu.py plus the emulations of csrc/vos.cu below), against the reference's loop
restated in oracle/davis_loop.py."""
import copy

import numpy as np
import pytest
import torch

import emu
from oracle import davis_loop as D
from psalm_b200 import synth
from psalm_b200.image_processor import nearest_pad_tables, pil_nearest_index
from psalm_b200.layout import PhiConfig, PsalmConfig
from psalm_b200.region import draw_point_indices, region_inputs, sample_region_points
from psalm_b200.structures import BitMasks, Instances

SMALL = PsalmConfig(phi=PhiConfig(hidden=256, layers=2, heads=4, inter=1024))


# ---- emulations of csrc/vos.cu ----------------------------------------------------------------------------------------
def pack_bits(m):
    """bool [M,Hp,Wp] -> int32 words [M,Hp,ceil(Wp/32)], bit x % 32 of word x // 32."""
    M, Hp, Wp = m.shape
    W32 = (Wp + 31) // 32
    x = torch.zeros(M, Hp, W32 * 32, dtype=torch.int64)
    x[..., :Wp] = m.long()
    words = (x.view(M, Hp, W32, 32) << torch.arange(32)).sum(-1)
    return torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32)


def unpack_bits(bits, Wp):
    b = ((bits.long() & 0xFFFFFFFF).unsqueeze(-1) >> torch.arange(32)) & 1
    return b.view(bits.shape[0], bits.shape[1], -1)[..., :Wp].bool()


def vos_pick(region_logits, stats):
    ms = stats[:, 1] / (stats[:, 0] + 1e-6)
    s = torch.sigmoid(region_logits.float()) * ms[None]
    K, Q = s.shape
    pick, score = torch.zeros(K, dtype=torch.int32), torch.zeros(K)
    taken, p, ps = [], 0, 0.0
    for k in range(K):
        for q in sorted(range(Q), key=lambda q: (-float(s[k, q]), q))[:10]:
            if q not in taken:
                taken.append(q)
                p, ps = q, float(s[k, q])
                break
        pick[k], score[k] = p, ps
    return pick, score


def vos_fuse(masks, src_row, src_col, bits, row_prefix, count, fill=None, labels=None, area=None, inter=None):
    on = masks.cpu() != 0
    K, H, W = on.shape
    r, c = src_row.cpu().long(), src_col.cpu().long()
    kept = on[:, r.clamp(min=0)][:, :, c.clamp(min=0)] & (r >= 0)[None, :, None] & (c >= 0)[None, None, :]
    bits.copy_(pack_bits(kept))
    rc = kept.sum(-1).int()
    row_prefix.zero_()
    row_prefix[:, 1:] = rc.cumsum(1)
    count.copy_(rc.sum(1))
    if labels is not None:
        lab = torch.zeros(H, W, dtype=torch.uint8)
        for k in range(K):
            lab[on[k]] = int(fill[k])
        labels.copy_(lab)
        f = on.view(K, -1).double()
        it = (f @ f.t()).int()
        inter.copy_(it)
        area.copy_(it.diagonal())


def region_points_gather(bits, row_prefix, sel, mask_of_region, Hp, Wp):
    m = unpack_bits(bits.cpu(), Wp)
    wh = torch.tensor([Hp, Wp])[None]
    return torch.stack([m[int(mask_of_region[r])].nonzero()[sel[r].long()] / wh for r in range(sel.shape[0])]).float()


def _install(monkeypatch):
    from psalm_b200 import kernels
    emu.install(monkeypatch)
    for name in ("vos_pick", "vos_fuse", "region_points_gather"):
        monkeypatch.setattr(kernels, name, globals()[name])
    monkeypatch.setattr(kernels, "postproc_fused", emu.postproc_fused)
    monkeypatch.setattr(kernels, "postproc_crop_supported", emu.postproc_crop_supported)


def _emu_model(monkeypatch, sd, use_cuda_graph=False):
    from psalm_b200.psalm import PSALMForDAVISEval
    _install(monkeypatch)

    class _EmuDAVIS(PSALMForDAVISEval):
        @staticmethod
        def _check_runtime(device):   # tests only: host-logic check with emulated kernels
            pass
    return _EmuDAVIS(sd, SMALL, torch.float32, "cpu", "region", use_cuda_graph=use_cuda_graph)


# ---- sample points ------------------------------------------------------------------------------------------------------
def test_points_from_host_drawn_indices_equal_sample_region_points():
    """n < 256 (repeats), n = 256, n > 256 (randperm), from the same generator state, bit for bit."""
    H, W = 61, 97
    m = torch.zeros(3, H, W, dtype=torch.bool)
    m[0, 3:9, 5:20] = True                     # 90 pixels
    m[1, 10:26, 30:46] = True                  # 256
    m[2, 20:60, 1:90] = True                   # 3560
    m[2, 33, 4] = False
    torch.manual_seed(123)
    ref = sample_region_points(m)
    torch.manual_seed(123)
    sel = draw_point_indices(m.flatten(1).sum(1).tolist())
    rp = torch.zeros(3, H + 1, dtype=torch.int32)
    rp[:, 1:] = m.sum(-1).cumsum(1)
    got = region_points_gather(pack_bits(m), rp, sel, torch.arange(3, dtype=torch.int32), H, W)
    assert got.dtype == ref.dtype and torch.equal(got, ref)


def test_empty_mask_raises_like_sample_region_points():
    m = torch.zeros(2, 8, 8, dtype=torch.bool)
    m[0, 1, 1] = True
    with pytest.raises(ValueError, match="empty region mask"):
        sample_region_points(m)
    with pytest.raises(ValueError, match="empty region mask"):
        draw_point_indices([1, 0])


# ---- nearest resize + padding ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("size", [(480, 854, 576, 1024, 1024, 1024), (480, 854, 1024, 1821, 1024, 1821),
                                  (7, 13, 5, 29, 8, 32), (333, 517, 1000, 771, 1000, 800), (90, 120, 144, 192, 192, 192)])
def test_nearest_resize_and_pad_equal_pillow(size):
    Image = pytest.importorskip("PIL.Image")
    H, W, oh, ow, Hp, Wp = size
    rng = np.random.default_rng(H * W)
    mask = (rng.random((H, W)) > 0.6).astype(np.uint8)
    ref = np.zeros((Hp, Wp), np.uint8)
    ref[:oh, :ow] = np.asarray(Image.fromarray(mask).resize((ow, oh), Image.NEAREST))
    rows, cols = nearest_pad_tables(H, W, (oh, ow), (Hp, Wp))
    bits, rp, cnt = torch.zeros(1, Hp, (Wp + 31) // 32, dtype=torch.int32), torch.zeros(1, Hp + 1, dtype=torch.int32), \
        torch.zeros(1, dtype=torch.int32)
    vos_fuse(torch.from_numpy(mask).float()[None], rows, cols, bits, rp, cnt)
    got = unpack_bits(bits, Wp)[0].numpy()
    assert np.array_equal(got, ref.astype(bool))
    assert int(cnt[0]) == int(ref.sum()) and np.array_equal(rp[0, 1:].numpy(), ref.sum(1).cumsum())
    assert np.array_equal(D.apply_segmentation(mask, (oh, ow), (Hp, Wp)), ref)
    row_ref = np.asarray(Image.fromarray(np.arange(H, dtype=np.int32)[:, None].repeat(W, 1)).resize((ow, oh), Image.NEAREST))
    assert np.array_equal(pil_nearest_index(H, oh), row_ref[:, 0])


# ---- pick, fuse, memory decision -------------------------------------------------------------------------------------------
def _pick_case(kind):
    g = torch.Generator().manual_seed(7)
    Q, K = 100, 4
    logits = torch.randn(K, Q, generator=g) * 3
    stats = torch.zeros(Q, 5)
    stats[:, 0] = torch.randint(1, 500, (Q,), generator=g).float()
    stats[:, 1] = stats[:, 0] * torch.rand(Q, generator=g)
    if kind == "ties":                # equal scores across queries: the lower query index goes first
        logits[:, 10:20] = 2.5
        stats[10:20, 0], stats[10:20, 1] = 100.0, 75.0
    elif kind == "all_taken":         # four objects with the same top 10 ... and a fifth: its 10 candidates are all taken
        logits = torch.randn(1, Q, generator=g).repeat(12, 1)
        logits[:, :10] = torch.linspace(9, 5, 10)
        stats[:10, 0], stats[:10, 1] = 10.0, 9.0
    return logits, stats


@pytest.mark.parametrize("kind", ["random", "ties", "all_taken"])
def test_pick_equals_the_reference_loop(kind):
    logits, stats = _pick_case(kind)
    pick, score = vos_pick(logits, stats)
    ms = stats[:, 1] / (stats[:, 0] + 1e-6)
    table = (torch.sigmoid(logits) * ms[None]).t().numpy()        # output['instances'].scores [Q,K]
    rp, rs = D.pick_objects(table)
    assert np.array_equal(pick.numpy(), rp) and np.array_equal(score.numpy(), rs)
    if kind == "all_taken":           # objects 10 and 11 keep object 9's pick (the reference's loop variables)
        assert rp[10] == rp[9] and rp[11] == rp[9] and len(set(rp[:10].tolist())) == 10


def _masks_case(kind, H=40, W=50):
    m = np.zeros((3, H, W), np.uint8)
    m[0, 0:10, 0:10] = 1
    if kind in ("above", "below"):    # two 100-pixel masks sharing 58 (IoU 58 / 142 = 0.408) or 57 pixels (0.399)
        shared = 58 if kind == "above" else 57
        a, b = np.divmod(np.arange(shared), 10), np.divmod(np.arange(100 - shared), 10)
        m[1, a[0], a[1]] = 1
        m[1, 30 + b[0], b[1]] = 1
    m[2, 20:30, 20:35] = 1
    if kind == "two_empty":           # masks 1 and 2 empty: 0 / 0 is NaN and fails no comparison
        m[2] = 0
    return m


@pytest.mark.parametrize("kind", ["above", "below", "two_empty"])
def test_fuse_and_memory_decision_equal_the_reference_loop(kind):
    from psalm_b200.psalm import memory_check
    m = _masks_case(kind)
    K, H, W = m.shape
    fills = torch.tensor([3, 200, 7], dtype=torch.int32)
    labels, area, inter = torch.zeros(H, W, dtype=torch.uint8), torch.zeros(K, dtype=torch.int32), torch.zeros(K, K, dtype=torch.int32)
    rows, cols = nearest_pad_tables(H, W, (H, W), (H, W))
    vos_fuse(torch.from_numpy(m).float(), rows, cols, torch.zeros(K, H, 2, dtype=torch.int32),
             torch.zeros(K, H + 1, dtype=torch.int32), torch.zeros(K, dtype=torch.int32), fills, labels, area, inter)
    assert np.array_equal(labels.numpy(), D.fuse_davis_mask(list(m), fills.tolist()))
    assert memory_check(area.numpy(), inter.numpy()) == D.memory_correct(list(m))
    assert D.memory_correct(list(m)) == (kind != "above")


# ---- the session against eval_video + the reference loop -----------------------------------------------------------------
H = W = 192
OUT_HW, RESIZED = (90, 120), (144, 192)


def _frame(seed, K):
    inp = synth.synth_inputs(batch=1, height=H, width=W, task="region", seed=seed, n_regions=K)
    pad = torch.ones(H, W, dtype=torch.bool)
    pad[:RESIZED[0], :RESIZED[1]] = False
    info = dict(padding_mask=pad, height=OUT_HW[0], width=OUT_HW[1])
    return inp, info


def _clip(K, n_frames=5):
    first, info = _frame(40, K)
    inst = first["seg_info"][0]["instances"]
    vp_masks = inst.region_masks.tensor.clone()
    fills = torch.arange(1, K + 1, dtype=torch.int64) * 37
    frames = []
    for t in range(n_frames):
        inp = first if t == 0 else _frame(40 + t, K)[0]
        frames.append(dict(images=inp["images"], seg_info=[dict(info)]))
    return first, vp_masks, fills, frames


def _eval_video_cpu(m, prompt, images, info, vp_images, vp_masks, fills):
    """eval_seg_async's region flow for one frame (plan, points drawn from vp_region_masks, forward, post-processing)."""
    inst = Instances(OUT_HW)
    inst.vp_region_masks = BitMasks(torch.as_tensor(vp_masks))
    inst.vp_fill_number = torch.as_tensor(fills)
    inst.gt_masks = torch.zeros(len(fills), H, W)
    si = [dict(info, instances=inst)]
    plan = copy.copy(m._cached_plan(prompt["input_ids"], prompt["attention_mask"], (H, W), None, None, None, None, None))
    pts, img, _ = region_inputs(si, None, "vp_region_masks")
    plan.region_points, plan.region_image, plan.vp_images = pts, img, vp_images
    out = m.forward_core(images, plan)
    return m.post_process(out, (H, W), si)[0]


@pytest.mark.parametrize("K,with_memory", [(1, True), (3, True), (3, False)])
def test_session_equals_eval_video_and_the_reference_loop(monkeypatch, K, with_memory):
    sd = synth.synth_state_dict(SMALL, seed=5)
    m = _emu_model(monkeypatch, sd)
    first, vp_masks, fills, frames = _clip(K)
    loop = D.DavisLoop(first["images"], vp_masks.numpy(), fills.tolist(), with_memory)
    torch.manual_seed(99)
    ref = []
    for f in frames:
        vp_img, vp_m, vp_f = loop.inputs()
        res = _eval_video_cpu(m, first, f["images"], f["seg_info"][0], vp_img, vp_m, vp_f)
        ref.append(loop.update(res, vp_f, f["images"], RESIZED, (H, W)))
    torch.manual_seed(99)
    vinst = Instances((H, W))
    vinst.vp_region_masks = BitMasks(vp_masks)
    vinst.vp_fill_number = fills
    vinfo = [dict(frames[0]["seg_info"][0], instances=vinst)]
    vid = m.open_video(first["images"], vinfo, first["input_ids"], first["attention_mask"], with_memory=with_memory)
    updates = 0
    for t, f in enumerate(frames):
        got = vid.step(f["images"], f["seg_info"])
        r = ref[t]
        assert np.array_equal(got.query_index.numpy(), r["pick"]), t
        assert np.array_equal(got.scores.numpy(), r["score"]), t
        assert np.array_equal(got.labels.numpy(), r["labels"]), t
        assert got.memory_updated == r["memory_updated"], t
        assert torch.equal(got.fill_numbers, fills)
        updates += got.memory_updated
    if K == 1 and with_memory:        # one object: the IoU check has no pair and always passes
        assert updates == len(frames)


def test_step_async_submits_the_next_frame_before_the_previous_is_read(monkeypatch):
    sd = synth.synth_state_dict(SMALL, seed=5)
    m = _emu_model(monkeypatch, sd)
    first, vp_masks, fills, frames = _clip(1, 3)
    vinst = Instances((H, W))
    vinst.vp_region_masks = BitMasks(vp_masks)
    vinst.vp_fill_number = fills
    vinfo = [dict(frames[0]["seg_info"][0], instances=vinst)]
    torch.manual_seed(5)
    vid = m.open_video(first["images"], vinfo, first["input_ids"], first["attention_mask"])
    a = [vid.step(f["images"], f["seg_info"]) for f in frames]
    torch.manual_seed(5)
    vid = m.open_video(first["images"], vinfo, first["input_ids"], first["attention_mask"])
    p0 = vid.step_async(frames[0]["images"], frames[0]["seg_info"])
    p1 = vid.step_async(frames[1]["images"], frames[1]["seg_info"])
    b0, b1 = p0.result(), p1.result()
    b2 = vid.step(frames[2]["images"], frames[2]["seg_info"])
    for x, y in zip(a, (b0, b1, b2)):
        assert torch.equal(x.labels, y.labels) and torch.equal(x.query_index, y.query_index)
        assert x.memory_updated == y.memory_updated


# ---- surface -------------------------------------------------------------------------------------------------------------
def _open(m, K=3, fills=None):
    first, vp_masks, f, frames = _clip(K, 1)
    vinst = Instances((H, W))
    vinst.vp_region_masks = BitMasks(vp_masks)
    vinst.vp_fill_number = f if fills is None else fills
    vinfo = [dict(frames[0]["seg_info"][0], instances=vinst)]
    return m.open_video(first["images"], vinfo, first["input_ids"], first["attention_mask"]), frames


def test_stale_session_raises(monkeypatch):
    m = _emu_model(monkeypatch, synth.synth_state_dict(SMALL, seed=5))
    vid, frames = _open(m)
    _open(m)
    with pytest.raises(RuntimeError, match="stale VideoSession"):
        vid.step(frames[0]["images"], frames[0]["seg_info"])
    vid, frames = _open(m)
    m.open_image(frames[0]["images"], frames[0]["seg_info"])
    with pytest.raises(RuntimeError, match="stale VideoSession"):
        vid.step(frames[0]["images"], frames[0]["seg_info"])


def test_more_than_32_objects_raise(monkeypatch):
    m = _emu_model(monkeypatch, synth.synth_state_dict(SMALL, seed=5))
    first, _, _, frames = _clip(3, 1)
    vinst = Instances((H, W))
    vinst.vp_region_masks = BitMasks(torch.ones(33, H, W, dtype=torch.bool))
    vinst.vp_fill_number = torch.arange(1, 34)
    vinfo = [dict(frames[0]["seg_info"][0], instances=vinst)]
    with pytest.raises(ValueError, match="1..32 objects"):
        m.open_video(first["images"], vinfo, first["input_ids"], first["attention_mask"])


def test_fill_number_above_255_raises(monkeypatch):
    m = _emu_model(monkeypatch, synth.synth_state_dict(SMALL, seed=5))
    with pytest.raises(ValueError, match="fill numbers"):
        _open(m, K=2, fills=torch.tensor([1, 256]))
    with pytest.raises(ValueError, match="fill numbers"):
        _open(m, K=2, fills=torch.tensor([0, 3]))
