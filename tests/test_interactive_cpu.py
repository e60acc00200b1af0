"""Interactive segmentation against one image (ImageSession.eval_seg with `visual_prompts`): the region-mask oracle
against the fixture the unmodified reference made, the disk test, the prompt cut of <region> prompts, and the session's
host orchestration with the CUDA entry points emulated (tests/emu.py plus the emulations of csrc/vos.cu below)."""
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import emu
from oracle import visual_prompt as VP
from psalm_b200 import sequence as SEQ
from psalm_b200 import synth
from psalm_b200.image_processor import nearest_pad_tables, resize_shortest_edge_shape
from psalm_b200.layout import PhiConfig, PsalmConfig
from psalm_b200.region import VISUAL_PROMPT_RADIUS, _rle_has_foreground, sample_region_points

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


def visual_prompt_raster(src, radius, src_row, src_col):
    """Seeds (== 1 with a radius, != 0 without) convolved with the integer disk, read through the NEAREST tables."""
    src = src.cpu()
    K = src.shape[0]
    r_, c_ = src_row.cpu().long(), src_col.cpu().long()
    kept = []
    for k in range(K):
        r = int(radius[k])
        seeds = (src[k] == 1) if r > 0 else (src[k] != 0)
        if r > 0:
            d = torch.arange(-r, r + 1)
            disk = (d[:, None] ** 2 + d[None, :] ** 2 <= r * r).double()
            seeds = F.conv2d(seeds.double()[None, None], disk[None, None], padding=r)[0, 0] > 0
        kept.append(seeds[r_.clamp(min=0)][:, c_.clamp(min=0)] & (r_ >= 0)[:, None] & (c_ >= 0)[None, :])
    kept = torch.stack(kept)
    rc = kept.sum(-1).int()
    row_prefix = torch.zeros(K, kept.shape[1] + 1, dtype=torch.int32)
    row_prefix[:, 1:] = rc.cumsum(1)
    return pack_bits(kept), row_prefix, rc.sum(1).int()


def region_points_gather(bits, row_prefix, sel, mask_of_region, Hp, Wp):
    m = unpack_bits(bits.cpu(), Wp)
    wh = torch.tensor([Hp, Wp])[None]
    return torch.stack([m[int(mask_of_region[r])].nonzero()[sel[r].long()] / wh for r in range(sel.shape[0])]).float()


def prefix_causal_attention(qkv, prefix_k, prefix_v, P, key_valid, B, T, nh, hd):
    q, k, v = (qkv[:, :, i].permute(0, 2, 1, 3).float() for i in range(3))
    pk = prefix_k[:, :P].float().unsqueeze(0).expand(B, -1, -1, -1)
    pv = prefix_v[:, :P].float().unsqueeze(0).expand(B, -1, -1, -1)
    kk, vv = torch.cat([pk, k], 2), torch.cat([pv, v], 2)
    s = (q @ kk.transpose(-2, -1)) * hd ** -0.5
    allowed = torch.cat([torch.ones(T, P, dtype=torch.bool), torch.tril(torch.ones(T, T, dtype=torch.bool))], 1)[None, None]
    if key_valid is not None:
        kv = torch.cat([torch.ones(B, P, dtype=torch.bool), key_valid.bool()], 1)
        allowed = allowed & kv[:, None, None, :]
    p = torch.nan_to_num(s.masked_fill(~allowed, float("-inf")).softmax(-1))
    return (p @ vv).permute(0, 2, 1, 3).reshape(B, T, nh * hd).to(qkv.dtype)


def mask_logits(mask_embed, feats, out_dtype=None):
    return emu.mask_logits(mask_embed, feats, out_dtype)


def mask_bits(mask_embed, feats):
    return emu.attn_mask_bits(mask_logits(mask_embed, feats, torch.float32))


def _install(monkeypatch):
    from psalm_b200 import kernels
    emu.install(monkeypatch)
    for name in ("visual_prompt_raster", "region_points_gather", "prefix_causal_attention", "mask_logits", "mask_bits"):
        monkeypatch.setattr(kernels, name, globals()[name])


def _emu_model(monkeypatch, sd, task="region"):
    from psalm_b200.psalm import PSALM
    _install(monkeypatch)

    class _EmuPSALM(PSALM):
        @staticmethod
        def _check_runtime(device):   # tests only: host-logic check with emulated kernels
            pass
    return _EmuPSALM(sd, SMALL, torch.float32, "cpu", task)


def rle_string(counts):
    """rleToString (the COCO compressed form) of run lengths `counts`."""
    out = []
    for i, x in enumerate(counts):
        if i > 2:
            x -= counts[i - 2]
        more = True
        while more:
            c = x & 0x1f
            x >>= 5
            more = (x != -1) if c & 0x10 else (x != 0)
            if more:
                c |= 0x20
            out.append(chr(c + 48))
    return "".join(out)


# ---- the region-mask oracle and the disk test ------------------------------------------------------------------------
def _golden_cases(golden):
    g = golden("visual_prompts.npz")
    for i in range(int(g["n"])):
        H, W = (int(v) for v in g["shape_%d" % i])
        src = np.unpackbits(g["src_%d" % i], axis=1, count=W)
        out = np.unpackbits(g["out_%d" % i], axis=1, count=W)
        yield str(g["kind_%d" % i]), src, out


def test_oracle_equals_the_reference_golden(golden):
    kinds = set()
    for kind, src, out in _golden_cases(golden):
        kinds.add(kind)
        r = VP.RADIUS[kind]
        got = VP.dilate(src, r) if r else src
        assert np.array_equal(got, out), kind
        if r and src.size <= 480 * 640:                     # the literal per-seed disks too, at the smaller sizes
            assert np.array_equal(VP.enhance_with_circles(src, r), out), kind
    assert kinds == set(VISUAL_PROMPT_RADIUS)


@pytest.mark.parametrize("r", [5, 10])
def test_integer_disk_test_equals_the_float64_sqrt(r):
    d2 = np.arange(0, 2 * r * r + 1)
    assert np.array_equal(d2 <= r * r, np.sqrt(d2.astype(np.float64)) <= r)


def test_emulated_raster_equals_the_oracle_on_the_golden(golden):
    for kind, src, _ in _golden_cases(golden):
        H, W = src.shape
        oh, ow = resize_shortest_edge_shape(H, W, 1024, 1024)
        rows, cols = nearest_pad_tables(H, W, (oh, ow), (1024, 1024))
        bits, rp, cnt = visual_prompt_raster(torch.from_numpy(src)[None], torch.tensor([VP.RADIUS[kind]]), rows, cols)
        want = VP.region_mask(kind, src, (oh, ow), (1024, 1024))
        assert np.array_equal(unpack_bits(bits, 1024)[0].numpy(), want), kind
        assert int(cnt[0]) == int(want.sum()) and np.array_equal(rp[0, 1:].numpy(), want.sum(1).cumsum())


def test_rle_foreground_check():
    assert _rle_has_foreground(rle_string([3, 4, 5, 1, 2]))
    assert not _rle_has_foreground(rle_string([480 * 640]))
    assert not _rle_has_foreground(rle_string([10, 0, 6]))
    assert _rle_has_foreground(rle_string([0, 100000, 7]).encode())


# ---- the prompt cut ----------------------------------------------------------------------------------------------------
def _region_prompt(K, head=(11, 12, 13), mid=(14, 15)):
    ids = list(head) + [SEQ.IMAGE_TOKEN_INDEX] + list(mid)
    for j in range(K):
        ids += [SEQ.REGION_TOKEN_INDEX, 20 + j]
    ids += [30, 31, SEQ.SEG_TOKEN_INDEX, 32]
    t = torch.tensor([ids])
    return dict(input_ids=t, attention_mask=torch.ones_like(t, dtype=torch.bool))


def test_suffix_plans_of_region_prompts_are_the_rows_of_the_full_plans():
    ps = [_region_prompt(K) for K in (1, 3, 2)]
    n_img, n_q = 16, 100
    sp = SEQ.split_prompts([dict(p, visual_prompts=[None] * K) for p, K in zip(ps, (1, 3, 2))], n_img, n_q)
    s, P, Ts = sp.suffix, sp.P, sp.suffix.T
    first = int(np.nonzero(ps[0]["input_ids"][0].numpy() == SEQ.REGION_TOKEN_INDEX)[0][0])
    assert len(sp.prefix_ids) == first and s.region_counts == (1, 3, 2)
    pos = 0
    for k, p in enumerate(ps):
        full = SEQ.build_plan(p["input_ids"], p["attention_mask"], n_img, n_q)
        n = full.T - P
        assert torch.equal(full.tok_ids[0, :P], sp.tok_ids[0])
        assert torch.equal(s.tok_ids[k, :n], full.tok_ids[0, P:])
        assert torch.equal(s.seg_pos[k * n_q:(k + 1) * n_q] - k * Ts + P, full.seg_pos)
        K = full.region_counts[0]
        assert s.region_counts[k] == K
        assert torch.equal(s.region_pos[pos:pos + K] - k * Ts + P, full.region_pos)
        pos += K


def test_graph_keys_of_plans_without_regions_are_unchanged():
    from psalm_b200.psalm import _plan_key
    inp = synth.synth_inputs(batch=1, height=64, width=64, task="referring", seed=3)
    plan = SEQ.build_plan(inp["input_ids"], inp["attention_mask"], 4, 100, token_refer_id=inp["token_refer_id"],
                          refer_embedding_indices=inp["refer_embedding_indices"])
    assert _plan_key(plan) == (plan.B, plan.T, plan.n_img, plan.any_padding, None, True, None)
    a = SEQ.build_plan(_region_prompt(2)["input_ids"], None, 4, 100)
    b = SEQ.build_plan(_region_prompt(3, head=(11,))["input_ids"], None, 4, 100)
    assert a.T == b.T and _plan_key(a) != _plan_key(b) and _plan_key(a)[-1] == (2,)


# ---- the session --------------------------------------------------------------------------------------------------------
def _masks(H, W, boxes):
    m = torch.zeros(len(boxes), H, W, dtype=torch.bool)
    for j, (y0, x0, y1, x1) in enumerate(boxes):
        m[j, y0:y1, x0:x1] = True
    return m


def test_session_indices_equal_per_prompt_region_inputs(monkeypatch):
    """Two prompts (2 and 3 regions, all kinds) at 333 x 500 padded to 1024^2: the session's points equal the points of
    per-prompt sample_region_points calls on the oracle's region masks, made in prompt order from the same seed."""
    from psalm_b200.psalm import ImageSession
    _install(monkeypatch)
    H, W = 333, 500
    oh, ow = resize_shortest_edge_shape(H, W, 1024, 1024)
    scrib = torch.zeros(H, W, dtype=torch.uint8)
    scrib[0, 10:200] = 1
    scrib[:80, 499] = 1
    blob = _masks(H, W, [(200, 100, 333, 260)])[0]
    prompts = [[("point", (5, 7)), ("box", (10, 20, 120, 300))],
               [("scribble", scrib), ("mask", blob), ("point", (332, 499))]]
    sess = ImageSession(types.SimpleNamespace(device=torch.device("cpu")), 0, 1, None, (1024, 1024),
                        [dict(height=H, width=W)], [(oh, ow)])
    torch.manual_seed(31)
    bits, prefix, sel = sess._region_inputs([r for p in prompts for r in p])
    got = region_points_gather(bits, prefix, sel, torch.arange(5, dtype=torch.int32), 1024, 1024)
    torch.manual_seed(31)
    ref = []
    for p in prompts:
        masks = []
        for kind, s in p:
            src = np.zeros((H, W), np.uint8)
            if kind == "point":
                src[s] = 1
            elif kind == "box":
                src = VP.paint_box(H, W, s)
            else:
                src = s.numpy().astype(np.uint8)
            masks.append(torch.from_numpy(VP.region_mask(kind, src, (oh, ow), (1024, 1024))))
        ref.append(sample_region_points(torch.stack(masks)))
    assert torch.equal(got, torch.cat(ref))


def _region_session(monkeypatch, H=192, W=192):
    sd = synth.synth_state_dict(SMALL, seed=9)
    inp = synth.synth_inputs(batch=1, height=H, width=W, task="region", seed=10)
    m = _emu_model(monkeypatch, sd)
    return m, inp, m.open_image(inp["images"], inp["seg_info"])


def _mask_prompt(inp):
    masks = inp["seg_info"][0]["instances"].region_masks.tensor
    return dict(input_ids=inp["input_ids"], attention_mask=inp["attention_mask"],
                visual_prompts=[("mask", mk) for mk in masks])


def test_single_prompt_session_matches_region_golden(monkeypatch, golden):
    """kind="mask" prompts equal to the region masks of e2e_region_192x192_b1.npz, points drawn from the seed the fixture
    was made with: the fixture's region logits and scores at the bars of tests/test_region_gpu.py."""
    g = golden("e2e_region_192x192_b1.npz")
    m, inp, sess = _region_session(monkeypatch)
    torch.manual_seed(1234)          # oracle/gen_golden_modules.py seeds region_pooling's draws with 1234
    pend = sess.eval_seg_async([_mask_prompt(inp)])
    logits = pend.parts[0][0]["pred_region_logits"][0]
    res = pend.result()
    assert np.allclose(logits.numpy(), g["pred_region_logits_0"], rtol=1e-3, atol=2e-3)
    inst = res[0]["instances"]
    assert tuple(inst.scores.shape) == g["region_scores"].shape
    assert np.allclose(inst.scores.numpy(), g["region_scores"], rtol=1e-3, atol=1e-4)
    assert np.abs(inst.pred_masks.flatten(1).sum(1).numpy() - g["region_mask_area"]).max() <= 2
    gt = res[0]["gt"].reshape(-1)[torch.from_numpy(g["region_gt_idx"])].numpy()
    assert np.allclose(gt, g["region_gt"], atol=1e-6)


def test_session_without_gt_masks_returns_no_gt(monkeypatch):
    sd = synth.synth_state_dict(SMALL, seed=9)
    inp = synth.synth_inputs(batch=1, height=96, width=96, task="region", seed=10)
    m = _emu_model(monkeypatch, sd)
    info = {k: v for k, v in inp["seg_info"][0].items() if k != "instances"}
    sess = m.open_image(inp["images"], [info])
    res = sess.eval_seg([_mask_prompt(inp)])
    assert "gt" not in res[0] and tuple(res[0]["instances"].scores.shape) == (100, 3)


# ---- errors --------------------------------------------------------------------------------------------------------------
def _no_launch(*a, **k):
    raise AssertionError("launched")


def test_errors(monkeypatch):
    m, inp, sess = _region_session(monkeypatch, 96, 96)
    p = _mask_prompt(inp)
    bare = dict(input_ids=inp["input_ids"], attention_mask=inp["attention_mask"])
    with pytest.raises(NotImplementedError, match="region"):             # no visual_prompts: as before
        sess.eval_seg([bare])
    with pytest.raises(ValueError, match="all have or all lack visual_prompts"):
        sess.eval_seg([p, bare])
    with pytest.raises(ValueError, match="3 <region> tokens"):
        sess.eval_seg([dict(p, visual_prompts=p["visual_prompts"][:2])])
    with pytest.raises(ValueError, match="kind"):
        sess.eval_seg([dict(p, visual_prompts=[("lasso", None)] * 3)])
    from psalm_b200 import kernels
    monkeypatch.setattr(kernels, "visual_prompt_raster", _no_launch)
    empty = [("mask", torch.zeros(96, 96)), ("box", (10, 10, 10, 40)), ("point", {"size": [96, 96], "counts": rle_string([96 * 96])}),
             ("scribble", torch.full((96, 96), 2, dtype=torch.uint8))]   # only pixels equal to 1 seed a disk
    for e in empty:
        vp = [e] + p["visual_prompts"][1:]
        with pytest.raises(ValueError, match="empty source mask"):
            sess.eval_seg([dict(p, visual_prompts=vp)])
    with pytest.raises(ValueError, match="outside"):
        sess.eval_seg([dict(p, visual_prompts=[("point", (96, 0))] + p["visual_prompts"][1:])])
    m.set_task("referring")
    with pytest.raises(ValueError, match="region"):
        sess.eval_seg([p])


def test_region_empty_after_the_resize_raises_like_draw_point_indices(monkeypatch):
    """A one-pixel mask on a source row that the NEAREST downscale skips (1333 x 1000 -> 1024 x 768)."""
    from psalm_b200.image_processor import pil_nearest_index
    m, inp, _ = _region_session(monkeypatch, 96, 96)
    H, W = 1333, 1000
    skipped = sorted(set(range(H)) - set(pil_nearest_index(H, 1024).tolist()))[0]
    pad = torch.ones(96, 96, dtype=torch.bool)
    pad[:74, :55] = False            # an un-padded box: the tables map the original size into it
    sess = m.open_image(inp["images"], [dict(padding_mask=pad, height=H, width=W)])
    one = torch.zeros(H, W, dtype=torch.uint8)
    one[skipped, 500] = 1
    vp = [("mask", one), ("box", (0, 0, 400, 400)), ("point", (700, 700))]
    with pytest.raises(ValueError, match="empty region mask"):
        sess.eval_seg([dict(input_ids=inp["input_ids"], attention_mask=inp["attention_mask"], visual_prompts=vp)])
