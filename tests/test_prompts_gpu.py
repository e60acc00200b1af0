"""Several prompts against one image on the GPU: the prefix-causal attention kernel, the stride-0 (shared image memory)
entries, and ImageSession.eval_seg against per-prompt eval_seg."""
import numpy as np
import pytest
import torch

from psalm_b200 import _lib, kernels
from psalm_b200 import sequence as SEQ
from psalm_b200 import synth
from psalm_b200.layout import PhiConfig, PsalmConfig

pytestmark = pytest.mark.gpu
DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
TOL = {"f32": 2e-5, "f16": 2e-3, "bf16": 1.2e-2}   # the bars of test_attn_gpu.py::test_rotary_and_causal_attention
SMALL = PsalmConfig(phi=PhiConfig(hidden=256, layers=2, heads=4, inter=1024))


def _close(out, ref, dt):
    out, ref = out.double(), ref.double()
    if out.numel() == 0:     # every query row is padding: only finiteness is asked of them
        return
    err = float((out - ref).abs().max() / (ref.abs().max() + 1e-30))
    assert err < TOL[dt], "rel-to-max error %.3e (tol %.1e)" % (err, TOL[dt])


def _ref_prefix_attention(qkv, pk, pv, P, kv, hd):
    """float64 torch reference on the device."""
    B, T, _, nh, _ = qkv.shape
    q, k, v = (qkv[:, :, i].permute(0, 2, 1, 3).double() for i in range(3))
    kk = torch.cat([pk[:, :P].double().unsqueeze(0).expand(B, -1, -1, -1), k], 2)
    vv = torch.cat([pv[:, :P].double().unsqueeze(0).expand(B, -1, -1, -1), v], 2)
    s = (q @ kk.transpose(-2, -1)) * hd ** -0.5
    dev = qkv.device
    allowed = torch.cat([torch.ones(T, P, dtype=torch.bool, device=dev),
                         torch.tril(torch.ones(T, T, dtype=torch.bool, device=dev))], 1)[None, None]
    if kv is not None:
        allowed = allowed & torch.cat([torch.ones(B, P, dtype=torch.bool, device=dev), kv.bool()], 1)[:, None, None, :]
    p = torch.nan_to_num(s.masked_fill(~allowed, float("-inf")).softmax(-1))
    return (p @ vv).permute(0, 2, 1, 3).reshape(B, T, nh * hd)


@pytest.mark.parametrize("dt", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("P", [0, 1, 63, 64, 65, 290])
@pytest.mark.parametrize("T", [1, 17, 64, 160])
@pytest.mark.parametrize("padded", [False, True])
def test_prefix_causal_attention(dt, B, P, T, padded):
    torch.manual_seed(P * 1000 + T * 10 + B)
    nh, hd = 4, 64
    ld = max(64, -(-P // 64) * 64)
    qkv = torch.randn(B, T, 3, nh, hd, device="cuda").to(DT[dt])
    pk = torch.randn(nh, ld, hd, device="cuda").to(DT[dt])
    pv = torch.randn(nh, ld, hd, device="cuda").to(DT[dt])
    kv = None
    if padded:
        kv = torch.ones(B, T, dtype=torch.uint8, device="cuda")
        kv[-1, T - min(T - 1, 9):] = 0
        if T == 1:
            kv[-1, 0] = 0 if P > 0 else 1
    out = kernels.prefix_causal_attention(qkv, pk, pv, P, kv, B, T, nh, hd)
    assert bool(torch.isfinite(out.float()).all())
    ref = _ref_prefix_attention(qkv, pk, pv, P, kv, hd)
    valid = torch.ones(B, T, dtype=torch.bool, device="cuda") if kv is None else kv.bool()
    _close(out.double()[valid], ref[valid], dt)
    # causal attention over [prefix | suffix] agrees on rows P.. (prefix keys rebuilt as qkv rows)
    full = torch.zeros(B, P + T, 3, nh, hd, device="cuda", dtype=DT[dt])
    full[:, :P, 1] = pk[:, :P].permute(1, 0, 2).unsqueeze(0)
    full[:, :P, 2] = pv[:, :P].permute(1, 0, 2).unsqueeze(0)
    full[:, P:] = qkv
    fkv = None if kv is None else torch.cat([torch.ones(B, P, dtype=torch.uint8, device="cuda"), kv], 1)
    cat = kernels.causal_attention(full.contiguous(), fkv, B, P + T, nh, hd)[:, P:]
    _close(cat.double()[valid], out.double()[valid], dt)


def _set(fn, v):
    _lib.check(getattr(_lib.lib(), fn)(v), fn)


@pytest.mark.parametrize("impl", [0, 1, 2])
@pytest.mark.parametrize("Lk", [1024, 4096, 16384])
@pytest.mark.parametrize("K", [1, 3, 16])
@pytest.mark.parametrize("dt", ["bf16", "f16"])
def test_masked_cross_attention_stride0_is_bit_identical(impl, Lk, K, dt):
    torch.manual_seed(Lk + K)
    C, Lq = 256, 100
    q = torch.randn(K, Lq, C, device="cuda").to(DT[dt])
    kv = torch.randn(1, Lk, 3 * C, device="cuda").to(DT[dt])     # a fused projection buffer: row stride 768
    k, v = kv[:, :, :C].expand(K, -1, -1), kv[:, :, C:2 * C].expand(K, -1, -1)
    bits = torch.randint(-2 ** 31, 2 ** 31 - 1, (K, Lq, (Lk + 31) // 32), dtype=torch.int32, device="cuda")
    row_open = (torch.rand(K, Lq, device="cuda") < 0.05).to(torch.uint8)
    _set("psalm_set_cross_impl", impl)
    try:
        a = kernels.masked_cross_attention(q, k, v, bits, row_open, 8)
        b = kernels.masked_cross_attention(q, k.contiguous(), v.contiguous(), bits, row_open, 8)
    finally:
        _set("psalm_set_cross_impl", 0)
    assert torch.equal(a, b)


@pytest.mark.parametrize("K", [1, 3, 16])
@pytest.mark.parametrize("P", [1024, 4096, 16384])
@pytest.mark.parametrize("impl", [1, 2])
def test_mask_bits_and_logits_stride0_are_bit_identical(K, P, impl):
    torch.manual_seed(K * P)
    me = torch.randn(K, 100, 256, device="cuda").bfloat16()
    f1 = torch.randn(1, P, 256, device="cuda").bfloat16()
    fe = f1.expand(K, -1, -1)
    a_bits, a_open = kernels.mask_bits(me, fe)
    b_bits, b_open = kernels.mask_bits(me, fe.contiguous())
    assert torch.equal(a_bits, b_bits) and torch.equal(a_open, b_open)
    _set("psalm_set_mask_proj_impl", impl)    # 1 = mma.sync, 2 = wgmma (one GEMM with M = K * Q at stride 0)
    try:
        a = kernels.mask_logits(me, fe)
        b = kernels.mask_logits(me, fe.contiguous())
    finally:
        _set("psalm_set_mask_proj_impl", 0)
    assert torch.equal(a, b)
    af = kernels.mask_logits(me.float(), fe.float(), out_dtype=torch.float32)    # SIMT fp32 kernel
    assert torch.equal(af, kernels.mask_logits(me.float(), fe.float().contiguous(), out_dtype=torch.float32))


# ---- sessions --------------------------------------------------------------------------------------------------------
def _prompt(inp):
    return {n: inp[n] for n in SEQ.PROMPT_KEYS if inp.get(n) is not None}


def _referring(refer_lens, H, W, seed=6):
    return [synth.synth_inputs(batch=1, height=H, width=W, task="referring", refer_len=n, seed=seed) for n in refer_lens]


def _eval(m, inp, **kw):
    return m.eval_seg(input_ids=inp["input_ids"], attention_mask=inp["attention_mask"], images=inp["images"],
                      seg_info=inp["seg_info"], class_name_ids=inp.get("class_name_ids"), cls_indices=inp.get("cls_indices"),
                      class_name_embedding_indices=inp.get("class_name_embedding_indices"),
                      token_refer_id=inp.get("token_refer_id"), refer_embedding_indices=inp.get("refer_embedding_indices"),
                      is_thing_list=inp.get("is_thing_list"), **kw)


def _core(m, inp):
    plan = m.make_plan(inp["input_ids"], inp["attention_mask"], inp["images"].shape[-2:], inp.get("class_name_ids"),
                       inp.get("cls_indices"), inp.get("class_name_embedding_indices"), inp.get("token_refer_id"),
                       inp.get("refer_embedding_indices")).to("cuda")
    trace = {}
    return m.forward_core(inp["images"].cuda(), plan, trace=trace), trace


def test_fp32_referring_session_matches_per_prompt_eval_seg(golden):
    from psalm_b200.psalm import PSALM
    H = W = 192
    sd = synth.synth_state_dict(SMALL, seed=5)
    m = PSALM(sd, SMALL, torch.float32, "cuda", "referring")
    ins = _referring([5, 12, 16], H, W)
    sess = m.open_image(ins[0]["images"], ins[0]["seg_info"])
    split, plan = m._cached_split([_prompt(i) for i in ins], (H, W))
    outs = m._prompts_forward(sess, split, plan)
    res = sess.eval_seg([_prompt(i) for i in ins])
    for k, inp in enumerate(ins):
        ref, _ = _core(m, inp)
        a, b = outs[k]["pred_masks"].float(), ref["pred_masks"].float()
        assert float((a - b).abs().max() / b.abs().max()) < 1e-3
        assert np.allclose(outs[k]["pred_SEG_logits"].cpu().numpy(), ref["pred_SEG_logits"].cpu().numpy(), rtol=1e-3, atol=2e-3)
        want = _eval(m, inp)[0]["instances"]
        got = res[k]["instances"]
        assert int(got.scores.argmax()) == int(want.scores.argmax())
    # K = 1 against the reference golden
    g = golden("e2e_referring_192x192_b1.npz")
    one = m._prompts_forward(sess, *m._cached_split([_prompt(ins[1])], (H, W)))[0]
    got = one["pred_masks"].reshape(-1)[torch.from_numpy(g["pred_masks_idx"]).cuda()].cpu().numpy()
    assert np.abs(got - g["pred_masks"]).max() / np.abs(g["pred_masks"]).max() < 2e-3


def test_fp32_panoptic_two_class_lists_match_per_prompt_eval_seg():
    from psalm_b200.psalm import PSALM
    H = W = 128
    sd = synth.synth_state_dict(SMALL, seed=8)
    m = PSALM(sd, SMALL, torch.float32, "cuda", "panoptic")
    m.object_mask_threshold = m.overlap_threshold = 0.0      # keep segments on random weights
    a = synth.synth_inputs(batch=1, height=H, width=W, task="panoptic", n_classes=9, seed=30)
    b = synth.synth_inputs(batch=1, height=H, width=W, task="panoptic", n_classes=6, seed=31)
    ia = a["input_ids"][0]
    first = int((ia == SEQ.CLS_TOKEN_INDEX).nonzero()[0])
    ib = b["input_ids"][0]
    b["input_ids"] = torch.cat([ia[:first], ib[int((ib == SEQ.CLS_TOKEN_INDEX).nonzero()[0]):]])[None]
    b["attention_mask"] = torch.ones_like(b["input_ids"], dtype=torch.bool)
    b["class_name_embedding_indices"] = (b["input_ids"] == SEQ.CLS_TOKEN_INDEX).long()
    b["images"], b["seg_info"] = a["images"], a["seg_info"]
    prompts = [dict(_prompt(a), is_thing_list=a["is_thing_list"]), dict(_prompt(b), is_thing_list=b["is_thing_list"])]
    res = m.open_image(a["images"], a["seg_info"]).eval_seg(prompts)
    for r, inp in zip(res, (a, b)):
        want = _eval(m, inp)[0]
        (pa, ia_), (pb, ib_) = r["panoptic_seg"], want["panoptic_seg"]
        assert float((pa != pb).float().mean()) < 2e-3
        assert [(d["id"], d["isthing"], d["category_id"]) for d in ia_] == [(d["id"], d["isthing"], d["category_id"]) for d in ib_]


def test_bf16_full_size_graph_session_matches_per_prompt_eval_seg():
    from psalm_b200.psalm import PSALM
    cfg = PsalmConfig()
    sd = synth.synth_state_dict(cfg, seed=2)
    m = PSALM(sd, cfg, torch.bfloat16, "cuda", "referring", use_cuda_graph=True)
    eager = PSALM(sd, cfg, torch.bfloat16, "cuda", "referring")
    del sd
    H = W = 1024
    ins = _referring([5, 9, 12, 16], H, W, seed=3)
    prompts = [_prompt(i) for i in ins]
    sess_e = eager.open_image(ins[0]["images"], ins[0]["seg_info"])
    split, plan = eager._cached_split(prompts, (H, W))
    out_e = eager._prompts_core(sess_e.state, sess_e.prefix_cache(split), plan)
    res = [r["instances"] for r in m.open_image(ins[0]["images"], ins[0]["seg_info"]).eval_seg(prompts)]
    res = [(r.scores.clone(), r.pred_masks.clone()) for r in res]
    n_q = eager.num_queries
    measured = []
    for k, inp in enumerate(ins):
        ref, trace = _core(eager, inp)
        if k == 0:   # the same kernels at the same batch: bitwise equal image-level stages
            for a, b in zip(sess_e.state["swin"], trace["swin"]):
                assert torch.equal(a, b)
            assert torch.equal(sess_e.state["mask_features"], trace["mask_features"])
        hs = out_e["seg_query"][k].float()
        hr = trace["seg_query"][0].float()
        assert hs.shape[0] == n_q
        rel = float((hs - hr).norm() / hr.norm())
        want = _eval(m, inp)[0]["instances"]
        top_s, top_r = int(res[k][0].argmax()), int(want.scores.argmax())
        # instances are in query order.  same-query IoU: the session's mask of the reference's top-1 query against the
        # reference's (asserted); top-1 IoU: the mask the session ranks first against the one eval_seg ranks first
        # (what a caller receives, although the two top-1 queries differ: they are near ties, see below)
        def iou_of(a, b):
            a, b = a > 0.5, b > 0.5
            return float((a & b).sum()) / max(float((a | b).sum()), 1.0)
        iou = iou_of(res[k][1][top_r], want.pred_masks[top_r])
        iou_top1 = iou_of(res[k][1][top_s], want.pred_masks[top_r])
        ls, lr = out_e["pred_SEG_logits"][k].float().flatten(), ref["pred_SEG_logits"][0].float().flatten()
        dlog = float((ls - lr).abs().max())                    # SEG-logit change of the split prefill
        margin = float(ls.max() - ls[top_r])                  # how far the reference's top-1 is behind in the session
        measured.append(dict(seg_query_l2rel=round(rel, 5), same_top1=top_s == top_r, iou=round(iou, 4),
                             top1_mask_iou=round(iou_top1, 4),
                             seg_logit_maxdiff=round(dlog, 4), seg_logit_absmax=round(float(lr.abs().max()), 3),
                             top1_logit_margin=round(margin, 4)))
    print("bf16 session vs eval_seg per prompt:", measured)
    for d in measured:
        assert d["seg_query_l2rel"] < 1e-2, d
        assert d["iou"] >= 0.95, d             # same query (the reference's top-1) in both
        assert d["top1_mask_iou"] >= 0.95, d   # each side's own top-1 mask: what a caller receives
        # Measured on an H100 80GB HBM3 (700 W): with synthetic weights the bf16 SEG logits sit near -14 (0.0625 apart in
        # bf16) and the referring scores of the best queries are near ties (1.7333e-6 / 1.7336e-6 for queries 47 / 51 of
        # prompt 0); the split prefill (seg-query l2-rel 8.0e-3) moves a logit by 2-4 bf16 steps (0.125-0.25), so the top-1
        # query differs for all four prompts.  The "same top-1 query" bar is NOT asserted here for that reason; the
        # logits are checked to agree within that bf16 rounding, and the mask of the reference's top-1 query by its
        # same-query IoU above.
        assert d["seg_logit_maxdiff"] < 2e-2 * d["seg_logit_absmax"], d


def test_graph_sessions_lanes_staleness_and_rle():
    from psalm_b200 import rle
    from psalm_b200.psalm import PSALM
    H = W = 192
    sd = synth.synth_state_dict(SMALL, seed=5)
    eager = PSALM(sd, SMALL, torch.bfloat16, "cuda", "referring")
    graphed = PSALM(sd, SMALL, torch.bfloat16, "cuda", "referring", use_cuda_graph=True)
    imgs = {s: _referring([5, 12, 16], H, W, seed=s) for s in (6, 7)}

    def snap(res):
        return [(r["instances"].scores.clone(), r["instances"].pred_masks.clone()) for r in res]
    want = {s: snap(eager.open_image(v[0]["images"], v[0]["seg_info"]).eval_seg([_prompt(i) for i in v]))
            for s, v in imgs.items()}
    for step in range(2):                           # lanes 0 / 1 alternate, the graphs replay on the second round
        sessions = {s: graphed.open_image(v[0]["images"], v[0]["seg_info"], lane=lane)
                    for lane, (s, v) in enumerate(imgs.items())}
        for s, sess in sessions.items():
            got = snap(sess.eval_seg([_prompt(i) for i in imgs[s]]))
            for (a, am), (b, bm) in zip(got, want[s]):
                assert torch.allclose(a, b, rtol=1e-5, atol=1e-7) and torch.equal(am, bm)
    stale = sessions[6]
    graphed.open_image(imgs[6][0]["images"], imgs[6][0]["seg_info"], lane=0)
    with pytest.raises(RuntimeError, match="stale"):
        stale.eval_seg([_prompt(imgs[6][0])])
    sess = graphed.open_image(imgs[7][0]["images"], imgs[7][0]["seg_info"], lane=0)
    res = sess.eval_seg([_prompt(i) for i in imgs[7]], mask_format="rle")
    for r in res:
        inst = r["instances"]
        dec = rle.decode(inst.pred_masks_rle)
        assert torch.equal(torch.as_tensor(dec).to(inst.pred_masks.device).bool(), inst.pred_masks.bool())
    pend = sess.eval_seg_async([_prompt(i) for i in imgs[7]])
    for a, (b, bm) in zip(snap(pend.result()), want[7]):
        assert torch.allclose(a[0], b, rtol=1e-5, atol=1e-7)


def test_graph_sessions_over_many_prompt_sets_of_one_template():
    """More prompt sets than the split cache holds (16), one template, a new session per set as in a RefCOCO loop: the
    prefix graph replays with its own copies of the prefix rows, and the graph sessions give the eager sessions' results
    and prefix K / V."""
    from psalm_b200.psalm import PSALM
    H = W = 192
    sd = synth.synth_state_dict(SMALL, seed=5)
    eager = PSALM(sd, SMALL, torch.bfloat16, "cuda", "referring")
    graphed = PSALM(sd, SMALL, torch.bfloat16, "cuda", "referring", use_cuda_graph=True)
    base = synth.synth_inputs(batch=1, height=H, width=W, task="referring", refer_len=9, seed=6)
    g = torch.Generator().manual_seed(0)

    def prompt_set():
        out = []
        for _ in range(2):
            r = base["token_refer_id"][0].clone()
            r[:-1] = torch.randint(5, 50000, (r.numel() - 1,), generator=g)
            out.append(dict(_prompt(base), token_refer_id=[r]))
        return out
    sets = [prompt_set() for _ in range(20)]
    for i, prompts in enumerate(sets):
        sess = graphed.open_image(base["images"], base["seg_info"])
        got = [(r["instances"].scores.clone(), r["instances"].pred_masks.clone()) for r in sess.eval_seg(prompts)]
        if i < len(sets) - 3:
            continue
        ref_sess = eager.open_image(base["images"], base["seg_info"])
        want = ref_sess.eval_seg(prompts)
        for (a, am), r in zip(got, want):
            assert torch.allclose(a, r["instances"].scores, rtol=1e-5, atol=1e-7)
            assert torch.equal(am, r["instances"].pred_masks)
        split, _ = graphed._cached_split(prompts, (H, W))
        gc, ec = sess.prefix_cache(split), ref_sess.prefix_cache(split)
        page = gc.k[0].shape[2]
        assert gc.length == ec.length == split.P
        for layer in range(SMALL.phi.layers):
            assert torch.equal(gc.k[layer][0, :, :split.P], ec.k[layer][0, :, :split.P])
            assert torch.equal(gc.v[layer][0, :, :split.P], ec.v[layer][0, :, :split.P])
        assert page % 64 == 0
    assert len(graphed._splits) == 16
