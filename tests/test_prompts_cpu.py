"""Several prompts against one image (PSALM.open_image / ImageSession.eval_seg): the prompt cut of
psalm_b200/sequence.py and the session's host orchestration, with the CUDA entry points emulated (tests/emu.py plus
emulations of the new wrappers below)."""
import numpy as np
import pytest
import torch

import emu
from psalm_b200 import sequence as SEQ
from psalm_b200 import synth
from psalm_b200.layout import PhiConfig, PsalmConfig

SMALL = PsalmConfig(phi=PhiConfig(hidden=256, layers=2, heads=4, inter=1024))


# ---- emulations of the wrappers the sessions add or extend ----------------------------------------------------------
def prefix_causal_attention(qkv, prefix_k, prefix_v, P, key_valid, B, T, nh, hd):
    """Attention over [prefix keys | own causal keys], float32 torch ops."""
    q, k, v = (qkv[:, :, i].permute(0, 2, 1, 3).float() for i in range(3))          # [B,nh,T,hd]
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
    """Accepts a stride-0 `expand` of one image's map, like the strided entry."""
    assert feats.shape[0] == mask_embed.shape[0] and feats.stride(0) in (0, feats.shape[1] * feats.shape[2])
    return emu.mask_logits(mask_embed, feats, out_dtype)


def mask_bits(mask_embed, feats):
    return emu.attn_mask_bits(mask_logits(mask_embed, feats, torch.float32))


def _install(monkeypatch):
    from psalm_b200 import kernels
    emu.install(monkeypatch)
    for name in ("prefix_causal_attention", "mask_logits", "mask_bits"):
        monkeypatch.setattr(kernels, name, globals()[name])


def _emu_model(monkeypatch, sd, task):
    from psalm_b200.psalm import PSALM
    _install(monkeypatch)

    class _EmuPSALM(PSALM):
        @staticmethod
        def _check_runtime(device):   # tests only: host-logic check with emulated kernels
            pass
    return _EmuPSALM(sd, SMALL, torch.float32, "cpu", task)


def _prompt(inp):
    return {n: inp[n] for n in SEQ.PROMPT_KEYS if inp.get(n) is not None}


def _referring(refer_lens, seed=6, H=192, W=192):
    ins = [synth.synth_inputs(batch=1, height=H, width=W, task="referring", refer_len=n, seed=seed) for n in refer_lens]
    assert all(torch.equal(i["images"], ins[0]["images"]) for i in ins)
    return ins


def _panoptic(n_classes_list, seed=21, H=96, W=96):
    return [synth.synth_inputs(batch=1, height=H, width=W, task="panoptic", n_classes=n, seed=seed + i)
            for i, n in enumerate(n_classes_list)]


# ---- the cut ---------------------------------------------------------------------------------------------------------
def test_referring_prompts_are_cut_at_refer():
    ins = _referring([5, 12, 16])
    ids = ins[0]["input_ids"][0].numpy()
    sp = SEQ.split_prompts([_prompt(i) for i in ins], 16, 100)
    L = int(np.nonzero(ids == SEQ.REFER_TOKEN_INDEX)[0][0])
    assert len(sp.prefix_ids) == L and np.array_equal(sp.prefix_ids, ids[:L])
    assert sp.P == L - 1 + 16 and sp.suffix.B == 3
    assert sp.n_classes == (0, 0, 0)


def test_panoptic_prompts_with_different_vocabularies_are_cut_at_the_first_cls():
    a, b = _panoptic([7, 5])
    b["input_ids"] = b["input_ids"].clone()
    ia = a["input_ids"][0]
    first = int((ia == SEQ.CLS_TOKEN_INDEX).nonzero()[0])
    b_ids = torch.cat([ia[:first], b["input_ids"][0][(b["input_ids"][0] == SEQ.CLS_TOKEN_INDEX).nonzero()[0]:]])
    b["input_ids"] = b_ids[None]
    b["attention_mask"] = torch.ones_like(b["input_ids"], dtype=torch.bool)
    b["class_name_embedding_indices"] = (b["input_ids"] == SEQ.CLS_TOKEN_INDEX).long()
    sp = SEQ.split_prompts([_prompt(a), _prompt(b)], 9, 100)
    assert len(sp.prefix_ids) == first and sp.n_classes == (7, 5)
    assert sp.suffix.cls_pool.shape[1] == 7 and float(sp.suffix.cls_pool[1, 5:].abs().sum()) == 0.0


def test_prompts_that_differ_before_the_image_raise():
    a, b = _referring([5, 5])
    b["input_ids"] = b["input_ids"].clone()
    b["input_ids"][0, 0] += 1
    with pytest.raises(ValueError, match="<image>"):
        SEQ.split_prompts([_prompt(a), _prompt(b)], 16, 100)


def test_masked_position_in_the_prefix_raises():
    a, b = _referring([5, 5])
    b["attention_mask"] = b["attention_mask"].clone()
    b["attention_mask"][0, 2] = False
    with pytest.raises(ValueError, match="masked position"):
        SEQ.split_prompts([_prompt(a), _prompt(b)], 16, 100)


def test_region_prompts_are_not_supported():
    r = synth.synth_inputs(batch=1, height=64, width=64, task="region", seed=3)
    with pytest.raises(NotImplementedError, match="region"):
        SEQ.split_prompts([_prompt(r)], 4, 100)


@pytest.mark.parametrize("kind", ["referring", "panoptic"])
def test_suffix_plans_are_the_rows_of_the_full_plans(kind):
    ins = _referring([5, 12, 16]) if kind == "referring" else _panoptic([7, 7, 7], seed=3)
    if kind == "panoptic":   # one template: same text, per-prompt class names
        for i in ins[1:]:
            i["input_ids"] = ins[0]["input_ids"]
            i["class_name_embedding_indices"] = ins[0]["class_name_embedding_indices"]
    n_img, n_q = 16, 100
    sp = SEQ.split_prompts([_prompt(i) for i in ins], n_img, n_q)
    s, P, Ts = sp.suffix, sp.P, sp.suffix.T
    for k, inp in enumerate(ins):
        full = SEQ.build_plan(inp["input_ids"], inp["attention_mask"], n_img, n_q, inp.get("class_name_ids"),
                              inp.get("cls_indices"), inp.get("class_name_embedding_indices"), inp.get("token_refer_id"),
                              inp.get("refer_embedding_indices"))
        n = full.T - P
        assert torch.equal(full.tok_ids[0, :P], sp.tok_ids[0])
        assert torch.equal(full.img_pos, sp.img_pos)
        assert torch.equal(s.tok_ids[k, :n], full.tok_ids[0, P:])
        assert bool(s.attention_mask[k, :n].all()) and not bool(s.attention_mask[k, n:].any())
        assert torch.equal(s.seg_pos[k * n_q:(k + 1) * n_q] - k * Ts + P, full.seg_pos)
        if full.refer_pool is not None:
            assert float(full.refer_pool[0, 0, :P].abs().sum()) == 0.0
            assert torch.equal(s.refer_pool[k, 0, :n], full.refer_pool[0, 0, P:])
        if full.cls_pool is not None:
            assert torch.equal(s.cls_pool[k, :, :n], full.cls_pool[0, :, P:])


# ---- host orchestration with emulated kernels -------------------------------------------------------------------------
def test_single_prompt_session_matches_referring_golden(monkeypatch, golden):
    """K = 1 on the inputs of e2e_referring_192x192_b1.npz, at the tolerances of test_host_pipeline_matches_golden."""
    H = W = 192
    sd = synth.synth_state_dict(SMALL, seed=5)
    inp = synth.synth_inputs(batch=1, height=H, width=W, task="referring", seed=6)
    m = _emu_model(monkeypatch, sd, "referring")
    g = golden("e2e_referring_192x192_b1.npz")
    state = m._image_core(inp["images"])
    sp = SEQ.split_prompts([_prompt(inp)], m.make_plan_n_img((H, W)), m.num_queries)
    out = m._prompts_core(state, m._prefix_core(state, sp), sp.suffix)
    H4, W4 = out["mask_size"]
    pm = out["pred_masks"].view(1, -1, H4, W4)
    assert list(pm.shape) == g["pred_masks_shape"].tolist()
    got = pm.reshape(-1)[torch.from_numpy(g["pred_masks_idx"])].numpy()
    assert np.abs(got - g["pred_masks"]).max() / np.abs(g["pred_masks"]).max() < 2e-3
    assert np.allclose(out["pred_SEG_logits"].numpy(), g["pred_SEG_logits"], rtol=1e-3, atol=2e-3)
    res = m.post_process(out, (H, W), inp["seg_info"])
    sc = res[0]["instances"].scores
    order = torch.argsort(sc, descending=True, stable=True)
    assert np.allclose(sc[order].numpy(), g["inst_scores_sorted"], rtol=1e-3, atol=1e-4)


def test_three_prompts_match_per_prompt_forward(monkeypatch):
    """K = 3 (one template, refer lengths 5 / 12 / 16): each prompt's result equals the emulated single-prompt pass."""
    H = W = 192
    sd = synth.synth_state_dict(SMALL, seed=5)
    ins = _referring([5, 12, 16])
    m = _emu_model(monkeypatch, sd, "referring")
    state = m._image_core(ins[0]["images"])
    sp = SEQ.split_prompts([_prompt(i) for i in ins], m.make_plan_n_img((H, W)), m.num_queries)
    out = m._prompts_core(state, m._prefix_core(state, sp), sp.suffix)
    for k, inp in enumerate(ins):
        plan = m.make_plan(inp["input_ids"], inp["attention_mask"], (H, W), token_refer_id=inp["token_refer_id"],
                           refer_embedding_indices=inp["refer_embedding_indices"])
        ref = m.forward_core(inp["images"], plan)
        a, b = out["pred_masks"][k], ref["pred_masks"][0]
        assert float((a - b).abs().max() / b.abs().max()) < 1e-5
        assert torch.equal(out["pred_SEG_logits"][k].argmax(0), ref["pred_SEG_logits"][0].argmax(0))
