"""CUDA attention / prediction-head kernels (through the C ABI) vs independent torch restatements
(tests/emu.py, fp32 CPU math on the storage-rounded inputs)."""
import pytest
import torch

import emu
from psalm_b200 import kernels

pytestmark = pytest.mark.gpu
DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
TOL = {"f32": 2e-5, "f16": 2e-3, "bf16": 1.2e-2}   # max |err| / max |ref|; 16-bit = output rounding


@pytest.fixture(params=["auto", "simt", "mma-workspace", "mma-cluster"], autouse=True)
def attn_impl(request):
    """auto = tensor-core (mma.sync) kernels for fp16/bf16 + SIMT for fp32; simt = fp32-math kernels for all;
    mma-workspace / mma-cluster = tensor cores with the split-K reduction forced through the workspace + combine
    kernel / through a thread-block cluster (distributed shared memory)."""
    from psalm_b200 import _lib
    _lib.check(_lib.lib().psalm_set_attention_impl({"auto": 0, "simt": 1, "mma-workspace": 2, "mma-cluster": 3}[request.param]), "set_attention_impl")
    yield request.param
    _lib.lib().psalm_set_attention_impl(0)


def _close(out, ref, dt, scale=1.0):
    out, ref = out.float().cpu(), ref.float().cpu()
    err = (out - ref).abs().max() / (ref.abs().max() + 1e-30)
    assert err < TOL[dt] * scale, "rel-to-max error %.3e (tol %.1e)" % (err, TOL[dt] * scale)


@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("H,W,shift", [(24, 24, 0), (24, 36, 6), (17, 29, 6), (50, 13, 6), (7, 5, 0)])
def test_window_attention(dt, H, W, shift):
    torch.manual_seed(H * 100 + W + shift)
    B, C, nh, ws = 2, 64, 2, 12
    qkv = torch.randn(B, H * W, 3 * C).to(DT[dt])
    bias = (torch.randn(3 * C) * 0.5).to(DT[dt])
    # compact relative-position bias table (the checkpoint's relative_position_bias_table, transposed); the emulation
    # expands it with the reference's relative_position_index (swin_trans.py:93-103, 131-134)
    rel = torch.randn(nh, (2 * ws - 1) ** 2)
    ref = emu.window_attention(qkv.float(), bias.float(), rel, B, H, W, C, nh, ws, shift)
    out = kernels.window_attention(qkv.cuda(), bias.cuda(), rel.cuda(), B, H, W, C, nh, ws, shift)
    _close(out, ref, dt)


@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("T,padded", [(77, False), (130, True), (33, True)])
def test_rotary_and_causal_attention(dt, T, padded):
    torch.manual_seed(T)
    B, nh, hd, rd = 2, 4, 64, 32
    qkv = torch.randn(B, T, 3, nh, hd).to(DT[dt])
    inv = 1.0 / (10000.0 ** (torch.arange(0, rd, 2).float() / rd))
    fr = torch.arange(T).float()[:, None] * inv[None]
    cos, sin = fr.cos().contiguous(), fr.sin().contiguous()
    kv = None
    if padded:
        kv = torch.ones(B, T, dtype=torch.uint8)
        kv[1, T - 9:] = 0
    ref_qkv = qkv.float().clone()
    emu.rotary_inplace(ref_qkv, cos, sin, B, T, nh, hd, rd)
    g = qkv.cuda()
    kernels.rotary_inplace(g, cos.cuda(), sin.cuda(), B, T, nh, hd, rd)
    _close(g, ref_qkv, dt)
    ref = emu.causal_attention(g.float().cpu(), kv, B, T, nh, hd)
    out = kernels.causal_attention(g, kv.cuda() if kv is not None else None, B, T, nh, hd)
    _close(out, ref, dt)


@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("Lq,Lk,splits", [(100, 1024, None), (100, 4096, 4), (100, 389, 3), (37, 100, 1), (100, 100, 1),
                                          (100, 4096, 16), (100, 16384, None), (100, 4096, 19), (100, 2048, 8),
                                          (100, 700, 2), (64, 4096, 5)])
def test_cross_attention_with_bit_mask(dt, Lq, Lk, splits):
    torch.manual_seed(Lq + Lk)
    B, nh, hd = 2, 8, 32
    C = nh * hd
    q, k, v = (torch.randn(B, n, C).to(DT[dt]) for n in (Lq, Lk, Lk))
    logits = torch.randn(B, Lq, Lk)
    logits[0, 3] = -1.0          # fully blocked row -> must attend everywhere (DEC:647)
    logits[1, 0] = 1.0           # fully open row
    bits, row_open = emu.attn_mask_bits(logits)
    assert int(row_open[0, 3]) == 1 and int(row_open[1, 0]) == 0
    ref = emu.cross_attention(q.float(), k.float(), v.float(), bits, row_open, nh)
    out = kernels.cross_attention(q.cuda(), k.cuda(), v.cuda(), bits.cuda(), row_open.cuda(), nh, splits=splits)
    _close(out, ref, dt)
    ref2 = emu.cross_attention(q.float(), k.float(), v.float(), None, None, nh)
    out2 = kernels.cross_attention(q.cuda(), k.cuda(), v.cuda(), None, None, nh, splits=splits)
    _close(out2, ref2, dt)


@pytest.mark.parametrize("impl", [0, 2, 1], ids=["auto", "tcgen05", "mma"])
@pytest.mark.parametrize("dt", ["f16", "bf16"])
@pytest.mark.parametrize("B,Lq,Lk,ld", [(2, 100, 1024, 256), (4, 100, 4096, 768), (1, 100, 16384, 768), (4, 100, 16384, 256),
                                        (2, 100, 27889, 768), (3, 37, 100, 256), (1, 112, 389, 768), (2, 1, 33, 256),
                                        (5, 100, 6400, 768), (1, 100, 31, 256)])
def test_masked_cross_attention_tma(impl, dt, B, Lq, Lk, ld):
    """The masked cross-attention kernels (auto: per-head flash kernel below 2048 keys, TMA-fed warp-level mma.sync
    kernel of csrc/xattn_tma.cu above; selectors 1 and 2 (the Blackwell tensor-memory kernel's slot, "tcgen05" in the
    ids): the TMA-fed kernel at every key count) vs the torch restatement: packed bit masks, fully blocked rows that
    re-open, fully open rows,
    ragged key counts (tail tile), row-strided K / V views of a fused projection buffer, single-CTA and split-K grids,
    and the no-mask case."""
    from psalm_b200 import _lib
    _lib.check(_lib.lib().psalm_set_cross_impl(impl), "psalm_set_cross_impl")
    try:
        _masked_cross_attention_case(dt, B, Lq, Lk, ld)
    finally:
        _lib.lib().psalm_set_cross_impl(0)


def _masked_cross_attention_case(dt, B, Lq, Lk, ld):
    torch.manual_seed(B * 1000 + Lq + Lk)
    nh, C = 8, 256
    q = torch.randn(B, Lq, C).to(DT[dt])
    kbuf, vbuf = torch.randn(B, Lk, ld).to(DT[dt]), torch.randn(B, Lk, ld).to(DT[dt])
    off = 0 if ld == 256 else 256
    logits = torch.randn(B, Lq, Lk)
    # spatially structured masks: long blocked runs (whole 16 x 32 blocks get skipped) and noise elsewhere
    logits[:, :, : Lk // 3] -= 4.0
    logits[0, min(3, Lq - 1)] = -1.0          # fully blocked row -> must attend everywhere (DEC:647)
    logits[B - 1, 0] = 1.0                     # fully open row
    bits, row_open = emu.attn_mask_bits(logits)
    kg, vg = kbuf.cuda(), vbuf.cuda()
    k, v = kg[:, :, off:off + C], vg[:, :, off:off + C]
    ref = emu.cross_attention(q.float(), kbuf[:, :, off:off + C].float(), vbuf[:, :, off:off + C].float(), bits, row_open, nh)
    out = kernels.masked_cross_attention(q.cuda(), k, v, bits.cuda(), row_open.cuda(), nh)
    torch.cuda.synchronize()
    _close(out, ref, dt)
    ref2 = emu.cross_attention(q.float(), kbuf[:, :, off:off + C].float(), vbuf[:, :, off:off + C].float(), None, None, nh)
    out2 = kernels.masked_cross_attention(q.cuda(), k, v, None, None, nh)
    _close(out2, ref2, dt)
    # same answer as the per-head kernel it replaces
    old = kernels.cross_attention(q.cuda(), k.contiguous(), v.contiguous(), bits.cuda(), row_open.cuda(), nh)
    _close(out, old.float().cpu(), dt)


@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
def test_mask_head_kernels(dt):
    torch.manual_seed(0)
    B, Q, C, H4, W4 = 2, 100, 256, 40, 52
    me = torch.randn(B, Q, C).to(DT[dt])
    mf = torch.randn(B, H4 * W4, C).to(DT[dt])
    ref = emu.mask_logits(me.float(), mf.float(), torch.float32)
    out = kernels.mask_logits(me.cuda(), mf.cuda(), out_dtype=torch.float32)
    _close(out, ref, "f32" if dt == "f32" else dt, scale=1.0)
    out_t = kernels.mask_logits(me.cuda(), mf.cuda())
    assert out_t.dtype == DT[dt]
    _close(out_t, ref, dt)
    for Ho, Wo in ((5, 7), (10, 13), (20, 26), (80, 104)):
        refb = emu.bilinear_tokens(mf.float(), H4, W4, Ho, Wo)
        outb = kernels.bilinear_tokens(mf.cuda(), H4, W4, Ho, Wo)
        _close(outb, refb, dt)
    lg = torch.randn(B, Q, 389)
    lg[1, 7] = -2.0
    bits_ref, ro_ref = emu.attn_mask_bits(lg)
    bits, ro = kernels.attn_mask_bits(lg.cuda())
    assert torch.equal(bits.cpu(), bits_ref) and torch.equal(ro.cpu(), ro_ref)


def test_pooled_mask_equals_reference_order():
    """interp(einsum(me, F)) vs einsum(me, interp(F)) (mask_decoder.py docstring): count sign flips of
    the resulting attention mask at the exact 2x/4x/8x factors and at a non-integer factor."""
    import torch.nn.functional as F
    torch.manual_seed(1)
    B, Q, C = 1, 100, 256
    me = torch.randn(B, Q, C).cuda()
    for (H4, W4), (Hl, Wl) in (((64, 64), (8, 8)), ((64, 64), (32, 32)), ((50, 66), (7, 9))):
        mf = torch.randn(B, H4 * W4, C).cuda()
        full = kernels.mask_logits(me, mf, out_dtype=torch.float32).view(B, Q, H4, W4)
        ref = F.interpolate(full, size=(Hl, Wl), mode="bilinear", align_corners=False).flatten(2) < 0
        pooled = kernels.bilinear_tokens(mf, H4, W4, Hl, Wl)
        got = kernels.mask_logits(me, pooled, out_dtype=torch.float32) < 0
        flips = (ref != got).float().mean().item()
        assert flips < 1e-4, flips


@pytest.mark.parametrize("dt", ["f16", "bf16"])
@pytest.mark.parametrize("P", [1024, 389, 4096 + 32])
def test_mask_bits_fused_and_mma_logits(dt, P, attn_impl):
    """Tensor-core mask projection: final logits equal the fp32 restatement within storage rounding; the
    fused bit mask equals thresholding those logits except where |logit| is at rounding level."""
    if attn_impl == "simt":
        pytest.skip("independent of the attention implementation switch")
    torch.manual_seed(P)
    B, Q, C = 2, 100, 256
    me = torch.randn(B, Q, C).to(DT[dt])
    f = torch.randn(B, P, C).to(DT[dt])
    ref = emu.mask_logits(me.float(), f.float(), torch.float32)
    if P % 2 == 0:
        out = kernels.mask_logits(me.cuda(), f.cuda())
        _close(out, ref, dt)
    bits, ro = kernels.mask_bits(me.cuda(), f.cuda())
    ref_bits, ref_ro = emu.attn_mask_bits(ref)
    got = ((bits.cpu().long() & 0xFFFFFFFF).unsqueeze(-1) >> torch.arange(32)) & 1
    want = ((ref_bits.long() & 0xFFFFFFFF).unsqueeze(-1) >> torch.arange(32)) & 1
    mism = (got != want).view(B, Q, -1)[..., :P]
    assert (mism & (ref.abs() > 1e-3)).sum() == 0      # flips only where the fp32 logit is ~0
    assert mism.float().mean() < 1e-4
    assert torch.equal(ro.cpu(), ref_ro)
    f2 = f.clone()
    me2 = me.clone()
    me2[0, 5] = 0
    me2[0, 5, 0] = 1.0
    f2[0, :, 0] = -1.0          # row 5 of batch 0: every key blocked -> row_open
    _, ro2 = kernels.mask_bits(me2.cuda(), f2.cuda())
    assert int(ro2[0, 5]) == 1


@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("B,Q,P", [(1, 100, 8192), (2, 100, 4096 + 96), (1, 128, 65536), (3, 7, 130)])
def test_mask_projection_tcgen05(dt, B, Q, P, attn_impl):
    """Large-P mask projection selector (2; the slot of the Blackwell tensor-memory kernel, on H100 the wgmma GEMM of
    csrc/gemm_wgmma.cu for P % 256 == 0, the mma.sync / generic kernels otherwise) vs the fp32 restatement; also
    vs the mma.sync selector (1) within the same tolerance (both accumulate in fp32, in different orders)."""
    if attn_impl == "simt":
        pytest.skip("independent of the attention implementation switch")
    from psalm_b200 import _lib
    torch.manual_seed(P + Q)
    me = torch.randn(B, Q, 256).to(DT[dt])
    f = torch.randn(B, P, 256).to(DT[dt])
    ref = emu.mask_logits(me.float(), f.float(), torch.float32)
    try:
        _lib.check(_lib.lib().psalm_set_mask_proj_impl(2), "set_mask_proj_impl")
        out = kernels.mask_logits(me.cuda(), f.cuda())
        _lib.check(_lib.lib().psalm_set_mask_proj_impl(1), "set_mask_proj_impl")
        out1 = kernels.mask_logits(me.cuda(), f.cuda())
        torch.cuda.synchronize()
    finally:
        _lib.lib().psalm_set_mask_proj_impl(0)
    _close(out, ref, dt)
    _close(out1, ref, dt)
    auto = kernels.mask_logits(me.cuda(), f.cuda())
    assert torch.equal(auto, out if P >= 8192 else out1)


@pytest.mark.parametrize("dt", ["f16", "bf16"])
@pytest.mark.parametrize("T,padded", [(64, False), (130, True), (257, False), (900, True), (1100, False), (1100, True), (2048, False)])
@pytest.mark.parametrize("impl", [1, 2])
def test_causal_attention_impls(dt, T, padded, impl):
    """Causal attention selectors 1 (mma.sync flash kernel) and 2 (the long-sequence tensor-core slot; on H100 the same
    flash kernel) against the fp32 restatement, up to the 2048-token prefill."""
    from psalm_b200 import _lib
    torch.manual_seed(T + impl)
    B, nh, hd = 2, 3, 64
    qkv = torch.randn(B, T, 3, nh, hd).to(DT[dt])
    kv = None
    if padded:
        kv = torch.ones(B, T, dtype=torch.uint8)
        kv[1, T - 9:] = 0
        kv[0, 5:40] = 0          # a hole inside the sequence
        kv[1, 0] = 0             # first key invalid: row 0 of batch 1 has no valid key at all
    ref = emu.causal_attention(qkv.float(), kv, B, T, nh, hd)
    try:
        _lib.check(_lib.lib().psalm_set_causal_impl(impl), "set_causal_impl")
        out = kernels.causal_attention(qkv.cuda(), kv.cuda() if kv is not None else None, B, T, nh, hd)
        out2 = kernels.causal_attention(qkv.cuda(), kv.cuda() if kv is not None else None, B, T, nh, hd)
    finally:
        _lib.lib().psalm_set_causal_impl(0)
    assert torch.equal(out, out2)
    valid = torch.ones(B, T, dtype=torch.bool) if kv is None else kv.bool()
    if kv is not None:
        valid[1, 0] = False      # fully-masked query row: implementation-defined (zeros here, NaN in torch)
    o, r = out.float().cpu()[valid], ref[valid]
    err = (o - r).abs().max() / (r.abs().max() + 1e-30)
    assert err < TOL[dt], "rel-to-max error %.3e" % err
