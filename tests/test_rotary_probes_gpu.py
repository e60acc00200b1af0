"""The rotary kernels, rotary composed with the attention kernels that consume it, and the linear_act epilogues on the
probes of tests/rotary_probe.py (references, bounds and their derivation: its docstring).

  rotary alone     exact probes bit for bit, float64 probes within the derived bound, and every element outside the
                   first rd dims of q and k bit-identical to its input, on every route (vector kernel, scalar kernel in
                   fp32 and in 16-bit) including grid-stride wraps.  Views with a storage offset take the scalar kernel
                   and give the aligned call's bits; malformed arguments are refused before any launch.
  chains           pre-rotary qkv through rotary_inplace and causal_attention (prefill), through rotary_inplace,
                   kv_cache_write into a one-page prefix cache and prefix_causal_attention (prompt suffix), and through
                   per-sequence prefill writes, the new token's rotary at row seq_len, kv_cache_write and
                   paged_decode_attention (decode).  The rotated rows and caches must equal q' / k' in value, and
                   the attention output must be within attn_probe.bound of the float64 attention of q', k', v.
  linear_act       relu bit for bit, gelu_tanh within its bound, at the model's fc1 / FFN / MLP shapes.

Largest err / bound observed on an NVIDIA H100 80GB HBM3 (700 W power limit), over every case of this file:
  rotary, vector kernel            bf16 1.000   fp16 1.000
  rotary, scalar kernel            bf16 1.000   fp16 1.000   fp32 0.986
  prefill chain                    bf16 0.017   fp16 0.126   fp32 0.048
  prompt-suffix chain              bf16 0.008   fp16 0.062   fp32 0.026
  decode chain                     bf16 0.039   fp16 0.148   fp32 0.004
  linear_act gelu_tanh             bf16 0.451   fp16 0.433
The rotary figures reach 1 because the storage half-ulp term of the bound is attained exactly by a round-to-nearest
tie; the exact probes, the relu probes and every rotated row of the chains matched their references exactly.  The
whole file runs in about 40 s on that GPU.
"""
import contextlib

import pytest
import torch

import attn_probe as ap
import rotary_probe as rp
from psalm_b200 import _lib, kernels
from rotary_probe import ACT_CASES, CAUSAL_CASES, DECODE_CASES, PREFIX_PS, ROTARY_CASES

pytestmark = pytest.mark.gpu
DT = {"bf16": torch.bfloat16, "f16": torch.float16, "f32": torch.float32}
INT = {torch.bfloat16: torch.int16, torch.float16: torch.int16, torch.float32: torch.int32}
DEV = torch.device("cuda")


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _bits(a, b):
    """Bit-for-bit equality of two tensors of one storage type."""
    return torch.equal(a.contiguous().view(INT[a.dtype]).cpu(), b.contiguous().view(INT[b.dtype]).cpu())


def _same(a, b):
    """Equality in value.  A quarter turn may give -0 where the post-rotary probe holds +0 (fp16 rounds a few of the
    probe's small key components to zero of either sign); attention cannot tell the two apart."""
    return torch.equal(a.cpu().double(), b.cpu().double())


@contextlib.contextmanager
def _attn_impl(impl):
    fn = _lib.lib().psalm_set_attention_impl
    _lib.check(fn(impl), "psalm_set_attention_impl")
    try:
        yield
    finally:
        fn(0)


def _report(tag, r):
    print("PROBE %s err/bound %.4f" % (tag, r))
    assert r <= 1.0, "%s: max err / bound = %.3f" % (tag, r)


# ---------------------------------------------------------------------------------------------------------------
# rotary alone
# ---------------------------------------------------------------------------------------------------------------
def _run_rotary(x, cos, sin, B, T, nh, hd, rd, dtype):
    """Rotate a device copy of x with rows 0..T-1 of the tables (a view at their start, as phi.py slices them)."""
    qkv = x.to(dtype).to(DEV)
    kernels.rotary_inplace(qkv, cos.to(DEV)[:T], sin.to(DEV)[:T], B, T, nh, hd, rd)
    torch.cuda.synchronize()
    return qkv


@pytest.mark.parametrize("dt", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("case", ROTARY_CASES, ids=lambda c: c[0])
def test_rotary_probe(case, dt):
    name, B, T, nh, hd, rd, P = case
    dtype = DT[dt]
    x, cos, sin = rp.exact_probe(B, T, nh, hd, rd, _g(T * 7 + rd))
    xs = x.to(dtype)
    out = _run_rotary(xs, cos, sin, B, T, nh, hd, rd, dtype)
    y = rp.rotate(x.to(DEV), cos, sin, rd)
    assert _bits(out, y.to(dtype)), "exact probe %s %s" % (name, dt)
    assert rp.untouched(out, xs, rd)
    x, cos, sin = rp.float_probe(B, T, nh, hd, rd, dtype, _g(T * 3 + rd), P=P)
    xs = x.to(dtype)
    out = _run_rotary(xs, cos, sin, B, T, nh, hd, rd, dtype)
    y, bnd = rp.bound(x.to(DEV), cos, sin, rd, dtype)
    assert rp.untouched(out, xs, rd)
    _report("rotary %s %s %s" % (name, dt, rp.route(dtype, hd, rd)), rp.ratio(out, y, bnd, rd))


def _offset_view(t, off):
    """A contiguous copy of t that starts `off` elements into its buffer."""
    buf = torch.empty(t.numel() + 8, dtype=t.dtype, device=DEV)
    v = buf[off:off + t.numel()].view(t.shape)
    v.copy_(t)
    return v


@pytest.mark.parametrize("dt", ["bf16", "f16"])
def test_rotary_offset_views_take_the_scalar_route(dt):
    B, T, nh, hd, rd, dtype = 2, 7, 32, 64, 32, DT[dt]
    assert rp.route(dtype, hd, rd) == "vec" and rp.route(dtype, hd, rd, aligned=False) == "scalar"
    x, cos, sin = rp.exact_probe(B, T, nh, hd, rd, _g(3))
    cos, sin = cos[:T].to(DEV), sin[:T].to(DEV)
    aligned = x.to(dtype).to(DEV)
    kernels.rotary_inplace(aligned, cos, sin, B, T, nh, hd, rd)
    assert _bits(aligned, rp.rotate(x, cos.cpu(), sin.cpu(), rd).to(dtype))
    for which in ("qkv", "cos", "sin"):
        q = _offset_view(x.to(dtype).to(DEV), 1) if which == "qkv" else x.to(dtype).to(DEV)
        c = _offset_view(cos, 1) if which == "cos" else cos
        s = _offset_view(sin, 1) if which == "sin" else sin
        assert (q.data_ptr() | c.data_ptr() | s.data_ptr()) % 16 != 0
        kernels.rotary_inplace(q, c, s, B, T, nh, hd, rd)
        torch.cuda.synchronize()
        assert _bits(q, aligned), which


def test_rotary_refuses_malformed_arguments():
    B, T, nh, hd, rd = 1, 5, 4, 64, 32
    x, cos, sin = rp.exact_probe(B, T, nh, hd, rd, _g(4))
    qkv = x.to(torch.bfloat16).to(DEV)
    before = qkv.clone()
    c, s = cos[:T].to(DEV), sin[:T].to(DEV)
    c6 = cos[:T + 1].to(DEV)
    bad = {
        "bf16 cos": (qkv, c.to(torch.bfloat16), s, B, T, nh, hd, rd),
        "short cos": (qkv, c[:T - 1], s, B, T, nh, hd, rd),
        "wide sin": (qkv, c, torch.zeros(T, rd // 2 + 1, device=DEV), B, T, nh, hd, rd),
        "short sin": (qkv, c, s[:T - 1], B, T, nh, hd, rd),
        "qkv too small": (qkv, c6, c6, B, T + 1, nh, hd, rd),
        "odd rd": (qkv, c[:, :15].contiguous(), s[:, :15].contiguous(), B, T, nh, hd, 31),
        "rd 0": (qkv, torch.zeros(T, 0, device=DEV), torch.zeros(T, 0, device=DEV), B, T, nh, hd, 0),
        "rd > hd": (qkv, torch.zeros(T, 33, device=DEV), torch.zeros(T, 33, device=DEV), B, T, nh, hd, 66),
    }
    torch.cuda.synchronize()
    n0 = kernels.launches()
    for name, args in bad.items():
        with pytest.raises(_lib.PsalmKernelError):
            kernels.rotary_inplace(*args)
        assert kernels.launches() == n0, name
    torch.cuda.synchronize()
    assert _bits(qkv, before)


# ---------------------------------------------------------------------------------------------------------------
# rotary composed with attention (quarter-turn tables: rotation is exact and invertible)
# ---------------------------------------------------------------------------------------------------------------
IMPLS = {"bf16": ("auto", "simt"), "f16": ("auto", "simt"), "f32": ("simt",)}   # fp32 always runs the SIMT kernels
ATTN = {"auto": 0, "simt": 1}


def _attn_check(tag, out_z, pb, dtype, hd, intended):
    ref = ap.attend(pb)
    assert float(ap.intended_weight(ref, intended.to(ref["w"].device)).min()) >= 0.99
    _report(tag, ap.ratio(out_z, ref, ap.bound(ref, dtype, hd)))


@pytest.mark.parametrize("dt", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("case", CAUSAL_CASES, ids=lambda c: "B%d_T%d_nh%d_pad%d" % c)
def test_prefill_chain(case, dt):
    B, T, nh, padded = case
    hd, rd, dtype = 64, 32, DT[dt]
    post, kv, intended = rp.causal_chain_probe(B, T, nh, hd, rd, padded, _g(T * 5 + padded))
    post = post.to(dtype)
    cos, sin = rp.quarter_tables(T, rd, _g(T))
    x = rp.unrotate(post, cos, sin, rd).to(dtype)
    kv_g = kv.to(DEV) if kv is not None else None
    pb = ap.causal_problem(post, kv, B, T, nh, hd)
    for impl in IMPLS[dt]:
        qkv = x.to(DEV, copy=True)
        kernels.rotary_inplace(qkv, cos.to(DEV), sin.to(DEV), B, T, nh, hd, rd)
        assert _same(qkv, post)
        with _attn_impl(ATTN[impl]):
            out = kernels.causal_attention(qkv, kv_g, B, T, nh, hd)
            torch.cuda.synchronize()
        _attn_check("prefill %s %s %s" % (case, dt, impl), ap.heads_out_z(out, B, T, nh, hd), pb, dtype, hd, intended)


@pytest.mark.parametrize("dt", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("shape", [(2, 17, 4), (1, 160, 32)], ids=lambda s: "B%d_T%d_nh%d" % s)
@pytest.mark.parametrize("P", PREFIX_PS)
def test_prompt_suffix_chain(P, shape, dt):
    B, T, nh = shape
    hd, rd, dtype = 64, 32, DT[dt]
    post, pk, pv, intended = rp.prefix_chain_probe(B, P, T, nh, hd, rd, _g(P * 3 + T))
    post, pk, pv = post.to(dtype), pk.to(dtype), pv.to(dtype)
    cos, sin = rp.quarter_tables(P + T, rd, _g(P + T))
    pre, suf = rp.prefix_inputs(post.double(), pk.double(), pv.double(), P, cos, sin, rd)
    cos_g, sin_g = cos.to(DEV), sin.to(DEV)
    page = pk.shape[1]
    # the one-page prefix cache: rows P.. hold the probe's poison; rows < P start as a constant the writes replace
    kc = pk.unsqueeze(0).to(DEV)
    vc = pv.unsqueeze(0).to(DEV)
    kc[:, :, :P] = -7.0
    vc[:, :, :P] = -7.0
    pre_g = pre.to(dtype).to(DEV)
    kernels.rotary_inplace(pre_g, cos_g[:P], sin_g[:P], 1, P, nh, hd, rd)
    zero = torch.zeros(1, dtype=torch.int32, device=DEV)
    kernels.kv_cache_write(pre_g, kc, vc, zero.view(1, 1), zero)
    assert page == -(-P // 64) * 64
    assert _same(kc[0], pk) and _same(vc[0], pv)
    pb = ap.prefix_problem(post, pk, pv, P, None, B, T, nh, hd)
    for impl in IMPLS[dt]:
        qkv = suf.to(dtype).to(DEV)
        kernels.rotary_inplace(qkv, cos_g[P:].contiguous(), sin_g[P:].contiguous(), B, T, nh, hd, rd)
        assert _same(qkv, post)
        with _attn_impl(ATTN[impl]):
            out = kernels.prefix_causal_attention(qkv, kc[0], vc[0], P, None, B, T, nh, hd)
            torch.cuda.synchronize()
        _attn_check("suffix P%d %s %s %s" % (P, shape, dt, impl), ap.heads_out_z(out, B, T, nh, hd), pb, dtype, hd,
                    intended)


@pytest.mark.parametrize("dt", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("case", DECODE_CASES, ids=lambda c: "ps%d_%s" % (c[1], "_".join(map(str, c[0]))))
def test_decode_chain(case, dt):
    lens, ps = case
    nh, hd, rd, dtype = 8, 64, 32, DT[dt]
    B = len(lens)
    q, kc, vc, bt, intended = rp.decode_chain_probe(lens, nh, hd, rd, ps, _g(ps + sum(lens)))
    q, kc, vc = q.to(dtype), kc.to(dtype), vc.to(dtype)
    cos, sin = rp.quarter_tables(max(lens) + 1, rd, _g(ps))
    pres, new = rp.decode_inputs(q.double(), kc.double(), vc.double(), bt, lens, cos, sin, rd)
    cos_g, sin_g, bt_g = cos.to(DEV), sin.to(DEV), bt.to(DEV)
    # the cache starts with only the lure slots seq_len + 1 written; every slot the chain writes holds -7
    kc_g, vc_g = kc.to(DEV), vc.to(DEV)
    for b, L in enumerate(lens):
        pos = torch.arange(L + 1)
        pg, sl = bt[b, pos // ps].long().to(DEV), (pos % ps).to(DEV)
        kc_g[pg, :, sl] = -7.0
        vc_g[pg, :, sl] = -7.0
    zero = torch.zeros(1, dtype=torch.int32, device=DEV)
    for b, L in enumerate(lens):                        # prefill of each sequence at rows 0..L-1
        pre = pres[b].to(dtype).to(DEV)
        kernels.rotary_inplace(pre, cos_g[:L], sin_g[:L], 1, L, nh, hd, rd)
        kernels.kv_cache_write(pre, kc_g, vc_g, bt_g[b:b + 1], zero)
    qkv = new.to(dtype).to(DEV)
    seq = torch.tensor(lens, dtype=torch.int32, device=DEV)
    if len(set(lens)) == 1:                             # one call for the batch, as PhiModel.decode_step makes it
        L = lens[0]
        kernels.rotary_inplace(qkv, cos_g[L:L + 1].contiguous(), sin_g[L:L + 1].contiguous(), B, 1, nh, hd, rd)
    else:
        for b, L in enumerate(lens):
            kernels.rotary_inplace(qkv[b:b + 1], cos_g[L:L + 1], sin_g[L:L + 1], 1, 1, nh, hd, rd)
    kernels.kv_cache_write(qkv, kc_g, vc_g, bt_g, seq)
    assert _same(qkv[:, 0, 0], q)
    assert _same(kc_g, kc) and _same(vc_g, vc)
    out = kernels.paged_decode_attention(qkv, kc_g, vc_g, bt_g, seq + 1)
    torch.cuda.synchronize()
    post_new = torch.zeros(B, 1, 3, nh, hd, dtype=dtype)
    post_new[:, 0, 0] = q
    pb = ap.decode_problem(post_new, kc, vc, bt, seq.cpu() + 1)
    _attn_check("decode %s %s" % (case, dt), out.to(torch.float64).view(B * nh, 1, hd), pb, dtype, hd, intended)


# ---------------------------------------------------------------------------------------------------------------
# linear_act
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("case", ACT_CASES, ids=lambda c: "M%d_N%d_K%d_%s" % c)
def test_linear_act_probe(case, dt):
    M, N, K, act = case
    dtype = DT[dt]
    x, w, b = rp.act_probe(M, N, K)
    out = kernels.linear_act(x.to(dtype).to(DEV), w.to(dtype).to(DEV), b.to(dtype).to(DEV), act)
    torch.cuda.synchronize()
    kidx = (37 * torch.arange(M)) % K
    z = (w[:, kidx].t() + b).to(DEV)                   # the exact pre-activation: one product per output
    o = out.to(torch.float64)
    assert torch.isfinite(o).all()
    if act == "relu":
        assert torch.equal(o, z.clamp(min=0)), "relu %s %s" % (case, dt)
    else:
        g = rp.gelu_new(z)
        _report("linear_act %s %s" % (case, dt), float(((o - g).abs() / rp.gelu_bound(z, g, dtype)).max()))


# ---------------------------------------------------------------------------------------------------------------
# the rows each Phi entry point hands the rotary kernel
# ---------------------------------------------------------------------------------------------------------------
def test_phi_entry_points_rotate_at_their_positions(monkeypatch):
    """PhiModel.forward rotates at rows 0..T-1, forward_suffix behind a P-row prefix at P..P+T-1, decode_step at the
    cache length: every call of every layer gets exactly those rows of the Phi tables."""
    from psalm_b200.generate import PagedKVCache
    from psalm_b200.layout import PhiConfig
    from psalm_b200.phi import PhiModel
    C, inter, nh, layers = 256, 512, 4, 2
    cfg = PhiConfig(hidden=C, layers=layers, heads=nh, inter=inter, vocab=16)
    g = _g(9)
    sd = {"model.embed_tokens.weight": torch.randn(16, C, generator=g)}

    def lin(name, o, i):
        sd[name + ".weight"] = torch.randn(o, i, generator=g) * 0.05
        sd[name + ".bias"] = torch.randn(o, generator=g) * 0.05

    def norm(name):
        sd[name + ".weight"], sd[name + ".bias"] = torch.ones(C), torch.zeros(C)

    for i in range(layers):
        p = "model.layers.%d." % i
        for n in ("q_proj", "k_proj", "v_proj", "dense"):
            lin(p + "self_attn." + n, C, C)
        lin(p + "mlp.fc1", inter, C)
        lin(p + "mlp.fc2", C, inter)
        norm(p + "input_layernorm")
    norm("model.final_layernorm")
    model = PhiModel(sd, cfg=cfg, dtype=torch.bfloat16, device="cuda")
    seen, real = [], kernels.rotary_inplace

    def spy(qkv, cos, sin, B, T, nh_, hd, rd):
        seen.append((cos.cpu(), sin.cpu()))
        real(qkv, cos, sin, B, T, nh_, hd, rd)

    monkeypatch.setattr(kernels, "rotary_inplace", spy)
    P, T, rd = 70, 9, cfg.head_dim // 2
    cos, sin = rp.phi_tables(P + T, rd)

    def expect(lo, hi):
        assert len(seen) == layers
        for c, s in seen:
            assert _bits(c, cos[lo:hi]) and _bits(s, sin[lo:hi]), (lo, hi)
        seen.clear()

    x = lambda B, L: torch.randn(B, L, C, generator=g).to(torch.bfloat16).cuda()   # noqa: E731
    prefix = PagedKVCache(cfg, 1, 128, torch.bfloat16, "cuda", page_size=128)      # one page, as psalm.py builds it
    model.forward(x(1, P), None, cache=prefix)
    prefix.length = P
    expect(0, P)
    model.forward_suffix(x(2, T), prefix)
    expect(P, P + T)
    cache = PagedKVCache(cfg, 2, 32, torch.bfloat16, "cuda", page_size=16)
    model.forward(x(2, 5), None, cache=cache)
    cache.advance(5)
    expect(0, 5)
    model.decode_step(x(2, 1), cache)
    expect(5, 6)
    torch.cuda.synchronize()
