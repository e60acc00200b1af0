"""Attention kernels on the probes of tests/attn_probe.py, against its float64 references and per-element bound.

Every case runs under each implementation selector that changes what it runs (psalm_set_attention_impl 0-3,
psalm_set_cross_impl 0-2, psalm_set_causal_impl 1), always restored in `finally`.  A case passes when every compared output is finite and
max |out - ref| / bound <= 1 (the bound and its constants: tests/attn_probe.py).  Largest err / bound observed on an
NVIDIA H100 80GB HBM3 (700 W power limit), over every case and selector of this file (the 16-bit figures are the
same under the tensor-core and SIMT selectors; fp32 storage always runs the SIMT kernels):
  window attention          bf16 0.153   fp16 0.167   fp32 0.398
  causal attention          bf16 0.100   fp16 0.156   fp32 0.105
  prefix-causal attention   bf16 0.008   fp16 0.062   fp32 0.026
  cross_attention           bf16 0.160   fp16 0.154   fp32 0.261
  masked, per-head kernel   bf16 0.160   fp16 0.157
  masked, TMA kernel        bf16 0.027   fp16 0.025
  paged decode              bf16 0.039   fp16 0.154   fp32 0.007
The whole file runs in about 1 min 55 s on that GPU.
"""
import contextlib

import pytest
import torch

import attn_probe as ap
from psalm_b200 import _lib, kernels

pytestmark = pytest.mark.gpu
DT = {"bf16": torch.bfloat16, "f16": torch.float16, "f32": torch.float32}
ATTN = {"auto": 0, "simt": 1, "mma-workspace": 2, "mma-cluster": 3}


@contextlib.contextmanager
def _selector(name, value):
    fn = getattr(_lib.lib(), name)
    _lib.check(fn(value), name)
    try:
        yield
    finally:
        fn(0)


def _check(tag, out_z, ref, bnd, rows=None, intended=None, pb_rows=None):
    if intended is not None:
        w = ap.intended_weight(ref, intended)
        if rows is not None:
            w = w[rows]
        assert float(w.min()) >= 0.99, (tag, float(w.min()))
    r = ap.ratio(out_z, ref, bnd, rows)
    print("PROBE %s err/bound %.4f" % (tag, r))
    assert r <= 1.0, "%s: max err / bound = %.3f" % (tag, r)


def _g(seed):
    return torch.Generator().manual_seed(seed)


# ---------------------------------------------------------------------------------------------------------------
# window attention (ws 12, hd 32): the head-pipelined tensor-core kernel at HPC = 1, 2 and 4, and the SIMT kernel
# ---------------------------------------------------------------------------------------------------------------
WINDOW_SHAPES = [  # B, H, W, C, nh, heads per CTA of launch_window
    (1, 24, 36, 128, 4, 1),
    (2, 30, 26, 64, 2, 1),
    (1, 256, 256, 128, 4, 2),        # Swin-B stage 0 at 1024^2
    (2, 256, 256, 128, 4, 4),
    (1, 128, 128, 256, 8, 2),        # stage 1
    (1, 64, 64, 512, 16, 2),         # stage 2
    (1, 32, 32, 1024, 32, 2),        # stage 3
    (1, 334, 334, 128, 4, 4),        # stage 0 at 1333^2: padded to 336
]


def test_window_shapes_cover_every_heads_per_cta():
    assert {s[-1] for s in WINDOW_SHAPES} == {1, 2, 4}
    for B, H, W, C, nh, hpc in WINDOW_SHAPES:
        assert ap.window_hpc(B, H, W, nh) == hpc


@pytest.mark.parametrize("impl", ["auto", "simt"])   # selectors 2 / 3 only change split-K, which this kernel lacks
@pytest.mark.parametrize("dt", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("shape", WINDOW_SHAPES, ids=lambda s: "B%dx%dx%d_C%d_nh%d_hpc%d" % s)
def test_window_attention_probe(shape, dt, impl):
    B, H, W, C, nh, hpc = shape
    if dt == "f32" and impl == "auto":
        pytest.skip("fp32 storage runs the SIMT kernel under both selectors")
    ws, dtype = 12, DT[dt]
    for shift in (0, 6):
        qkv, bias, rel, _ = ap.window_probe(B, H, W, C, nh, ws, shift, dtype, _g(H * 7 + nh + shift))
        with _selector("psalm_set_attention_impl", ATTN[impl]):
            out = kernels.window_attention(qkv.cuda(), bias.cuda(), rel.cuda(), B, H, W, C, nh, ws, shift)
            torch.cuda.synchronize()
        pb = ap.window_problem(qkv, bias, rel, B, H, W, C, nh, ws, shift)
        ref = ap.attend(pb)
        bnd = ap.bound(ref, dtype, C // nh)
        _check("window %s %s shift%d %s" % (shape, dt, shift, impl), ap.window_out_z(out, pb), ref, bnd, pb["rows"],
               pb["bias"].argmax(-1))


# ---------------------------------------------------------------------------------------------------------------
# causal prefill (hd 64): mma.sync flash kernel (KG = 1 and 2) and the SIMT kernel
# ---------------------------------------------------------------------------------------------------------------
# psalm_set_causal_impl 1 and 2 both select the same mma.sync flash kernel on sm_90a (the selector only validates its
# argument), so one of them is run; the flash kernel's one / two key groups per CTA follow from T (two once a CTA walks
# more than two 64-key tiles), which the T sweep covers.
CAUSAL_IMPLS = [("mma", 1), ("simt", 1)]


@pytest.mark.parametrize("impl", CAUSAL_IMPLS, ids=lambda p: "%s-c%d" % p)
@pytest.mark.parametrize("dt", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("padded", [False, True])
@pytest.mark.parametrize("T", [1, 63, 64, 65, 128, 129, 900, 1100, 2048])
def test_causal_attention_probe(T, padded, dt, impl):
    if dt == "f32" and impl[0] == "mma":
        pytest.skip("fp32 storage always runs the SIMT kernel")
    nh = 32 if T in (900, 2048) else 4                 # Phi-1.5's 32 heads, and a small head count
    B, hd, dtype = (2 if padded else 1), 64, DT[dt]
    qkv, kv, intended = ap.causal_probe(B, T, nh, hd, padded, _g(T * 3 + padded))
    qkv = qkv.to(dtype)
    with _selector("psalm_set_attention_impl", ATTN["simt" if impl[0] == "simt" else "auto"]), \
            _selector("psalm_set_causal_impl", impl[1]):
        out = kernels.causal_attention(qkv.cuda(), kv.cuda() if kv is not None else None, B, T, nh, hd)
        torch.cuda.synchronize()
    pb = ap.causal_problem(qkv, kv, B, T, nh, hd)
    ref = ap.attend(pb)
    _check("causal T%d pad%d %s %s" % (T, padded, dt, impl), ap.heads_out_z(out, B, T, nh, hd), ref,
           ap.bound(ref, dtype, hd), intended=intended)


# ---------------------------------------------------------------------------------------------------------------
# prefix-causal prefill: rows P..ld_rows-1 of the prefix buffer are poison
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", ["auto", "simt"])
@pytest.mark.parametrize("dt", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("T", [1, 17, 64, 160])
@pytest.mark.parametrize("P", [1, 63, 64, 65, 290])
def test_prefix_causal_attention_probe(P, T, dt, impl):
    if dt == "f32" and impl == "auto":
        pytest.skip("fp32 storage runs the SIMT kernel under both selectors")
    B, nh, hd, dtype = 2, 4, 64, DT[dt]
    qkv, pk, pv, ld, intended = ap.prefix_probe(B, P, T, nh, hd, _g(P * 11 + T))
    qkv, pk, pv = qkv.to(dtype), pk.to(dtype), pv.to(dtype)
    with _selector("psalm_set_attention_impl", ATTN[impl]):
        out = kernels.prefix_causal_attention(qkv.cuda(), pk.cuda(), pv.cuda(), P, None, B, T, nh, hd)
        torch.cuda.synchronize()
    pb = ap.prefix_problem(qkv, pk, pv, P, None, B, T, nh, hd)
    ref = ap.attend(pb)
    _check("prefix P%d T%d %s %s" % (P, T, dt, impl), ap.heads_out_z(out, B, T, nh, hd), ref, ap.bound(ref, dtype, hd),
           intended=intended)


# ---------------------------------------------------------------------------------------------------------------
# cross attention with packed bit masks
# ---------------------------------------------------------------------------------------------------------------
def _flash_boundaries(Lk, splits, tile=64):
    nt = -(-Lk // tile)
    tps = -(-nt // splits)
    return [sp * tps * tile for sp in range(1, splits) if sp * tps * tile < Lk]


def _tma_boundaries(B, Lk, sms=132):
    """Split boundaries of the TMA kernel (restates xa_splits in csrc/xattn_tma.cu for an H100's 132 SMs)."""
    steps = -(-Lk // 32)
    s = min(2 * sms // (2 * B), (steps + 3) // 4)
    s = max(s, 1, -(-steps // 16))
    per = -(-steps // s)
    return [i * per * 32 for i in range(1, -(-steps // per))]


def _thin(xs, n=8):
    """At most n boundaries (the probe has hd - 4 designated keys): spread over the list."""
    if len(xs) <= n:
        return xs
    return [xs[int(i * (len(xs) - 1) / (n - 1))] for i in range(n)]


CROSS_CASES = [  # B, Lq, Lk, splits
    (2, 100, 100, 1), (1, 37, 31, 1), (2, 65, 389, 3), (5, 64, 2047, 4), (1, 112, 2048, 16), (2, 100, 4096 + 31, 19),
    (1, 1, 16384, 16), (2, 100, 27889, 4),
]


@pytest.mark.parametrize("impl", list(ATTN))
@pytest.mark.parametrize("dt", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("case", CROSS_CASES, ids=lambda c: "B%d_Lq%d_Lk%d_s%d" % c)
def test_cross_attention_probe(case, dt, impl):
    if dt == "f32" and impl not in ("auto", "simt"):
        pytest.skip("fp32 storage runs the SIMT kernel")
    if dt == "f32" and impl == "auto":
        pytest.skip("fp32 storage runs the SIMT kernel under both selectors")
    B, Lq, Lk, splits = case
    dtype = DT[dt]
    q, k, v, bits, ro, intended = ap.cross_probe(B, Lq, Lk, _g(Lk + Lq), boundaries=_thin(_flash_boundaries(Lk, splits)))
    q, k, v = q.to(dtype), k.to(dtype), v.to(dtype)
    with _selector("psalm_set_attention_impl", ATTN[impl]):
        out = kernels.cross_attention(q.cuda(), k.cuda(), v.cuda(), bits.cuda(), ro.cuda(), 8, splits=splits)
        torch.cuda.synchronize()
    pb = ap.cross_problem(q, k, v, bits, ro, 8)
    ref = ap.attend(pb)
    _check("cross %s %s %s" % (case, dt, impl), ap.heads_out_z(out, B, Lq, 8, 32), ref, ap.bound(ref, dtype, 32),
           intended=intended)


MASKED_CASES = [  # B, Lq, Lk, K / V row stride, stride-0 batch
    (1, 100, 31, 256, False), (2, 37, 100, 768, False), (5, 65, 389, 256, False), (2, 112, 2047, 768, False),
    (1, 64, 2048, 256, False), (2, 100, 4096 + 31, 768, False), (1, 1, 16384, 256, False), (2, 100, 27889, 768, False),
    (5, 100, 6400 + 17, 256, False), (3, 100, 4096 + 31, 256, True), (4, 100, 389, 768, True),
]


@pytest.mark.parametrize("cross", [0, 1, 2])
@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("case", MASKED_CASES, ids=lambda c: "B%d_Lq%d_Lk%d_ld%d%s" % (c[:4] + ("_shared" if c[4] else "",)))
def test_masked_cross_attention_probe(case, dt, cross):
    """Per-head flash kernel (auto below 2048 keys) and the TMA-fed kernel: K / V are row-strided views of buffers
    whose other columns hold NaN; with B > 1 image b+1's first rows lure image b; stride-0 batches share one K / V.
    The probe has hd - 4 = 28 key directions, so at most 8 split boundaries (spread over the kernel's list by _thin)
    get a one-open-key row on each side: at 27889 keys the TMA kernel has 63 splits and most of their boundaries are
    not probed.  The Lq = 1 case has a single all-open row (it intends key 0): it checks the grid and the combine at
    16384 keys, not boundaries, tails or masks."""
    B, Lq, Lk, ld, shared = case
    dtype = DT[dt]
    tma = cross != 0 or Lk >= 2048
    bnds = _tma_boundaries(B, Lk) if tma else _flash_boundaries(Lk, kernels_small_splits(B, Lk))
    q, k, v, bits, ro, intended = ap.cross_probe(B, Lq, Lk, _g(Lk * 3 + Lq), boundaries=_thin(bnds), shared_kv=shared)
    q, k, v = q.to(dtype), k.to(dtype), v.to(dtype)
    nb = k.shape[0]
    off = 0 if ld == 256 else 256
    kbuf = torch.full((nb, Lk, ld), float("nan"), dtype=dtype)
    vbuf = torch.full((nb, Lk, ld), float("nan"), dtype=dtype)
    kbuf[:, :, off:off + 256], vbuf[:, :, off:off + 256] = k, v
    kg, vg = kbuf.cuda()[:, :, off:off + 256], vbuf.cuda()[:, :, off:off + 256]
    if shared:
        kg, vg = kg.expand(B, Lk, 256), vg.expand(B, Lk, 256)
    with _selector("psalm_set_cross_impl", cross):
        out = kernels.masked_cross_attention(q.cuda(), kg, vg, bits.cuda(), ro.cuda(), 8)
        torch.cuda.synchronize()
    pb = ap.cross_problem(q, k.expand(B, Lk, 256), v.expand(B, Lk, 256), bits, ro, 8)
    ref = ap.attend(pb)
    _check("masked %s %s cross%d" % (case, dt, cross), ap.heads_out_z(out, B, Lq, 8, 32), ref,
           ap.bound(ref, dtype, 32, q_rounded=tma), intended=intended)


def kernels_small_splits(B, Lk):
    """Split count of the per-head kernel behind masked_cross_attention below 2048 keys (restates small_splits)."""
    want = -(-2 * 132 // (B * 16))
    return max(1, min(want, (Lk + 255) // 256, 16))


# ---------------------------------------------------------------------------------------------------------------
# paged decode
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("ps", [4, 8, 16])
@pytest.mark.parametrize("hd", [32, 64])
def test_paged_decode_attention_probe(hd, ps, dt):
    lens, nh, dtype = [1, 31, 32, 33, 127, 128, 129, 921, 2048], 8, DT[dt]
    qkv, kc, vc, bt, seq, intended = ap.decode_probe(lens, nh, hd, ps, _g(hd * 10 + ps))
    qkv, kc, vc = qkv.to(dtype), kc.to(dtype), vc.to(dtype)
    out = kernels.paged_decode_attention(qkv.cuda(), kc.cuda(), vc.cuda(), bt.cuda(), seq.cuda())
    torch.cuda.synchronize()
    pb = ap.decode_problem(qkv, kc, vc, bt, seq)
    ref = ap.attend(pb)
    _check("decode hd%d ps%d %s" % (hd, ps, dt), out.to(torch.float64).view(len(lens) * nh, 1, hd), ref,
           ap.bound(ref, dtype, hd), intended=intended)
