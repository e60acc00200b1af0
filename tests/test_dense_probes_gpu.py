"""Dense kernels on the probes of tests/dense_probe.py: the wgmma linear kernel, every mask projection path, the mask
bits, add_layernorm, patch_merge_layernorm and groupnorm_tokens.

The exact probes (linear_fused, mask_logits, mask_bits, attn_mask_bits) must equal the float64 reference rounded once
to storage, bit for bit; every output buffer is poisoned with NaN / all-ones bits before the call, so an unwritten
element shows.  The float64 probes (the norms) must stay within the per-element bound of tests/dense_probe.py, and
constant LayerNorm rows must give the bias exactly.  The mask projection runs under each psalm_set_mask_proj_impl
selector (0 auto, 1 mma.sync, 2 wgmma), restored in `finally`.

Largest err / bound observed on an NVIDIA H100 80GB HBM3 (700 W power limit), over every case of this file:
  linear_fused GELU epilogue                       0.840 (every other linear / mask output: bit-exact)
  add_layernorm                  bf16 0.996   fp16 0.994   fp32 0.453
  patch_merge_layernorm          0.996 over all types
  groupnorm_tokens               bf16 0.996   fp16 0.997   fp32 0.817
The 16-bit figures sit at the output rounding u |y|.  The earlier groupnorm_tokens (fp32 sums of x and x^2, then
E[x^2] - mean^2) failed this file's GroupNorm probes from mean / std 10 on, in every storage type: fp32 by 35x at
mean / std 10, 388x at 30 and 15766x at 300.  The whole file runs in about 2 min 10 s on that GPU."""
import contextlib
import math

import pytest
import torch

import dense_probe as dp
from psalm_b200 import _lib, kernels

pytestmark = pytest.mark.gpu
DT = {"bf16": torch.bfloat16, "f16": torch.float16, "f32": torch.float32}
CUDA = torch.device("cuda")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@contextlib.contextmanager
def _poisoned(*shapes_dtypes):
    """Fill the allocator's next blocks of these sizes with 0xFF bytes (NaN in every float type, all bits set in
    the integer outputs), so that the kernel under test must overwrite every element it owns."""
    blocks = [torch.full((math.prod(s) * torch.empty((), dtype=d).element_size(),), 255, dtype=torch.uint8, device=CUDA)
              for s, d in shapes_dtypes]
    ptrs = {b.data_ptr() for b in blocks}
    del blocks
    yield ptrs


def _check_poisoned(t, ptrs):
    assert t.data_ptr() in ptrs, "the output did not reuse the poisoned block"


@contextlib.contextmanager
def _mask_proj_impl(v):
    fn = _lib.lib().psalm_set_mask_proj_impl
    _lib.check(fn(v), "psalm_set_mask_proj_impl")
    try:
        yield
    finally:
        fn(0)


def _dev(*ts):
    return [None if t is None else t.to(CUDA) for t in ts]


# ---------------------------------------------------------------------------------------------------------------
# linear_fused
# ---------------------------------------------------------------------------------------------------------------
def _run_linear(a, w, b, dtype, epilogue="bias", S=0, x=None):
    """linear_fused on storage copies of float64 operands, output poisoned first."""
    x = a.to(dtype) if x is None else x
    wt, bt = w.to(dtype), (None if b is None else b.to(dtype))
    M, N = a.shape[0], w.shape[0]
    shape = (M // S, N // 32, S, 32) if epilogue == "head_major" else (M, N)
    with _poisoned((shape, dtype)) as ptrs:
        out = kernels.linear_fused(x, wt, bt, epilogue, S)
    _check_poisoned(out, ptrs)
    return out


def _exact_linear(a, w, b, dtype, tag):
    a, w, b = _dev(a, w, b)
    out = _run_linear(a, w, b, dtype)
    ref = dp.stored(dp.linear_ref(a, w, b), dtype)
    assert dp.same(out, ref), "%s: %d elements differ" % (tag, int((out.double() != ref).sum()))


def _gelu_linear(a, w, b, dtype, tag):
    a, w, b = _dev(a, w, b)
    out = _run_linear(a, w, b, dtype, "gelu_erf")
    g = dp.gelu(dp.linear_ref(a, w, b))
    r = dp.ratio(out, g.cpu(), dp.gelu_bound(g, dtype).cpu())
    print("PROBE %s gelu err/bound %.4f" % (tag, r))
    assert r <= 1.0, (tag, r)


@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("kblocks", [1, 2, 3, 4, 5])
def test_linear_more_tiles_than_sms(dt, kblocks):
    """Every CTA runs >= 2 tiles, so the 3-stage ring wraps at every phase alignment of kblocks against 3."""
    dtype, K, N = DT[dt], 64 * kblocks, 256
    M = 2 * _sms() * 128 + 37                                     # ragged last tile
    assert -(-M // 128) * (N // 256) >= 2 * _sms()
    tag = "linear M%d N%d K%d %s" % (M, N, K, dt)
    _exact_linear(*dp.address_probe(M, N, K), dtype, tag + " address")
    _exact_linear(*dp.dense_probe(M, N, K, torch.Generator().manual_seed(kblocks)), dtype, tag + " dense")
    _gelu_linear(*dp.address_probe(M, N, K, scale=2.0 ** -4), dtype, tag)


@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("N", [256, 1024, 4096])
@pytest.mark.parametrize("M", [1, 63, 64, 65, 127, 129])
def test_linear_small_m(dt, N, M):
    dtype, K = DT[dt], 192
    tag = "linear M%d N%d K%d %s" % (M, N, K, dt)
    _exact_linear(*dp.address_probe(M, N, K), dtype, tag + " address")
    _exact_linear(*dp.dense_probe(M, N, K, torch.Generator().manual_seed(M + N)), dtype, tag + " dense")
    if N == 1024:
        _gelu_linear(*dp.address_probe(M, N, K, scale=2.0 ** -4), dtype, tag)


@pytest.mark.parametrize("dt", ["bf16", "f16"])
def test_linear_dense_k1024(dt):
    a, w, b = dp.dense_probe(777, 1024, 1024, torch.Generator().manual_seed(3))
    _exact_linear(a, w, b, DT[dt], "linear dense K1024 " + dt)
    _exact_linear(dp.address_a(777, 1024), dp.w_code(1024, 1024), None, DT[dt], "linear address K1024 no bias " + dt)


@pytest.mark.parametrize("dt", ["bf16", "f16"])
def test_linear_row_strided_view(dt):
    dtype = DT[dt]
    M, N, K = 1000, 512, 128
    a, w, b = _dev(*dp.address_probe(M, N, K))
    wide = torch.full((M, 384), float("nan"), dtype=dtype, device=CUDA)      # neighbouring columns must not be read
    wide[:, 128:256] = a.to(dtype)
    out = _run_linear(a, w, b, dtype, x=wide[:, 128:256])
    assert dp.same(out, dp.stored(dp.linear_ref(a, w, b), dtype))


@pytest.mark.parametrize("dt", ["bf16", "f16"])
def test_linear_head_major_lands_at_image_head_row(dt):
    """S % 128 != 0 (tiles straddle images), two column tiles of 8 heads, more tiles than SMs."""
    dtype, S, N, K = DT[dt], 2720, 512, 192
    B = -(-2 * _sms() * 128 // S) + 1
    a, w, b = _dev(*dp.address_probe(B * S, N, K))
    assert kernels.linear_fused_supported(a.to(dtype), w.to(dtype), "head_major", S)
    out = _run_linear(a, w, b, dtype, "head_major", S)
    ref = dp.head_major(dp.stored(dp.linear_ref(a, w, b), dtype), S)
    assert out.shape == (B, N // 32, S, 32)
    assert dp.same(out, ref)


# ---------------------------------------------------------------------------------------------------------------
# mask projection: every path, exact
# ---------------------------------------------------------------------------------------------------------------
MP_Q = [1, 7, 100, 112, 128]
MP_P = [32, 130, 389, 4096 + 96, 8192, 65536]


def _mask_logits(me, feats, dtype, out_dtype):
    B, Q, _ = me.shape
    P = feats.shape[1]
    m, f = me.to(dtype), feats.to(dtype)
    if f.shape[0] == 1 and B > 1:
        f = f.expand(B, P, f.shape[2])                            # stride-0 view of one image's map
    with _poisoned(((B, Q, P), out_dtype)) as ptrs:
        out = kernels.mask_logits(m, f, out_dtype=out_dtype)
    _check_poisoned(out, ptrs)
    return out


@pytest.mark.parametrize("impl", [0, 1, 2])
@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("P", MP_P)
def test_mask_logits_paths_exact(impl, dt, P):
    dtype = DT[dt]
    probes = {}
    for shared in (False, True):
        B = 3 if shared else 2
        probes[shared, "address"] = _dev(*dp.mask_proj_probe(B, max(MP_Q), P, shared=shared, bits_rows=False))
        me, feats = _dev(*dp.mask_proj_dense(B, max(MP_Q), P, torch.Generator().manual_seed(P + shared)))
        probes[shared, "dense"] = (me, feats[:1] if shared else feats)
    with _mask_proj_impl(impl):
        for Q in MP_Q:
            for shared in (False, True):
                for probe in ("address", "dense"):
                    me, feats = probes[shared, probe]
                    me = me[:, :Q].contiguous()                   # query q's row does not depend on Q
                    ref = dp.mask_logits_ref(me, feats)
                    for out_dtype in (dtype, torch.float32):
                        out = _mask_logits(me, feats, dtype, out_dtype)
                        tag = "impl %d %s Q%d P%d shared %d %s out %s" % (impl, dt, Q, P, shared, probe, out_dtype)
                        assert dp.same(out, dp.stored(ref, out_dtype)), tag


@pytest.mark.parametrize("P", [32, 130, 389, 4096 + 96])
def test_mask_logits_fp32_simt_exact(P):
    for Q in (1, 7, 100, 128):
        for C in (256, 80):                                       # 80: a partial 32-wide K chunk
            me, feats = _dev(*dp.mask_proj_probe(2, Q, P, C=C, bits_rows=False))
            out = _mask_logits(me, feats, torch.float32, torch.float32)
            assert dp.same(out, dp.mask_logits_ref(me, feats)), (Q, P, C)


# ---------------------------------------------------------------------------------------------------------------
# mask bits: logit < 0 blocks, 0 is open, bits past P are 0, row_open = every valid key blocked
# ---------------------------------------------------------------------------------------------------------------
def _bits_call(fn, B, Q, P, *args, poison_checked=True):
    """poison_checked = False where the call also allocates an intermediate (mask_bits through fp32 logits), which may
    take a poisoned block first; attn_mask_bits itself is checked directly."""
    W32 = (P + 31) // 32
    with _poisoned(((B, Q, W32), torch.int32), ((B, Q), torch.uint8)) as ptrs:
        bits, ro = fn(*args)
    if poison_checked:
        _check_poisoned(bits, ptrs)
        _check_poisoned(ro, ptrs)
    return bits, ro


@pytest.mark.parametrize("dt", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("P", [32, 130, 389, 4096 + 96])
def test_mask_bits_exact(dt, P):
    dtype = DT[dt]
    for Q in MP_Q:
        for shared in (False, True):
            B = 3 if shared else 2
            me, feats = _dev(*dp.mask_proj_probe(B, Q, P, shared=shared))
            bits_ref, ro_ref = dp.mask_bits_ref(dp.mask_logits_ref(me, feats).cpu())
            f = feats.to(dtype)
            f = f.expand(B, P, f.shape[2]) if shared else f
            fused = dtype != torch.float32 and Q <= 112           # the mma.sync kernel writes bits straight away
            bits, ro = _bits_call(kernels.mask_bits, B, Q, P, me.to(dtype), f, poison_checked=fused)
            tag = "%s Q%d P%d shared %d" % (dt, Q, P, shared)
            assert torch.equal(bits.cpu(), bits_ref), tag
            assert torch.equal(ro.cpu(), ro_ref), tag


@pytest.mark.parametrize("dt", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("P", [1, 31, 32, 33, 389])
def test_attn_mask_bits_exact(dt, P):
    x = dp.bits_logits_probe(13, P, torch.Generator().manual_seed(P))
    bits_ref, ro_ref = dp.mask_bits_ref(x)
    bits, ro = _bits_call(kernels.attn_mask_bits, 1, 13, P, x.to(DT[dt]).to(CUDA))
    assert torch.equal(bits.cpu(), bits_ref)
    assert torch.equal(ro.cpu(), ro_ref)


# ---------------------------------------------------------------------------------------------------------------
# norms: float64 references and the per-element bound
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("C", [128, 256, 512, 1024, 2048])
def test_add_layernorm_probe(dt, C):
    dtype = DT[dt]
    worst = 0.0
    for R in (1, 3, 4 * 24 + 1):
        for nres in (0, 1, 2):
            ins, w, b = dp.ln_probe(R, C, nres, dtype, torch.Generator().manual_seed(R * 7 + nres + C))
            ins, (w, b) = _dev(*ins), _dev(w, b)
            xs = [t.to(dtype) for t in ins] + [None] * (3 - len(ins))
            for rs in (False, True):
                out = kernels.add_layer_norm(xs[0], w.to(dtype), b.to(dtype), dp.EPS, xs[1], xs[2], return_sum=rs)
                s, y = out if rs else (None, out)
                ref = dp.ln_ref(ins, w, b, dtype, rs)
                bnd = dp.ln_bound(ref, w, dtype)
                r = dp.ratio(y, ref["y"].cpu(), bnd.cpu())
                worst = max(worst, r)
                tag = "LN %s C%d R%d nres%d sum%d" % (dt, C, R, nres, rs)
                assert r <= 1.0, (tag, r)
                const = ref["const"].squeeze(-1)
                assert torch.equal(y[const].double(), b.expand(R, C)[const]), tag + ": constant row is not the bias"
                if rs:
                    if dtype == torch.float32:
                        assert bool(((s.double() - ref["s"]).abs() <= 2 * dp.U32 * ref["ain"]).all()), tag
                    else:
                        assert dp.same(s, ref["s"]), tag + ": returned sum"
    print("PROBE LN %s C%d err/bound %.4f" % (dt, C, worst))


@pytest.mark.parametrize("dt", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("C", [128, 256, 512])
def test_patch_merge_layernorm_probe(dt, C):
    dtype = DT[dt]
    worst = 0.0
    for B, H, W in ((2, 9, 7), (1, 1, 1), (1, 8, 6), (3, 5, 12)):
        x, w, b = _dev(*dp.patch_merge_probe(B, H, W, C, dtype, torch.Generator().manual_seed(H * W + C)))
        y = kernels.patch_merge_layer_norm(x.to(dtype), H, W, w.to(dtype), b.to(dtype), dp.EPS)
        ref = dp.ln_ref([dp.patch_merge_gather(x, H, W)], w, b, dtype, False)
        r = dp.ratio(y, ref["y"].cpu(), dp.ln_bound(ref, w, dtype).cpu())
        worst = max(worst, r)
        assert r <= 1.0, (B, H, W, r)
        const = ref["const"].squeeze(-1)
        assert torch.equal(y[const].double(), b.expand(y.shape)[const])
    print("PROBE patch-merge LN %s C%d err/bound %.4f" % (dt, C, worst))


@pytest.mark.parametrize("dt", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("C", [128, 256, 512, 1024])
def test_groupnorm_tokens_probe(dt, C):
    """B = 3 with per-(batch, group) offsets and scales, mean / std 0 .. 300, a +-50 pre_bias, ReLU on and off, and
    bitwise determinism.  Every case is run before asserting, so that the printout lists each one."""
    dtype = DT[dt]
    fails = []
    for groups in [g for g in (32, 16, 64) if C % (4 * g) == 0]:
        for ni, N in enumerate((1, 255, 256, 257, 5000)):
            for ri, ratio_ms in enumerate((0, 10, 30, 100, 300)):
                pre, relu = bool(ri % 2), bool(ni % 2)
                gen = torch.Generator().manual_seed(N + ratio_ms + groups)
                x, pb, w, b = _dev(*dp.gn_probe(3, N, C, groups, ratio_ms, dtype, gen, pre_bias=pre))
                args = (x.to(dtype), w.to(dtype), b.to(dtype), groups, dp.EPS, relu)
                kw = dict(pre_bias=pb.to(dtype) if pre else None)
                y = kernels.group_norm_tokens(*args, **kw)
                y2 = kernels.group_norm_tokens(*args, **kw)
                ref = dp.gn_ref(x, pb, w, b, groups, relu)
                r = dp.ratio(y, ref["y"].cpu(), dp.gn_bound(ref, w, dtype, C, groups, pre).cpu())
                err = float((y.double() - ref["y"]).abs().max())
                tag = "GN %s C%d G%d N%d mean/std %d pre_bias %d relu %d" % (dt, C, groups, N, ratio_ms, pre, relu)
                print("PROBE %s err/bound %.4f max err %.3e" % (tag, r, err))
                if r > 1.0:
                    fails.append((tag, r))
                assert torch.equal(y, y2), tag + ": not deterministic"
    assert not fails, fails
