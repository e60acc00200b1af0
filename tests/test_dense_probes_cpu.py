"""The dense-kernel probes of tests/dense_probe.py can fail: each exact probe differs from every named mutant in at
least one bit, and each float64 probe misses every named mutant by >= 10x the bound that tests/test_dense_probes_gpu.py
applies to the kernels.  The storage-rounded references and fp32 emulations of the kernels' summation orders pass the
same bounds.  No kernel runs here."""
import pytest
import torch

import dense_probe as dp

DT16 = [torch.bfloat16, torch.float16]
DTYPES = DT16 + [torch.float32]


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _differs(mut, ref_stored):
    return not torch.equal(mut, ref_stored)


# ---------------------------------------------------------------------------------------------------------------
# GEMM
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DT16)
@pytest.mark.parametrize("kblocks", [1, 3, 5])
def test_gemm_address_probe_rejects_mutants(dtype, kblocks):
    M, N, K = 321, 256, 64 * kblocks
    a, w, b = dp.address_probe(M, N, K)
    ref = dp.linear_ref(a, w, b)
    assert ref.abs().max() <= 189 and torch.equal(dp.stored(ref, dtype), ref)          # exact in storage
    st = lambda t: dp.stored(t, dtype)                                                   # noqa: E731
    ks = {0, K // 2 // 64 * 64, K - 64}                                                  # first, interior, last k-block
    for k0 in ks:
        assert _differs(st(dp.drop_k(a, w, b, k0, k0 + 64)), st(ref)), ("k-block", k0)
    for step in range(4):                                                                # each 16-wide k-step
        assert _differs(st(dp.drop_k(a, w, b, 16 * step, 16 * step + 16)), st(ref)), ("k-step", step)
    assert _differs(st(dp.linear_ref(a, dp.swizzle_wrong_rows(w), b)), st(ref))          # W box columns permuted
    assert _differs(st(dp.linear_ref(dp.swizzle_wrong_rows(a), w, b)), st(ref))          # A box columns permuted
    assert _differs(st(dp.linear_ref(a, w, dp.bias_shift(b))), st(ref))
    assert _differs(dp.tail_unwritten(st(ref)), st(ref))
    # every row's result is distinct from a neighbouring row's, so a row-store mix-up shows too
    assert _differs(st(ref).roll(1, 0), st(ref))


@pytest.mark.parametrize("dtype", DT16)
def test_gemm_dense_probe_is_exact_and_rejects_dropped_blocks(dtype):
    M, N, K = 200, 256, 1024
    a, w, b = dp.dense_probe(M, N, K, _gen(1))
    ref = dp.linear_ref(a, w, b)
    assert ref.abs().max() <= K + 64
    if dtype == torch.float16:
        assert torch.equal(dp.stored(ref, dtype), ref)
    for k0 in (0, 512, K - 64):
        assert _differs(dp.stored(dp.drop_k(a, w, b, k0, k0 + 64), dtype), dp.stored(ref, dtype))


def test_gemm_head_major_probe_rejects_image_and_head_shifts():
    B, S, N, K = 3, 160, 512, 128
    a, w, b = dp.address_probe(B * S, N, K)
    hm = dp.head_major(dp.linear_ref(a, w, b), S)
    assert hm.shape == (B, N // 32, S, 32)
    assert _differs(dp.head_major_off_by_one(hm, 0), hm)
    assert _differs(dp.head_major_off_by_one(hm, 1), hm)
    # the image shift would still show without the NaN of the unwritten first image: images differ row for row
    assert not torch.equal(hm[1:], hm[:-1]) and not torch.equal(hm[:, 1:], hm[:, :-1])


@pytest.mark.parametrize("dtype", DT16)
def test_gelu_probe_bound(dtype):
    a, w, b = dp.address_probe(512, 256, 128, scale=2.0 ** -4)
    z = dp.linear_ref(a, w, b)
    assert torch.equal(dp.stored(z, dtype), z)                                           # pre-activation exact
    g = dp.gelu(z)
    bnd = dp.gelu_bound(g, dtype)
    assert float(((dp.stored(g, dtype) - g).abs() / bnd).max()) <= 1.0
    # an epilogue that forgot the bias column shift or used tanh-GELU is far outside
    tanh = 0.5 * z * (1 + torch.tanh(0.7978845608028654 * (z + 0.044715 * z ** 3)))
    assert float(((dp.stored(tanh, dtype) - g).abs() / bnd).max()) >= 1.0
    assert float(((dp.stored(dp.gelu(z.roll(8, 1)), dtype) - g).abs() / bnd).max()) >= 10


# ---------------------------------------------------------------------------------------------------------------
# mask projection and mask bits
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", [130, 389])
def test_mask_proj_probe_rejects_mutants(P):
    B, Q = 2, 7
    me, feats = dp.mask_proj_probe(B, Q, P)
    ref = dp.mask_logits_ref(me, feats)
    assert ref.abs().max() <= 125
    assert _differs(dp.mask_logits_ref(me, feats.roll(1, 0)), ref)                        # wrong image's map
    assert _differs(dp.mask_logits_ref(me, dp.swizzle_wrong_rows(feats[0])[None].expand(B, -1, -1)), ref)
    bits, ro = dp.mask_bits_ref(ref)
    assert int(ro[:, 0].min()) == 1 and int(ro[:, 1:].max()) == 0                        # row 0 all blocked, row 1 open
    assert int(bits[:, 1].abs().max()) == 0                                              # exact zeros stay open
    for mut in (dict(rule="le0"), dict(tail=True), dict(open_over_padded=True)):
        mb, mro = dp.mask_bits_ref(ref, **mut)
        assert not (torch.equal(mb, bits) and torch.equal(mro, ro)), mut


def test_mask_bits_direct_probe_rejects_mutants():
    x = dp.bits_logits_probe(12, 389, _gen(3))
    assert bool((x == 0).any()) and bool(torch.signbit(x[x == 0]).any())                # +0 and -0 logits present
    bits, ro = dp.mask_bits_ref(x)
    assert int(ro.sum()) == 3                                                            # rows 0, 4, 8
    for dt in (torch.bfloat16, torch.float16, torch.float32):
        assert torch.equal(dp.stored(x, dt), x)                                          # exact in every storage type
    for mut in (dict(rule="le0"), dict(tail=True), dict(open_over_padded=True)):
        mb, mro = dp.mask_bits_ref(x, **mut)
        assert not (torch.equal(mb, bits) and torch.equal(mro, ro)), mut


def test_pack_bits_layout():
    blocked = torch.zeros(1, 1, 40, dtype=torch.bool)
    blocked[0, 0, [0, 31, 33]] = True
    bits = dp.pack_bits(blocked)
    assert bits.tolist() == [[[1 | -(1 << 31), 2]]]


# ---------------------------------------------------------------------------------------------------------------
# LayerNorm
# ---------------------------------------------------------------------------------------------------------------
def _worst(out, ref, bnd, rows=None):
    r = (out - ref).abs() / bnd
    return float(r.max() if rows is None else r[rows].max())


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("C", [128, 2048])
def test_layernorm_probe_bound_and_mutants(dtype, C):
    R = 4 * 24 + 1
    one_pass = []
    for nres in (0, 1, 2):
        ins, w, b = dp.ln_probe(R, C, nres, dtype, _gen(C + nres))
        if dtype != torch.float32:   # the probes' residual sums are exact in fp32: the returned sum is exact
            s32 = dp.kernel_sum32(ins, torch.float32, False).to(dp.F64)
            assert torch.equal(s32, sum(ins))
        for rs in (False, True):
            ref = dp.ln_ref(ins, w, b, dtype, rs)
            bnd = dp.ln_bound(ref, w, dtype)
            assert bool(ref["const"].any())
            assert _worst(dp.stored(ref["y"], dtype), ref["y"], bnd) <= 1.0
            emu = dp.ln_fp32(dp.kernel_sum32(ins, dtype, rs), w, b, dtype)                # the kernel's order
            assert _worst(emu, ref["y"], bnd) <= 1.0
            const = ref["const"].squeeze(-1)
            assert torch.equal(emu[const], b.expand(R, C)[const])                      # constant rows: y = bias
            # one-pass E[x^2] - m^2: 16-bit storage cannot hold mean / std = 1e3 (bf16 keeps 8 bits), so the offset
            # rows reach it through the fp32 sum of residuals, i.e. when the sum is not rounded back to storage
            if dtype == torch.float32 or (nres and not rs):
                one = dp.ln_fp32(dp.kernel_sum32(ins, dtype, rs), w, b, dtype, one_pass=True)
                one_pass.append(_worst(one, ref["y"], bnd))
            assert _worst(dp.stored(dp.ln_eps_outside(ref, w, b), dtype), ref["y"], bnd) >= 10, "eps outside"
            if rs and nres and dtype != torch.float32:   # x alone is already in storage: rounding changes nothing
                unrounded = dp.ln_ref(ins, w, b, dtype, False)
                assert _worst(dp.stored(unrounded["y"], dtype), ref["y"], bnd) >= 10, "sum not rounded"
            # a row mix-up (row i normalised with row i+1's statistics)
            mix = (ref["s"] - ref["mu"].roll(1, 0)) * ref["r"].roll(1, 0) * w + b
            assert _worst(dp.stored(mix, dtype), ref["y"], bnd) >= 10
    assert max(one_pass) >= 10, ("one-pass E[x^2] - m^2", one_pass)       # the probe set rejects it


@pytest.mark.parametrize("dtype", DTYPES)
def test_patch_merge_probe_bound(dtype):
    x, w, b = dp.patch_merge_probe(2, 9, 7, 128, dtype, _gen(11))
    g = dp.patch_merge_gather(x, 9, 7)
    ref = dp.ln_ref([g], w, b, dtype, False)
    bnd = dp.ln_bound(ref, w, dtype)
    B, R, C4 = g.shape
    emu = dp.ln_fp32(g.view(-1, C4).to(torch.float32), w, b, dtype).view(B, R, C4)
    assert _worst(emu, ref["y"], bnd) <= 1.0
    assert bool(ref["const"].any())
    if dtype == torch.float32:   # 16-bit storage cannot hold the offset that exposes it (bf16 keeps 8 bits)
        one = dp.ln_fp32(g.view(-1, C4).to(torch.float32), w, b, dtype, one_pass=True).view(B, R, C4)
        assert _worst(one, ref["y"], bnd) >= 10
    assert _worst(dp.stored(dp.ln_eps_outside(ref, w, b), dtype), ref["y"], bnd) >= 10


# ---------------------------------------------------------------------------------------------------------------
# GroupNorm
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_groupnorm_centred_scheme_passes_every_offset(dtype):
    B, N, C, G = 3, 300, 256, 32
    for ratio in (0, 10, 30, 100, 300):
        for pre in (False, True):
            x, pb, w, b = dp.gn_probe(B, N, C, G, ratio, dtype, _gen(ratio + pre), pre_bias=pre)
            ref = dp.gn_ref(x, pb, w, b, G, relu=False)
            bnd = dp.gn_bound(ref, w, dtype, C, G, pre)
            assert _worst(dp.stored(ref["y"], dtype), ref["y"], bnd) <= 1.0
            emu = dp.gn_fp32(x, pb, w, b, G, dtype, relu=False)
            assert _worst(emu, ref["y"], bnd) <= 1.0, (ratio, pre)


@pytest.mark.parametrize("N", [512, 5000])
def test_groupnorm_raw_moment_mutant_fails_from_offset_30_in_fp32(N):
    """The earlier kernel's statistics (fp32 sums of x and x^2, then E[x^2] - mean^2) miss the bound by >= 10x at
    mean / std >= 30 in fp32 storage."""
    B, C, G = 1, 256, 32
    for ratio in (30, 100, 300):
        x, pb, w, b = dp.gn_probe(B, N, C, G, ratio, torch.float32, _gen(ratio))
        ref = dp.gn_ref(x, pb, w, b, G, relu=False)
        bnd = dp.gn_bound(ref, w, torch.float32, C, G, False)
        raw = dp.gn_fp32(x, pb, w, b, G, torch.float32, relu=False, scheme="raw")
        assert _worst(raw, ref["y"], bnd) >= 10, ratio


def test_groupnorm_raw_moment_mutant_fails_in_fp16_at_offset_300():
    B, N, C, G = 1, 5000, 256, 32
    x, pb, w, b = dp.gn_probe(B, N, C, G, 300, torch.float16, _gen(7))
    ref = dp.gn_ref(x, pb, w, b, G, relu=False)
    bnd = dp.gn_bound(ref, w, torch.float16, C, G, False)
    raw = dp.gn_fp32(x, pb, w, b, G, torch.float16, relu=False, scheme="raw")
    assert _worst(raw, ref["y"], bnd) >= 10


@pytest.mark.parametrize("dtype", DTYPES)
def test_groupnorm_wrong_batch_or_group_statistics(dtype):
    B, N, C, G = 3, 257, 256, 32
    x, pb, w, b = dp.gn_probe(B, N, C, G, 10, dtype, _gen(5), pre_bias=True)
    ref = dp.gn_ref(x, pb, w, b, G, relu=True)
    bnd = dp.gn_bound(ref, w, dtype, C, G, True)
    for kw in (dict(stat_batch=torch.arange(B).roll(1)), dict(stat_group=torch.arange(G).roll(1))):
        mut = dp.gn_ref(x, pb, w, b, G, relu=True, **kw)
        assert _worst(dp.stored(mut["y"], dtype), ref["y"], bnd) >= 10, kw
    # pre_bias left out
    mut = dp.gn_ref(x, None, w, b, G, relu=True)
    assert _worst(dp.stored(mut["y"], dtype), ref["y"], bnd) >= 10
