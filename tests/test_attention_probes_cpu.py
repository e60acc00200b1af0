"""The attention probes of tests/attn_probe.py can fail: at small shapes, for each probe family, the intended key
carries >= 0.99 of the weight in the float64 reference, the reference rounded to storage passes its own bound, and
every named mutant semantics (computed with the same float64 code) misses the reference by >= 10x the bound that
tests/test_attention_probes_gpu.py applies to the kernels.  For the TMA cross-attention kernel, whose bound also
carries its q-rounding term, this is shown for its tile and split mutants (last / interior 32-key tile, a dropped
split, empty splits combined with m = 0) and for the next image's tail rows; the row_open mutant is shown under the
bound of the per-head kernels, which apply the same rule.  No kernel runs here."""
import pytest
import torch

import attn_probe as ap

DTYPES = [torch.bfloat16, torch.float16, torch.float32]
CPU = torch.device("cpu")


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _self_check(pb, ref, dtype, hd, intended=None, q_rounded=False):
    """The intended key wins, and the storage-rounded reference is within its own bound."""
    if intended is not None:
        w = ap.intended_weight(ref, intended)
        rows = pb.get("rows")
        w = w[rows] if rows is not None else w
        assert float(w.min()) >= 0.99, float(w.min())
    bnd = ap.bound(ref, dtype, hd, q_rounded)
    assert ap.ratio(ap.stored(ref["out"], dtype), ref, bnd, pb.get("rows")) <= 1.0
    return bnd


def _mutant_fails(out_mut, ref, bnd, rows=None):
    r = (out_mut - ref["out"]).abs() / bnd
    if rows is not None:
        r = r[rows]
    return float(r.max())


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_window_probe_and_mutants(dtype):
    B, H, W, C, nh, ws = 1, 30, 26, 128, 4, 12          # padded to 36 x 36: padded keys carry qkv_bias
    for shift in (0, 6):
        qkv, bias, rel, _ = ap.window_probe(B, H, W, C, nh, ws, shift, dtype, _gen(shift))
        pb = ap.window_problem(qkv, bias, rel, B, H, W, C, nh, ws, shift, dev=CPU)
        ref = ap.attend(pb)
        intended = pb["bias"].argmax(-1)                 # +20 offset key if visible (and in the region), else self
        bnd = _self_check(pb, ref, dtype, C // nh, intended)
        # every head of a 2-head CTA reads the table of its first head
        mut = ap.attend(ap.window_problem(qkv, bias, rel, B, H, W, C, nh, ws, shift, rel_heads=[0, 0, 2, 2], dev=CPU))
        assert _mutant_fails(mut["out"], ref, bnd, pb["rows"]) >= 10
        mut = ap.attend(ap.window_problem(qkv, bias, rel, B, H, W, C, nh, ws, shift, rel_heads=[0, 0, 0, 0], dev=CPU))
        assert _mutant_fails(mut["out"], ref, bnd, pb["rows"]) >= 10
        if shift:
            # the offset key in another shift region is favoured by 8 nats but masked by -100
            mut = ap.attend(ap.window_problem(qkv, bias, rel, B, H, W, C, nh, ws, shift, shift_mask=False, dev=CPU))
            assert _mutant_fails(mut["out"], ref, bnd, pb["rows"]) >= 10


def test_window_hpc_rule_covers_1_2_4():
    assert ap.window_hpc(1, 24, 36, 4) == 1
    assert ap.window_hpc(1, 256, 256, 4) == 2
    assert ap.window_hpc(2, 256, 256, 4) == 4
    assert ap.window_hpc(1, 334, 334, 4) == 4
    assert [ap.window_hpc(1, s, s, n) for s, n in ((128, 8), (64, 16), (32, 32))] == [2, 2, 2]


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("padded", [False, True])
def test_causal_probe_and_mutants(dtype, padded):
    B, T, nh, hd = 2, 200, 4, 64
    qkv, kv, intended = ap.causal_probe(B, T, nh, hd, padded, _gen(T + padded))
    qkv = ap.stored(qkv, dtype)
    pb = ap.causal_problem(qkv, kv, B, T, nh, hd, dev=CPU)
    ref = ap.attend(pb)
    bnd = _self_check(pb, ref, dtype, hd, intended)
    # causal mask off by one key: the lured future key wins
    mut = ap.attend(ap.causal_problem(qkv, kv, B, T, nh, hd, future=1, dev=CPU))
    assert _mutant_fails(mut["out"], ref, bnd) >= 10
    if padded:
        mut = ap.attend(ap.causal_problem(qkv, kv, B, T, nh, hd, ignore_valid=True, dev=CPU))
        assert _mutant_fails(mut["out"], ref, bnd) >= 10
    # the last key tile (192..199 holds T-2, T-1) and an interior tile (64..127) skipped
    assert _mutant_fails(ap.attend(ap.drop_keys(pb, 192, 256))["out"], ref, bnd) >= 10
    assert _mutant_fails(ap.attend(ap.drop_keys(pb, 64, 128))["out"], ref, bnd) >= 10
    # tile-by-tile online softmax: equal to the reference; one skipped rescale (the last tile of the rising ladder)
    assert _mutant_fails(ap.online(pb, 64), ref, bnd) <= 1e-6
    assert _mutant_fails(ap.online(pb, 64, skip_rescale=3), ref, bnd) >= 10
    # the rising ladder rescales at every tile of every row; the other ladder keeps its tile-0 maximum
    rise, first = (nh - 2, nh - 1)
    assert _mutant_fails(ap.online(pb, 64, skip_rescale=3)[rise], dict(out=ref["out"][rise]), bnd[rise]) >= 10
    assert _mutant_fails(ap.attend(ap.drop_keys(pb, 0, 64))["out"][first], dict(out=ref["out"][first]), bnd[first]) >= 10


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("P,T", [(1, 17), (65, 64), (130, 33)])
def test_prefix_probe_and_mutants(dtype, P, T):
    B, nh, hd = 2, 3, 64
    qkv, pk, pv, ld, intended = ap.prefix_probe(B, P, T, nh, hd, _gen(P * 7 + T))
    qkv, pk, pv = (ap.stored(x, dtype) for x in (qkv, pk, pv))
    pb = ap.prefix_problem(qkv, pk, pv, P, None, B, T, nh, hd, dev=CPU)
    ref = ap.attend(pb)
    bnd = _self_check(pb, ref, dtype, hd, intended)
    # the padding rows P..ld_rows-1 of the prefix buffer take part
    mut = ap.attend(ap.prefix_problem(qkv, pk, pv, P, None, B, T, nh, hd, prefix_rows=ld, dev=CPU))
    assert _mutant_fails(mut["out"], ref, bnd) >= 10
    # causal mask of the own keys off by one
    n = P + T
    a = pb["allowed"].clone()
    a[:, torch.arange(T - 1), P + torch.arange(1, T)] = True
    if T > 1:
        assert _mutant_fails(ap.attend(dict(pb, allowed=a))["out"], ref, bnd) >= 10
    # the first own-key tile and the prefix tile skipped
    assert _mutant_fails(ap.attend(ap.drop_keys(pb, P, min(n, P + 64)))["out"], ref, bnd) >= 10
    assert _mutant_fails(ap.attend(ap.drop_keys(pb, 0, min(P, 64)))["out"], ref, bnd) >= 10


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_cross_probe_and_mutants(dtype):
    B, Lq, Lk, nh, hd = 2, 37, 389, 8, 32
    splits = 4                                        # 7 tiles of 64 -> 2 per split: splits [0,128) [128,256) ...
    q, k, v, bits, ro, intended = ap.cross_probe(B, Lq, Lk, _gen(5), boundaries=(128, 256, 384, 96, 352))
    q, k, v = (ap.stored(x, dtype) for x in (q, k, v))
    pb = ap.cross_problem(q, k, v, bits, ro, nh, dev=CPU)
    ref = ap.attend(pb)
    tma = dtype != torch.float32                      # the TMA kernel rounds q * scale * log2e to 16 bits
    bnd = _self_check(pb, ref, dtype, hd, intended)
    bnd_t = _self_check(pb, ref, dtype, hd, intended, q_rounded=True) if tma else bnd
    # combine with one split left out; empty splits entering the combine with m = 0
    assert _mutant_fails(ap.online(pb, 64, splits), ref, bnd) <= 1e-6
    assert _mutant_fails(ap.online(pb, 64, splits, drop_split=1), ref, bnd) >= 10
    assert _mutant_fails(ap.online(pb, 64, splits, empty_split_m0=True), ref, bnd) >= 10
    # the same two mutants of the TMA kernel's combine (32-key tiles, 4 tiles per split: the same split boundaries
    # 128 / 256 / 384), under its bound, on the rows built to catch them: open keys in one split, scores 128 nats down
    r = torch.arange(Lq)
    one_split = ((r % 4 == 2) & (r != 2)).expand(B * nh, Lq)
    assert _mutant_fails(ap.online(pb, 32, splits), ref, bnd_t, one_split) <= 1e-6
    assert _mutant_fails(ap.online(pb, 32, splits, drop_split=1), ref, bnd_t, one_split) >= 10
    assert _mutant_fails(ap.online(pb, 32, splits, empty_split_m0=True), ref, bnd_t, one_split) >= 10
    # last tile (64 keys flash, 32 keys TMA; both hold Lk-1), an interior tile
    assert _mutant_fails(ap.attend(ap.drop_keys(pb, 384, Lk))["out"], ref, bnd) >= 10
    assert _mutant_fails(ap.attend(ap.drop_keys(pb, 320, 384))["out"], ref, bnd) >= 10
    assert _mutant_fails(ap.attend(ap.drop_keys(pb, 384, Lk))["out"], ref, bnd_t) >= 10
    assert _mutant_fails(ap.attend(ap.drop_keys(pb, 32, 64))["out"], ref, bnd_t) >= 10
    # the row_open row applies its all-blocking bits
    assert _mutant_fails(ap.attend(ap.cross_problem(q, k, v, bits, ro, nh, ignore_row_open=True, dev=CPU))["out"],
                         ref, bnd) >= 10
    # a 32-key tile load past Lk = 389 reads 27 rows of image b+1, which lure image b's rows
    mut = ap.attend(ap.cross_problem(q, k, v, bits, ro, nh, tail=(-Lk) % 32, dev=CPU))
    assert _mutant_fails(mut["out"], ref, bnd_t) >= 10


def test_cross_probe_shared_memory_batch():
    B, Lq, Lk = 3, 20, 100
    q, k, v, bits, ro, intended = ap.cross_probe(B, Lq, Lk, _gen(9), shared_kv=True)
    assert k.shape[0] == 1
    pb = ap.cross_problem(ap.stored(q, torch.bfloat16), ap.stored(k, torch.bfloat16).expand(B, Lk, 256),
                          ap.stored(v, torch.bfloat16).expand(B, Lk, 256), bits, ro, 8, dev=CPU)
    ref = ap.attend(pb)
    _self_check(pb, ref, torch.bfloat16, 32, intended, q_rounded=True)


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("hd,ps", [(32, 4), (64, 16)])
def test_decode_probe_and_mutants(dtype, hd, ps):
    lens, nh = [1, 33, 129, 200], 8
    qkv, kc, vc, bt, seq, intended = ap.decode_probe(lens, nh, hd, ps, _gen(hd + ps))
    qkv, kc, vc = (ap.stored(x, dtype) for x in (qkv, kc, vc))
    pb = ap.decode_problem(qkv, kc, vc, bt, seq, dev=CPU)
    ref = ap.attend(pb)
    bnd = _self_check(pb, ref, dtype, hd, intended)
    # slot seq_len read too
    mut = ap.attend(ap.decode_problem(qkv, kc, vc, bt, seq, extra=1, dev=CPU))
    assert _mutant_fails(mut["out"][:, :, :], ref, bnd) >= 10
    # the keys of lane 127 / 128 (and the page holding them) dropped
    assert _mutant_fails(ap.attend(ap.drop_keys(pb, 128, 129))["out"], ref, bnd) >= 10
