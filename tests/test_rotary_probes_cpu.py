"""The rotary, rotary-plus-attention and linear_act probes of tests/rotary_probe.py can fail.  On the CPU, with the
float64 code of rotary_probe: the exact probes differ from every structural mutant in at least one element, the float64
probes and the attention chains miss every named mutant by >= 10x their bound, a correct fp32 evaluation (with and
without FMA) passes the float64 bound, and the shapes of tests/test_rotary_probes_gpu.py reach every kernel route and
wrap every grid-stride loop.  No kernel runs here."""
import pytest
import torch

import attn_probe as ap
import rotary_probe as rp
from rotary_probe import ACT_CASES, CAUSAL_CASES, DECODE_CASES, PREFIX_PS, ROTARY_CASES

DTYPES = [torch.bfloat16, torch.float16, torch.float32]
CPU = torch.device("cpu")


def _g(seed):
    return torch.Generator().manual_seed(seed)


# mutants of the rotary kernel alone that apply to a case: name -> keyword arguments of rotary_probe.rotate
def _mutants(B, T, hd, rd, rt):
    t = torch.arange(T).expand(B, T)
    m = {
        "interleave": dict(pairing="interleave"),
        "sin sign": dict(sin_sign=-1.0),
        "c/s swapped": dict(swap=True),
        "row pos+1": dict(pos=t + 1),
        "row pos-1": dict(pos=t - 1),
        "v rotated": dict(which=(0, 1, 2)),
        "only q": dict(which=(0,)),
        "only k": dict(which=(1,)),
    }
    if rd == 2:    # one pair: (0, 1) is both the half pairing and the interleaved one
        del m["interleave"]
    if T == 1:     # one token: pos +- 1 wraps to the same (only) row, so no input can tell
        del m["row pos+1"], m["row pos-1"]
    if B > 1:
        m["flat token index"] = dict(pos=torch.arange(B * T).view(B, T))
    if rd < hd:
        m["all hd dims"] = dict(pairing="all")
        m["half = hd/2"] = dict(pairing="head")
    if rt == "vec":
        if rd // 2 > 8:
            m["chunk column c"] = dict(chunk_cols=True)
        m["last chunk unwritten"] = dict(last_chunk=False)
    return m


SMALL_CASES = [  # (B, T, nh, hd, rd): the CPU-sized counterparts of every GPU case's route and mutant set
    (1, 1, 4, 64, 32), (1, 7, 4, 64, 32), (1, 61, 4, 64, 32), (2, 9, 2, 64, 64), (3, 17, 2, 64, 32),
    (2, 19, 2, 64, 24), (1, 9, 2, 64, 2), (2, 11, 2, 36, 16),
]


def test_routes_and_wraps_are_reached():
    reached, wrapped = set(), set()
    for name, B, T, nh, hd, rd, P in ROTARY_CASES:
        for dt in DTYPES:
            rt = rp.route(dt, hd, rd)
            key = (rt, dt == torch.float32)
            reached.add(key)
            if rp.wraps(rt, B, T, nh, rd):
                wrapped.add(key)
    want = {("vec", False), ("scalar", False), ("scalar", True)}
    assert reached == want and wrapped == want
    assert rp.route(torch.bfloat16, 64, 32, aligned=False) == "scalar"
    # the wrap cases each run more than one pass: B 4, T 2100, nh 32 launches 1.07M vector work items
    assert rp.work_items("vec", 4, 2100, 32, 32) == 1075200 > rp.GRID
    # the 16-bit scalar route is reached by each of its three conditions
    assert {(hd, rd) for _, _, _, _, hd, rd, _ in ROTARY_CASES if rp.route(torch.float16, hd, rd) == "scalar"} >= \
        {(64, 24), (64, 2), (36, 16)}
    for case in SMALL_CASES:
        assert any(rp.route(torch.bfloat16, c[4], c[5]) == rp.route(torch.bfloat16, case[3], case[4])
                   for c in ROTARY_CASES)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", SMALL_CASES, ids=lambda c: "B%d_T%d_nh%d_hd%d_rd%d" % c)
def test_exact_probe_rejects_structural_mutants(case, dtype):
    B, T, nh, hd, rd = case
    x, cos, sin = rp.exact_probe(B, T, nh, hd, rd, _g(T + rd))
    y = rp.rotate(x, cos, sin, rd)
    assert torch.equal(rp.stored(y, dtype), y)                     # exact in storage
    assert (y[:, :, :2, :, :rd] * 4 == torch.round(y[:, :, :2, :, :rd] * 4)).all() and y.abs().max() <= 30
    assert torch.equal(rp.fp32_kernel(x, cos, sin, rd, dtype, True), y)
    assert torch.equal(rp.fp32_kernel(x, cos, sin, rd, dtype, False), y)
    assert torch.equal(rp.rotate(x, cos, sin, rd, round_to=dtype), y)     # not a structural mutant: equal here
    for name, mut in _mutants(B, T, hd, rd, rp.route(dtype, hd, rd)).items():
        ym = rp.rotate(x, cos, sin, rd, **mut)
        assert int((ym != y).sum()) >= 1, name


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", SMALL_CASES + [(1, 7, 4, 64, 32, 2093)], ids=str)
def test_float_probe_bound_and_mutants(case, dtype):
    B, T, nh, hd, rd = case[:5]
    P = case[5] if len(case) > 5 else 1000
    x, cos, sin = rp.float_probe(B, T, nh, hd, rd, dtype, _g(T * 3 + rd), P=P)
    y, bnd = rp.bound(x, cos, sin, rd, dtype)
    for fma in (True, False):
        assert rp.ratio(rp.fp32_kernel(x, cos, sin, rd, dtype, fma), y, bnd, rd) <= 1.0
    assert rp.ratio(rp.stored(y, dtype), y, bnd, rd) <= 1.0
    muts = _mutants(B, T, hd, rd, rp.route(dtype, hd, rd))
    if dtype != torch.float32:
        muts["products rounded to storage"] = dict(round_to=dtype)
    for name, mut in muts.items():
        ym = rp.rotate(x, cos, sin, rd, **mut)
        if name in ("v rotated", "all hd dims"):         # changes elements outside the rotated set
            assert not rp.untouched(ym, x, rd), name
            continue
        r = rp.ratio(ym, y, bnd, rd)
        assert r >= 10, (name, r)


# ---------------------------------------------------------------------------------------------------------------
# chains
# ---------------------------------------------------------------------------------------------------------------
def _common_mutants():
    return {"interleave": dict(pairing="interleave"), "sin sign": dict(sin_sign=-1.0),
            "q not rotated": dict(q_rot=False), "k not rotated": dict(k_rot=False)}


def _chain_fails(ref, mut, bnd):
    return float(((mut["out"] - ref["out"]).abs() / bnd).max())


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("padded", [False, True])
def test_causal_chain_rejects_mutants(padded, dtype):
    B, T, nh, hd, rd = 2, 67, 4, 64, 32
    post, kv, intended = rp.causal_chain_probe(B, T, nh, hd, rd, padded, _g(T + padded))
    post = rp.stored(post, dtype)
    cos, sin = rp.quarter_tables(T + 2, rd, _g(5))
    x = rp.unrotate(post, cos, sin, rd)
    assert torch.equal(rp.stored(x, dtype), x)
    ref = ap.attend(ap.causal_problem(post, kv, B, T, nh, hd, dev=CPU))
    assert float(ap.intended_weight(ref, intended).min()) >= 0.99
    bnd = ap.bound(ref, dtype, hd)
    good = rp.causal_chain(x, kv, cos, sin, rd)
    assert torch.equal(good["out"], ref["out"])
    muts = dict(_common_mutants())
    for d in (1, -1):
        muts["q row %+d" % d] = dict(q_shift=d)
        muts["k row %+d" % d] = dict(k_shift=d)
        muts["q and k row %+d" % d] = dict(q_shift=d, k_shift=d)
    for name, mut in muts.items():
        r = _chain_fails(ref, rp.causal_chain(x, kv, cos, sin, rd, **mut), bnd)
        assert r >= 10, (name, r)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("P", PREFIX_PS)
def test_prefix_chain_rejects_mutants(P, dtype):
    B, T, nh, hd, rd = 2, 17, 4, 64, 32
    post, pk, pv, intended = rp.prefix_chain_probe(B, P, T, nh, hd, rd, _g(P))
    post, pk, pv = rp.stored(post, dtype), rp.stored(pk, dtype), rp.stored(pv, dtype)
    cos, sin = rp.quarter_tables(2 * P + T + 2, rd, _g(P + 1))
    pre, suf = rp.prefix_inputs(post, pk, pv, P, cos, sin, rd)
    ref = ap.attend(ap.prefix_problem(post, pk, pv, P, None, B, T, nh, hd, dev=CPU))
    assert float(ap.intended_weight(ref, intended).min()) >= 0.99
    bnd = ap.bound(ref, dtype, hd)
    good = rp.prefix_chain(pre, suf, pk, pv, P, cos, sin, rd)
    assert torch.equal(good["out"], ref["out"])
    muts = dict(_common_mutants())
    for d in (1, -1):
        muts["q row %+d" % d] = dict(q_shift=d)
        muts["k row %+d" % d] = dict(k_shift=d)
        muts["q and k row %+d" % d] = dict(q_shift=d, k_shift=d)
    muts["suffix from row 0"] = dict(suf_start=0)
    muts["prefix from row P"] = dict(pre_start=P)
    for name, mut in muts.items():
        r = _chain_fails(ref, rp.prefix_chain(pre, suf, pk, pv, P, cos, sin, rd, **mut), bnd)
        assert r >= 10, (name, r)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("ps", [4, 16])
def test_decode_chain_rejects_mutants(ps, dtype):
    lens, nh, hd, rd = [1, 17, 33, 130], 4, 64, 32
    q, kc, vc, bt, intended = rp.decode_chain_probe(lens, nh, hd, rd, ps, _g(ps))
    q, kc, vc = rp.stored(q, dtype), rp.stored(kc, dtype), rp.stored(vc, dtype)
    cos, sin = rp.quarter_tables(max(lens) + 3, rd, _g(ps + 1))
    pres, new = rp.decode_inputs(q, kc, vc, bt, lens, cos, sin, rd)
    post_new = torch.zeros_like(new)
    post_new[:, 0, 0] = q
    seq = torch.tensor(lens, dtype=torch.int32) + 1
    ref = ap.attend(ap.decode_problem(post_new, kc, vc, bt, seq, dev=CPU))
    assert float(ap.intended_weight(ref, intended).min()) >= 0.99
    bnd = ap.bound(ref, dtype, hd)
    good = rp.decode_chain(pres, new, kc, vc, bt, lens, cos, sin, rd)
    assert torch.equal(good["out"], ref["out"])
    muts = dict(_common_mutants())
    for d in (1, -1):
        muts["q row %+d" % d] = dict(q_shift=d)
        muts["k row %+d" % d] = dict(pre_shift=d, newk_shift=d)
        muts["q and k row %+d" % d] = dict(pre_shift=d, q_shift=d, newk_shift=d)
        muts["new token at seq_len %+d" % d] = dict(q_shift=d, newk_shift=d)
    for name, mut in muts.items():
        r = _chain_fails(ref, rp.decode_chain(pres, new, kc, vc, bt, lens, cos, sin, rd, **mut), bnd)
        assert r >= 10, (name, r)


def test_gpu_chain_cases_fit_the_probe():
    """Every GPU chain case has room for its designated keys in the rd key directions."""
    for B, T, nh, padded in CAUSAL_CASES:
        rp.causal_chain_probe(B, T, nh, 64, 32, padded, _g(1))
    for lens, ps in DECODE_CASES:
        rp.decode_chain_probe(lens, 2, 64, 32, ps, _g(1))


# ---------------------------------------------------------------------------------------------------------------
# linear_act
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_act_probe_exact_and_mutants(dtype):
    for M, N, K, act in ACT_CASES:
        M = min(M, 300)
        x, w, b = rp.act_probe(M, N, K)
        z = x @ w.t() + b
        for t in (x, w, b, z):
            assert torch.equal(rp.stored(t, dtype), t)
        assert float(z.min()) <= -8 and float(z.max()) >= 8
    M, N, K = 300, 8192, 2048
    x, w, b = rp.act_probe(M, N, K)
    z = x @ w.t() + b
    g = rp.gelu_new(z)
    bnd = rp.gelu_bound(z, g, dtype)
    assert float(((rp.stored(g, dtype) - g).abs() / bnd).max()) <= 1.0
    xw = x @ w.t()
    muts = {"bias dropped": rp.gelu_new(xw), "bias after activation": rp.gelu_new(xw) + b, "relu": z.clamp(min=0)}
    for name, gm in muts.items():
        r = float(((rp.stored(gm, dtype) - g).abs() / bnd).max())
        assert r >= 10, (name, r)
    # erf-GELU passes the same bound: the probe does not distinguish it from gelu_new
    erf = 0.5 * z * (1.0 + torch.erf(z / 2.0 ** 0.5))
    assert float(((rp.stored(erf, dtype) - g).abs() / bnd).max()) <= 1.0
