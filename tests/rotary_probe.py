"""Float64 references, per-element bounds and probe inputs for the Phi-1.5 partial rotary embedding
(psalm_rotary_inplace: rotary_kernel and rotary_vec_kernel in csrc/attn_simt.cu), for rotary composed with the attention
that consumes it (prefill, prompt suffix behind a cached prefix, paged decode), and for the fc1 gelu_new / FFN relu
epilogues of kernels.linear_act.

No kernel is called here, and nothing is shared with tests/emu.py.  tests/test_rotary_probes_cpu.py shows that each
probe rejects its named mutants; tests/test_rotary_probes_gpu.py runs the kernels on the same probes.

Rotary reference (modeling_phi apply_rotary_pos_emb / rotate_half on the first rd dims of q and k, half = rd / 2):

    y[i] = x[i] c - x[i + half] s,   y[i + half] = x[i + half] c + x[i] s,   i < half

with (c, s) = (cos, sin)[pos, i]; v and dims rd..hd-1 are unchanged.  `rotate` computes it in float64 for any table
rows, and carries the named mutants as keyword arguments.

Exact probes.  Inputs are integers with 1 <= |x| <= 15 (no zeros, so the sign of zero never matters) and the tables
hold c, s drawn independently per (row, pair) from {+-1/4, +-1/2, +-3/4, +-1} (not rotations: the kernel takes any
fp32 table).  Every y is a multiple of 1/4 with |y| <= 30, i.e. at most 7 significant bits: exact in fp32 products
and sums (with or without FMA) and in bf16, fp16 and fp32 storage.  The output must equal the reference bit for bit,
and every element outside the first rd dims of q and k must equal its input bit for bit.

Float64 probes.  Real Phi tables (PhiModel.rope_tables: fp32 theta^(-2i/rd) times the position, cos / sin in fp32) at
positions up to 2100, storage-rounded Gaussian inputs, and cancelling rows in which x[i + half] is the storage
rounding of x[i] c / s, so that y[i] = x[i] c - x[i + half] s is a few ulp of its products.  The kernel evaluates
each output as two fp32 products and a sum of exact (storage) inputs and fp32 table entries, with or without FMA,
then rounds once to storage.  With m = |x1 c| + |x2 s| (the output's product magnitudes) and u32 = 2^-24:

    fp32 evaluation   |y^ - y| <= u32 m + u32 |y^ - product error| <= u32 (|y| + (1 + u32) m) = e32
                      (each product rounds with error <= u32 |product|, the sum with <= u32 |y^|; an FMA drops one
                      product rounding, which only lowers the error)
    storage           |out - y^| <= half_ulp_s(|y^|) <= half_ulp_s(|y| + e32)   (0 for fp32 storage)

    |out - y| <= e32 + half_ulp_s(|y| + e32)

half_ulp_s(v) is half the storage type's ulp at v (bf16 8, fp16 11 significant bits; fp16's subnormal spacing 2^-24
below 2^-14).  Rounding each product to 16-bit storage before the sum (the reference's own bf16 arithmetic) changes
the cancelling outputs by up to half_ulp_s of the products, far above half_ulp_s(|y|): the float64 probes reject it;
on the exact probes it equals the reference.

Routes.  `route` restates psalm_rotary_inplace: 16-bit storage with half % 8 == 0, hd % 8 == 0 and 16-byte aligned
qkv, cos and sin takes the vector kernel (one work item per 8 pairs), everything else the scalar kernel (one work item
per pair).  Both launch at most 132 x 16 blocks of 256 threads (GRID work items per pass); `wraps` says when the
grid-stride loop runs more than one pass.

Composition with attention.  Tables are quarter turns: (c, s) per (row, pair) drawn from {(1,0), (0,1), (-1,0),
(0,-1)}.  The rotation is then a signed permutation: exact in every storage type and exactly invertible (`rotate`
with sin_sign = -1 undoes it).  The tables are not R(p theta), so scores depend on absolute positions, and shifting q
and k together is caught too.  The probes build post-rotary q', k', v as tests/attn_probe.py does (intended keys 16
nats above the rest, +-1 V codes, lures), with every key-selection direction in the first rd dims, round them to
storage and un-rotate q' and k' per position to get the inputs.  A wrong table row turns a row's query direction (or a
key's) by a quarter turn with probability 3/4, which moves the intended score from 16 nats to 0 or -16: the output
moves by O(1).  The reference is attn_probe.attend on q', k', v under attn_probe.bound.

linear_act probes.  x has one 1 per row, at k_m = 37 m mod K; W[n, k] = (((131 n + 17 k) mod 257) - 128) / 16 and
bias[n] = (((29 n) mod 33) - 16) / 16, so z = x W^T + b = W[n, k_m] + bias[n] is a multiple of 1/16 in [-9, 9]: one
product per output, exact in fp32 in any summation order, and representable in bf16 and fp16 (at most 8 significant
bits), whether the library applies the activation in its epilogue or to a rounded GEMM output.
  relu       must equal max(z, 0) exactly.
  gelu_tanh  checked against float64 gelu_new(z) = z / 2 (1 + tanh(sqrt(2 / pi) (z + 0.044715 z^3))) with the bound
             half_ulp_s(|g|) + |z| u_s (u_s = 2^-8 bf16, 2^-11 fp16).  That is the error the reference's own
             NewGELUActivation admits in the storage type: its 1 + tanh(.) lies in [0, 2] and is rounded to storage
             (absolute error <= 2 u_s), which z / 2 scales to |z| u_s; the product is rounded once more (half an ulp
             of g).  erf-GELU differs from gelu_new by < 5e-4; rounded to storage it stays within this bound on the
             probe's z grid (err / bound 0.45 in bf16, 0.58 in fp16), so the probe cannot tell the two apart.  It
             does reject a dropped bias, a bias added after the activation and relu in place of gelu.
"""
import math

import torch

import attn_probe as ap

F64 = torch.float64
UNIT = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 2.0 ** -24}
PREC = {torch.bfloat16: 8, torch.float16: 11}      # significant bits of 16-bit storage
EMIN = {torch.bfloat16: -126, torch.float16: -14}  # smallest normal exponent
U32 = 2.0 ** -24
GRID = 132 * 16 * 256                              # work items of one grid-stride pass of either rotary kernel
QUARTERS = (0.25, 0.5, 0.75, 1.0, -0.25, -0.5, -0.75, -1.0)

# shapes of tests/test_rotary_probes_gpu.py (the CPU file checks what they reach)
ROTARY_CASES = [  # name, B, T, nh, hd, rd, first Phi table row of the float64 probe
    ("phi_T1", 1, 1, 32, 64, 32, 2099), ("phi_T7", 1, 7, 32, 64, 32, 2093), ("phi_T921", 1, 921, 32, 64, 32, 0),
    ("rd64", 2, 33, 4, 64, 64, 100), ("B3", 3, 17, 8, 64, 32, 500), ("wrap", 4, 2100, 32, 64, 32, 0),
    ("rd24", 2, 19, 4, 64, 24, 7), ("rd24_wrap", 2, 1100, 32, 64, 24, 1000), ("rd2", 1, 9, 4, 64, 2, 3),
    ("hd36", 2, 11, 4, 36, 16, 50),
]
CAUSAL_CASES = [(1, 1, 4, False), (2, 65, 4, True), (2, 129, 4, False), (1, 921, 32, False), (2, 300, 32, True)]
PREFIX_PS = [1, 63, 64, 65, 290]
DECODE_CASES = [([1, 31, 32, 33, 127, 128, 129, 921], 4), ([5, 64, 300], 8), ([921, 921], 16), ([2048, 17], 16)]
ACT_CASES = [  # M, N, K, activation: Phi-1.5 fc1 (prefill, decode), pixel-decoder FFN, mask-decoder FFN and MLP
    (921, 8192, 2048, "gelu_tanh"), (1, 8192, 2048, "gelu_tanh"), (21504, 1024, 256, "relu"),
    (100, 2048, 256, "relu"), (100, 256, 256, "relu"),
]


def stored(x, dtype):
    """Storage rounding, back to float64."""
    return x.to(dtype).to(F64)


def half_ulp(v, dtype):
    """Half the storage type's ulp at |v| >= 0 (0 for fp32 storage: the kernel's fp32 result is stored as is)."""
    if dtype == torch.float32:
        return torch.zeros_like(v)
    _, e = torch.frexp(v)                          # v = m 2^e, m in [0.5, 1)
    e = torch.where(v > 0, e - 1, torch.full_like(e, EMIN[dtype])).clamp(min=EMIN[dtype])
    return torch.pow(2.0, (e - PREC[dtype]).to(F64))


# ---------------------------------------------------------------------------------------------------------------
# routes (restates psalm_rotary_inplace)
# ---------------------------------------------------------------------------------------------------------------
def route(dtype, hd, rd, aligned=True):
    if dtype != torch.float32 and (rd // 2) % 8 == 0 and hd % 8 == 0 and aligned:
        return "vec"
    return "scalar"


def work_items(rt, B, T, nh, rd):
    return B * T * 2 * nh * (rd // 16 if rt == "vec" else rd // 2)


def wraps(rt, B, T, nh, rd):
    return work_items(rt, B, T, nh, rd) > GRID


# ---------------------------------------------------------------------------------------------------------------
# reference and mutants
# ---------------------------------------------------------------------------------------------------------------
def _pairs(hd, rd, pairing):
    """(first, second, table column) of every rotated pair."""
    half = rd // 2
    i = torch.arange(half)
    if pairing == "half":
        return i, i + half, i
    if pairing == "interleave":                    # GPT-J: (2i, 2i + 1)
        return 2 * i, 2 * i + 1, i
    if pairing == "head":                          # half = hd / 2: (i, i + hd / 2), i < rd / 2
        return i, i + hd // 2, i
    if pairing == "all":                           # all hd dims rotated: (i, i + hd / 2), i < hd / 2
        j = torch.arange(hd // 2)
        return j, j + hd // 2, j % half
    raise ValueError(pairing)


def rotate(qkv, cos, sin, rd, pos=None, which=(0, 1), pairing="half", sin_sign=1.0, swap=False, chunk_cols=False,
           last_chunk=True, round_to=None, magnitude=False):
    """Float64 rotary of qkv [B,T,3,nh,hd] (any dtype) by the table rows pos [B,T] (default: row t; rows past the
    table wrap around) of cos / sin [rows, rd/2].  Mutants: `which` = the parts rotated (0 q, 1 k, 2 v); `pairing`
    (see _pairs); `sin_sign` = -1 flips the sine (with the correct tables: the inverse rotation); `swap` exchanges c
    and s; `chunk_cols`: the vector kernel reads table column c + j for lane j of 8-pair chunk c (instead of 8 c + j);
    `last_chunk=False` leaves the last 8-pair chunk unwritten; `round_to` rounds each product to that storage type
    before the sum.  magnitude=True returns |x1 c| + |x2 s| per rotated element instead (for the bound)."""
    x = qkv.to(F64)
    B, T = x.shape[:2]
    hd = x.shape[-1]
    dev = x.device
    ia, ib, col = (t.to(dev) for t in _pairs(hd, rd, pairing))
    if chunk_cols:
        col = col // 8 + col % 8
    c, s = cos.to(dev, F64), sin.to(dev, F64) * sin_sign
    if swap:
        c, s = s, c
    if pos is None:
        pos = torch.arange(T, device=dev).expand(B, T)
    pos = pos.to(dev) % c.shape[0]
    cc, ss = c[pos][..., col].unsqueeze(2), s[pos][..., col].unsqueeze(2)        # [B, T, 1, pairs]
    keep = (torch.arange(len(ia), device=dev) >= rd // 2 - 8) if not last_chunk else None
    y = x.clone()
    for w in which:
        x1, x2 = x[:, :, w][..., ia], x[:, :, w][..., ib]
        p = [x1 * cc, x2 * ss, x2 * cc, x1 * ss]
        if magnitude:
            y1, y2 = p[0].abs() + p[1].abs(), p[2].abs() + p[3].abs()
        else:
            if round_to is not None:
                p = [stored(t, round_to) for t in p]
            y1, y2 = p[0] - p[1], p[2] + p[3]
        if keep is not None:
            y1 = torch.where(keep, x1, y1)
            y2 = torch.where(keep, x2, y2)
        yw = y[:, :, w]
        yw[..., ia] = y1
        yw[..., ib] = y2
    return y


def rotated_mask(shape, rd, device=None):
    """True on the elements the kernel may change: the first rd dims of q and k."""
    m = torch.zeros(shape, dtype=torch.bool, device=device)
    m[:, :, :2, :, :rd] = True
    return m


def bound(qkv, cos, sin, rd, dtype, pos=None):
    """(float64 reference y, per-element bound) of the kernel's output on storage inputs qkv."""
    y = rotate(qkv, cos, sin, rd, pos)
    m = rotate(qkv, cos, sin, rd, pos, magnitude=True)
    e32 = U32 * (y.abs() + (1 + U32) * m)
    return y, e32 + half_ulp(y.abs() + e32, dtype)


def ratio(out, y, bnd, rd):
    """max |out - y| / bound over the rotated elements."""
    o = out.to(y.device, F64)
    assert torch.isfinite(o).all(), "non-finite kernel output"
    m = rotated_mask(y.shape, rd, y.device)
    return float(((o - y).abs() / bnd)[m].max())


def untouched(out, qkv, rd):
    """Every element outside the first rd dims of q and k equals its input bit for bit."""
    m = ~rotated_mask(qkv.shape, rd, out.device)
    a, b = out[m], qkv.to(out.device)[m]
    if a.dtype in (torch.bfloat16, torch.float16):
        a, b = a.view(torch.int16), b.view(torch.int16)
    elif a.dtype == torch.float32:
        a, b = a.view(torch.int32), b.view(torch.int32)
    return torch.equal(a, b)


def fp32_kernel(qkv, cos, sin, rd, dtype, fma):
    """The kernel's arithmetic emulated in fp32 (with or without FMA), rounded to storage: it must pass `bound`."""
    x = qkv.to(F64)
    half = rd // 2
    c = cos.to(x.device, F64)[:x.shape[1]].view(1, -1, 1, half)
    s = sin.to(x.device, F64)[:x.shape[1]].view(1, -1, 1, half)
    f = lambda t: t.to(torch.float32).to(F64)        # noqa: E731
    y = x.clone()
    for w in (0, 1):
        x1, x2 = x[:, :, w, :, :half], x[:, :, w, :, half:rd]
        if fma:       # x1 c is exact in float64 (24 x 24 bits): one rounding of x1 c - fl(x2 s)
            y1, y2 = f(x1 * c - f(x2 * s)), f(x2 * c + f(x1 * s))
        else:
            y1, y2 = f(f(x1 * c) - f(x2 * s)), f(f(x2 * c) + f(x1 * s))
        y[:, :, w, :, :half], y[:, :, w, :, half:rd] = y1, y2
    return stored(y, dtype)


# ---------------------------------------------------------------------------------------------------------------
# rotary probes
# ---------------------------------------------------------------------------------------------------------------
def exact_probe(B, T, nh, hd, rd, gen):
    """(qkv float64 [B,T,3,nh,hd], cos, sin fp32 [B*T+1, rd/2]).  The kernel gets rows 0..T-1 (a view at the start of
    the table); the rows after them are what a kernel reading past its T rows (a flat token index, row t + 1) finds."""
    mag = torch.randint(1, 16, (B, T, 3, nh, hd), generator=gen).to(F64)
    x = torch.where(torch.rand(B, T, 3, nh, hd, generator=gen) < 0.5, -mag, mag)
    q = torch.tensor(QUARTERS, dtype=torch.float32)
    cos = q[torch.randint(0, 8, (B * T + 1, rd // 2), generator=gen)]
    sin = q[torch.randint(0, 8, (B * T + 1, rd // 2), generator=gen)]
    return x, cos, sin


def phi_tables(n, rd, theta=10000.0):
    """cos / sin [n, rd/2] fp32 as PhiModel.rope_tables builds them."""
    inv = 1.0 / (theta ** (torch.arange(0, rd, 2, dtype=torch.int64).float() / rd))
    fr = torch.arange(n).float()[:, None] * inv[None, :]
    return fr.cos().contiguous(), fr.sin().contiguous()


def float_probe(B, T, nh, hd, rd, dtype, gen, P=0):
    """(storage-rounded qkv float64, cos, sin [B*T+1, rd/2]): Phi table rows from P on, of which the kernel gets the
    first T (as in exact_probe).  In q and k of every even head and even token, x[i + half] is the storage rounding
    of x[i] c / s (|s| >= 1/64): y[i] cancels."""
    half = rd // 2
    cos, sin = phi_tables(P + B * T + 1, rd)
    cos, sin = cos[P:].contiguous(), sin[P:].contiguous()
    x = torch.randn(B, T, 3, nh, hd, generator=gen, dtype=F64) * 2.0
    x = stored(x, dtype)
    c, s = cos[:T].to(F64).view(1, T, 1, half), sin[:T].to(F64).view(1, T, 1, half)
    for w in (0, 1):
        x1 = x[:, 0::2, w, 0::2, :half]
        cc, sc = c[:, 0::2], s[:, 0::2]
        ok = sc.abs() >= 1 / 64
        canc = stored(x1 * cc / torch.where(ok, sc, torch.ones_like(sc)), dtype)
        x[:, 0::2, w, 0::2, half:rd] = torch.where(ok, canc, x[:, 0::2, w, 0::2, half:rd])
    return x, cos, sin


# ---------------------------------------------------------------------------------------------------------------
# rotary composed with attention: quarter-turn tables, post-rotary probes, their inputs
# ---------------------------------------------------------------------------------------------------------------
def quarter_tables(n, rd, gen):
    """cos / sin [n, rd/2] fp32: a random quarter turn per (row, pair)."""
    k = torch.randint(0, 4, (n, rd // 2), generator=gen)
    cos = torch.tensor([1.0, 0.0, -1.0, 0.0])[k]
    sin = torch.tensor([0.0, 1.0, 0.0, -1.0])[k]
    return cos.contiguous(), sin.contiguous()


def unrotate(qkv, cos, sin, rd, pos=None):
    """Inputs whose rotation at rows pos is qkv (exact for quarter-turn tables)."""
    return rotate(qkv, cos, sin, rd, pos, sin_sign=-1.0)


def rotate_qk(qkv, cos, sin, rd, q_pos, k_pos, **mut):
    """q rotated at table rows q_pos and k at k_pos ([B,T] long; None = not rotated), with the mutants of `rotate`."""
    y = qkv.to(F64)
    if q_pos is not None:
        y = rotate(y, cos, sin, rd, q_pos, which=(0,), **mut)
    if k_pos is not None:
        y = rotate(y, cos, sin, rd, k_pos, which=(1,), **mut)
    return y


def rows(B, T, start=0):
    return (torch.arange(T) + start).expand(B, T)


def causal_chain_probe(B, T, nh, hd, rd, padded, gen):
    """Post-rotary (qkv' [B,T,3,nh,hd] float64, key_valid uint8 [B,T] or None, intended [B*nh, T]) built as
    attn_probe.causal_probe builds its probe (designated keys, future and invalid-key lures), without ladders and with
    every key direction in the first rd dims."""
    scale = hd ** -0.5
    kv = None
    if padded:
        kv = torch.ones(B, T, dtype=torch.uint8)
        if B > 1 and T > 12:
            kv[1, T - 9:] = 0
    Z = B * nh
    choice = torch.zeros(Z, T, dtype=torch.long)
    lure = torch.full((Z, T), -1, dtype=torch.long)
    t = torch.arange(T)
    for b in range(B):
        cand = sorted({p for p in ap.SPECIAL if p < T} | {T - 2, T - 1} - {-1} |
                      set(torch.randint(0, T, (4,), generator=gen).tolist()))
        if padded:
            bad = [p + 1 for p in cand[1::3] if p + 1 < T and p + 1 not in cand][:3]
            kv[b, bad] = 0
        valid = [p for p in cand if kv is None or kv[b, p]][: rd - 6]
        vt = torch.tensor(valid)
        n_le = torch.searchsorted(vt, t, right=True)
        for h in range(nh):
            z = b * nh + h
            choice[z] = vt[(t + h) % n_le]
            choice[z, vt] = vt
            pv = vt[vt >= 1]
            lure[z, pv - 1] = pv
            if padded:
                for p in valid:
                    if p + 1 < T and not kv[b, p + 1]:
                        r = (choice[z] == p).nonzero().flatten()
                        lure[z, r[r >= p + 1]] = p + 1
    q, k, v, _ = ap.keyed(Z, T, T, hd, scale, choice, lure, reserved=hd - rd, gen=gen)
    qkv = torch.stack([ap.heads_in(q, B, nh), ap.heads_in(k, B, nh), ap.heads_in(v, B, nh)], 2)
    return qkv, kv, choice


def prefix_chain_probe(B, P, T, nh, hd, rd, gen):
    """Post-rotary (qkv' [B,T,3,nh,hd] of the suffix, pk', pv [nh, page, hd] of a one-page prefix cache of
    page = P rounded up to 64 rows, intended [B*nh, T] in the key axis [P | own]), built as attn_probe.prefix_probe
    builds its probe with every key direction in the first rd dims.  Rows P..page-1 of the page are poison (they lure
    rows and carry V = +-8) when P is not a multiple of 64."""
    scale = hd ** -0.5
    ld = -(-P // 64) * 64
    Lk = ld + T
    pre = sorted({p for p in (0, 1, 31, 62, 63, 64, 65, 127, 200, 289) if p < P} | {P - 1})
    own = sorted({u for u in (0, 1, 15, 16, 63, 64, 100, 159) if u < T} | {T - 1})
    poison = sorted({p for p in (P, P + 1, ld - 1) if P <= p < ld})
    choice = torch.zeros(nh, T, dtype=torch.long)
    lure = torch.full((nh, T), -1, dtype=torch.long)
    for h in range(nh):
        for r in range(T):
            ol = [u for u in own if u <= r]
            choice[h, r] = ld + ol[(r + h) % len(ol)] if r % 2 == 1 and ol else pre[(r + h) % len(pre)]
            if r + 1 in own:
                lure[h, r] = ld + r + 1
            elif poison:
                lure[h, r] = poison[(r + h) % len(poison)]
    q, k, v, _ = ap.keyed(nh, T, Lk, hd, scale, choice, lure, reserved=hd - rd, gen=gen)
    v[:, poison] *= 8.0
    pk, pv = k[:, :ld].clone(), v[:, :ld].clone()
    qkv = torch.stack([ap.heads_in(q, 1, nh), ap.heads_in(k[:, ld:], 1, nh), ap.heads_in(v[:, ld:], 1, nh)],
                      2).repeat(B, 1, 1, 1, 1)
    for b in range(1, B):
        qkv[b, :, 2, :, 1:] = torch.where(torch.rand(T, nh, hd - 1, generator=gen) < 0.5, -1.0, 1.0).double()
    intended = torch.where(choice >= ld, choice - ld + P, choice).repeat(B, 1)
    return qkv, pk, pv, intended


def prefix_inputs(qkv_s, pk_s, pv_s, P, cos, sin, rd, pre_start=0, suf_start=None):
    """Pre-rotary inputs of the prompt-suffix chain from storage-rounded post-rotary values: the prefix
    qkv [1,P,3,nh,hd] (q = 0; k un-rotated at rows pre_start..; v) and the suffix qkv (q, k un-rotated at rows
    suf_start.. (default P))."""
    nh, hd = pk_s.shape[0], pk_s.shape[2]
    B, T = qkv_s.shape[:2]
    pre = torch.zeros(1, P, 3, nh, hd, dtype=F64)
    pre[0, :, 1] = pk_s[:, :P].transpose(0, 1)
    pre[0, :, 2] = pv_s[:, :P].transpose(0, 1)
    pre = unrotate(pre, cos, sin, rd, rows(1, P, pre_start))
    suf = unrotate(qkv_s, cos, sin, rd, rows(B, T, P if suf_start is None else suf_start))
    return pre, suf


def decode_chain_probe(lens, nh, hd, rd, ps, gen):
    """Post-rotary paged decode: sequence b has lens[b] cached tokens and its new token at slot lens[b] (attention over
    lens[b] + 1 keys); slot lens[b] + 1 holds a lure with V = +-4.  Returns (q' [B, nh, hd], kc', vc
    [pages, nh, ps, hd] (every slot 0..lens[b] + 1 written, the rest 0), block_table [B, max_pages] int32 (pages in
    random order), intended [B*nh, 1]).  Head h of sequence b intends one of key 0, the page boundaries, 31 / 32,
    127 / 128 / 129, lens[b] - 1 and lens[b] (its own key)."""
    B = len(lens)
    scale = hd ** -0.5
    max_pages = -(-(max(lens) + 2) // ps) + 1
    bt = torch.randperm(B * max_pages, generator=gen).view(B, max_pages).to(torch.int32)
    kc = torch.zeros(B * max_pages, nh, ps, hd, dtype=F64)
    vc = torch.zeros_like(kc)
    q = torch.zeros(B, nh, hd, dtype=F64)
    intended = torch.zeros(B * nh, 1, dtype=torch.long)
    for b, L in enumerate(lens):
        cand = sorted({p for p in (0, ps - 1, ps, 2 * ps - 1, 2 * ps, 31, 32, 127, 128, 129, L - 1, L) if 0 <= p <= L})
        choice = torch.tensor([[cand[(h * 5 + b) % len(cand)]] for h in range(nh)])
        qz, kz, vz, _ = ap.keyed(nh, 1, L + 2, hd, scale, choice, torch.full((nh, 1), L + 1), reserved=hd - rd,
                                 gen=gen)
        vz[:, L + 1] *= 4.0
        q[b] = qz[:, 0]
        intended[b * nh:(b + 1) * nh] = choice
        pos = torch.arange(L + 2)
        pg, sl = bt[b, pos // ps].long(), pos % ps
        kc[pg, :, sl] = kz.transpose(0, 1)
        vc[pg, :, sl] = vz.transpose(0, 1)
    return q, kc, vc, bt, intended


def gather_rows(cache, bt, b, n):
    """Slots 0..n-1 of sequence b: [n, nh, hd]."""
    ps = cache.shape[2]
    pos = torch.arange(n)
    return cache[bt[b, pos // ps].long(), :, pos % ps]


def decode_inputs(q_s, kc_s, vc_s, bt, lens, cos, sin, rd):
    """Pre-rotary inputs of the decode chain from storage-rounded post-rotary values: per sequence the prefill
    qkv [1,L,3,nh,hd] (q = 0, k un-rotated at rows 0..L-1, v) and the new tokens qkv [B,1,3,nh,hd] (q and k
    un-rotated at row L).  The lure slot L + 1 is not an input: it stays in the cache as written."""
    B, nh, hd = q_s.shape
    pres = []
    new = torch.zeros(B, 1, 3, nh, hd, dtype=F64)
    for b, L in enumerate(lens):
        kk, vv = gather_rows(kc_s, bt, b, L + 1), gather_rows(vc_s, bt, b, L + 1)
        pre = torch.zeros(1, L, 3, nh, hd, dtype=F64)
        pre[0, :, 1], pre[0, :, 2] = kk[:L], vv[:L]
        pres.append(unrotate(pre, cos, sin, rd))
        one = torch.zeros(1, 1, 3, nh, hd, dtype=F64)
        one[0, 0, 0], one[0, 0, 1], one[0, 0, 2] = q_s[b], kk[L], vv[L]
        new[b] = unrotate(one, cos, sin, rd, torch.tensor([[L]]))[0]
    return pres, new


# chain emulators (float64): the kernels' composition with one named mistake; no arguments = the correct chain -------
def _pos(B, T, start, on):
    return rows(B, T, start) if on else None


def causal_chain(qkv_in, kv, cos, sin, rd, q_shift=0, k_shift=0, q_rot=True, k_rot=True, **mut):
    B, T, _, nh, hd = qkv_in.shape
    y = rotate_qk(qkv_in, cos, sin, rd, _pos(B, T, q_shift, q_rot), _pos(B, T, k_shift, k_rot), **mut)
    return ap.attend(ap.causal_problem(y, kv, B, T, nh, hd, dev=torch.device("cpu")))


def prefix_chain(pre, suf, pk_s, pv_s, P, cos, sin, rd, pre_start=0, suf_start=None, q_shift=0, k_shift=0,
                 q_rot=True, k_rot=True, **mut):
    B, T, _, nh, hd = suf.shape
    suf_start = P if suf_start is None else suf_start
    pre_y = rotate_qk(pre, cos, sin, rd, None, _pos(1, P, pre_start + k_shift, k_rot), **mut)
    pk = pk_s.clone()
    pk[:, :P] = pre_y[0, :, 1].transpose(0, 1)
    y = rotate_qk(suf, cos, sin, rd, _pos(B, T, suf_start + q_shift, q_rot), _pos(B, T, suf_start + k_shift, k_rot),
                  **mut)
    return ap.attend(ap.prefix_problem(y, pk, pv_s, P, None, B, T, nh, hd, dev=torch.device("cpu")))


def decode_chain(pres, new, kc_s, vc_s, bt, lens, cos, sin, rd, pre_shift=0, q_shift=0, newk_shift=0, q_rot=True,
                 k_rot=True, **mut):
    """pre_shift: the prefill keys at rows t + pre_shift; q_shift / newk_shift: the new token's q / k at row
    lens[b] + shift."""
    kc = kc_s.clone()
    ps = kc.shape[2]
    y_new = torch.zeros_like(new)
    for b, L in enumerate(lens):
        pre_y = rotate_qk(pres[b], cos, sin, rd, None, _pos(1, L, pre_shift, k_rot), **mut)
        one = rotate_qk(new[b:b + 1], cos, sin, rd, _pos(1, 1, L + q_shift, q_rot), _pos(1, 1, L + newk_shift, k_rot),
                        **mut)
        y_new[b] = one[0]
        pos = torch.arange(L + 1)
        kc[bt[b, pos // ps].long(), :, pos % ps] = torch.cat([pre_y[0, :, 1], one[0, :, 1]], 0)
    seq = torch.tensor(lens, dtype=torch.int32) + 1
    return ap.attend(ap.decode_problem(y_new, kc, vc_s, bt, seq, dev=torch.device("cpu")))


# ---------------------------------------------------------------------------------------------------------------
# linear_act
# ---------------------------------------------------------------------------------------------------------------
def act_probe(M, N, K):
    """(x [M, K], W [N, K], bias [N]) float64, exact in bf16 and fp16; z = x W^T + b in [-9, 9] in steps of 1/16."""
    x = torch.zeros(M, K, dtype=F64)
    x[torch.arange(M), (37 * torch.arange(M)) % K] = 1.0
    n = torch.arange(N, dtype=torch.int64)[:, None]
    k = torch.arange(K, dtype=torch.int64)[None]
    w = (((131 * n + 17 * k) % 257) - 128).to(F64) / 16
    b = (((29 * torch.arange(N, dtype=torch.int64)) % 33) - 16).to(F64) / 16
    return x, w, b


def gelu_new(z):
    return 0.5 * z * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (z + 0.044715 * z ** 3)))


def gelu_bound(z, g, dtype):
    return half_ulp(g.abs(), dtype) + z.abs() * UNIT[dtype]
