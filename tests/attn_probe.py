"""Float64 attention references, a per-element error bound, and probe inputs for the attention kernels.

No kernel is called here.  tests/test_attention_probes_cpu.py shows that every probe fails (by >= 10x its bound) the
mutant semantics a subtly wrong tiled / split / masked kernel would compute; tests/test_attention_probes_gpu.py runs
the kernels on the same probes.

The references are written independently of tests/emu.py (the CPU tests install emu as the kernels, so a bug shared
by the two would never show).  They take the storage-rounded inputs, compute in float64 on the device when one is
present, and work in one layout: Z = independent (image / window, head) instances, q [Z, Lq, d], k / v [Z, Lk, d],
`allowed` [Z, Lq, Lk] and an optional additive score bias.  Each family maps its kernel layout to that layout
(`*_problem`) and the kernel's output back into it (`*_out_z`).

Rows with no open key are defined as 0 (every kernel writes zeros there); the probes never build such rows.

Error bound (per output element, `bound`).  Attention output is a convex combination of the V rows a row may
attend, so it is scaled by vmax = max_j max_d |v_jd| over those keys, not by the output:

    |o - o_ref| <= vmax * (c_u * u + sub + expm1(2 * delta)) + 2^-24

  u      unit roundoff of the storage type (bf16 2^-8, fp16 2^-11).
  c_u    3 for 16-bit storage: 1 for P rounded to 16 bits before the PV product (each weight gets a relative error
         <= u, so the output moves by <= u * vmax), 1 for rounding the output (|o| <= vmax), and 1 of slack for the
         fp32 sums of l and O and ex2.approx: every kernel sums <= ~500 terms per fp32 chain (tiles of 32 / 64 keys
         per split, <= 128 keys per decode lane), i.e. <= 500 * 2^-24 = 3e-5 < 2^-11.
         fp32 storage (SIMT kernels): u = 2^-24 and c_u = 2 * (ceil(n_open / 32) + 32) + 8: the sequential chains
         of the tile-by-tile l and O updates (one per 32-key tile plus 32 terms inside a tile), expf and the output.
  sub    fp16 only: P below 2^-14 is subnormal and rounds with an absolute error <= 2^-25 each; l >= 1 (the row's
         maximum key contributes 1), so n_open * 2^-25 bounds their effect.  bf16 has fp32's exponent range.
  delta  error (nats) of the scores: hd * 2^-24 * scale * max_j sum_d |q_d k_jd| for the fp32 accumulation of the
         products of 16-bit operands (exact products), plus u * scale * max_j sum_d |q_d k_jd| where the kernel rounds
         an operand after scaling (the TMA cross-attention kernel stores q * scale * log2e as 16 bits).  For the
         latter k_jd is replaced by k_jd - kbar_d (kbar = the mean key of the instance): q_d (1 + e_d) kbar_d adds the
         same amount to every score of the row, which cancels in the softmax and in every split combine, so only
         the key-dependent part counts (a dimension in which all keys are equal contributes nothing).  Score
         errors <= delta move every weight by a factor in [e^-2delta, e^2delta] (numerator and normaliser), and
         since the weight changes sum to 0 the output moves by <= expm1(2 delta) * vmax.
  2^-24  absolute floor for outputs near zero (fp16 subnormal outputs round with absolute error 2^-25).

Probes.  Each query row (per head) puts >= 0.99 of its weight on one intended key.  V rows carry a +-1 code: column
0 is +1 for keys some row intends and -1 for every other key; columns 1.. are random signs per key.  Attending a
wrong key, a mixture, or nothing therefore moves some output element by O(1), not O(1/L).  Scores come from one-hot
directions: the intended keys of an instance each own one dimension (k = 8 e_m), a row intending key m has q =
alpha e_m with alpha * 8 * scale = 16 nats, and every other key has |k| ~ 0.02 noise, so the intended key is 16 nats
above the rest (enough for 0.99 at 27889 keys) and sum_d |q_d k_d| stays ~16 nats.  A row may also carry a lure:
1.5x the attraction (24 nats) towards a key it must not see (a future key, an invalid key, a padding row of the
prefix, a slot past seq_len, the next image's rows); if the kernel lets it in, it wins.
"""
import torch

UNIT = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 2.0 ** -24}
G = 16.0            # nats between an intended key and the rest
BETA = 8.0          # |k| of a designated key along its own direction
LURE = 1.5          # attraction of a lure relative to the intended key (24 nats against 16)


def device():
    return torch.device("cuda") if torch.cuda.is_available() else torch.device("cpu")


def stored(x, dtype):
    """Storage rounding, back to float64."""
    return x.to(dtype).to(torch.float64)


# ---------------------------------------------------------------------------------------------------------------
# core reference, bound and check
# ---------------------------------------------------------------------------------------------------------------
def _scores(pb):
    s = torch.matmul(pb["q"], pb["k"].transpose(-1, -2)) * pb["scale"]
    if pb.get("bias") is not None:
        s = s + pb["bias"]
    return s.masked_fill(~pb["allowed"], float("-inf"))


def attend(pb):
    """Float64 attention of a problem dict -> dict(out, w, vmax, sabs, nopen) in the Z layout."""
    s = _scores(pb)
    w = torch.softmax(s, -1).nan_to_num(0.0)      # rows without an open key: 0, as the kernels write
    out = torch.matmul(w, pb["v"])
    allowed = pb["allowed"].expand(s.shape)
    vabs = pb["v"].abs().amax(-1)                   # [Z, Lk]
    vmax = torch.where(allowed, vabs.unsqueeze(-2), torch.zeros((), dtype=vabs.dtype, device=vabs.device)).amax(-1)
    sabs = torch.matmul(pb["q"].abs(), pb["k"].abs().transpose(-1, -2)) * pb["scale"]
    zero = torch.zeros((), dtype=sabs.dtype, device=sabs.device)
    sabs = torch.where(allowed, sabs, zero).amax(-1)
    # the same against K centred on its mean key: the part of a q-rounding error that is common to all keys of a row
    kc = pb["k"] - pb["k"].mean(-2, keepdim=True)
    sabs_c = torch.matmul(pb["q"].abs(), kc.abs().transpose(-1, -2)) * pb["scale"]
    sabs_c = torch.where(allowed, sabs_c, zero).amax(-1)
    return dict(out=out, w=w, vmax=vmax, sabs=sabs, sabs_c=sabs_c, nopen=allowed.sum(-1))


def bound(ref, dtype, hd, q_rounded=False):
    """Per-row bound [Z, Lq, 1] (see the module docstring for every term)."""
    u = UNIT[dtype]
    n = ref["nopen"].to(torch.float64)
    delta = ref["sabs"] * hd * 2.0 ** -24 + (u * ref["sabs_c"] if q_rounded else 0.0)
    if dtype == torch.float32:
        cu = 2.0 * (torch.ceil(n / 32) + 32) + 8
        sub = 0.0
    else:
        cu = 3.0
        sub = n * 2.0 ** -25 if dtype == torch.float16 else 0.0
    return (ref["vmax"] * (cu * u + sub + torch.expm1(2 * delta)) + 2.0 ** -24).unsqueeze(-1)


def ratio(out_z, ref, bnd, rows=None):
    """max |out - ref| / bound over the compared rows (out_z in the Z layout, any float type); asserts finiteness."""
    o = out_z.to(torch.float64)
    assert torch.isfinite(o if rows is None else o[rows]).all(), "non-finite kernel output"
    r = (o - ref["out"]).abs() / bnd
    if rows is not None:
        r = r[rows]
    return float(r.max()) if r.numel() else 0.0


def intended_weight(ref, intended):
    """Weight each row puts on its intended key ([Z, Lq] long)."""
    return ref["w"].gather(-1, intended.unsqueeze(-1).to(ref["w"].device)).squeeze(-1)


# ---------------------------------------------------------------------------------------------------------------
# generic mutants: the same float64 code with one semantic changed
# ---------------------------------------------------------------------------------------------------------------
def drop_keys(pb, lo, hi):
    """A kernel that skips keys [lo, hi) (a whole key tile)."""
    a = pb["allowed"].expand(pb["allowed"].shape[:-2] + (pb["q"].shape[-2], pb["k"].shape[-2])).clone()
    a[..., lo:hi] = False
    return dict(pb, allowed=a)


def online(pb, tile, splits=1, skip_rescale=None, drop_split=None, empty_split_m0=False):
    """Tile-by-tile online softmax with split-K over contiguous tile ranges and a (m, l, O) combine, as the kernels
    run it, in float64.  Mutants: `skip_rescale` = a tile whose running-max rescale is skipped, `drop_split` = a split
    left out of the combine, `empty_split_m0` = a split without open keys enters the combine with m = 0 instead of
    being skipped (its exp weights then underflow in fp32 as in the kernel)."""
    s, v = _scores(pb), pb["v"]
    Lk = s.shape[-1]
    nt = -(-Lk // tile)
    tps = -(-nt // splits)
    parts = []
    for sp in range(splits):
        m = torch.full(s.shape[:-1] + (1,), float("-inf"), dtype=s.dtype, device=s.device)
        l = torch.zeros_like(m)
        o = torch.zeros(s.shape[:-1] + (v.shape[-1],), dtype=s.dtype, device=s.device)
        for t in range(sp * tps, min(nt, (sp + 1) * tps)):
            st = s[..., t * tile:(t + 1) * tile]
            m_new = torch.maximum(m, st.amax(-1, keepdim=True))
            fin = torch.isfinite(m_new)
            corr = torch.where(fin & torch.isfinite(m), torch.exp(m - m_new), torch.zeros_like(m))
            corr = torch.where(fin, corr, torch.ones_like(m))
            if skip_rescale == t:
                corr = torch.ones_like(m)
            p = torch.where(fin, torch.exp(st - torch.where(fin, m_new, torch.zeros_like(m_new))), torch.zeros_like(st))
            l = l * corr + p.sum(-1, keepdim=True)
            o = o * corr + torch.matmul(p, v[..., t * tile:(t + 1) * tile, :])
            m = m_new
        parts.append((m, l, o))
    if drop_split is not None:
        parts.pop(drop_split)
    ms = torch.stack([p[0] for p in parts])
    if empty_split_m0:
        ms = torch.where(torch.isfinite(ms), ms, torch.zeros_like(ms))
    M = ms.amax(0)
    e = torch.exp((ms - torch.where(torch.isfinite(M), M, torch.zeros_like(M))).float()).double()   # fp32 as in the combine
    e = torch.where(torch.isfinite(ms), e, torch.zeros_like(e))
    L = sum(e[i] * parts[i][1] for i in range(len(parts)))
    O = sum(e[i] * parts[i][2] for i in range(len(parts)))
    return torch.where(L > 0, O / torch.where(L > 0, L, torch.ones_like(L)), torch.zeros_like(O))


# ---------------------------------------------------------------------------------------------------------------
# probe inputs in the Z layout
# ---------------------------------------------------------------------------------------------------------------
def keyed(Z, Lq, Lk, hd, scale, choice, lure=None, reserved=2, gen=None):
    """q [Z,Lq,hd], k / v [Z,Lk,hd] (float64, before storage rounding): row r of instance z intends key choice[z, r];
    lure[z, r] >= 0 adds a 1.5x stronger attraction to that key.  Dimensions hd-reserved.. are left for callers
    (ladders, baselines, cross-image lures).  Returns (q, k, v, designated keys per instance)."""
    D = hd - reserved
    alpha = G / (BETA * scale)
    k = torch.randn(Z, Lk, hd, generator=gen, dtype=torch.float64) * 0.02
    k[..., D:] = 0
    q = torch.zeros(Z, Lq, hd, dtype=torch.float64)
    v = torch.where(torch.rand(Z, Lk, hd, generator=gen) < 0.5, -1.0, 1.0).to(torch.float64)
    v[..., 0] = -1.0
    rows = torch.arange(Lq)
    keys = []
    for z in range(Z):
        ch = choice[z]
        lz = lure[z] if lure is not None else torch.full((Lq,), -1, dtype=torch.long)
        allk = torch.unique(torch.cat([ch, lz[lz >= 0]]))
        if allk.numel() > D:
            raise ValueError("probe: %d designated keys, %d directions" % (allk.numel(), D))
        pos = torch.full((Lk,), -1, dtype=torch.long)
        pos[allk] = torch.randperm(D, generator=gen)[:allk.numel()]   # per instance: heads differ in K, not just V
        k[z, allk] = 0
        k[z, allk, pos[allk]] = BETA
        q[z, rows, pos[ch]] = alpha
        lr = lz >= 0
        q[z, rows[lr], pos[lz[lr]]] = LURE * alpha
        v[z, ch, 0] = 1.0
        keys.append(allk)
    return q, k, v, keys


def ladder(q, k, v, z, kind, tile, scale, span=100):
    """Turn instance z into a ladder (all its rows; dimension hd-2).  "rise": the row maximum climbs by 8 nats with
    every key tile of the last `span` tiles (a peak key at the start of each such tile, 12 nats above that tile's
    plateau), so the running max is rescaled at every tile; "first": the maximum is key 0 and every later tile sits
    20 nats below tile 0.  Returns the intended key of a row that sees keys [0, n): see ladder_intended."""
    hd, Lk = q.shape[-1], k.shape[-2]
    L = hd - 2
    c = 4.0                                           # nats per unit of k[:, L]: integers <= 256 stay exact in bf16
    q[z] = 0
    q[z, :, L] = c / scale
    j = torch.arange(Lk)
    t = j // tile
    nt = -(-Lk // tile)
    k[z, :, L] = 0
    v[z, :, 0] = -1.0
    if kind == "rise":
        t0 = max(0, nt - span)
        climb = t >= t0
        peak = climb & (j % tile == 0)
        k[z, :, L] = torch.where(climb, 2.0 * (t - t0 + 1), torch.zeros(Lk, dtype=torch.float64)) + 3.0 * peak
        v[z, peak, 0] = 1.0
    else:
        k[z, :, L] = torch.where(t == 0, 0.0, -5.0).to(torch.float64)
        k[z, 0, L] = 3.0
        v[z, 0, 0] = 1.0


def ladder_intended(kind, tile, Lk, last, span=100):
    """Intended key of a ladder row whose last visible key is `last` (tensor)."""
    if kind == "first":
        return torch.zeros_like(last)
    nt = -(-Lk // tile)
    t0 = max(0, nt - span)
    return torch.clamp(last // tile, min=t0) * tile


# ---------------------------------------------------------------------------------------------------------------
# window attention (Swin W-MSA / SW-MSA): qkv [B, H*W, 3C], qkv_bias [3C], compact rel table [nh, (2ws-1)^2]
# ---------------------------------------------------------------------------------------------------------------
def rel_index(ws):
    y, x = torch.meshgrid(torch.arange(ws), torch.arange(ws), indexing="ij")
    y, x = y.reshape(-1), x.reshape(-1)
    return (y[:, None] - y[None, :] + ws - 1) * (2 * ws - 1) + (x[:, None] - x[None, :] + ws - 1)


def _regions(Hp, Wp, ws, shift):
    """Shift-mask region of every padded position (the reference's three slices per axis)."""
    ry = torch.where(torch.arange(Hp) < Hp - ws, 0, torch.where(torch.arange(Hp) < Hp - shift, 1, 2))
    rx = torch.where(torch.arange(Wp) < Wp - ws, 0, torch.where(torch.arange(Wp) < Wp - shift, 1, 2))
    return ry[:, None] * 3 + rx[None, :]


def _partition(x, B, Hp, Wp, ws, nh):
    """[B, Hp, Wp, nh*hd] -> [B*nW*nh, ws*ws, hd]."""
    hd = x.shape[-1] // nh
    x = x.reshape(B, Hp // ws, ws, Wp // ws, ws, nh, hd).permute(0, 1, 3, 5, 2, 4, 6)
    return x.reshape(-1, ws * ws, hd)


def window_problem(qkv, qkv_bias, rel, B, H, W, C, nh, ws, shift, rel_heads=None, shift_mask=True, dev=None):
    """rel_heads: head -> table row (mutant: every head of a CTA reads its first head's row); shift_mask=False: the
    mutant that drops the -100 mask."""
    dev = dev or device()
    Hp, Wp = -(-H // ws) * ws, -(-W // ws) * ws
    x = qkv_bias.to(dev, torch.float64).view(1, 1, 1, 3 * C).repeat(B, Hp, Wp, 1)
    x[:, :H, :W] = qkv.to(dev, torch.float64).view(B, H, W, 3 * C)
    real = torch.zeros(B, Hp, Wp, 1, dtype=torch.float64, device=dev)
    real[:, :H, :W] = 1
    if shift:
        x = torch.roll(x, (-shift, -shift), (1, 2))
        real = torch.roll(real, (-shift, -shift), (1, 2))
    q, k, v = (_partition(x[..., i * C:(i + 1) * C], B, Hp, Wp, ws, nh) for i in range(3))
    N, nW = ws * ws, (Hp // ws) * (Wp // ws)
    table = rel.to(dev, torch.float64)
    if rel_heads is not None:
        table = table[torch.as_tensor(rel_heads, device=dev)]
    bias = table[:, rel_index(ws).to(dev)].unsqueeze(0).expand(B * nW, nh, N, N)
    if shift and shift_mask:
        reg = _partition(_regions(Hp, Wp, ws, shift).to(dev, torch.float64)[None, :, :, None].repeat(1, 1, 1, 1),
                         1, Hp, Wp, ws, 1)[:, :, 0]                                  # [nW, N]
        m = torch.where(reg[:, :, None] != reg[:, None, :], -100.0, 0.0).to(dev, torch.float64)
        bias = bias + m.repeat(B, 1, 1).unsqueeze(1)
    rows = _partition(real.expand(B, Hp, Wp, nh), B, Hp, Wp, ws, nh)[..., 0] > 0
    allowed = torch.ones(1, N, N, dtype=torch.bool, device=dev)
    return dict(q=q, k=k, v=v, allowed=allowed, bias=bias.reshape(-1, N, N), scale=(C // nh) ** -0.5, rows=rows,
                geom=(B, H, W, C, nh, ws, shift))


def window_out_z(out, pb):
    """Kernel output [B, H*W, C] -> Z layout of the problem (padded rows are zero and not compared)."""
    B, H, W, C, nh, ws, shift = pb["geom"]
    Hp, Wp = -(-H // ws) * ws, -(-W // ws) * ws
    x = torch.zeros(B, Hp, Wp, C, dtype=torch.float64, device=pb["q"].device)
    x[:, :H, :W] = out.to(pb["q"].device, torch.float64).view(B, H, W, C)
    if shift:
        x = torch.roll(x, (-shift, -shift), (1, 2))
    return _partition(x, B, Hp, Wp, ws, nh)


def window_hpc(B, H, W, nh, ws=12):
    """Heads per CTA the tensor-core window kernel picks (restates launch_window in csrc/attn_mma.cu)."""
    windows = B * (-(-H // ws)) * (-(-W // ws))
    if nh % 4 == 0 and windows * (nh // 4) >= 600:
        return 4
    if nh % 2 == 0 and windows * (nh // 2) >= 132:
        return 2
    return 1


def window_probe(B, H, W, C, nh, ws, shift, dtype, gen, qk_std=0.1):
    """Per-head rel-bias probe: head h's table is +20 at its own offset (dy_h, dx_h) and +12 at (0, 0); Q / K are
    small.  A row whose offset key lies inside its window (and, shifted, in its own region) intends that key (8 nats
    above self, 20 above the rest); any other row intends itself (12 nats above the rest).  Where the offset key
    lies in another shift region it is favoured by 8 but masked by -100.  V is a +-1 code per token; padded tokens
    carry the qkv bias, whose V part is a +-1 code too."""
    R = 2 * ws - 1
    qkv = torch.randn(B, H * W, 3 * C, generator=gen, dtype=torch.float64) * qk_std
    qkv[..., 2 * C:] = torch.where(torch.rand(B, H * W, C, generator=gen) < 0.5, -1.0, 1.0).double()
    bias = torch.randn(3 * C, generator=gen, dtype=torch.float64) * qk_std
    bias[2 * C:] = torch.where(torch.rand(C, generator=gen) < 0.5, -1.0, 1.0).double()
    rel = torch.randn(nh, R * R, generator=gen, dtype=torch.float64) * 0.1
    offs = []
    for h in range(nh):
        dy, dx = 1 + (h * 5) % (ws - 2), -((h * 3) % (ws - 1))   # distinct for the heads of a CTA (and mostly overall)
        if h % 3 == 2:
            dy = -dy
        offs.append((dy, dx))
        rel[h, (dy + ws - 1) * R + (dx + ws - 1)] = 20.0
        rel[h, (ws - 1) * R + (ws - 1)] = 12.0
    return qkv.to(dtype), bias.to(dtype), rel.float(), offs


# ---------------------------------------------------------------------------------------------------------------
# causal / prefix-causal prefill: qkv [B, T, 3, nh, hd]
# ---------------------------------------------------------------------------------------------------------------
def causal_problem(qkv, key_valid, B, T, nh, hd, future=0, ignore_valid=False, dev=None):
    """future=1: the mutant that lets key t+1 in; ignore_valid: the mutant that ignores key_valid."""
    dev = dev or device()
    x = qkv.to(dev, torch.float64)
    q, k, v = (x[:, :, i].permute(0, 2, 1, 3).reshape(B * nh, T, hd) for i in range(3))
    t = torch.arange(T, device=dev)
    allowed = (t[None, :] <= t[:, None] + future).unsqueeze(0).expand(B, T, T)
    if key_valid is not None and not ignore_valid:
        allowed = allowed & key_valid.to(dev).bool()[:, None, :]
    allowed = allowed.unsqueeze(1).expand(B, nh, T, T).reshape(B * nh, T, T)
    return dict(q=q, k=k, v=v, allowed=allowed, scale=hd ** -0.5)


def heads_out_z(out, B, T, nh, hd, dev=None):
    """[B, T, nh*hd] -> [B*nh, T, hd]."""
    dev = dev or device()
    return out.to(dev, torch.float64).view(B, T, nh, hd).permute(0, 2, 1, 3).reshape(B * nh, T, hd)


def heads_in(x, B, nh):
    """[B*nh, L, hd] -> [B, L, nh, hd]."""
    Z, L, hd = x.shape
    return x.view(B, nh, L, hd).permute(0, 2, 1, 3)


SPECIAL = (0, 1, 31, 32, 62, 63, 64, 65, 126, 127, 128, 129, 255, 256, 511, 512, 899, 900, 1023, 1024, 1099, 2047)


def causal_probe(B, T, nh, hd, padded, gen, ladders=("rise", "first")):
    """qkv [B,T,3,nh,hd] float64, key_valid uint8 [B,T] or None, intended [B*nh, T] long.
    Designated keys: SPECIAL positions below T, T-2, T-1 and a few random ones (valid ones only).  Row t intends t
    itself when t is designated, otherwise one of the designated keys <= t (cycling with the head).  Rows s-1 are
    lured to the future key s for designated s; with `padded`, a key next to a designated one is invalid and lures
    the rows that intend its neighbour, and sequence 1 ends in 9 invalid keys.  The last len(ladders) heads are
    ladders (64-key tiles)."""
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
        cand = sorted({p for p in SPECIAL if p < T} | {T - 2, T - 1} - {-1} |
                      set(torch.randint(0, T, (6,), generator=gen).tolist()))
        if padded:   # invalid neighbours of designated keys (never a ladder peak, which sits at a multiple of 64)
            bad = [p + 1 for p in cand[1::3] if p + 1 < T and p + 1 not in cand and (p + 1) % 64][:4]
            kv[b, bad] = 0
        valid = [p for p in cand if kv is None or kv[b, p]][: hd - 8]
        vt = torch.tensor(valid)
        n_le = torch.searchsorted(vt, t, right=True)        # designated keys <= t (key 0 is one)
        for h in range(nh):
            z = b * nh + h
            choice[z] = vt[(t + h) % n_le]
            choice[z, vt] = vt                                 # a designated row intends itself
            pv = vt[vt >= 1]
            lure[z, pv - 1] = pv                               # the future key p is the most attractive key of row p-1
            if padded:
                for p in valid:
                    if p + 1 < T and not kv[b, p + 1]:
                        rows = (choice[z] == p).nonzero().flatten()
                        lure[z, rows[rows >= p + 1]] = p + 1   # invalid neighbour, causally visible
    q, k, v, _ = keyed(Z, T, T, hd, scale, choice, lure, gen=gen)
    intended = choice.clone()
    for i, kind in enumerate(ladders):      # ladder heads of sequence 0 (never right-padded)
        z = nh - len(ladders) + i
        if z < 0:
            continue
        ladder(q, k, v, z, kind, 64, scale)
        intended[z] = ladder_intended(kind, 64, T, t)
        if kv is not None:
            assert bool(kv[0, intended[z]].all())
    qkv = torch.stack([heads_in(q, B, nh), heads_in(k, B, nh), heads_in(v, B, nh)], 2)
    return qkv, kv, intended


def prefix_problem(qkv, pk, pv, P, key_valid, B, T, nh, hd, prefix_rows=None, dev=None):
    """Key axis [prefix rows 0..prefix_rows-1 | own keys]; prefix_rows > P is the mutant that lets the padding rows of
    the prefix buffer in."""
    dev = dev or device()
    n = P if prefix_rows is None else prefix_rows
    x = qkv.to(dev, torch.float64)
    q, ko, vo = (x[:, :, i].permute(0, 2, 1, 3) for i in range(3))          # [B, nh, T, hd]
    kp = pk.to(dev, torch.float64)[:, :n].unsqueeze(0).expand(B, nh, n, hd)
    vp = pv.to(dev, torch.float64)[:, :n].unsqueeze(0).expand(B, nh, n, hd)
    k = torch.cat([kp, ko], 2).reshape(B * nh, n + T, hd)
    v = torch.cat([vp, vo], 2).reshape(B * nh, n + T, hd)
    t = torch.arange(T, device=dev)
    own = (t[None, :] <= t[:, None]).unsqueeze(0).expand(B, T, T)
    if key_valid is not None:
        own = own & key_valid.to(dev).bool()[:, None, :]
    allowed = torch.cat([torch.ones(B, T, n, dtype=torch.bool, device=dev), own], 2)
    allowed = allowed.unsqueeze(1).expand(B, nh, T, n + T).reshape(B * nh, T, n + T)
    return dict(q=q.reshape(B * nh, T, hd), k=k, v=v, allowed=allowed, scale=hd ** -0.5)


def prefix_probe(B, P, T, nh, hd, gen):
    """(qkv [B,T,3,nh,hd], pk, pv [nh, ld_rows, hd], ld_rows, intended [B*nh, T] in the axis [P | own]).
    ld_rows = P rounded up to 64, plus 64: rows P..ld_rows-1 are poison (they lure rows and have V = +-8).  Even rows
    intend a prefix key, odd rows an own key <= t (or a prefix key when none is designated yet).  Row t-1 of a
    designated own key t is lured to it (a future key); every other row to a poison row."""
    scale = hd ** -0.5
    ld = -(-P // 64) * 64 + 64
    Lk = ld + T                                         # probe axis [ld_rows | own]
    pre = sorted({p for p in (0, 1, 31, 62, 63, 64, 65, 127, 200, 289) if p < P} | {P - 1})
    own = sorted({u for u in (0, 1, 15, 16, 63, 64, 100, 159) if u < T} | {T - 1})
    poison = sorted({p for p in (P, P + 1, ld - 1)})
    Z = nh
    choice = torch.zeros(Z, T, dtype=torch.long)
    lure = torch.full((Z, T), -1, dtype=torch.long)
    for h in range(nh):
        for r in range(T):
            ol = [u for u in own if u <= r]
            if r % 2 == 1 and ol:
                choice[h, r] = ld + ol[(r + h) % len(ol)]
            else:
                choice[h, r] = pre[(r + h) % len(pre)]
            lure[h, r] = ld + r + 1 if r + 1 in own else poison[(r + h) % len(poison)]   # future own key or poison
    q, k, v, _ = keyed(Z, T, Lk, hd, scale, choice, lure, gen=gen)
    v[:, poison] *= 8.0
    pk, pv = k[:, :ld].clone(), v[:, :ld].clone()
    qkv = torch.stack([heads_in(q, 1, nh), heads_in(k[:, ld:], 1, nh), heads_in(v[:, ld:], 1, nh)], 2).repeat(B, 1, 1, 1, 1)
    for b in range(1, B):                               # other sequences: same scores, their own V codes
        qkv[b, :, 2, :, 1:] = torch.where(torch.rand(T, nh, hd - 1, generator=gen) < 0.5, -1.0, 1.0).double()
    intended = torch.where(choice >= ld, choice - ld + P, choice).repeat(B, 1)
    return qkv, pk, pv, ld, intended


# ---------------------------------------------------------------------------------------------------------------
# cross attention: q [B, Lq, C], k / v [B, Lk, C], packed bits (1 = blocked) [B, Lq, ceil(Lk/32)], row_open [B, Lq]
# ---------------------------------------------------------------------------------------------------------------
def pack_bits(blocked):
    """bool [B, Lq, Lk] -> int32 words [B, Lq, ceil(Lk/32)] (bit j of word w = key 32 w + j)."""
    B, Lq, Lk = blocked.shape
    W32 = -(-Lk // 32)
    x = torch.zeros(B, Lq, W32 * 32, dtype=torch.int64)
    x[..., :Lk] = blocked.long()
    words = (x.view(B, Lq, W32, 32) << torch.arange(32)).sum(-1)
    return torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32)


def unpack_bits(bits, Lk):
    w = bits.long() & 0xFFFFFFFF
    return (((w.unsqueeze(-1) >> torch.arange(32, device=bits.device)) & 1).flatten(-2)[..., :Lk]).bool()


def cross_problem(q, k, v, bits, row_open, nh, ignore_row_open=False, tail=0, dev=None):
    """tail > 0: the mutant that lets the first `tail` K / V rows of image b+1 in for image b (the rows a tile load
    past Lk brings in); ignore_row_open: the mutant that applies the bits of a row_open row."""
    dev = dev or device()
    B, Lq, C = q.shape
    Lk = k.shape[1]
    hd = C // nh
    qh = q.to(dev, torch.float64).view(B, Lq, nh, hd).permute(0, 2, 1, 3)
    kk, vv = k.to(dev, torch.float64), v.to(dev, torch.float64)
    allowed = torch.ones(B, Lq, Lk, dtype=torch.bool, device=dev)
    if bits is not None:
        blk = unpack_bits(bits.to(dev), Lk)
        if row_open is not None and not ignore_row_open:
            blk = blk & ~row_open.to(dev).bool().unsqueeze(-1)
        allowed = ~blk
    if tail:
        nxt = torch.cat([kk[1:, :tail], torch.zeros_like(kk[:1, :tail])], 0)
        nxv = torch.cat([vv[1:, :tail], torch.zeros_like(vv[:1, :tail])], 0)
        kk, vv = torch.cat([kk, nxt], 1), torch.cat([vv, nxv], 1)
        extra = torch.zeros(B, Lq, tail, dtype=torch.bool, device=dev)
        extra[:-1] = True
        allowed = torch.cat([allowed, extra], 2)
    kh = kk.reshape(B, -1, nh, hd).permute(0, 2, 1, 3)
    vh = vv.reshape(B, -1, nh, hd).permute(0, 2, 1, 3)
    allowed = allowed.unsqueeze(1).expand(B, nh, Lq, allowed.shape[-1])
    n = kh.shape[2]
    return dict(q=qh.reshape(B * nh, Lq, hd), k=kh.reshape(B * nh, n, hd), v=vh.reshape(B * nh, n, hd),
                allowed=allowed.reshape(B * nh, Lq, n), scale=hd ** -0.5)


def cross_probe(B, Lq, Lk, gen, nh=8, hd=32, boundaries=(), shared_kv=False):
    """(q [B,Lq,C], k, v [B or 1,Lk,C] float64, bits, row_open, intended [B*nh, Lq]).

    Designated keys: 0, 31, 32, 63, 64, both sides of the given split / tile boundaries, Lk-1 and two random keys,
    sorted and cut to the first hd-4 (key directions are scarce: with many boundaries the later ones are not probed,
    and callers pass a thinned list).  Only the rows that exist are probed: with Lq = 1 there is one all-open row,
    which intends key 0.  Row r intends designated key (r // 4 + 3 (r % 4)) mod n, the same for every head (the mask is
    head independent; the key directions are permuted per head).  Rows by r % 4: 0 all open; 1 only the intended key
    open; 2 at most 6 keys around the intended one open, all inside its 32-key tile (so inside one split), with every
    score 128 nats down (a combine that rescales the empty splits against m = 0 underflows in fp32) and the intended
    key 8 nats above the other <= 5 (enough for 0.99, and it keeps the TMA kernel's q-rounding term small); 3 a random half
    of the keys blocked.  Row 2 is blocked everywhere with row_open set (it must attend everything, no offset).
    With B > 1 the first 64 key rows of image b+1 (the rows past Lk a 32- or 64-key tile load reads) lure the r % 4
    == 0 rows of image b by 24 nats.  shared_kv: one K / V for all images (a stride-0 batch)."""
    C = nh * hd
    scale = hd ** -0.5
    des = {0, 31, 32, 63, 64, Lk - 1}
    for x in boundaries:
        des |= {x - 1, x}
    des = sorted({p for p in des if 0 <= p < Lk} | set(torch.randint(0, Lk, (2,), generator=gen).tolist()))[: hd - 4]
    ni = 1 if shared_kv else B
    rows_per = Lq * (B if shared_kv else 1)
    r = torch.arange(rows_per)
    pick = torch.tensor(des)[(r // 4 + 3 * (r % 4)) % len(des)]
    choice = pick.repeat(ni * nh, 1)
    q, k, v, _ = keyed(ni * nh, rows_per, Lk, hd, scale, choice, reserved=4, gen=gen)
    D = hd - 4
    blocked = torch.zeros(ni, rows_per, Lk, dtype=torch.bool)
    row_open = torch.zeros(ni, rows_per, dtype=torch.uint8)
    for i in range(ni):
        rnd = torch.rand(rows_per, Lk, generator=gen) < 0.5
        for j in range(rows_per):
            c, kind = int(pick[j]), j % 4
            if kind == 1:
                blocked[i, j] = True
            elif kind == 2:
                blocked[i, j] = True
                t0 = (c // 32) * 32
                blocked[i, j, max(t0, c - 3):min(Lk, t0 + 32, c + 3)] = False
            elif kind == 3:
                blocked[i, j] = rnd[j]
            blocked[i, j, c] = False
        if rows_per > 2:
            blocked[i, 2] = True
            row_open[i, 2] = 1
    for z in range(ni * nh):
        k[z, :, hd - 1] = 8.0
        q[z, 2::4, hd - 1] = -128.0 / (8.0 * scale)
        q[z, 2::4, :D] *= 0.5
        if rows_per > 2:
            q[z, 2, hd - 1] = 0.0
            q[z, 2, :D] *= 2.0
    if not shared_kv:
        for b in range(B - 1):
            dim = D + (b % 2)                 # alternate: image b+1's own lured rows use the other dimension
            for h in range(nh):
                k[(b + 1) * nh + h, :min(64, Lk), dim] = BETA
                q[b * nh + h, 0::4, dim] = LURE * G / (BETA * scale)
    qq = heads_in(q, ni, nh).reshape(ni, rows_per, C)
    kk = heads_in(k, ni, nh).reshape(ni, Lk, C)
    vv = heads_in(v, ni, nh).reshape(ni, Lk, C)
    bits = pack_bits(blocked)
    intended = choice
    if shared_kv:
        qq = qq.view(B, Lq, C)
        bits = bits.view(B, Lq, -1)
        row_open = row_open.view(B, Lq)
        intended = pick.view(B, 1, Lq).expand(B, nh, Lq).reshape(B * nh, Lq)
    return qq, kk, vv, bits, row_open, intended


# ---------------------------------------------------------------------------------------------------------------
# paged decode: one query per sequence, K / V pages [num_pages, nh, page, hd] through a block table
# ---------------------------------------------------------------------------------------------------------------
def decode_problem(qkv, kc, vc, bt, seq_lens, extra=0, dev=None):
    """extra=1: the mutant that reads slot seq_len too."""
    dev = dev or device()
    B, _, _, nh, hd = qkv.shape
    ps = kc.shape[2]
    n = int(seq_lens.max()) + extra
    npg = -(-n // ps)
    btl = bt[:, :npg].long().to(dev)
    k = kc.to(dev, torch.float64)[btl].permute(0, 2, 1, 3, 4).reshape(B, nh, npg * ps, hd)[:, :, :n]
    v = vc.to(dev, torch.float64)[btl].permute(0, 2, 1, 3, 4).reshape(B, nh, npg * ps, hd)[:, :, :n]
    q = qkv.to(dev, torch.float64)[:, 0, 0].reshape(B * nh, 1, hd)
    allowed = torch.arange(n, device=dev)[None, :] < (seq_lens.to(dev).long() + extra)[:, None]
    allowed = allowed[:, None, None, :].expand(B, nh, 1, n).reshape(B * nh, 1, n)
    return dict(q=q, k=k.reshape(B * nh, n, hd), v=v.reshape(B * nh, n, hd), allowed=allowed, scale=hd ** -0.5)


def decode_probe(seq_lens, nh, hd, ps, gen):
    """(qkv [B,1,3,nh,hd], kc, vc, block_table, intended [B*nh, 1]): pages in random order; head h of sequence b
    intends one of key 0, the page boundaries, 127 / 128 (the 128 lanes of the kernel own keys k mod 128) and
    seq_len-1; slot seq_len (in the last page) holds a lure with V = +-4."""
    B = len(seq_lens)
    scale = hd ** -0.5
    n = max(seq_lens) + 1
    max_pages = -(-n // ps) + 1
    perm = torch.randperm(B * max_pages, generator=gen)
    bt = perm.view(B, max_pages).to(torch.int32)
    kc = torch.zeros(B * max_pages, nh, ps, hd, dtype=torch.float64)
    vc = torch.zeros_like(kc)
    q = torch.zeros(B, nh, hd, dtype=torch.float64)
    intended = torch.zeros(B * nh, 1, dtype=torch.long)
    for b, L in enumerate(seq_lens):
        cand = sorted({p for p in (0, ps - 1, ps, 2 * ps - 1, 2 * ps, 31, 32, 127, 128, 129, L - 1) if p < L})
        choice = torch.tensor([[cand[(h * 5 + b) % len(cand)]] for h in range(nh)])
        lure = torch.full((nh, 1), L)
        qz, kz, vz, _ = keyed(nh, 1, L + 1, hd, scale, choice, lure, gen=gen)
        vz[:, L] *= 4.0
        q[b] = qz[:, 0]
        intended[b * nh:(b + 1) * nh] = choice
        pos = torch.arange(L + 1)
        pg, sl = bt[b, pos // ps].long(), pos % ps
        kc[pg, :, sl] = kz.transpose(0, 1)
        vc[pg, :, sl] = vz.transpose(0, 1)
    qkv = torch.zeros(B, 1, 3, nh, hd, dtype=torch.float64)
    qkv[:, 0, 0] = q
    return qkv, kc, vc, bt, torch.tensor(seq_lens, dtype=torch.int32), intended
