"""Exact and float64 probes for the kernels that sample and resample maps: MSDeformAttn (csrc/msda.cu: msda_vec_kernel,
msda_scalar_kernel, msda_encoder_fused_kernel), bilinear_tokens (csrc/mask_head.cu), region_pool (csrc/region.cu) and
the fused task heads (csrc/postproc.cu: postproc_fused_kernel plain and COMPOSED; csrc/postproc_fast.cu).

No kernel is called here.  tests/test_resample_probes_cpu.py shows that each probe rejects named mutants: by at least
one wrong bit for the exact probes, by >= 10x its bound for the float64 probes.  tests/test_resample_probes_gpu.py runs
the kernels on the same probes.  The references are float64 restatements of each operation from its definition,
written apart from tests/emu.py and oracle/ (the CPU tests install emu as the kernels, so a shared bug would never
show).  Index arithmetic that ATen defines in float32 (the source index of upsample_bilinear2d) is kept in float32.

Exact probes.  Every operation is a bilinear blend.  Values are small integers (|v| <= 127, exact in bf16) coded from
their coordinates, ((a level + b y + c x + d head + e channel + f image) mod 251) - 125, so that reading a neighbouring
pixel, level, head, channel or image changes the value.  Positions are dyadic, so every bilinear weight, every product
and every fp32 partial sum is exact in any order, and the kernel's fp32 result equals the float64 reference; one
round-to-nearest-even to storage follows in both, so outputs compare with torch.equal.
  MSDA vec / scalar   x = loc_x W - 0.5 on the 1/8 grid (power-of-two levels, loc = (8x + 4) / 8W) or the 1/32 grid
                      (odd levels, loc = j / 32), including x = -1 and x = W (excluded), -1 + 1/8, -0.5, 0, W - 1,
                      W - 1 + 1/8 and W - 1/8, in both axes.  Attention weights are multiples of 1/4 in [0, 1].  The
                      corner weights are then multiples of 2^-12 (2^-10 for c = hy hx aw on the 1/8 grid), products with
                      |v| <= 125 and sums over L P <= 16 samples stay below 2^11 in magnitude: at most 23 significant
                      bits, exact in fp32.  16-bit `loc` is rounded to storage first and the reference reads the
                      stored value: rounding an 11-bit dyadic to 8 or 11 bits gives a coarser dyadic, so the grid bound
                      still holds (every edge case survives for W <= 16).
  MSDA fused          power-of-two levels; x = (qx + 0.5) W_l / W_q + ox - 0.5 is exact when ox is a multiple of 1/8
                      (bf16 `ow`: ox rounded to bf16 first, still on the 1/8 grid).  The softmax is exact: one-hot (one
                      logit 0, the others -200; expf(-200) = 0 in fp32, so the kernel's weight is exactly 1; the
                      float64 reference differs from 1 by < 16 e^-200, far below any storage unit) or k-hot with k a
                      power of two (weights exactly 1/k).
  bilinear_tokens     ratios x2, /2, /4, /8 (odd sizes where the ratio is still a power of two): the source index is
                      exact in fp32 and the weights are multiples of 1/4 per axis; with accumulate the old value (a
                      storage value) plus the exact blend is rounded once in both.
  region_pool         h - 1 and w - 1 powers of two, points (k / 8) / (h - 1): sample positions on the 1/8 grid,
                      P = 256 so that the mean's 1/P is exact; sums stay below 2^15 with granularity 2^-6.
  task heads          integer logits in [-127, 127], up-sampling x1, x2, x4 or x8 (weights multiples of 1/(2r) per
                      axis, products multiples of 1/256, exact in bf16 as the fast kernel's A operand, e.g. 225/256):
                      x is exact in both kernels, so count(x > 0), count(x >= 0), in_mask, area, intersection and the
                      instance masks compare exactly.  Exact zeros come from cancelling taps: source columns (m, -K m)
                      with K = 2r - 1 give x = (1 - 1/2r) m - (1/2r) K m = 0 at the output column with l = 1/2r,
                      planted only in the upper source rows so that some warps see a zero and others do not.  The
                      composed crop path is exact when Hp / H4 and oh / H are powers of two.
  panoptic ids        v_q = wq_q sigma(x_q) + negq_q.  Both kernels' sigmoids (__expf + __fdividef; ex2.approx +
                      rcp.approx) are within 2^-20 of sigma for |x| <= 127 (2 ulp each, and the rounding of x log2(e)
                      moves the exponent by <= |x| 2^-23, scaled by sigma (1 - sigma) |x| <= 0.23), fmaf adds 2^-24, so
                      a winner that leads by more than IDS_MARGIN = 2^-18 > 2 (2^-20 + 2^-24) is decided.  Kept queries
                      have distinct wq = (205 + 5 (37 q mod 113)) / 1024; tie pairs (identical maps, equal wq) sit
                      across the even / odd halves, the quad lanes (q, q + 2) and the n-tiles (q, q + 8): the lower
                      index must win.  Non-kept queries (wq = 0, negq = -1) include saturated logits 127.

Float64 probes.
  sem_seg             sem[c, p] = sum_q P[c, q] sigma(x_q(p)).  The kernels round sigma to fp16 (relative 2^-11, or
                      absolute 2^-25 below 2^-14), after the approximate sigmoid (2^-20, see above), and accumulate
                      exact fp16 x fp16 products in fp32 over 112 queries (<= 112 2^-24 relative):
                          |sem - ref| <= (2^-11 + 2^-15) sum_q P_q sigma_q + 2^-19 sum_q P_q + 2^-24 |ref|.
  sum(sigma [x > 0])  fast kernel, over n pixels with x > 0 (sigma in [1/2, 1]): ex2.approx (2^-22 relative on
                      e <= 1) and rcp.approx (2^-24 on [1/2, 1]) with the rounding of x log2(e) (<= 2^-25 after the
                      factor e / (1 + e)^2) give 2^-21.4, the 2^-22 fixed point 2^-23: n 2^-21 together; the per-CTA
                      total converted to fp32 (2^-24 relative), then the fp32 sum of `rows` per-CTA partials:
                      n 2^-21 + (rows + 1) 2^-24 ref.  Generic kernel: fp16 sigma (2^-11 sigma + 2^-20 per pixel),
                      fp32 chains of 128 pixels per tile, then `rows` tiles: 2^-11 ref + n 2^-20 + (129 + rows) 2^-24
                      ref.  The exact count(x > 0) is what catches a lost pixel on the generic kernel; the fast bound
                      is below a 16-pixel tile row of sigma >= 1/2 by 10x at 256^2.
  bilinear_tokens     non-power-of-two ratios: the kernel may contract scale (d + 0.5) - 0.5 into one fma, so its
                      source index can differ from ATen's float32 one by 1 ulp (<= 2^-23 max(Hi, Wi)); the blend is
                      Lipschitz in the index with constant max |adjacent difference| <= 250; three levels of fp32
                      products and sums add 3 2^-24 max |corner|:  u |ref| + 2^-24 (|old| + 3 max|v|) + 250 2 ulp.
  MSDA fused          non-power-of-two levels: rx = (qx + 0.5) / W_q, ox / W_l, their sum, the product with W_l and
                      the -0.5 are five fp32 roundings on magnitudes <= W_l + |ox| + 1: |dx| <= 2^-21 (W_l + |ox| + 1)
                      (likewise y).  Bilinear with zero padding is Lipschitz in x with constant max |adjacent
                      difference| <= 250 (the step to the zero padding included), so a sample moves by <= aw 250
                      (|dx| + |dy|); the fp32 accumulation of 4 L P products adds 4 L P 2^-24 125, the output rounding
                      u |ref|.
  composed crop       up-sample x 4 (exact), crop, resize to a non-power-of-two size (the down / up / portrait /
                      coco-1024 geometries): x is within bx of the reference (crop_x_bound: one ulp of the second
                      stage's source index times the cropped map's slope, plus the fp32 4 x 4 blend).  Counts lie
                      between count(x_ref > bx) and count(x_ref >= -bx); masks and in_mask are exact where
                      |x_ref| > bx; ids are decided beyond 2 (bx / 4 + 2^-20 + 2^-24); sem_seg and sum(sigma [x > 0])
                      get bx / 4 per term (sigma is 1/4-Lipschitz) and 1/2 + bx / 4 per pixel that may flip.
For a threshold near 0 on a float64 path, the bound decides which pixels may flip; every other pixel must match.
"""
import math

import numpy as np
import torch

F64 = torch.float64
UNIT = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 2.0 ** -24}
U32 = 2.0 ** -24
IDS_MARGIN = 2.0 ** -18
MSDA_TW = 8   # the fused / patch kernels' tile width (queries); tile height 256 / G / 8
PP_TH, PP_TW = 8, 16


def stored(x, dtype):
    """Storage rounding, back to float64."""
    return x.to(dtype).to(F64)


def same(out, ref):
    """Bit-for-bit equality of a kernel output (any dtype) with a float64 reference already rounded to storage."""
    return torch.equal(out.to(F64).cpu(), ref.to(F64).cpu())


def err_over_bound(out, ref, bound):
    return ((out.to(F64) - ref).abs() / bound).max().item()


def level_starts(shapes):
    st, s = [], 0
    for h, w in shapes:
        st.append(s)
        s += h * w
    return st


def code(*terms):
    """((sum of coefficient * index) mod 251) - 125 as float64: |v| <= 125."""
    acc = 0
    for c, t in terms:
        acc = acc + c * t
    return (acc % 251 - 125).to(F64)


def _ar(n, device):
    return torch.arange(n, dtype=torch.int64, device=device)


# ---------------------------------------------------------------------------------------------------------------
# MSDeformAttn
# ---------------------------------------------------------------------------------------------------------------
# `>= -1` / `<= W` for `> -1` / `< W` are equivalent mutants: at x = -1 (x = W) the one corner inside the map has
# bilinear weight 0, so no finite input tells them apart; the CPU tests assert that they equal the reference.
MSDA_EQUIVALENT = ("ge_minus1", "le_W")
MSDA_MUTANTS = ("far_corner", "no_half", "swap_xy", "next_level_start", "head_shift",
                "batch_shift", "drop_last_point", "drop_last_level")
FUSED_MUTANTS = ("softmax_per_level", "ref_no_half", "ragged_wrap")


def msda_value(B, shapes, M, D, device="cpu"):
    """[B, S, M, D] coded values (reference layout)."""
    parts = []
    for l, (h, w) in enumerate(shapes):
        y = _ar(h, device).view(1, h, 1, 1, 1)
        x = _ar(w, device).view(1, 1, w, 1, 1)
        m = _ar(M, device).view(1, 1, 1, M, 1)
        c = _ar(D, device).view(1, 1, 1, 1, D)
        b = _ar(B, device).view(B, 1, 1, 1, 1)
        parts.append(code((37, l), (11, y), (3, x), (53, m), (7, c), (89, b)).reshape(B, h * w, M, D))
    return torch.cat(parts, 1)


def edge_positions(n):
    """The predicates' edge cases for a level extent n: -1 and n are excluded, the rest are inside."""
    return [-1.0, -1.0 + 2 ** -3, -0.5, 0.0, n - 1.0, n - 1.0 + 2 ** -3, n - 2 ** -3, float(n)]


def msda_probe(B, shapes, M, Lq, P, gen, loc_dtype=torch.float32, device="cpu"):
    """(loc [B, Lq, M, L, P, 2], aw [B, Lq, M, L, P]) stored in loc_dtype, as float64.  Power-of-two levels: x, y on the
    1/8 grid, two thirds of the samples on an edge case of edge_positions (x and y cycled with co-prime strides), the rest
    uniform over [-1.25, n + 0.25]; other levels: loc = j / 32.  Weights are multiples of 1/4."""
    L = len(shapes)
    loc = torch.empty(B, Lq, M, L, P, 2, dtype=F64)
    n = B * Lq * M * P
    idx = torch.arange(n, dtype=torch.int64).view(B, Lq, M, P)
    for l, (h, w) in enumerate(shapes):
        for a, ext, stride in ((0, w, 1), (1, h, 3)):
            if ext & (ext - 1) == 0:
                edges = torch.tensor(edge_positions(ext), dtype=F64)
                pick = edges[(idx * stride + l) % len(edges)]
                rnd = torch.randint(-10, 8 * ext + 3, (B, Lq, M, P), generator=gen).to(F64) / 8
                pos = torch.where((idx + l) % 3 != 0, pick, rnd)
                loc[..., l, :, a] = (pos + 0.5) / ext
            else:
                loc[..., l, :, a] = torch.randint(-4, 37, (B, Lq, M, P), generator=gen).to(F64) / 32
    aw = torch.randint(0, 5, (B, Lq, M, L, P), generator=gen).to(F64) / 4
    return stored(loc, loc_dtype).to(device), stored(aw, loc_dtype).to(device)


def msda_ref(value, shapes, loc, aw, mutant=None):
    """value [B, S, M, D], loc [B, Lq, M, L, P, 2] (x, y) in [0, 1] units, aw [B, Lq, M, L, P] -> [B, Lq, M * D]:
    sum over levels and points of aw * bilinear(value_l, loc_x W - 0.5, loc_y H - 0.5), zero outside the map."""
    B, S, M, D = value.shape
    _, Lq, _, L, P, _ = loc.shape
    dev = value.device
    starts = level_starts(shapes)
    bi = _ar(B, dev).view(B, 1, 1, 1)
    mi = _ar(M, dev).view(1, 1, M, 1)
    if mutant == "batch_shift":
        bi = (bi + 1) % B
    if mutant == "head_shift":
        mi = (mi + 1) % M
    out = torch.zeros(B, Lq, M, D, dtype=F64, device=dev)
    pts = P - 1 if mutant == "drop_last_point" else P
    for l in range(L - 1 if mutant == "drop_last_level" else L):
        H, W = shapes[l]
        st = starts[(l + 1) % L] if mutant == "next_level_start" else starts[l]
        lx, ly = loc[..., l, :pts, 0], loc[..., l, :pts, 1]
        if mutant == "swap_xy":
            lx, ly = ly, lx
        half = 0.0 if mutant == "no_half" else 0.5
        x, y = lx * W - half, ly * H - half
        if mutant == "ge_minus1":
            inside = (x >= -1) & (y >= -1) & (x < W) & (y < H)
        elif mutant == "le_W":
            inside = (x > -1) & (y > -1) & (x <= W) & (y <= H)
        else:
            inside = (x > -1) & (y > -1) & (x < W) & (y < H)
        x0, y0 = torch.floor(x), torch.floor(y)
        fx, fy = x - x0, y - y0
        a = aw[..., l, :pts]
        for dy in (0, 1):
            for dx in (0, 1):
                yy, xx = y0 + dy, x0 + dx
                xok = (xx < W - 1) if (mutant == "far_corner" and dx == 1) else (xx <= W - 1)
                ok = inside & (yy >= 0) & (yy <= H - 1) & (xx >= 0) & xok
                wgt = torch.where(ok, (fy if dy else 1 - fy) * (fx if dx else 1 - fx) * a, torch.zeros_like(a))
                pix = (st + yy.clamp(0, H - 1).long() * W + xx.clamp(0, W - 1).long()) % S
                out += (wgt.unsqueeze(-1) * value[bi, pix, mi]).sum(-2)
    return out.reshape(B, Lq, M * D)


def query_grid(shapes, device="cpu"):
    """(level, qy, qx) of every query of the pixel grid (Lq == S)."""
    ls, ys, xs = [], [], []
    for l, (h, w) in enumerate(shapes):
        yy, xx = torch.meshgrid(_ar(h, device), _ar(w, device), indexing="ij")
        ls.append(torch.full((h * w,), l, dtype=torch.int64, device=device))
        ys.append(yy.reshape(-1))
        xs.append(xx.reshape(-1))
    return torch.cat(ls), torch.cat(ys), torch.cat(xs)


def fused_probe(B, shapes, M, gen, hot=1, ow_dtype=torch.float32, P=4, device="cpu"):
    """ow [B, S, M L P 3] (offsets | logits) as float64 stored in ow_dtype.  Power-of-two levels: each offset puts the
    sample on an edge case of edge_positions or on a 1/8-grid point; other levels: offsets uniform multiples of 1/8.
    Logits: `hot` equal logits 0 (hot = 1, 2, 4, 16), the rest -200."""
    L = len(shapes)
    LP = L * P
    S = sum(h * w for h, w in shapes)
    ql, qy, qx = query_grid(shapes)
    Wq = torch.tensor([w for _, w in shapes], dtype=F64)[ql]
    Hq = torch.tensor([h for h, _ in shapes], dtype=F64)[ql]
    off = torch.empty(B, S, M, L, P, 2, dtype=F64)
    idx = torch.arange(B * S * M * P, dtype=torch.int64).view(B, S, M, P)
    for l, (h, w) in enumerate(shapes):
        for a, ext, qc, qext, stride in ((0, w, qx, Wq, 1), (1, h, qy, Hq, 3)):
            base = (qc.to(F64) + 0.5) * ext / qext - 0.5              # where offset 0 samples, level-l pixels
            if ext & (ext - 1) == 0 and all((e & (e - 1)) == 0 for s in shapes for e in s):
                edges = torch.tensor(edge_positions(ext), dtype=F64)
                tgt = edges[(idx * stride + l) % len(edges)]
                rnd = torch.randint(-10, 8 * ext + 3, (B, S, M, P), generator=gen).to(F64) / 8
                tgt = torch.where((idx + l) % 3 != 0, tgt, rnd)
                off[..., l, :, a] = tgt - base.view(1, S, 1, 1)
            else:
                off[..., l, :, a] = torch.randint(-24, 25, (B, S, M, P), generator=gen).to(F64) / 8
    lg = torch.full((B, S, M, LP), -200.0, dtype=F64)
    start = torch.randint(0, LP, (B, S, M, 1), generator=gen)
    for k in range(hot):
        lg.scatter_(-1, (start + k * (LP // hot)) % LP, 0.0)
    ow = torch.cat([off.reshape(B, S, M * LP * 2), lg.reshape(B, S, M * LP)], -1)
    return stored(ow, ow_dtype).to(device)


def fused_locations(ow, shapes, M, P=4, mutant=None):
    """The fused variant's definition: aw = softmax over the L P logits of a head, ref = ((qx + 0.5) / W_q,
    (qy + 0.5) / H_q), loc = ref + off / (W_l, H_l)."""
    B, S, _ = ow.shape
    L = len(shapes)
    LP = L * P
    dev = ow.device
    off = ow[..., :M * LP * 2].reshape(B, S, M, L, P, 2)
    lg = ow[..., M * LP * 2:].reshape(B, S, M, L, P)
    if mutant == "softmax_per_level":
        aw = torch.softmax(lg, -1)
    else:
        aw = torch.softmax(lg.reshape(B, S, M, LP), -1).reshape(B, S, M, L, P)
    ql, qy, qx = query_grid(shapes, dev)
    Wq = torch.tensor([w for _, w in shapes], dtype=F64, device=dev)[ql]
    Hq = torch.tensor([h for h, _ in shapes], dtype=F64, device=dev)[ql]
    qxf, qyf = qx.to(F64), qy.to(F64)
    if mutant == "ragged_wrap":
        # a query of a ragged tile (qx >= W) that is not masked off writes the pixel (qy + 1, qx - W) with its own
        # reference point: pixel (y, x), y >= 1, x < pad, gets the reference point of (y - 1, x + W)
        pad = ((Wq.long() + MSDA_TW - 1) // MSDA_TW) * MSDA_TW - Wq.long()
        hit = (qy >= 1) & (qx < pad)
        qxf = torch.where(hit, qxf + Wq, qxf)
        qyf = torch.where(hit, qyf - 1, qyf)
    half = 0.0 if mutant == "ref_no_half" else 0.5
    rx, ry = (qxf + half) / Wq, (qyf + half) / Hq
    Wl = torch.tensor([w for _, w in shapes], dtype=F64, device=dev).view(1, 1, 1, L, 1)
    Hl = torch.tensor([h for h, _ in shapes], dtype=F64, device=dev).view(1, 1, 1, L, 1)
    lx = rx.view(1, S, 1, 1, 1) + off[..., 0] / Wl
    ly = ry.view(1, S, 1, 1, 1) + off[..., 1] / Hl
    return torch.stack([lx, ly], -1), aw


def msda_fused_ref(value_hm, ow, shapes, P=4, mutant=None):
    """value_hm [B, M, S, D] head-major, ow [B, S, M L P 3] -> [B, S, M D]."""
    M = value_hm.shape[1]
    loc, aw = fused_locations(ow, shapes, M, P, mutant)
    return msda_ref(value_hm.permute(0, 2, 1, 3), shapes, loc, aw)


def fused_bound(value_hm, ow, shapes, ref, dtype, P=4):
    """Per-element bound of the fused kernel on any levels (module docstring)."""
    B, M, S, D = value_hm.shape
    L = len(shapes)
    LP = L * P
    vmax = value_hm.abs().max().item()
    lip = 2 * vmax
    loc, aw = fused_locations(ow, shapes, M, P)
    off = ow[..., :M * LP * 2].reshape(B, S, M, L, P, 2).abs()
    Wl = torch.tensor([w for _, w in shapes], dtype=F64, device=ow.device).view(1, 1, 1, L, 1)
    Hl = torch.tensor([h for h, _ in shapes], dtype=F64, device=ow.device).view(1, 1, 1, L, 1)
    dx = 2.0 ** -21 * (Wl + off[..., 0] + 1)
    dy = 2.0 ** -21 * (Hl + off[..., 1] + 1)
    move = (aw * lip * (dx + dy)).sum((-1, -2))                             # [B, S, M]
    b = move.unsqueeze(-1).expand(B, S, M, D).reshape(B, S, M * D)
    return UNIT[dtype] * ref.abs() + b + 4 * LP * U32 * vmax


# ---------------------------------------------------------------------------------------------------------------
# bilinear_tokens (upsample_bilinear2d, align_corners = False) and region_pool (grid_sample, align_corners = True)
# ---------------------------------------------------------------------------------------------------------------
BILINEAR_MUTANTS = ("align_corners", "no_clamp", "upper_unclamped", "accumulate_drops_old")
REGION_MUTANTS = ("align_corners", "swap_yx", "wrong_image")


def _taps(n_in, n_out, mutant=None):
    """(i0, i1, w0, w1) of every output index: ATen's source index in float32, then float64 weights."""
    f = np.float32
    d = np.arange(n_out, dtype=np.float32)
    if mutant == "align_corners":
        s = d * f((n_in - 1) / (n_out - 1) if n_out > 1 else 0.0)
    else:
        s = f(f(n_in) / f(n_out)) * (d + f(0.5)) - f(0.5)
        if mutant != "no_clamp":
            s = np.maximum(s, f(0))
    i0 = s.astype(np.int64)                    # truncation, as the kernels' (int) cast
    i1 = i0 + 1 if mutant == "upper_unclamped" else i0 + (i0 < n_in - 1)
    lam = (s - i0.astype(np.float32)).astype(np.float64)
    return torch.from_numpy(i0), torch.from_numpy(i1), torch.from_numpy(1 - lam), torch.from_numpy(lam)


def bilinear_ref(x, Hi, Wi, Ho, Wo, old=None, mutant=None):
    """x [B, Hi Wi, C] token-major float64 -> [B, Ho Wo, C]; with `old`, old + blend (accumulate).  Taps past the map
    (the upper_unclamped mutant) read the next token of the flat buffer, zero past its end."""
    B, _, C = x.shape
    dev = x.device
    yi0, yi1, wy0, wy1 = (t.to(dev) for t in _taps(Hi, Ho, mutant))
    xi0, xi1, wx0, wx1 = (t.to(dev) for t in _taps(Wi, Wo, mutant))
    flat = torch.cat([x.reshape(B * Hi * Wi, C), torch.zeros(Wi + 1, C, dtype=F64, device=dev)])
    base = (_ar(B, dev) * Hi * Wi).view(B, 1, 1)
    out = torch.zeros(B, Ho, Wo, C, dtype=F64, device=dev)
    for yi, wy in ((yi0, wy0), (yi1, wy1)):
        for xi, wx in ((xi0, wx0), (xi1, wx1)):
            idx = (base + yi.view(1, Ho, 1) * Wi + xi.view(1, 1, Wo)).clamp(max=flat.shape[0] - 1)
            out += (wy.view(1, Ho, 1, 1) * wx.view(1, 1, Wo, 1)) * flat[idx]
    out = out.reshape(B, Ho * Wo, C)
    if old is not None and mutant != "accumulate_drops_old":
        out = old + out
    return out


def bilinear_bound(x, Hi, Wi, ref, out_dtype, old=None):
    vmax = x.abs().max().item()
    lip = 2 * vmax
    ulp = 2.0 ** -23 * max(Hi, Wi)
    b = UNIT[out_dtype] * ref.abs() + U32 * 3 * vmax + lip * 2 * ulp
    if old is not None:
        b = b + U32 * old.abs()
    return b


def tokens_probe(B, Hi, Wi, C, device="cpu"):
    b = _ar(B, device).view(B, 1, 1, 1)
    y = _ar(Hi, device).view(1, Hi, 1, 1)
    x = _ar(Wi, device).view(1, 1, Wi, 1)
    c = _ar(C, device).view(1, 1, 1, C)
    return code((89, b), (11, y), (3, x), (7, c)).reshape(B, Hi * Wi, C)


def region_probe(B, h, w, C, R, P, gen, device="cpu"):
    """tokens [B, h w, C], points [R, P, 2] (y, x) with h - 1, w - 1 powers of two, region_image [R] int32 (unsorted)."""
    assert (h - 1) & (h - 2) == 0 and (w - 1) & (w - 2) == 0
    tokens = tokens_probe(B, h, w, C, device)
    iy = torch.randint(0, 8 * (h - 1) + 1, (R, P), generator=gen).to(F64) / 8
    ix = torch.randint(0, 8 * (w - 1) + 1, (R, P), generator=gen).to(F64) / 8
    iy[:, 0], ix[:, 0] = 0, 0                         # first row / column
    iy[:, 1], ix[:, 1] = h - 1, w - 1                 # last row / column
    iy[:, 2], ix[:, 2] = h - 1, 0
    iy[:, 3], ix[:, 3] = 0.5, w - 1.5
    pts = torch.stack([iy / (h - 1), ix / (w - 1)], -1)
    img = (torch.arange(R) * 7 + 3) % B
    return tokens, pts.to(device), img.to(torch.int32).to(device)


def region_ref(tokens, h, w, points, region_image, mutant=None):
    """mean over P of grid_sample(map, 2 (x, y) - 1, align_corners = True, zero padding); points are (y, x)."""
    B, N, C = tokens.shape
    R, P, _ = points.shape
    py, px = points[..., 0], points[..., 1]
    if mutant == "swap_yx":
        py, px = px, py
    if mutant == "align_corners":
        iy, ix = py * h - 0.5, px * w - 0.5
    else:
        iy, ix = py * (h - 1), px * (w - 1)
    img = region_image.long()
    if mutant == "wrong_image":
        img = (img + 1) % B
    y0, x0 = torch.floor(iy), torch.floor(ix)
    fy, fx = iy - y0, ix - x0
    out = torch.zeros(R, C, dtype=F64, device=tokens.device)
    for dy in (0, 1):
        for dx in (0, 1):
            yy, xx = y0 + dy, x0 + dx
            ok = (yy >= 0) & (yy < h) & (xx >= 0) & (xx < w)
            wgt = torch.where(ok, (fy if dy else 1 - fy) * (fx if dx else 1 - fx), torch.zeros_like(fy))
            pix = yy.clamp(0, h - 1).long() * w + xx.clamp(0, w - 1).long()
            out += (wgt.unsqueeze(-1) * tokens[img.view(R, 1), pix]).sum(1)
    return out / P


# ---------------------------------------------------------------------------------------------------------------
# task heads
# ---------------------------------------------------------------------------------------------------------------
HEADS_MUTANTS = ("gt_ge_swap", "tie_high", "last_tile_row", "last_tile_col", "tap_shift", "sem_class_shift",
                 "sem_pixel_shift", "drop_last_qtile", "drop_last_ctile", "slot_reverse")


def resize(img, Ho, Wo, mutant=None):
    """[N, Hi, Wi] float64 -> [N, Ho, Wo] by upsample_bilinear2d(align_corners = False) as two dense tap matrices.
    tap_shift: every row tap reads one source row lower (clamped)."""
    N, Hi, Wi = img.shape

    def mat(n_in, n_out, shift=0):
        i0, i1, w0, w1 = _taps(n_in, n_out)
        i0, i1 = (i0 + shift).clamp(max=n_in - 1), (i1 + shift).clamp(max=n_in - 1)
        m = torch.zeros(n_out, n_in, dtype=F64)
        r = torch.arange(n_out)
        m.index_put_((r, i0), w0, accumulate=True)
        m.index_put_((r, i1), w1, accumulate=True)
        return m.to(img.device)

    Ry = mat(Hi, Ho, 1 if mutant == "tap_shift" else 0)
    Rx = mat(Wi, Wo)
    return torch.einsum("oh,nhw,pw->nop", Ry, img, Rx)


def heads_x(logits, H, W, crop=None, mutant=None):
    if crop is None:
        return resize(logits, H, W, mutant)
    Hp, Wp, oh, ow = crop
    return resize(resize(logits, Hp, Wp, mutant)[:, :oh, :ow].contiguous(), H, W)


def wq_code(Q, kept):
    q = torch.arange(Q)
    wq = (205 + 5 * ((37 * q) % 113)).to(F64) / 1024
    return torch.where(kept, wq, torch.zeros_like(wq)), torch.where(kept, torch.zeros(Q, dtype=F64), -torch.ones(Q, dtype=F64))


TIE_PAIRS = ((10, 11), (20, 22), (30, 38), (41, 43), (64, 65), (96, 104))


def heads_probe(Q, H4, W4, ratio, ncls, K, zeros=True, device="cpu"):
    """(logits [Q, H4, W4], probsT [144, 112], wq [Q], negq [Q], slot_query [K]) as float64 / int64.  `ratio` is the
    up-sampling factor of the plain path (for exact zeros)."""
    q = torch.arange(Q).view(Q, 1, 1)
    y = torch.arange(H4).view(1, H4, 1)
    x = torch.arange(W4).view(1, 1, W4)
    logits = ((17 * q + 29 * y + 13 * x + (q * y * x) % 7) % 255 - 127).to(F64)
    logits[logits == 0] = 1.0                                      # zeros only where planted
    if zeros:   # cancelling taps (m, -K m) at source columns (8 j + 3, 8 j + 4), upper source rows only
        Kc = 2 * ratio - 1
        top = max(1, H4 // 2)
        for qq in range(0, Q, 3):
            m = 1 + qq % 8
            for c in range(3, W4 - 1, 8):
                if ratio == 1:
                    logits[qq, :top, c] = 0.0
                else:
                    logits[qq, :top, c] = float(m)
                    logits[qq, :top, c + 1] = float(-Kc * m)
    kept = (torch.arange(Q) % 3 != 2)
    logits[~kept & (torch.arange(Q) % 6 == 5)] = 127.0            # not kept, saturated
    wq, negq = wq_code(Q, kept)
    for a, b in TIE_PAIRS:
        if b < Q:
            logits[b] = logits[a]
            kept[a] = kept[b] = True
            wq[b] = wq[a] = (205 + 5 * ((37 * a) % 113)) / 1024
            negq[a] = negq[b] = 0.0
    c = torch.arange(144).view(144, 1)
    qq = torch.arange(112).view(1, 112)
    probsT = (((7 * c + 3 * qq) % 17 + 1).to(F64) / 64) * ((c < ncls) & (qq < Q))
    k = torch.arange(K)
    slots = (k * 37) % Q
    slots[(k % 7) == 3] = -1                                       # holes
    if K > 4:
        slots[4] = slots[1]                                        # a duplicate
    return logits.to(device), probsT.to(device), wq.to(device), negq.to(device), slots.to(device)


def heads_ref(x, probsT, wq, negq, slots, ncls, mutant=None, rows=1):
    """Task-head outputs from the up-sampled logits x [Q, H, W] (float64, from heads_x):
    stats [Q, 5] = count(x > 0), sum(sigma [x > 0]), count(x >= 0), area, intersection; sem [ncls, H, W]; ids, in_mask;
    inst [K, H, W] ([x > 0] per slot, hole slots left as NaN).  Mutants model a kernel with one named mistake; the
    unwritten-output ones leave NaN / -1 / 255 (the poison) in place."""
    Q, H, W = x.shape
    live = torch.ones(Q, dtype=torch.bool, device=x.device)
    if mutant == "drop_last_qtile":
        live[((Q - 1) // 8) * 8:] = False
    sig = torch.sigmoid(x)
    if mutant == "gt_ge_swap":
        pos, ge = x >= 0, x > 0
    else:
        pos, ge = x > 0, x >= 0
    pos, ge = pos & live.view(Q, 1, 1), ge & live.view(Q, 1, 1)
    out = {}
    stats = torch.zeros(Q, 5, dtype=F64, device=x.device)
    stats[:, 0] = pos.flatten(1).sum(1)
    stats[:, 1] = (sig * pos).flatten(1).sum(1)
    stats[:, 2] = ge.flatten(1).sum(1)
    if probsT is not None:
        P = probsT[:, :Q]
        if mutant == "sem_class_shift":
            P = torch.roll(P, -1, 0)
        s = sig * live.view(Q, 1, 1)
        if mutant == "sem_pixel_shift":
            s = torch.roll(s, -1, 2)
        sem = torch.einsum("cq,qhw->chw", P[:ncls], s)
        if mutant == "drop_last_ctile":
            sem[((ncls - 1) // 8) * 8:] = 0.0
        out["sem"] = sem
        out["sem_bound"] = (2.0 ** -11 + 2.0 ** -15) * sem.abs() + 2.0 ** -19 * P[:ncls].sum(1).view(-1, 1, 1) + U32 * sem.abs()
    if wq is not None:
        v = wq.view(Q, 1, 1) * sig + negq.view(Q, 1, 1)
        v = torch.where(live.view(Q, 1, 1), v, torch.full_like(v, -2.0))
        if mutant == "tie_high":
            ids = Q - 1 - torch.flip(v, (0,)).argmax(0)
        else:
            ids = v.argmax(0)                                    # first maximum
        xm = x.gather(0, ids.unsqueeze(0))[0]
        inm = (xm > 0) if mutant == "gt_ge_swap" else (xm >= 0)
        stats[:, 3] = torch.bincount(ids.flatten(), minlength=Q).to(F64)
        stats[:, 4] = torch.bincount(ids.flatten(), weights=inm.flatten().to(F64), minlength=Q)
        out["ids"], out["in_mask"] = ids.to(torch.int64), inm.to(torch.uint8)
        best = v.max(0).values
        cand = v >= best - IDS_MARGIN
        out["ids_clear"] = (cand.sum(0) == 1) | ((v == best) | ~cand).all(0)
        out["ids_cand"] = cand
    if slots is not None:
        sl = torch.flip(slots, (0,)) if mutant == "slot_reverse" else slots
        inst = torch.full((slots.shape[0], H, W), float("nan"), dtype=F64, device=x.device)
        has = sl >= 0
        inst[has] = (x[sl[has]] > 0).to(F64) * live[sl[has]].view(-1, 1, 1)
        out["inst"] = inst
    if mutant in ("last_tile_row", "last_tile_col"):
        sel = (slice(None), slice(((H - 1) // PP_TH) * PP_TH, None)) if mutant == "last_tile_row" else \
              (slice(None), slice(None), slice(((W - 1) // PP_TW) * PP_TW, None))
        for k, poison in (("ids", -1), ("in_mask", 255), ("inst", float("nan")), ("sem", float("nan"))):
            if k in out:
                t = out[k].unsqueeze(0) if out[k].dim() == 2 else out[k]
                t[sel] = poison
    n, ref = stats[:, 0], stats[:, 1]
    out["sig_bound_fast"] = n * 2.0 ** -21 + (rows + 1) * U32 * ref
    out["sig_bound_generic"] = 2.0 ** -11 * ref + n * 2.0 ** -20 + (129 + rows) * U32 * ref
    out["stats"], out["x"], out["wq"], out["negq"] = stats, x, wq, negq
    return out


def probe_properties(x, ref, Q):
    """What makes a task-head probe sharp: exact zeros in some output rows (warps of the fast kernel) and not in others,
    and a tie pair that wins at least one pixel (so the lower-index tie-break is observable)."""
    rows_with_zero = (x == 0).any(0).any(1)
    tie_wins = any(bool((ref["ids"] == a).any()) for a, b in TIE_PAIRS if b < Q)
    return dict(zero_rows=bool(rows_with_zero.any()), zero_free_rows=not bool(rows_with_zero.all()), tie_wins=tie_wins,
                decided=bool(ref["ids_clear"].all()))


def crop_x_bound(logits, crop, H, W):
    """Bound on |x_kernel - x_ref| on the composed crop path, whose first stage (x Hp / H4, a power of two) is exact.
    The second stage's source index can differ from ATen's float32 one by 1 ulp (fma contraction), <= 2^-23 oh (rows)
    and 2^-23 ow (columns); the cropped map is Lipschitz with constant (max adjacent logit difference) / (Hp / H4) per
    row (likewise columns); the kernel's 4 x 4 fp32 blend (4 weight products, two chains of 4 fmas, on magnitudes
    <= max |logit|) adds at most 16 2^-24 max |logit|."""
    Hp, Wp, oh, ow = crop
    Q, H4, W4 = logits.shape
    dy = (logits[:, 1:] - logits[:, :-1]).abs().max().item() if H4 > 1 else 0.0
    dx = (logits[:, :, 1:] - logits[:, :, :-1]).abs().max().item() if W4 > 1 else 0.0
    return dy / (Hp / H4) * 2.0 ** -23 * oh + dx / (Wp / W4) * 2.0 ** -23 * ow + 16 * U32 * logits.abs().max().item()


def crop_violations(got, ref, probsT, ncls, slots, bx, scale=1.0):
    """Which outputs of a composed-crop run break the float64 bound (every bound times `scale`).  Pixels with
    |x_ref| <= b = scale bx may fall on either side of 0; everything else is exact.  A panoptic winner is decided when
    it leads by more than 2 (b / 4 + 2^-20 + 2^-24) (sigma is 1/4-Lipschitz); otherwise any query within that margin
    may win, and in_mask, area and intersection must follow the chosen query."""
    bad = []
    x = ref["x"]
    Q = x.shape[0]
    b = bx * scale
    st, rs = got["stats"].to(F64), ref["stats"]
    flip = x.abs() <= b
    for col in (0, 2):
        lo, hi = (x > b).flatten(1).sum(1), (x >= -b).flatten(1).sum(1)
        if not bool(((st[:, col] >= lo) & (st[:, col] <= hi)).all()):
            bad.append("count %d" % col)
    has = slots >= 0
    inst = got["inst"][has].to(F64)
    xs = x[slots[has]]
    if not torch.equal(inst[~flip[slots[has]]], (xs > 0).to(F64)[~flip[slots[has]]]):
        bad.append("inst")
    ids = got["ids"].long()
    sig = torch.sigmoid(x)
    wq, negq = ref["wq"], ref["negq"]
    v = wq.view(Q, 1, 1) * sig + negq.view(Q, 1, 1)
    best = v.max(0).values
    cand = v >= best - 2 * (b / 4 + 2.0 ** -20 + 2.0 ** -24)
    clear = (cand.sum(0) == 1) | ((v == best) | ~cand).all(0)
    ok_ids = bool((ids >= 0).all() and (ids < Q).all())
    if not ok_ids or not torch.equal(ids[clear], v.argmax(0)[clear]) or \
            not bool(cand.gather(0, ids.clamp(0, Q - 1).unsqueeze(0)).all()):
        bad.append("ids")
    else:
        xa = x.gather(0, ids.unsqueeze(0))[0]
        sure = xa.abs() > b
        if not torch.equal(got["in_mask"][sure].long(), (xa[sure] >= 0).long()):
            bad.append("in_mask")
        inm = got["in_mask"].to(F64)
        if not (torch.equal(st[:, 3], torch.bincount(ids.flatten(), minlength=Q).to(F64)) and
                torch.equal(st[:, 4], torch.bincount(ids.flatten(), weights=inm.flatten(), minlength=Q))):
            bad.append("area")
    P = probsT[:ncls, :Q]
    sem_b = scale * (ref["sem_bound"] + (P * (b / 4)).sum(1).view(-1, 1, 1))
    d = (got["sem"].to(F64) - ref["sem"]).abs()
    if not bool((d <= sem_b).all()):
        bad.append("sem")
    nflip = flip.flatten(1).sum(1)
    npos = (x > -b).flatten(1).sum(1)
    sig_b = scale * ref["sig_bound_generic"] + npos * b / 4 + nflip * (0.5 + b / 4)
    if not bool(((st[:, 1] - rs[:, 1]).abs() <= sig_b).all()):
        bad.append("sum(sigma)")
    return bad


def constant_heads(Q, H4, W4, consts, device="cpu"):
    """Logit maps constant per query: the up-sampled map is the constant itself, so every output is closed form."""
    return torch.tensor(consts, dtype=F64).view(Q, 1, 1).expand(Q, H4, W4).contiguous().to(device)


# ---------------------------------------------------------------------------------------------------------------
# the fast kernel's fixed-point sum of sigma [x > 0]
# ---------------------------------------------------------------------------------------------------------------
def fixed_point_payload(s):
    """Bits of (s + 2.0f) minus 0x40000000 for s in [0, 1]: round(s 2^22)."""
    f = np.float32(np.float32(s) + np.float32(2.0))
    return int(np.array([f], dtype=np.float32).view(np.uint32)[0]) - 0x40000000


def fixed_point_total(payloads_per_tile, carry=lambda it: (it << 31) & 0xFFFFFFFF):
    """CPU emulation of one accumulator slot: per tile one wrapping 32-bit add of two fixed-point values, each carrying
    0x40000000 of exponent bits, then the carry of `it` tiles removed.  payloads_per_tile: [(p0, p1)] per tile."""
    acc = 0
    for p0, p1 in payloads_per_tile:
        acc = (acc + (0x40000000 + p0) + (0x40000000 + p1)) & 0xFFFFFFFF
    it = len(payloads_per_tile)
    return (acc - carry(it)) & 0xFFFFFFFF


def fast_max_tiles_geometry(sms):
    """(H4, W4, H, W) at x8 up-sampling whose 8 x 16 tile count is 255 per CTA of the fast kernel's 2 CTAs per SM:
    the largest the fixed-point accumulators admit."""
    H, W = 8 * 255, 16 * 2 * sms
    return H // 8, W // 8, H, W


def sigmoid(c):
    return 1.0 / (1.0 + math.exp(-c))
