"""Exact and float64 probes for the dense kernels: the wgmma linear kernel (csrc/gemm_wgmma.cu), the mask projection
paths and mask bits (csrc/mask_head.cu, csrc/mask_head_mma.cu) and the normalisation kernels (csrc/norm.cu).

No kernel is called here.  tests/test_dense_probes_cpu.py shows that each probe rejects named mutants: by at least one
wrong bit for the exact probes, by >= 10x its bound for the float64 probes.  tests/test_dense_probes_gpu.py runs the
kernels on the same probes.  The references are written independently of tests/emu.py (the CPU tests install emu as the
kernels, so a bug shared by the two would never show).

Exact probes (GEMM, mask projection, mask bits).  Operands are small integers (times 2^-4 for the GELU probe), so every
product is exact and every partial fp32 sum is an integer (a multiple of 2^-8) below 2^24: exact in any accumulation
order.  The kernel's fp32 accumulator therefore equals the float64 result, and one round-to-nearest-even to the storage
type follows in both, so the outputs are compared with torch.equal.
  address probe   row m of A holds a single 1 at k_m = 37 m mod K (37 is odd, so every k, hence every k-block and
                  every 16-wide k-step, is hit once M >= K).  W[n, k] = ((131 n + 17 k) mod 251) - 125 and bias[n] =
                  ((29 n) mod 129) - 64, so out[m, n] = W[n, k_m] + bias[n] with |out| <= 189: exact in bf16 and fp16.
                  Two columns of W are equal only 251 apart, two rows only 251 apart, so reading the wrong k (a dropped
                  k-block or k-step, a permuted swizzle chunk), the wrong n, the wrong bias column or storing to the
                  wrong place changes the bits.
  dense probe     A, W in {-1, 0, 1}, integer bias: |out| <= K + 64 <= 1088 for K <= 1024.  Integers up to 2048 are
                  exact in fp16; in bf16 the reference rounds the same exact integer, so the comparison stays exact.
                  This covers accumulation across all k-blocks at once.
  GELU            the same exact pre-activation z (address probe scaled by 2^-4, |z| <= 11.8 in steps of 1/16); the
                  reference is float64 GELU.  The epilogue's polynomial has absolute error < 1.5e-6 everywhere
                  (header of csrc/gemm_wgmma.cu); rounding the result to storage adds u |g| (u = 2^-8 bf16, 2^-11
                  fp16), and fp16 subnormal outputs an absolute 2^-25: bound u (|g| + 1.5e-6) + 1.5e-6 + 2^-24.
  mask bits       logits from the address probe of the mask projection, with reserved feature columns: column 0 is
                  -1 everywhere (a row whose every valid logit is negative: row_open = 1), column 1 is 0 everywhere
                  (logit exactly 0 is open: sigmoid = 0.5 is not < 0.5), column 2 cycles -1, 0, 1.  bits = logit < 0
                  packed 32 keys per word, bits past P are 0, row_open = every valid logit < 0.  No flip tolerance.

Float64 probes (LayerNorm, patch-merge LayerNorm, GroupNorm).  The reference is float64 normalisation of the
storage-rounded inputs; add_layernorm's sum x + r1 + r2 is rounded to storage first only when it is returned (the
kernel normalises what the next consumer reads).  Per element, with u the unit roundoff of the storage type, u32 =
2^-24, x^ = (s - mean) * rstd the float64 normalised value, r = rstd and w the weight:

    |y - y_ref| <= u |y_ref| + u32 |w| (c_x |x^| + c_0) + 2^-24

  u |y_ref|   rounding of the output to storage (for fp32 storage the final fp32 add).
  c_x |x^|    errors proportional to the normalised value, i.e. relative errors of rstd and of the epilogue:
              L / 2 for the fp32 sum of squares (non-negative terms summed in chains of <= L adds have relative error
              <= L u32, and rstd = var^-1/2 halves it), 8 for rsqrtf (2 ulp = 4 u32), the rounding of var + eps and the
              three fp32 products and differences of the epilogue, plus the effect on the variance of input
              errors e_i (Cauchy-Schwarz: |2/n sum d_i e_i| <= 2 sigma max|e|, i.e. a relative rstd error <= max|e| r):
              2 A r for LayerNorm (A = max over the row of |x| + |r1| + |r2|, two fp32 adds of the residuals) and, with
              a pre_bias, A r for GroupNorm (A = max over the group of |x + pre_bias|, one fp32 add).
              LayerNorm: c_x = L / 2 + 8 + 2 A r + (L a r)^2 u32 / 2: 8 = 4 for rsqrtf (2 ulp), 1 for var + eps, 3 for
              the epilogue's difference and two products; the last term is the variance taken around an fp32 mean
              that is off by L a u32 (a = mean |s| of the row).
              GroupNorm: c_x = L / 2 + 9 + GN_AGREE / (2 u32) (+ A r with a pre_bias): 4 for rsqrtf, 1 for var + eps,
              1 for x - pivot rounded once per value, 3 for the epilogue, and the kernel may keep raw-moment
              statistics whose variance is within GN_AGREE (var + eps) of the centred one (rstd within GN_AGREE / 2).
  c_0         errors independent of x^, moving the element by an absolute amount times r: LayerNorm 2 |x|+|r1|+|r2|
              of the element (its fp32 sum) plus L a (the fp32 mean); GroupNorm A for the mean rounded to fp32, A
              more with a pre_bias (x + pre_bias in fp32 in the apply pass), L (the fp32 sum of the centred values
              moves the mean by <= L u32 sigma), and GN_AGREE / u32 for a kept raw mean within GN_AGREE sqrt(var + eps).
  L           the longest fp32 chain of the statistics.  add_layernorm / patch_merge_layernorm: one warp per row, each
              lane adds its C / 32 values in sequence, then 5 butterfly levels: L = C / 32 + 5.  groupnorm_tokens:
              each thread adds its C / 4 tokens of the 256-token slice per channel in two chains (even / odd tokens),
              3 adds merge them and its 4 channels, and 256 / groups thread sums make a group:
              L = C / 8 + 256 / groups + 5 (the slices are combined in double).
  2^-24       absolute floor for outputs near zero (fp16 subnormal outputs round with absolute error 2^-25).

ReLU is 1-Lipschitz, so the GroupNorm bound of the pre-activation covers the activated output.
"""
import math

import torch

UNIT = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 2.0 ** -24}
U32 = 2.0 ** -24
GELU_ABS = 1.5e-6
EPS = 1e-5
GN_AGREE = 2.0 ** -19   # groupnorm_tokens keeps the raw-moment statistics where they agree with the centred ones
F64 = torch.float64


def stored(x, dtype):
    """Storage rounding, back to float64."""
    return x.to(dtype).to(F64)


def same(out, ref):
    """Bit-for-bit equality of a kernel output (any dtype) with a float64 reference already rounded to storage."""
    return torch.equal(out.to(F64).cpu(), ref.cpu())


# ---------------------------------------------------------------------------------------------------------------
# exact GEMM probes
# ---------------------------------------------------------------------------------------------------------------
def w_code(N, K, shift=0):
    n = torch.arange(N, dtype=torch.int64)[:, None] + shift
    k = torch.arange(K, dtype=torch.int64)[None]
    return ((131 * n + 17 * k) % 251 - 125).to(F64)


def bias_code(N):
    return ((29 * torch.arange(N, dtype=torch.int64)) % 129 - 64).to(F64)


def address_a(M, K, offset=0):
    """[M, K] one-hot rows: row m reads column k_m = 37 (m + offset) mod K."""
    a = torch.zeros(M, K, dtype=F64)
    a[torch.arange(M), (37 * (torch.arange(M) + offset)) % K] = 1.0
    return a


def address_probe(M, N, K, scale=1.0):
    return address_a(M, K), w_code(N, K) * scale, bias_code(N) * scale


def dense_probe(M, N, K, gen):
    a = torch.randint(-1, 2, (M, K), generator=gen).to(F64)
    w = torch.randint(-1, 2, (N, K), generator=gen).to(F64)
    return a, w, torch.randint(-64, 65, (N,), generator=gen).to(F64)


def linear_ref(a, w, b):
    out = a @ w.t()
    return out if b is None else out + b


def gelu(z):
    return 0.5 * z * (1.0 + torch.erf(z / math.sqrt(2.0)))


def gelu_bound(ref, dtype):
    u = UNIT[dtype]
    return u * (ref.abs() + GELU_ABS) + GELU_ABS + 2.0 ** -24


def head_major(out2d, S):
    """[B*S, N] -> [B, N/32, S, 32], the value layout of the sampling kernel."""
    M, N = out2d.shape
    return out2d.reshape(M // S, S, N // 32, 32).permute(0, 2, 1, 3).contiguous()


# GEMM mutants: float64 semantics of a kernel with one named mistake ----------------------------------------------
def drop_k(a, w, b, k0, k1):
    """k columns [k0, k1) never accumulated (a dropped k-block or 16-wide k-step)."""
    a = a.clone()
    a[:, k0:k1] = 0
    return linear_ref(a, w, b)


def swizzle_wrong_rows(t):
    """The 16-byte chunk c of row r in a 64-column box read from chunk c ^ (r & 7) ^ ((r >> 1) & 7): the 128-B swizzle
    XORed with the wrong row bits, i.e. columns permuted inside each box."""
    R, K = t.shape
    r = torch.arange(R)[:, None]
    k = torch.arange(K)[None]
    c = (k % 64) // 8
    src = (k // 64) * 64 + ((c ^ (r & 7) ^ ((r >> 1) & 7)) * 8) + k % 8
    return t.gather(1, src.expand(R, K))


def bias_shift(b, s=8):
    return torch.roll(b, -s)


def tail_unwritten(out, box=64):
    """Rows of the last, partly filled 64-row box never stored (they keep the NaN poison)."""
    out = out.clone()
    M = out.shape[0]
    if M % box:
        out[M - M % box:] = float("nan")
    return out


def head_major_off_by_one(hm, axis):
    """The head-major store lands one image (axis 0) or one head (axis 1) further; the first one stays unwritten."""
    mut = torch.full_like(hm, float("nan"))
    if axis == 0:
        mut[1:] = hm[:-1]
    else:
        mut[:, 1:] = hm[:, :-1]
    return mut


# ---------------------------------------------------------------------------------------------------------------
# exact mask projection and mask-bit probes
# ---------------------------------------------------------------------------------------------------------------
def mask_proj_probe(B, Q, P, C=256, shared=False, bits_rows=True):
    """mask_embed [B, Q, C] one-hot, feats [B or 1, P, C] integer codes (image b shifted by 3 b pixels).  With
    bits_rows, queries 0 / 1 / 2 read the reserved columns 0 / 1 / 2 (all -1, all 0, cycling -1 0 1)."""
    nb = 1 if shared else B
    feats = torch.stack([w_code(P, C, shift=3 * i) for i in range(nb)])
    p = torch.arange(P)
    feats[:, :, 0] = -1.0
    feats[:, :, 1] = 0.0
    feats[:, :, 2] = (p % 3 - 1).to(F64)
    me = torch.zeros(B, Q, C, dtype=F64)
    for b in range(B):
        k = 3 + (37 * torch.arange(Q) + 11 * b) % (C - 3)
        if bits_rows:
            k[:min(Q, 3)] = torch.arange(min(Q, 3))
        me[b, torch.arange(Q), k] = 1.0
    return me, feats


def mask_proj_dense(B, Q, P, gen, C=256):
    me = torch.randint(-1, 2, (B, Q, C), generator=gen).to(F64)
    return me, torch.randint(-1, 2, (B, P, C), generator=gen).to(F64)


def mask_logits_ref(me, feats):
    return torch.matmul(me, feats.expand(me.shape[0], -1, -1).transpose(1, 2))


def pack_bits(blocked):
    """bool [..., P] -> int32 words [..., ceil(P/32)] (bit j of word w = key 32 w + j), zero past P."""
    P = blocked.shape[-1]
    W32 = (P + 31) // 32
    pad = torch.zeros(blocked.shape[:-1] + (W32 * 32,), dtype=torch.int64)
    pad[..., :P] = blocked.to(torch.int64)
    words = (pad.view(blocked.shape[:-1] + (W32, 32)) << torch.arange(32)).sum(-1)
    return torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32)


def mask_bits_ref(logits, rule="lt0", tail=False, open_over_padded=False):
    """(bits, row_open) of float64 logits [B, Q, P].  The reference is rule 'lt0'; the keyword arguments are the named
    mutants: rule 'le0' (<= 0 blocks), tail (bits past P set), open_over_padded (row_open over the padded width)."""
    blocked = logits < 0 if rule == "lt0" else logits <= 0
    bits = pack_bits(blocked)
    P = logits.shape[-1]
    if tail and P % 32:
        bits[..., -1] |= torch.tensor(-(1 << (P % 32)), dtype=torch.int32)     # bits P % 32 .. 31 of the last word
    row_open = blocked.all(-1)
    if open_over_padded:
        W32 = bits.shape[-1]
        keys = (bits.to(torch.int64).unsqueeze(-1) >> torch.arange(32)) & 1
        row_open = keys.view(bits.shape[:-1] + (W32 * 32,)).bool().all(-1)
    return bits, row_open.to(torch.uint8)


def bits_logits_probe(R, P, gen):
    """Direct attn_mask_bits input [1, R, P]: rows cycle through every-valid-negative, exactly-zero / -0.0 mixtures,
    tiny negatives and integer codes."""
    x = torch.randint(-3, 4, (R, P), generator=gen).to(F64)
    for r in range(R):
        kind = r % 4
        if kind == 0:
            x[r] = -torch.randint(1, 5, (P,), generator=gen).to(F64)          # every valid key blocked
        elif kind == 1:
            x[r] = 0.0
            x[r, ::2] = -0.0                                                    # -0.0 is not < 0: open
        elif kind == 2:
            x[r, ::3] = -(2.0 ** -14)                                           # tiny negatives block (fp16 normal)
    return x.unsqueeze(0)


# ---------------------------------------------------------------------------------------------------------------
# LayerNorm
# ---------------------------------------------------------------------------------------------------------------
def _z(C, gen):
    """Gaussian-shaped values kept away from 0 (|z| >= 1/4), so that every row spans few binades and x + r1 + r2 of
    16-bit inputs is exact in fp32 (the returned, rounded sum then equals the reference bit for bit)."""
    z = torch.randn(C, generator=gen, dtype=F64)
    return torch.sign(z) * (0.25 + z.abs())


LN_KINDS = ("scale", "offset", "outlier", "constant", "cancel", "small")


def ln_probe(R, C, nres, dtype, gen):
    """Rows cycling through LN_KINDS, with residuals: returns (inputs list of float64 [R, C] storage-rounded, w, b).
    scale: Gaussian rows of std 1e-3 .. 1e3 (a row mix-up moves the output by O(1)); offset: mean / std 10 .. 1e3;
    outlier: one channel 1e3x the rest; constant: x + r1 + r2 = 3.25 exactly (y must be the bias); cancel: r1 = -x +
    O(1), x ~ 100; small: std 2e-3, where eps = 1e-5 matters."""
    n_in = 1 + nres
    ins = [torch.zeros(R, C, dtype=F64) for _ in range(n_in)]
    for i in range(R):
        kind = LN_KINDS[i % len(LN_KINDS)]
        z = [_z(C, gen) for _ in range(n_in)]
        if kind == "scale":
            sig = 10.0 ** (((i // len(LN_KINDS)) % 7) - 3)
            rows = [sig * t for t in z]
        elif kind == "offset":
            ratio = (10.0, 100.0, 1000.0)[(i // len(LN_KINDS)) % 3] * (-1) ** i
            rows = [ratio + z[0]] + [0.5 * t for t in z[1:]]
        elif kind == "outlier":
            rows = [t.clone() for t in z]
            rows[0][(37 * i) % C] *= 1000.0
        elif kind == "constant":
            rows = [torch.full((C,), v, dtype=F64) for v in ((3.25,), (2.0, 1.25), (2.0, 1.0, 0.25))[nres]]
        elif kind == "cancel":
            big = stored(100.0 * z[0], dtype)
            rows = [big] + ([stored(-big + z[1], dtype)] + z[2:nres + 1] if nres else [])
            if not nres:
                rows = [z[0]]
        else:
            rows = [2e-3 * t for t in z]
        for k in range(n_in):
            ins[k][i] = stored(rows[k], dtype)
    w = stored(1.0 + 0.5 * torch.randn(C, generator=gen, dtype=F64), dtype)
    b = stored(0.5 * torch.randn(C, generator=gen, dtype=F64), dtype)
    return ins, w, b


def ln_ref(ins, w, b, dtype, return_sum, eps=EPS):
    """Float64 add + LayerNorm over the last dim; the sum is rounded to storage first only when it is returned."""
    s = sum(ins)
    if return_sum and dtype != torch.float32:   # fp32 storage: the returned sum is the kernel's fp32 sum itself
        s = stored(s, dtype)
    mu = s.mean(-1, keepdim=True)
    var = ((s - mu) ** 2).mean(-1, keepdim=True)
    r = 1.0 / torch.sqrt(var + eps)
    xh = (s - mu) * r
    ain = sum(t.abs() for t in ins)
    return dict(s=s, y=xh * w + b, xhat=xh, r=r, var=var, mu=mu, a=s.abs().mean(-1, keepdim=True), ain=ain,
                A=ain.amax(-1, keepdim=True), const=(var == 0))


def ln_chain(C):
    return C / 32 + 5


def ln_bound(ref, w, dtype):
    u = UNIT[dtype]
    L = ln_chain(ref["s"].shape[-1])
    r = ref["r"]
    ar = ref["a"] * r
    cx = L / 2 + 8 + 2 * ref["A"] * r + 0.5 * (L * ar) ** 2 * U32
    c0 = r * (2 * ref["ain"] + L * ref["a"])
    return u * ref["y"].abs() + U32 * w.abs() * (cx * ref["xhat"].abs() + c0) + 2.0 ** -24


def ratio(out, ref_y, bnd):
    o = out.to(F64).cpu()
    assert torch.isfinite(o).all(), "non-finite kernel output"
    return float(((o - ref_y) / bnd).abs().max())


def ln_eps_outside(ref, w, b, eps=EPS):
    """Mutant: 1 / (sqrt(var) + eps) instead of 1 / sqrt(var + eps)."""
    return (ref["s"] - ref["mu"]) / (torch.sqrt(ref["var"]) + eps) * w + b


def _butterfly(s):
    for o in (16, 8, 4, 2, 1):
        s = s + s[..., torch.arange(32) ^ o]
    return s


def _fma32(a, b, c):
    return (a.to(F64) * b.to(F64) + c.to(F64)).to(torch.float32)


def ln_fp32(s32, w, b, dtype, eps=EPS, one_pass=False):
    """fp32 emulation of add_layernorm_kernel's statistics in its order (lane l holds elements (32 c + l) * 4 + i,
    adds them in (c, i) order, then 5 butterfly levels) on the fp32 row s32 [R, C]; one_pass = the mutant that sums
    x and x^2 and takes E[x^2] - mean^2.  Returns the output rounded to storage, as float64."""
    R, C = s32.shape
    v = s32.view(R, C // 128, 32, 4)
    s = torch.zeros(R, 32, dtype=torch.float32)
    q = torch.zeros(R, 32, dtype=torch.float32)
    for c in range(C // 128):
        for i in range(4):
            s = s + v[:, c, :, i]
            if one_pass:
                q = _fma32(v[:, c, :, i], v[:, c, :, i], q)
    inv = torch.tensor(1.0 / C, dtype=torch.float32)
    mean = (_butterfly(s)[:, :1] * inv)
    if one_pass:
        var = torch.clamp(_butterfly(q)[:, :1] * inv - mean * mean, min=0)
    else:
        d = s32 - mean
        dv = d.view(R, C // 128, 32, 4)
        q = torch.zeros(R, 32, dtype=torch.float32)
        for c in range(C // 128):
            for i in range(4):
                q = _fma32(dv[:, c, :, i], dv[:, c, :, i], q)
        var = _butterfly(q)[:, :1] * inv
    rstd = (1.0 / torch.sqrt((var + torch.tensor(eps, dtype=torch.float32)).to(F64))).to(torch.float32)
    y = (s32 - mean) * rstd * w.to(torch.float32) + b.to(torch.float32)
    return stored(y, dtype)


def kernel_sum32(ins, dtype, return_sum):
    """The kernel's fp32 row: x (+ r1) (+ r2) added in fp32, rounded to storage when it is returned."""
    s = ins[0].to(torch.float32)
    for t in ins[1:]:
        s = s + t.to(torch.float32)
    return s.to(dtype).to(torch.float32) if return_sum else s


# patch merge: the 2x2 gather of swin PatchMerging, zero padded to even H / W -------------------------------------
def patch_merge_gather(x, H, W):
    """x [B, H*W, C] float64 -> [B, ceil(H/2)*ceil(W/2), 4C] (cat of x[2i,2j], x[2i+1,2j], x[2i,2j+1], x[2i+1,2j+1])."""
    B, _, C = x.shape
    xm = x.view(B, H, W, C)
    xm = torch.nn.functional.pad(xm, (0, 0, 0, W % 2, 0, H % 2))
    xm = torch.cat([xm[:, 0::2, 0::2], xm[:, 1::2, 0::2], xm[:, 0::2, 1::2], xm[:, 1::2, 1::2]], -1)
    return xm.reshape(B, -1, 4 * C)


def patch_merge_probe(B, H, W, C, dtype, gen):
    """Pixels take the kind of their output row (LN_KINDS without the residual-only 'cancel'), so every gathered
    row is a scale / offset / outlier / constant / small row (rows touching the zero padding mix in zeros)."""
    H2, W2 = (H + 1) // 2, (W + 1) // 2
    x = torch.zeros(B, H, W, C, dtype=F64)
    kinds = ("scale", "offset", "outlier", "constant", "small")
    for bi in range(B):
        for yy in range(H):
            for xx in range(W):
                i = (bi * H2 + yy // 2) * W2 + xx // 2
                kind = kinds[i % len(kinds)]
                z = _z(C, gen)
                if kind == "scale":
                    v = 10.0 ** ((i % 7) - 3) * z
                elif kind == "offset":
                    v = 1000.0 * (-1) ** i + z
                elif kind == "outlier":
                    v = z.clone()
                    v[(37 * i) % C] *= 1000.0
                elif kind == "constant":
                    v = torch.full((C,), 3.25, dtype=F64)
                else:
                    v = 2e-3 * z
                x[bi, yy, xx] = stored(v, dtype)
    w = stored(1.0 + 0.5 * torch.randn(4 * C, generator=gen, dtype=F64), dtype)
    b = stored(0.5 * torch.randn(4 * C, generator=gen, dtype=F64), dtype)
    return x.view(B, H * W, C), w, b


# ---------------------------------------------------------------------------------------------------------------
# GroupNorm
# ---------------------------------------------------------------------------------------------------------------
def gn_probe(B, N, C, groups, ratio_ms, dtype, gen, pre_bias=False):
    """x [B, N, C] with x + pre_bias ~ mean + std z per (batch, group): std 2^((3 b + 5 g) % 7 - 3), mean = +-ratio_ms
    * std (sign by group).  pre_bias: a per-channel bias in [-50, 50] that the stored x compensates, so the
    offset of x + pre_bias stays the designed one.  Returns (x, pb or None, w, b), float64 storage-rounded."""
    cpg = C // groups
    g = torch.arange(C) // cpg
    std = torch.stack([2.0 ** (((3 * bi + 5 * g) % 7) - 3).to(F64) for bi in range(B)])     # [B, C]
    mean = ratio_ms * std * torch.where(g % 2 == 0, 1.0, -1.0).to(F64)
    target = mean[:, None, :] + std[:, None, :] * torch.randn(B, N, C, generator=gen, dtype=F64)
    pb = None
    if pre_bias:
        pb = stored(torch.linspace(-50, 50, C, dtype=F64)[torch.randperm(C, generator=gen)], dtype)
        x = stored(target - pb, dtype)
    else:
        x = stored(target, dtype)
    w = stored(1.0 + 0.5 * torch.randn(C, generator=gen, dtype=F64), dtype)
    b = stored(0.5 * torch.randn(C, generator=gen, dtype=F64), dtype)
    return x, pb, w, b


def gn_ref(x, pb, w, b, groups, relu, eps=EPS, stat_batch=None, stat_group=None):
    """Float64 GroupNorm of x + pre_bias over (tokens, channels of the group).  stat_batch / stat_group (index maps)
    are the mutants that normalise with another batch's or group's statistics."""
    B, N, C = x.shape
    v = x if pb is None else x + pb
    vg = v.view(B, N, groups, C // groups)
    mu = vg.mean(dim=(1, 3))                                          # [B, G]
    var = ((vg - mu[:, None, :, None]) ** 2).mean(dim=(1, 3))
    if stat_batch is not None:
        mu, var = mu[stat_batch], var[stat_batch]
    if stat_group is not None:
        mu, var = mu[:, stat_group], var[:, stat_group]
    r = 1.0 / torch.sqrt(var + eps)
    xh = ((vg - mu[:, None, :, None]) * r[:, None, :, None]).view(B, N, C)
    y = xh * w + b
    A = vg.abs().amax(dim=(1, 3))
    rr = r[:, None, :, None].expand(B, N, groups, C // groups).reshape(B, N, C)
    AA = A[:, None, :, None].expand(B, N, groups, C // groups).reshape(B, N, C)
    return dict(y=y.clamp(min=0) if relu else y, y_pre=y, xhat=xh, r=rr, A=AA, mu=mu, var=var)


def gn_chain(C, groups):
    return C / 8 + 256 / groups + 5


def gn_bound(ref, w, dtype, C, groups, pre_bias):
    u = UNIT[dtype]
    L = gn_chain(C, groups)
    Ar = ref["A"] * ref["r"]
    cx = L / 2 + 9 + GN_AGREE / (2 * U32) + (Ar if pre_bias else 0.0)
    c0 = (2 * Ar if pre_bias else Ar) + L + GN_AGREE / U32
    return u * ref["y_pre"].abs() + U32 * w.abs() * (cx * ref["xhat"].abs() + c0) + 2.0 ** -24


def gn_fp32(x, pb, w, b, groups, dtype, relu, eps=EPS, scheme="kernel"):
    """fp32 emulation of groupnorm_tokens in its summation order (256-token slices).  scheme 'kernel': the kernel of
    csrc/norm.cu, i.e. the raw moments where they agree with the centred statistics (pivot = slice mean, two
    accumulators per channel, Chan combine in double) to GN_AGREE, the centred ones elsewhere.  scheme 'raw': the
    mutant that always takes the raw moments (fp32 sums of x and x^2 per thread, its 4 channels in one chain, then
    E[x^2] - mean^2 in double), i.e. the earlier kernel.  Returns the output rounded to storage, as float64."""
    B, N, C = x.shape
    f32 = torch.float32
    pbv = torch.zeros(C, dtype=f32) if pb is None else pb.to(f32)
    chunks, cpg = C // 4, C // groups
    tpb, cpgc = 256 // chunks, cpg // 4
    T = 256
    nparts = (N + T - 1) // T
    Np = nparts * T
    xp = (-pbv).expand(B, Np, C).clone()                     # padding tokens: x + pre_bias = 0 exactly
    xp[:, :N] = x.to(f32)
    J = T // tpb
    # token t0 + trow + j tpb of slice p, chunk cidx, element i
    v = (xp + pbv).view(B, nparts, J, tpb, chunks, 4)
    cnt = torch.clamp(N - torch.arange(nparts) * T, max=T).to(F64) * cpg        # [nparts]
    n = float(N * cpg)

    def group_reduce(t):                                    # [B, P, tpb, chunks] -> [B, P, G] in the kernel's order
        out = torch.zeros(B, nparts, groups, dtype=f32)
        tg = t.view(B, nparts, tpb, groups, cpgc)
        for rr in range(tpb):
            for c in range(cpgc):
                out = out + tg[:, :, rr, :, c]
        return out

    # raw moments
    s = torch.zeros(B, nparts, tpb, chunks, dtype=f32)
    q = torch.zeros_like(s)
    for j in range(J):
        for i in range(4):
            f = v[:, :, j, :, :, i]
            s = s + f
            q = _fma32(f, f, q)
    gs = group_reduce(s)
    mean_raw = gs.to(F64).sum(1) / n
    var_raw = torch.clamp(group_reduce(q).to(F64).sum(1) / n - mean_raw * mean_raw, min=0)
    if scheme == "raw":
        mean, var = mean_raw, var_raw
    else:
        piv = (gs.to(F64) / cnt[None, :, None]).to(f32)                              # [B, P, G]
        pc = piv.repeat_interleave(cpg, dim=2).view(B, nparts, 1, chunks, 4)
        d1 = torch.zeros(2, B, nparts, tpb, chunks, 4, dtype=f32)             # even / odd tokens of a thread
        d2 = torch.zeros_like(d1)
        tok = (torch.arange(nparts)[:, None, None] * T + torch.arange(J)[None, :, None] * tpb
               + torch.arange(tpb)[None, None, :])                                # [P, J, tpb]
        for j in range(J):
            valid = (tok[:, j] < N).view(1, nparts, tpb, 1, 1)
            d = torch.where(valid, v[:, :, j] - pc, torch.zeros((), dtype=f32))
            d1[j % 2] = d1[j % 2] + d
            d2[j % 2] = _fma32(d, d, d2[j % 2])
        e1, e2 = d1[0] + d1[1], d2[0] + d2[1]
        g1 = group_reduce((e1[..., 0] + e1[..., 1]) + (e1[..., 2] + e1[..., 3])).to(F64)
        g2 = group_reduce((e2[..., 0] + e2[..., 1]) + (e2[..., 2] + e2[..., 3])).to(F64)
        pm = piv.to(F64) + g1 / cnt[None, :, None]
        pm2 = g2 - g1 * g1 / cnt[None, :, None]
        mean_c = (cnt[None, :, None] * pm).sum(1) / n
        var_c = torch.clamp((pm2 + cnt[None, :, None] * (pm - mean_c[:, None]) ** 2).sum(1), min=0) / n
        ve = var_c + eps
        agree = ((mean_raw - mean_c).abs() <= GN_AGREE * ve.sqrt()) & ((var_raw - var_c).abs() <= GN_AGREE * ve)
        mean, var = torch.where(agree, mean_raw, mean_c), torch.where(agree, var_raw, var_c)
    rstd = (1.0 / torch.sqrt(var.to(f32).to(F64) + eps)).to(f32)              # rsqrtf((float)var + eps)
    mr = mean.to(f32).repeat_interleave(cpg, dim=1)[:, None, :]
    rr = rstd.repeat_interleave(cpg, dim=1)[:, None, :]
    y = ((x.to(f32) + pbv) - mr) * rr * w.to(f32) + b.to(f32)
    if relu:
        y = y.clamp(min=0)
    return stored(y, dtype)
