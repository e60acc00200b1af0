// Generic fused attention (scores -> policy bias/mask -> online softmax -> PV) in fp32 SIMT math.
//
// This is the exact-arithmetic tier of the attention family: storage type T in {fp32, fp16, bf16},
// all math in fp32 with accurate expf.  It serves (a) fp32 parity runs against the oracle and (b) as
// the correctness anchor for the tensor-core kernels.  Three policies share one kernel:
//   WindowPolicy  Swin W-MSA / SW-MSA   (reference multimodal_encoder/swin_trans.py:117-149,194-253)
//                 window partition, cyclic shift, zero padding after norm1, relative-position bias and
//                 the -100 shift mask are all folded into addressing — no roll / pad / partition copies.
//   CausalPolicy  Phi prefill attention (transformers modeling_phi.py eager_attention_forward;
//                 call site language_model/llava_phi.py:1354-1363) with key padding mask.
//   CrossPolicy   Mask2Former masked cross-attention / query self-attention
//                 (transformer_decoder/mask2former_transformer_decoder.py:93-105, 35-45) with a packed
//                 bit mask (1 = blocked) and the "fully blocked row attends everywhere" rule (:647).
// Split-K over the keys (partials + combine) keeps 100-query problems on all 132 SMs.
#include "common.cuh"

namespace psalm {

struct AttnDims {
  int B, H, Lq, Lk, splits;
  float scale;
};

constexpr int kBQ = 32, kBK = 32, kNT = 256;

template <typename T>
__device__ __forceinline__ float4 ld4(const T* p) {
  if constexpr (sizeof(T) == 4) {
    return __ldg(reinterpret_cast<const float4*>(p));
  } else {
    const uint2 v = __ldg(reinterpret_cast<const uint2*>(p));
    float4 r;
    unpack2<T>(v.x, r.x, r.y);
    unpack2<T>(v.y, r.z, r.w);
    return r;
  }
}

// ------------------------------------------------------------------------------------------------
template <typename T>
struct WindowPolicy {
  const T* qkv;        // [B, H*W, 3, nh, hd]
  const T* qkv_bias;   // [3*C]  (value of a zero-padded token after the qkv Linear)
  const float* rel;    // [nh, (2 ws - 1)^2] compact relative-position bias table (checkpoint table, transposed)
  T* out;              // [B, H*W, C]
  int H, W, Hp, Wp, ws, shift, nh, hd, C, nWx, nW;

  __device__ __forceinline__ bool token(int z, int n, int& tok, int& region) const {
    const int win = z % nW, bi = z / nW;
    const int wy = win / nWx, wx = win - wy * nWx;
    const int i = n / ws, j = n - i * ws;
    const int py = wy * ws + i, px = wx * ws + j;
    const int rh = py < Hp - ws ? 0 : (py < Hp - shift ? 1 : 2);
    const int rw = px < Wp - ws ? 0 : (px < Wp - shift ? 1 : 2);
    region = rh * 3 + rw;
    int oy = py + shift, ox = px + shift;
    if (oy >= Hp) oy -= Hp;
    if (ox >= Wp) ox -= Wp;
    tok = (bi * H + oy) * W + ox;
    return oy < H && ox < W;
  }
  __device__ __forceinline__ float4 load(int which, int z, int h, int n, int d0) const {
    int tok, reg;
    const int col = which * C + h * hd + d0;
    if (token(z, n, tok, reg)) return ld4<T>(qkv + (size_t)tok * 3 * C + col);
    return ld4<T>(qkv_bias + col);
  }
  __device__ __forceinline__ float4 load_q4(int z, int h, int n, int d0) const { return load(0, z, h, n, d0); }
  __device__ __forceinline__ float4 load_k4(int z, int h, int n, int d0) const { return load(1, z, h, n, d0); }
  __device__ __forceinline__ float4 load_v4(int z, int h, int n, int d0) const { return load(2, z, h, n, d0); }
  __device__ __forceinline__ float score(int z, int h, int qi, int kj, float s) const {
    // relative_position_index[qi, kj] = (yi - yj + ws - 1) * (2 ws - 1) + (xi - xj + ws - 1)  (swin_trans.py:93-103)
    const int R = 2 * ws - 1;
    const int yi = qi / ws, xi = qi - yi * ws, yj = kj / ws, xj = kj - yj * ws;
    s += __ldg(rel + (size_t)h * R * R + (yi - yj + ws - 1) * R + (xi - xj + ws - 1));
    if (shift > 0) {
      int t, rq, rk;
      token(z, qi, t, rq);
      token(z, kj, t, rk);
      if (rq != rk) s += -100.0f;  // swin_trans.py:387
    }
    return s;
  }
  __device__ __forceinline__ int key_tile_end(int q0, int kt1) const { return kt1; }
  __device__ __forceinline__ void store(int z, int h, int n, int d, float v) const {
    int tok, reg;
    if (token(z, n, tok, reg)) out[(size_t)tok * C + h * hd + d] = from_f32<T>(v);
  }
};

template <typename T>
struct CausalPolicy {
  const T* qkv;              // [B, T, 3, nh, hd] (rotary already applied to q, k)
  const uint8_t* key_valid;  // [B, T] or null
  T* out;                    // [B, T, nh*hd]
  int T_, nh, hd;
  __device__ __forceinline__ float4 load(int which, int b, int h, int n, int d0) const {
    return ld4<T>(qkv + (((size_t)b * T_ + n) * 3 + which) * nh * hd + h * hd + d0);
  }
  __device__ __forceinline__ float4 load_q4(int b, int h, int n, int d0) const { return load(0, b, h, n, d0); }
  __device__ __forceinline__ float4 load_k4(int b, int h, int n, int d0) const { return load(1, b, h, n, d0); }
  __device__ __forceinline__ float4 load_v4(int b, int h, int n, int d0) const { return load(2, b, h, n, d0); }
  __device__ __forceinline__ float score(int b, int h, int qi, int kj, float s) const {
    if (kj > qi) return -INFINITY;
    if (key_valid && !key_valid[(size_t)b * T_ + kj]) return -INFINITY;
    return s;
  }
  __device__ __forceinline__ int key_tile_end(int q0, int kt1) const {
    const int e = (q0 + kBQ - 1) / kBK + 1;
    return e < kt1 ? e : kt1;
  }
  __device__ __forceinline__ void store(int b, int h, int n, int d, float v) const {
    out[((size_t)b * T_ + n) * nh * hd + h * hd + d] = from_f32<T>(v);
  }
};

// Causal prefill of prompt suffixes behind a shared prefix (key axis = [P prefix keys | own keys]): the prefix K / V are
// head-major [nh, ld_rows, hd] and shared by all B sequences; query t attends the prefix and its own keys u <= t.
template <typename T>
struct PrefixCausalPolicy {
  const T* qkv;              // [B, T, 3, nh, hd], rotary applied at positions P + t
  const T *pk, *pv;          // [nh, ld_rows, hd]
  const uint8_t* key_valid;  // [B, T] or null
  T* out;                    // [B, T, nh*hd]
  int T_, nh, hd, P, ld_rows;
  __device__ __forceinline__ float4 load_q4(int b, int h, int n, int d0) const {
    return ld4<T>(qkv + (((size_t)b * T_ + n) * 3) * nh * hd + h * hd + d0);
  }
  __device__ __forceinline__ float4 load_k4(int b, int h, int kj, int d0) const {
    if (kj < P) return ld4<T>(pk + ((size_t)h * ld_rows + kj) * hd + d0);
    return ld4<T>(qkv + (((size_t)b * T_ + kj - P) * 3 + 1) * nh * hd + h * hd + d0);
  }
  __device__ __forceinline__ float4 load_v4(int b, int h, int kj, int d0) const {
    if (kj < P) return ld4<T>(pv + ((size_t)h * ld_rows + kj) * hd + d0);
    return ld4<T>(qkv + (((size_t)b * T_ + kj - P) * 3 + 2) * nh * hd + h * hd + d0);
  }
  __device__ __forceinline__ float score(int b, int h, int qi, int kj, float s) const {
    if (kj < P) return s;
    const int u = kj - P;
    if (u > qi) return -INFINITY;
    if (key_valid && !key_valid[(size_t)b * T_ + u]) return -INFINITY;
    return s;
  }
  __device__ __forceinline__ int key_tile_end(int q0, int kt1) const {
    const int e = (P + q0 + kBQ - 1) / kBK + 1;
    return e < kt1 ? e : kt1;
  }
  __device__ __forceinline__ void store(int b, int h, int n, int d, float v) const {
    out[((size_t)b * T_ + n) * nh * hd + h * hd + d] = from_f32<T>(v);
  }
};

template <typename T>
struct CrossPolicy {
  const T *q, *k, *v;        // [B, Lq, nh*hd], [B, Lk, nh*hd] x2
  const uint32_t* bits;      // [B, Lq, W32] 1 = blocked, or null
  const uint8_t* row_open;   // [B, Lq] 1 = every key blocked -> ignore the mask (DEC:647), or null
  T* out;                    // [B, Lq, nh*hd]
  int Lq, Lk, nh, hd, W32;
  __device__ __forceinline__ float4 load_q4(int b, int h, int n, int d0) const {
    return ld4<T>(q + ((size_t)b * Lq + n) * nh * hd + h * hd + d0);
  }
  __device__ __forceinline__ float4 load_k4(int b, int h, int n, int d0) const {
    return ld4<T>(k + ((size_t)b * Lk + n) * nh * hd + h * hd + d0);
  }
  __device__ __forceinline__ float4 load_v4(int b, int h, int n, int d0) const {
    return ld4<T>(v + ((size_t)b * Lk + n) * nh * hd + h * hd + d0);
  }
  __device__ __forceinline__ float score(int b, int h, int qi, int kj, float s) const {
    if (bits) {
      const size_t row = (size_t)b * Lq + qi;
      if (!(row_open && row_open[row]) && ((__ldg(bits + row * W32 + (kj >> 5)) >> (kj & 31)) & 1u)) return -INFINITY;
    }
    return s;
  }
  __device__ __forceinline__ int key_tile_end(int q0, int kt1) const { return kt1; }
  __device__ __forceinline__ void store(int b, int h, int n, int d, float v) const {
    out[((size_t)b * Lq + n) * nh * hd + h * hd + d] = from_f32<T>(v);
  }
};

// ------------------------------------------------------------------------------------------------
// grid = (q_tiles * splits, H, B'), block = 256: thread (r = tid/8, c = tid%8) owns query row r,
// keys {c, c+8, c+16, c+24} of each key tile and output dims {c + 8 i}.
// ------------------------------------------------------------------------------------------------
template <typename Policy, int HD>
__global__ void __launch_bounds__(kNT) attn_simt_kernel(Policy pol, AttnDims dm, float* __restrict__ part) {
  __shared__ float Qs[kBQ][HD + 1];
  __shared__ float Ks[kBK][HD + 1];
  __shared__ float Vs[kBK][HD + 1];
  __shared__ float Ps[kBQ][kBK + 1];
  const int tid = threadIdx.x, r = tid >> 3, c = tid & 7;
  const int qt = blockIdx.x / dm.splits, sp = blockIdx.x - qt * dm.splits;
  const int h = blockIdx.y, b = blockIdx.z;
  const int q0 = qt * kBQ;
  const int ktiles = (dm.Lk + kBK - 1) / kBK;
  const int tps = (ktiles + dm.splits - 1) / dm.splits;
  const int kt0 = sp * tps;
  int kt1 = kt0 + tps < ktiles ? kt0 + tps : ktiles;
  kt1 = pol.key_tile_end(q0, kt1);

  for (int i = tid; i < kBQ * HD / 4; i += kNT) {
    const int row = i / (HD / 4), d0 = (i % (HD / 4)) * 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q0 + row < dm.Lq) v = pol.load_q4(b, h, q0 + row, d0);
    Qs[row][d0] = v.x; Qs[row][d0 + 1] = v.y; Qs[row][d0 + 2] = v.z; Qs[row][d0 + 3] = v.w;
  }
  float m_run = -INFINITY, l_run = 0.f;
  float o[HD / 8];
#pragma unroll
  for (int i = 0; i < HD / 8; ++i) o[i] = 0.f;
  const int qi = q0 + r;

  for (int kt = kt0; kt < kt1; ++kt) {
    __syncthreads();
    for (int i = tid; i < kBK * HD / 4; i += kNT) {
      const int row = i / (HD / 4), d0 = (i % (HD / 4)) * 4;
      float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
      const int kj = kt * kBK + row;
      if (kj < dm.Lk) {
        kv = pol.load_k4(b, h, kj, d0);
        vv = pol.load_v4(b, h, kj, d0);
      }
      Ks[row][d0] = kv.x; Ks[row][d0 + 1] = kv.y; Ks[row][d0 + 2] = kv.z; Ks[row][d0 + 3] = kv.w;
      Vs[row][d0] = vv.x; Vs[row][d0 + 1] = vv.y; Vs[row][d0 + 2] = vv.z; Vs[row][d0 + 3] = vv.w;
    }
    __syncthreads();
    float s[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 8
    for (int d = 0; d < HD; ++d) {
      const float qv = Qs[r][d];
#pragma unroll
      for (int j = 0; j < 4; ++j) s[j] = fmaf(qv, Ks[c + 8 * j][d], s[j]);
    }
    float tmax = -INFINITY;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int kj = kt * kBK + c + 8 * j;
      s[j] = (qi < dm.Lq && kj < dm.Lk) ? pol.score(b, h, qi, kj, s[j] * dm.scale) : -INFINITY;
      tmax = fmaxf(tmax, s[j]);
    }
#pragma unroll
    for (int off = 1; off < 8; off <<= 1) tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, off));
    const float m_new = fmaxf(m_run, tmax);
    float corr = 1.f, psum = 0.f;
    float p[4] = {0.f, 0.f, 0.f, 0.f};
    if (m_new != -INFINITY) {
      corr = (m_run == -INFINITY) ? 0.f : expf(m_run - m_new);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        p[j] = (s[j] == -INFINITY) ? 0.f : expf(s[j] - m_new);
        psum += p[j];
      }
    }
#pragma unroll
    for (int off = 1; off < 8; off <<= 1) psum += __shfl_xor_sync(0xffffffffu, psum, off);
    l_run = l_run * corr + psum;
    m_run = m_new;
#pragma unroll
    for (int j = 0; j < 4; ++j) Ps[r][c + 8 * j] = p[j];
    __syncwarp();
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) o[i] *= corr;
#pragma unroll 8
    for (int k = 0; k < kBK; ++k) {
      const float pv = Ps[r][k];
#pragma unroll
      for (int i = 0; i < HD / 8; ++i) o[i] = fmaf(pv, Vs[k][c + 8 * i], o[i]);
    }
  }
  if (qi >= dm.Lq) return;
  if (dm.splits == 1) {
    const float inv = l_run > 0.f ? 1.f / l_run : 0.f;
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) pol.store(b, h, qi, c + 8 * i, o[i] * inv);
  } else {
    float* pr = part + ((((size_t)b * dm.H + h) * dm.splits + sp) * dm.Lq + qi) * (HD + 2);
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) pr[c + 8 * i] = o[i];
    if (c == 0) {
      pr[HD] = m_run;
      pr[HD + 1] = l_run;
    }
  }
}

template <typename Policy, int HD>
__global__ void attn_combine_kernel(Policy pol, AttnDims dm, const float* __restrict__ part) {
  const long long n = (long long)dm.B * dm.H * dm.Lq * HD;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < n;
       idx += (long long)gridDim.x * blockDim.x) {
    long long t = idx;
    const int d = (int)(t % HD); t /= HD;
    const int qi = (int)(t % dm.Lq); t /= dm.Lq;
    const int h = (int)(t % dm.H);
    const int b = (int)(t / dm.H);
    const float* base = part + (((size_t)b * dm.H + h) * dm.splits * dm.Lq + qi) * (HD + 2);
    const size_t stride = (size_t)dm.Lq * (HD + 2);
    float M = -INFINITY;
    for (int s = 0; s < dm.splits; ++s) M = fmaxf(M, base[s * stride + HD]);
    float L = 0.f, O = 0.f;
    if (M != -INFINITY) {
      for (int s = 0; s < dm.splits; ++s) {
        const float ms = base[s * stride + HD];
        if (ms == -INFINITY) continue;
        const float e = expf(ms - M);
        L += base[s * stride + HD + 1] * e;
        O += base[s * stride + d] * e;
      }
    }
    pol.store(b, h, qi, d, L > 0.f ? O / L : 0.f);
  }
}

template <typename Policy>
static int launch_attn(const Policy& pol, AttnDims dm, int zdim, int hd, float* workspace, cudaStream_t st,
                       const char* what) {
  dim3 grid(((dm.Lq + kBQ - 1) / kBQ) * dm.splits, dm.H, zdim);
  PSALM_REQUIRE(dm.H <= 65535 && zdim <= 65535, "%s: grid too large (H=%d, z=%d)", what, dm.H, zdim);
  PSALM_REQUIRE(dm.splits == 1 || workspace != nullptr, "%s: split-K needs a workspace", what);
  if (hd == 32) {
    attn_simt_kernel<Policy, 32><<<grid, kNT, 0, st>>>(pol, dm, workspace);
    if (dm.splits > 1) attn_combine_kernel<Policy, 32><<<132 * 4, 256, 0, st>>>(pol, dm, workspace);
  } else if (hd == 64) {
    attn_simt_kernel<Policy, 64><<<grid, kNT, 0, st>>>(pol, dm, workspace);
    if (dm.splits > 1) attn_combine_kernel<Policy, 64><<<132 * 4, 256, 0, st>>>(pol, dm, workspace);
  } else {
    set_error("%s: head_dim %d unsupported (32 or 64)", what, hd);
    return PSALM_E_UNSUPPORTED;
  }
  return check_launch(what);
}

// ------------------------------------------------------------------------------------------------
// partial rotary embedding, in place on q and k of a [B,T,3,nh,hd] buffer
// (modeling_phi.py apply_rotary_pos_emb on the first `rd` dims; cos/sin [T, rd/2] fp32)
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void rotary_kernel(T* __restrict__ qkv, const float* __restrict__ cs, const float* __restrict__ sn,
                              int B, int T_, int nh, int hd, int rd) {
  const int half = rd / 2;
  const long long n = (long long)B * T_ * 2 * nh * half;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < n;
       idx += (long long)gridDim.x * blockDim.x) {
    long long t = idx;
    const int i = (int)(t % half); t /= half;
    const int h = (int)(t % nh); t /= nh;
    const int which = (int)(t % 2); t /= 2;
    const int pos = (int)(t % T_);
    const int b = (int)(t / T_);
    T* p = qkv + ((((size_t)b * T_ + pos) * 3 + which) * nh + h) * hd;
    const float c = cs[(size_t)pos * half + i], s = sn[(size_t)pos * half + i];
    const float x1 = to_f32<T>(p[i]), x2 = to_f32<T>(p[i + half]);
    p[i] = from_f32<T>(x1 * c - x2 * s);
    p[i + half] = from_f32<T>(x2 * c + x1 * s);
  }
}

// 16-byte vector form for 16-bit storage and rd / 2 a multiple of 8: one thread rotates 8 (x1, x2) pairs
// (the scalar kernel moved 2 bytes per load: 28 us per layer at 4 x 920 tokens against ~5 us of HBM time)
template <typename T>
__global__ void __launch_bounds__(256) rotary_vec_kernel(T* __restrict__ qkv, const float* __restrict__ cs,
                                                         const float* __restrict__ sn, int B, int T_, int nh, int hd, int rd) {
  const int half = rd / 2, chunks = half / 8;
  const long long n = (long long)B * T_ * 2 * nh * chunks;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
    long long t = idx;
    const int c = (int)(t % chunks); t /= chunks;
    const int h = (int)(t % nh); t /= nh;
    const int which = (int)(t % 2); t /= 2;
    const int pos = (int)(t % T_);
    const int b = (int)(t / T_);
    T* p = qkv + ((((size_t)b * T_ + pos) * 3 + which) * nh + h) * hd + c * 8;
    float x1[8], x2[8], co[8], si[8], y1[8], y2[8];
    load16_as_f32<T>(p, x1);
    load16_as_f32<T>(p + half, x2);
    const float4* c4 = reinterpret_cast<const float4*>(cs + (size_t)pos * half + c * 8);
    const float4* s4 = reinterpret_cast<const float4*>(sn + (size_t)pos * half + c * 8);
    const float4 ca = __ldg(c4), cb = __ldg(c4 + 1), sa = __ldg(s4), sb = __ldg(s4 + 1);
    co[0] = ca.x; co[1] = ca.y; co[2] = ca.z; co[3] = ca.w; co[4] = cb.x; co[5] = cb.y; co[6] = cb.z; co[7] = cb.w;
    si[0] = sa.x; si[1] = sa.y; si[2] = sa.z; si[3] = sa.w; si[4] = sb.x; si[5] = sb.y; si[6] = sb.z; si[7] = sb.w;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      y1[i] = x1[i] * co[i] - x2[i] * si[i];
      y2[i] = x2[i] * co[i] + x1[i] * si[i];
    }
    store16_from_f32<T>(p, y1);
    store16_from_f32<T>(p + half, y2);
  }
}

}  // namespace psalm

namespace psalm {
// tensor-core paths (attn_mma.cu)
int mma_causal_attention(const void*, const uint8_t*, void*, int, int, int, int, int, cudaStream_t);
int mma_cross_attention(const void*, const void*, const void*, const uint32_t*, const uint8_t*, void*, float*, int,
                        int, int, int, int, int, int, cudaStream_t, int kv_ld = 0, long long kv_bstride = -1);
int mma_prefix_causal_attention(const void*, const void*, const void*, int, int, const uint8_t*, void*, int, int, int, int,
                                int, cudaStream_t);
int mma_window_attention(const void*, const void*, const float*, void*, int, int, int, int, int, int, int,
                         cudaStream_t);
extern int g_splitk_mode;
static int g_attn_impl = 0;  // 0 = auto (tensor cores for 16-bit storage), 1 = force the fp32 SIMT kernels
}  // namespace psalm

using namespace psalm;

extern "C" int psalm_set_attention_impl(int impl) {
  PSALM_REQUIRE(impl >= 0 && impl <= 3, "set_attention_impl: 0 (auto), 1 (simt), 2 (split-K via workspace) or 3 (split-K via cluster)");
  g_attn_impl = impl == 1 ? 1 : 0;
  g_splitk_mode = impl == 2 ? 1 : (impl == 3 ? 2 : 0);
  return PSALM_OK;
}

extern "C" int psalm_set_causal_impl(int impl) {
  PSALM_REQUIRE(impl >= 0 && impl <= 2, "set_causal_impl: 0 (auto), 1 (mma.sync) or 2 (long-sequence tensor-core kernel); all "
                                        "select the mma.sync flash kernel on sm_90a");
  return PSALM_OK;
}

#define DISPATCH_T(dt, ...)                                           \
  switch (dt) {                                                       \
    case PSALM_F32: { using T = float; __VA_ARGS__; } break;          \
    case PSALM_F16: { using T = __half; __VA_ARGS__; } break;         \
    case PSALM_BF16: { using T = __nv_bfloat16; __VA_ARGS__; } break; \
    default: set_error("unknown dtype %d", dt); return PSALM_E_ARG;   \
  }

extern "C" int psalm_window_attention(const void* qkv, const void* qkv_bias, const float* rel_bias, void* out,
                                      int B, int H, int W, int C, int nh, int ws, int shift, int dtype,
                                      void* stream) {
  PSALM_REQUIRE(qkv && qkv_bias && rel_bias && out, "window_attention: null pointer");
  PSALM_REQUIRE(C % nh == 0 && ws > 0 && shift >= 0 && shift < ws, "window_attention: bad C/nh/ws/shift");
  const int hd = C / nh;
  const int Hp = (H + ws - 1) / ws * ws, Wp = (W + ws - 1) / ws * ws;
  const int nWx = Wp / ws, nW = nWx * (Hp / ws);
  if (dtype != PSALM_F32 && g_attn_impl == 0 && ws == 12 && hd == 32)
    return mma_window_attention(qkv, qkv_bias, rel_bias, out, B, H, W, C, nh, shift, dtype, (cudaStream_t)stream);
  AttnDims dm{B * nW, nh, ws * ws, ws * ws, 1, 1.0f / sqrtf((float)hd)};
  int rc = PSALM_OK;
  DISPATCH_T(dtype, {
    WindowPolicy<T> pol{(const T*)qkv, (const T*)qkv_bias, rel_bias, (T*)out, H, W, Hp, Wp, ws, shift, nh, hd, C, nWx, nW};
    rc = launch_attn(pol, dm, B * nW, hd, nullptr, (cudaStream_t)stream, "window_attention");
  });
  return rc;
}

extern "C" int psalm_causal_attention(const void* qkv, const uint8_t* key_valid, void* out, int B, int T_,
                                      int nh, int hd, int dtype, void* stream) {
  PSALM_REQUIRE(qkv && out, "causal_attention: null pointer");
  if (dtype != PSALM_F32 && g_attn_impl == 0 && (hd == 32 || hd == 64))
    return mma_causal_attention(qkv, key_valid, out, B, T_, nh, hd, dtype, (cudaStream_t)stream);
  AttnDims dm{B, nh, T_, T_, 1, 1.0f / sqrtf((float)hd)};
  int rc = PSALM_OK;
  DISPATCH_T(dtype, {
    CausalPolicy<T> pol{(const T*)qkv, key_valid, (T*)out, T_, nh, hd};
    rc = launch_attn(pol, dm, B, hd, nullptr, (cudaStream_t)stream, "causal_attention");
  });
  return rc;
}

extern "C" int psalm_prefix_causal_attention(const void* qkv, const void* prefix_k, const void* prefix_v, int P,
                                             int prefix_ld_rows, const uint8_t* key_valid, void* out, int B, int T_, int nh,
                                             int hd, int dtype, void* stream) {
  PSALM_REQUIRE(qkv && out, "prefix_causal_attention: null pointer");
  PSALM_REQUIRE(P >= 0 && prefix_ld_rows >= P && (P == 0 || (prefix_k && prefix_v)),
                "prefix_causal_attention: bad prefix (P=%d, ld_rows=%d)", P, prefix_ld_rows);
  PSALM_REQUIRE(B >= 1 && T_ >= 1 && nh >= 1 && hd % 4 == 0, "prefix_causal_attention: bad B / T / nh / hd");
  if (dtype != PSALM_F32 && g_attn_impl == 0 && (hd == 32 || hd == 64)) {
    PSALM_REQUIRE(((uintptr_t)qkv & 15) == 0 && ((uintptr_t)prefix_k & 15) == 0 && ((uintptr_t)prefix_v & 15) == 0,
                  "prefix_causal_attention: pointers must be 16-byte aligned");
    PSALM_REQUIRE((P + 63) / 64 * 64 + T_ <= 128 * 64, "prefix_causal_attention: padded prefix + T must be <= 8192 keys");
    return mma_prefix_causal_attention(qkv, prefix_k, prefix_v, P, prefix_ld_rows, key_valid, out, B, T_, nh, hd, dtype,
                                       (cudaStream_t)stream);
  }
  AttnDims dm{B, nh, T_, P + T_, 1, 1.0f / sqrtf((float)hd)};
  int rc = PSALM_OK;
  DISPATCH_T(dtype, {
    PrefixCausalPolicy<T> pol{(const T*)qkv, (const T*)prefix_k, (const T*)prefix_v, key_valid, (T*)out, T_, nh, hd, P,
                              prefix_ld_rows};
    rc = launch_attn(pol, dm, B, hd, nullptr, (cudaStream_t)stream, "prefix_causal_attention");
  });
  return rc;
}

extern "C" int psalm_rotary_inplace(void* qkv, const float* cos_t, const float* sin_t, int B, int T_, int nh,
                                    int hd, int rd, int dtype, void* stream) {
  PSALM_REQUIRE(qkv && cos_t && sin_t, "rotary: null pointer");
  PSALM_REQUIRE(rd > 0 && rd % 2 == 0 && rd <= hd, "rotary: bad rotary dim %d (head dim %d)", rd, hd);
  // the vector kernel makes 16-byte loads of qkv and cos / sin: a tensor with a storage offset takes the scalar kernel
  const bool aligned = (((uintptr_t)qkv | (uintptr_t)cos_t | (uintptr_t)sin_t) & 15) == 0;
  if (dtype != PSALM_F32 && (rd / 2) % 8 == 0 && hd % 8 == 0 && aligned) {
    const long long nv = (long long)B * T_ * 2 * nh * (rd / 16);
    const int vb = (int)((nv + 255) / 256 < 132 * 16 ? (nv + 255) / 256 : 132 * 16);
    if (dtype == PSALM_BF16) rotary_vec_kernel<__nv_bfloat16><<<vb > 0 ? vb : 1, 256, 0, (cudaStream_t)stream>>>((__nv_bfloat16*)qkv, cos_t, sin_t, B, T_, nh, hd, rd);
    else rotary_vec_kernel<__half><<<vb > 0 ? vb : 1, 256, 0, (cudaStream_t)stream>>>((__half*)qkv, cos_t, sin_t, B, T_, nh, hd, rd);
    return check_launch("rotary_vec_kernel");
  }
  const long long n = (long long)B * T_ * 2 * nh * (rd / 2);
  const int blocks = (int)((n + 255) / 256 < 132 * 16 ? (n + 255) / 256 : 132 * 16);
  DISPATCH_T(dtype, {
    rotary_kernel<T><<<blocks > 0 ? blocks : 1, 256, 0, (cudaStream_t)stream>>>((T*)qkv, cos_t, sin_t, B, T_, nh, hd, rd);
  });
  return check_launch("rotary_kernel");
}

extern "C" size_t psalm_cross_attention_workspace_bytes(int B, int nh, int hd, int Lq, int splits) {
  return splits > 1 ? (size_t)B * nh * splits * Lq * (hd + 2) * sizeof(float) : 0;
}

extern "C" int psalm_cross_attention(const void* q, const void* k, const void* v, const uint32_t* mask_bits,
                                     const uint8_t* row_open, void* out, float* workspace, int B, int Lq,
                                     int Lk, int nh, int hd, int splits, int dtype, void* stream) {
  PSALM_REQUIRE(q && k && v && out, "cross_attention: null pointer");
  PSALM_REQUIRE(splits >= 1, "cross_attention: splits must be >= 1");
  if (dtype != PSALM_F32 && g_attn_impl == 0 && (hd == 32 || hd == 64))
    return mma_cross_attention(q, k, v, mask_bits, row_open, out, workspace, B, Lq, Lk, nh, hd, splits, dtype,
                               (cudaStream_t)stream);
  AttnDims dm{B, nh, Lq, Lk, splits, 1.0f / sqrtf((float)hd)};
  int rc = PSALM_OK;
  DISPATCH_T(dtype, {
    CrossPolicy<T> pol{(const T*)q, (const T*)k, (const T*)v, mask_bits, row_open, (T*)out, Lq, Lk, nh, hd, (Lk + 31) / 32};
    rc = launch_attn(pol, dm, B, hd, workspace, (cudaStream_t)stream, "cross_attention");
  });
  return rc;
}
