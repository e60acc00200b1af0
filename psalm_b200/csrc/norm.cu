// Normalisation kernels of the hot path (HBM-bound streaming work, fp32 statistics):
//   add_layernorm   s = x (+ r1) (+ r2);  y = LayerNorm(s) * w + b;  optionally also writes s.
//                   Replaces the residual `add` + nn.LayerNorm pairs of SwinTransformerBlock
//                   (swin_trans.py:207,247-251), PhiDecoderLayer (attn + mlp + residual, then the next
//                   input_layernorm), the encoder / decoder post-norm layers (msdeformattn.py:59-65,
//                   mask2former_transformer_decoder.py:42-43,102-103,160-161).  One warp per row,
//                   the row lives in registers (two-pass mean / variance like ATen), 16-byte accesses.
//   groupnorm_tokens  GroupNorm(32) on a TOKEN-MAJOR map [B, N, C] (+ optional ReLU): deterministic
//                   per-CTA partial sums -> fixed-order finalize (double) -> streaming apply pass (msdeformattn.py:199-203,244-252 conv+GN(+ReLU) blocks).
#include "common.cuh"

namespace psalm {

template <typename T>
__device__ __forceinline__ void load4(const T* p, float (&f)[4]) {
  if constexpr (sizeof(T) == 4) {
    const float4 v = *reinterpret_cast<const float4*>(p);
    f[0] = v.x; f[1] = v.y; f[2] = v.z; f[3] = v.w;
  } else {
    const uint2 v = *reinterpret_cast<const uint2*>(p);
    unpack2<T>(v.x, f[0], f[1]);
    unpack2<T>(v.y, f[2], f[3]);
  }
}
template <typename T>
__device__ __forceinline__ void store4(T* p, const float (&f)[4]) {
  if constexpr (sizeof(T) == 4) {
    *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
  } else {
    uint2 v;
    v.x = pack2<T>(f[0], f[1]);
    v.y = pack2<T>(f[2], f[3]);
    *reinterpret_cast<uint2*>(p) = v;
  }
}

// CPL = 4-element chunks per lane; C = 128 * CPL
template <typename T, int CPL>
__global__ void __launch_bounds__(128) add_layernorm_kernel(const T* __restrict__ x, const T* __restrict__ r1,
                                                            const T* __restrict__ r2, const T* __restrict__ w,
                                                            const T* __restrict__ b, T* __restrict__ sum_out,
                                                            T* __restrict__ y, long long rows, float eps) {
  constexpr int C = 128 * CPL;
  const long long row = (long long)blockIdx.x * 4 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const size_t base = (size_t)row * C;
  float v[CPL][4];
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < CPL; ++c) {
    const int off = (c * 32 + lane) * 4;
    load4<T>(x + base + off, v[c]);
    if (r1) {
      float t[4];
      load4<T>(r1 + base + off, t);
#pragma unroll
      for (int i = 0; i < 4; ++i) v[c][i] += t[i];
    }
    if (r2) {
      float t[4];
      load4<T>(r2 + base + off, t);
#pragma unroll
      for (int i = 0; i < 4; ++i) v[c][i] += t[i];
    }
    if (sum_out) {
      // the residual stream is stored in T: normalise what the next consumer will actually read
      store4<T>(sum_out + base + off, v[c]);
      if constexpr (sizeof(T) == 2) {
#pragma unroll
        for (int i = 0; i < 4; ++i) v[c][i] = to_f32<T>(from_f32<T>(v[c][i]));
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) s += v[c][i];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s * (1.f / C);
  float q = 0.f;
#pragma unroll
  for (int c = 0; c < CPL; ++c)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float d = v[c][i] - mean;
      q = fmaf(d, d, q);
    }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q * (1.f / C) + eps);
#pragma unroll
  for (int c = 0; c < CPL; ++c) {
    const int off = (c * 32 + lane) * 4;
    float g[4], bb[4], o4[4];
    load4<T>(w + off, g);
    load4<T>(b + off, bb);
#pragma unroll
    for (int i = 0; i < 4; ++i) o4[i] = (v[c][i] - mean) * rstd * g[i] + bb[i];
    store4<T>(y + base + off, o4);
  }
}

// ---- PatchMerging gather + LayerNorm (swin_trans.py:269-296) -----------------------------------------
// y[b, i, j, :] = LN(cat(x[b, 2i, 2j], x[b, 2i+1, 2j], x[b, 2i, 2j+1], x[b, 2i+1, 2j+1])) over 4C channels, pixels beyond
// an odd H / W are zeros (F.pad before the slicing) and take part in the statistics.  Replaces the four strided slices +
// torch.cat (a 4C-wide copy of the map) in front of the norm.  CPL = 4-element chunks per lane over the 4C row.
template <typename T, int CPL>
__global__ void __launch_bounds__(128) patch_merge_layernorm_kernel(const T* __restrict__ x, const T* __restrict__ w,
                                                                    const T* __restrict__ b, T* __restrict__ y, int B, int H,
                                                                    int W, float eps) {
  constexpr int C4 = 128 * CPL, C = C4 / 4;
  const int H2 = (H + 1) / 2, W2 = (W + 1) / 2;
  const long long rows = (long long)B * H2 * W2;
  const long long row = (long long)blockIdx.x * 4 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int j = (int)(row % W2), i = (int)((row / W2) % H2), bi = (int)(row / ((long long)W2 * H2));
  float v[CPL][4];
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < CPL; ++c) {
    const int off = (c * 32 + lane) * 4;
    const int q = off / C, cc = off - q * C;
    const int yy = 2 * i + (q & 1), xx = 2 * j + (q >> 1);
    if (yy < H && xx < W) load4<T>(x + (((size_t)bi * H + yy) * W + xx) * C + cc, v[c]);
    else v[c][0] = v[c][1] = v[c][2] = v[c][3] = 0.f;
#pragma unroll
    for (int e = 0; e < 4; ++e) s += v[c][e];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s * (1.f / C4);
  float qd = 0.f;
#pragma unroll
  for (int c = 0; c < CPL; ++c)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float d = v[c][e] - mean;
      qd = fmaf(d, d, qd);
    }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) qd += __shfl_xor_sync(0xffffffffu, qd, o);
  const float rstd = rsqrtf(qd * (1.f / C4) + eps);
#pragma unroll
  for (int c = 0; c < CPL; ++c) {
    const int off = (c * 32 + lane) * 4;
    float g[4], bb[4], o4[4];
    load4<T>(w + off, g);
    load4<T>(b + off, bb);
#pragma unroll
    for (int e = 0; e < 4; ++e) o4[e] = (v[c][e] - mean) * rstd * g[e] + bb[e];
    store4<T>(y + (size_t)row * C4 + off, o4);
  }
}

template <typename T>
static int launch_pm(const void* x, const void* w, const void* b, void* y, int B, int H, int W, int C, float eps, cudaStream_t st) {
  const long long rows = (long long)B * ((H + 1) / 2) * ((W + 1) / 2);
  const unsigned grid = (unsigned)((rows + 3) / 4);
#define PM(CPL) patch_merge_layernorm_kernel<T, CPL><<<grid, 128, 0, st>>>((const T*)x, (const T*)w, (const T*)b, (T*)y, B, H, W, eps)
  switch (C) {
    case 128: PM(4); break;
    case 256: PM(8); break;
    case 512: PM(16); break;
    default: set_error("patch_merge_layernorm: C=%d unsupported (128/256/512)", C); return PSALM_E_UNSUPPORTED;
  }
#undef PM
  return check_launch("patch_merge_layernorm_kernel");
}

// ---- GroupNorm on token-major maps -----------------------------------------------------------------
// Deterministic (no atomics): (1) per-CTA partial (sum, sumsq) per group over a slice of 256 tokens,
// reduced inside the CTA in a fixed order; (2) a finalize kernel adds the partials of each (batch, group)
// in a fixed order in double and emits (mean, rstd); (3) streaming apply.
// C <= 1024, C % (4*groups) == 0, 256 % (C/4) == 0.
template <typename T>
__global__ void __launch_bounds__(256) groupnorm_partial_kernel(const T* __restrict__ x, const T* __restrict__ pre_bias,
                                                                float2* __restrict__ part,
                                                                int N, int C, int groups, int tokens_per_cta) {
  __shared__ float ts[256], tq[256];
  const int b = blockIdx.y;
  const int t0 = blockIdx.x * tokens_per_cta;
  const int t1 = min(N, t0 + tokens_per_cta);
  const int cpg = C / groups;
  const int chunks = C / 4;                    // 4-element chunks per token
  const int tpb = 256 / chunks;                // tokens processed concurrently
  const int cidx = threadIdx.x % chunks, trow = threadIdx.x / chunks;
  float s = 0.f, q = 0.f;
  if (trow < tpb) {
    float pb[4] = {0.f, 0.f, 0.f, 0.f};        // per-channel bias of the producing conv / linear, folded in here
    if (pre_bias) load4<T>(pre_bias + cidx * 4, pb);
    for (int t = t0 + trow; t < t1; t += tpb) {
      float f[4];
      load4<T>(x + ((size_t)b * N + t) * C + cidx * 4, f);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        f[i] += pb[i];
        s += f[i];
        q = fmaf(f[i], f[i], q);
      }
    }
  }
  ts[threadIdx.x] = s;
  tq[threadIdx.x] = q;
  __syncthreads();
  if (threadIdx.x < groups) {
    const int g = threadIdx.x;
    const int cpgc = cpg / 4;                  // chunks per group
    float gs = 0.f, gq = 0.f;
    for (int r = 0; r < tpb; ++r)
      for (int c = 0; c < cpgc; ++c) {
        const int t = r * chunks + g * cpgc + c;
        gs += ts[t];
        gq += tq[t];
      }
    part[((size_t)b * groups + g) * gridDim.x + blockIdx.x] = make_float2(gs, gq);
  }
}

__global__ void groupnorm_finalize_kernel(const float2* __restrict__ part, float2* __restrict__ mean_rstd, int n_bg,
                                          int n_part, double count, float eps) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_bg) return;
  double s = 0.0, q = 0.0;
  for (int k = 0; k < n_part; ++k) {
    const float2 v = part[(size_t)i * n_part + k];
    s += (double)v.x;
    q += (double)v.y;
  }
  const double m = s / count;
  double var = q / count - m * m;
  if (var < 0) var = 0;
  mean_rstd[i] = make_float2((float)m, rsqrtf((float)var + eps));
}

template <typename T>
__global__ void groupnorm_apply_kernel(const T* __restrict__ x, const T* __restrict__ pre_bias,
                                       const float2* __restrict__ mean_rstd,
                                       const T* __restrict__ w, const T* __restrict__ bias, T* __restrict__ y,
                                       int B, int N, int C, int groups, int relu) {
  const int cpg = C / groups;
  const long long n4 = (long long)B * N * C / 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const long long e = i * 4;
    const int c = (int)(e % C);
    const int b = (int)(e / ((long long)N * C));
    const float2 mr = mean_rstd[(size_t)b * groups + c / cpg];
    float f[4], gw[4], gb[4], o[4], pb[4] = {0.f, 0.f, 0.f, 0.f};
    load4<T>(x + e, f);
    load4<T>(w + c, gw);
    load4<T>(bias + c, gb);
    if (pre_bias) load4<T>(pre_bias + c, pb);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      o[k] = (f[k] + pb[k] - mr.x) * mr.y * gw[k] + gb[k];
      if (relu) o[k] = fmaxf(o[k], 0.f);
    }
    store4<T>(y + e, o);
  }
}

template <typename T>
static int launch_ln(const void* x, const void* r1, const void* r2, const void* w, const void* b, void* sum_out,
                     void* y, long long rows, int C, float eps, cudaStream_t st) {
  const unsigned grid = (unsigned)((rows + 3) / 4);
#define LN(CPL)                                                                                               \
  add_layernorm_kernel<T, CPL><<<grid, 128, 0, st>>>((const T*)x, (const T*)r1, (const T*)r2, (const T*)w,     \
                                                     (const T*)b, (T*)sum_out, (T*)y, rows, eps)
  switch (C) {
    case 128: LN(1); break;
    case 256: LN(2); break;
    case 512: LN(4); break;
    case 1024: LN(8); break;
    case 2048: LN(16); break;
    default: set_error("add_layernorm: C=%d unsupported (128/256/512/1024/2048)", C); return PSALM_E_UNSUPPORTED;
  }
#undef LN
  return check_launch("add_layernorm_kernel");
}

template <typename T>
static int launch_gn(const void* x, const void* pre_bias, const void* w, const void* b, void* y, double* workspace, int B, int N, int C,
                     int groups, float eps, int relu, cudaStream_t st) {
  const int tokens_per_cta = 256;
  const int n_part = (N + tokens_per_cta - 1) / tokens_per_cta;
  float2* mean_rstd = reinterpret_cast<float2*>(workspace);                    // [B*groups]
  float2* part = mean_rstd + (size_t)B * groups;                               // [B*groups][n_part]
  dim3 g1(n_part, B);
  groupnorm_partial_kernel<T><<<g1, 256, 0, st>>>((const T*)x, (const T*)pre_bias, part, N, C, groups, tokens_per_cta);
  const int n_bg = B * groups;
  groupnorm_finalize_kernel<<<(n_bg + 127) / 128, 128, 0, st>>>(part, mean_rstd, n_bg, n_part,
                                                              (double)N * (C / groups), eps);
  const long long n4 = (long long)B * N * C / 4;
  const int blocks = (int)((n4 + 255) / 256 < 132 * 16 ? (n4 + 255) / 256 : 132 * 16);
  groupnorm_apply_kernel<T><<<blocks > 0 ? blocks : 1, 256, 0, st>>>((const T*)x, (const T*)pre_bias, mean_rstd, (const T*)w, (const T*)b,
                                                                     (T*)y, B, N, C, groups, relu);
  return check_launch("groupnorm_tokens");
}

}  // namespace psalm

using namespace psalm;

extern "C" int psalm_add_layernorm(const void* x, const void* r1, const void* r2, const void* weight,
                                   const void* bias, void* sum_out, void* y, long long rows, int C, float eps,
                                   int dtype, void* stream) {
  PSALM_REQUIRE(x && weight && bias && y, "add_layernorm: null pointer");
  PSALM_REQUIRE(rows > 0 && rows < (1ll << 33), "add_layernorm: bad row count");
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case PSALM_F32: return launch_ln<float>(x, r1, r2, weight, bias, sum_out, y, rows, C, eps, st);
    case PSALM_F16: return launch_ln<__half>(x, r1, r2, weight, bias, sum_out, y, rows, C, eps, st);
    case PSALM_BF16: return launch_ln<__nv_bfloat16>(x, r1, r2, weight, bias, sum_out, y, rows, C, eps, st);
  }
  set_error("add_layernorm: unknown dtype %d", dtype);
  return PSALM_E_ARG;
}

extern "C" int psalm_groupnorm_tokens(const void* x, const void* pre_bias, const void* weight, const void* bias, void* y,
                                      double* stats_workspace, int B, int N, int C, int groups, float eps,
                                      int relu, int dtype, void* stream) {
  PSALM_REQUIRE(x && weight && bias && y && stats_workspace, "groupnorm_tokens: null pointer");
  PSALM_REQUIRE(groups > 0 && groups <= 64 && C % (4 * groups) == 0 && C <= 1024 && 256 % (C / 4) == 0,
                "groupnorm_tokens: unsupported C=%d groups=%d", C, groups);
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case PSALM_F32: return launch_gn<float>(x, pre_bias, weight, bias, y, stats_workspace, B, N, C, groups, eps, relu, st);
    case PSALM_F16: return launch_gn<__half>(x, pre_bias, weight, bias, y, stats_workspace, B, N, C, groups, eps, relu, st);
    case PSALM_BF16: return launch_gn<__nv_bfloat16>(x, pre_bias, weight, bias, y, stats_workspace, B, N, C, groups, eps, relu, st);
  }
  set_error("groupnorm_tokens: unknown dtype %d", dtype);
  return PSALM_E_ARG;
}

extern "C" int psalm_patch_merge_layernorm(const void* x, const void* weight, const void* bias, void* y, int B, int H, int W,
                                           int C, float eps, int dtype, void* stream) {
  PSALM_REQUIRE(x && weight && bias && y, "patch_merge_layernorm: null pointer");
  PSALM_REQUIRE(B > 0 && H > 0 && W > 0, "patch_merge_layernorm: bad shape");
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case PSALM_F32: return launch_pm<float>(x, weight, bias, y, B, H, W, C, eps, st);
    case PSALM_F16: return launch_pm<__half>(x, weight, bias, y, B, H, W, C, eps, st);
    case PSALM_BF16: return launch_pm<__nv_bfloat16>(x, weight, bias, y, B, H, W, C, eps, st);
  }
  set_error("patch_merge_layernorm: unknown dtype %d", dtype);
  return PSALM_E_ARG;
}
