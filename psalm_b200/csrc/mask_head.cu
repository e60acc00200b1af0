// Prediction-head kernels of the masked-attention decoder
// (reference transformer_decoder/mask2former_transformer_decoder.py:695-762):
//   mask_logits      outputs_mask = einsum("bqc,bchw->bqhw", mask_embed, mask_features)   (DEC:750)
//                    on a TOKEN-MAJOR feature map [B, HW, C] (C contiguous = K-major for both operands)
//   bilinear_tokens  F.interpolate(..., mode="bilinear", align_corners=False) on [B,H,W,C] maps
//                    (DEC:754 attention-mask target sizes; pixel_decoder/msdeformattn.py:306 FPN up-sampling)
//   attn_mask_bits   (sigmoid(x) < 0.5) == (x < 0), packed 1 bit / key (1 = blocked), plus the per-row
//                    "every key blocked" flag that DEC:647 turns into "attend everywhere"
// Since interpolation and the einsum are both linear, the 9 intermediate heads evaluate
//   mask_embed . bilinear(mask_features)  on the 3 pooled maps instead of 9 full-resolution einsums.
#include "common.cuh"

namespace psalm {

// ---- C[q, p] = sum_c A[q, c] * F[p, c]  (A: [B,Q,C], F: [B,P,C], out: [B,Q,P]) -------------------
// SIMT fp32 tile kernel: CTA = 32 queries x 128 pixels, K chunks of 32; thread = 2 q x 8 p.
template <typename T, typename TO>
__global__ void __launch_bounds__(256) mask_logits_kernel(const T* __restrict__ A, const T* __restrict__ F,
                                                          TO* __restrict__ out, int Q, int P, int C, long long fbs) {
  constexpr int TQ = 32, TP = 128, TK = 32;
  __shared__ float As[TK][TQ + 1];
  __shared__ float Fs[TK][TP + 1];
  const int b = blockIdx.z;
  const int q0 = blockIdx.y * TQ, p0 = blockIdx.x * TP;
  const int tid = threadIdx.x;
  const int tq = tid / 16, tp = tid % 16;  // thread computes q = tq*2 + {0,1}, p = tp + 16*j (j<8)
  float acc[2][8];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  const T* Ab = A + (size_t)b * Q * C;
  const T* Fb = F + (size_t)b * fbs;   // fbs = P * C, or 0: one feature map for every query set
  for (int k0 = 0; k0 < C; k0 += TK) {
    for (int i = tid; i < TQ * TK; i += 256) {
      const int qq = i / TK, kk = i % TK;
      As[kk][qq] = (q0 + qq < Q && k0 + kk < C) ? to_f32<T>(Ab[(size_t)(q0 + qq) * C + k0 + kk]) : 0.f;
    }
    for (int i = tid; i < TP * TK; i += 256) {
      const int pp = i / TK, kk = i % TK;
      Fs[kk][pp] = (p0 + pp < P && k0 + kk < C) ? to_f32<T>(Fb[(size_t)(p0 + pp) * C + k0 + kk]) : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int kk = 0; kk < TK; ++kk) {
      const float a0 = As[kk][tq * 2], a1 = As[kk][tq * 2 + 1];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float f = Fs[kk][tp + 16 * j];
        acc[0][j] = fmaf(a0, f, acc[0][j]);
        acc[1][j] = fmaf(a1, f, acc[1][j]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int q = q0 + tq * 2 + i;
    if (q >= Q) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int p = p0 + tp + 16 * j;
      if (p < P) out[((size_t)b * Q + q) * P + p] = from_f32<TO>(acc[i][j]);
    }
  }
}

// ---- bilinear resize of a token-major map, align_corners = False (ATen upsample_bilinear2d) ------
template <typename T, typename TO>
__global__ void bilinear_tokens_kernel(const T* __restrict__ in, TO* __restrict__ out, int B, int Hi, int Wi,
                                       int Ho, int Wo, int C, int accumulate) {
  const float sh = (float)Hi / (float)Ho, sw = (float)Wi / (float)Wo;
  const long long n = (long long)B * Ho * Wo * C;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < n;
       idx += (long long)gridDim.x * blockDim.x) {
    long long t = idx;
    const int c = (int)(t % C); t /= C;
    const int x = (int)(t % Wo); t /= Wo;
    const int y = (int)(t % Ho);
    const int b = (int)(t / Ho);
    float sy = sh * ((float)y + 0.5f) - 0.5f, sx = sw * ((float)x + 0.5f) - 0.5f;
    sy = sy < 0.f ? 0.f : sy;
    sx = sx < 0.f ? 0.f : sx;
    const int y0 = (int)sy, x0 = (int)sx;
    const int y1 = y0 + (y0 < Hi - 1 ? 1 : 0), x1 = x0 + (x0 < Wi - 1 ? 1 : 0);
    const float ly = sy - (float)y0, lx = sx - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
    const T* ib = in + (size_t)b * Hi * Wi * C + c;
    const float v = hy * (hx * to_f32<T>(ib[((size_t)y0 * Wi + x0) * C]) + lx * to_f32<T>(ib[((size_t)y0 * Wi + x1) * C])) +
                    ly * (hx * to_f32<T>(ib[((size_t)y1 * Wi + x0) * C]) + lx * to_f32<T>(ib[((size_t)y1 * Wi + x1) * C]));
    if (accumulate) out[idx] = from_f32<TO>(to_f32<TO>(out[idx]) + v);
    else out[idx] = from_f32<TO>(v);
  }
}

// same op, one thread per 16-byte channel vector of an output pixel (same-type output, C a multiple of the vector width):
// the scalar kernel above moves 2 bytes per thread per corner and ran at ~1 TB/s of input on the 256^2 x 256 mask features
template <typename T>
__global__ void __launch_bounds__(256) bilinear_tokens_vec_kernel(const T* __restrict__ in, T* __restrict__ out, int B, int Hi,
                                                                  int Wi, int Ho, int Wo, int C, int accumulate) {
  constexpr int CH = Vec16<T>::CH;
  const float sh = (float)Hi / (float)Ho, sw = (float)Wi / (float)Wo;
  const int cv = C / CH;
  const long long n = (long long)B * Ho * Wo * cv;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < n;
       idx += (long long)gridDim.x * blockDim.x) {
    long long t = idx;
    const int c = (int)(t % cv) * CH; t /= cv;
    const int x = (int)(t % Wo); t /= Wo;
    const int y = (int)(t % Ho);
    const int b = (int)(t / Ho);
    float sy = sh * ((float)y + 0.5f) - 0.5f, sx = sw * ((float)x + 0.5f) - 0.5f;
    sy = sy < 0.f ? 0.f : sy;
    sx = sx < 0.f ? 0.f : sx;
    const int y0 = (int)sy, x0 = (int)sx;
    const int y1 = y0 + (y0 < Hi - 1 ? 1 : 0), x1 = x0 + (x0 < Wi - 1 ? 1 : 0);
    const float ly = sy - (float)y0, lx = sx - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
    const T* ib = in + (size_t)b * Hi * Wi * C + c;
    float f00[CH], f01[CH], f10[CH], f11[CH], o[CH];
    load16_as_f32<T>(ib + ((size_t)y0 * Wi + x0) * C, f00);
    load16_as_f32<T>(ib + ((size_t)y0 * Wi + x1) * C, f01);
    load16_as_f32<T>(ib + ((size_t)y1 * Wi + x0) * C, f10);
    load16_as_f32<T>(ib + ((size_t)y1 * Wi + x1) * C, f11);
    T* op = out + idx * CH;
    if (accumulate) load16_as_f32<T>(op, o);
#pragma unroll
    for (int e = 0; e < CH; ++e) {   // the scalar kernel's expression
      const float v = hy * (hx * f00[e] + lx * f01[e]) + ly * (hx * f10[e] + lx * f11[e]);
      o[e] = accumulate ? o[e] + v : v;
    }
    store16_from_f32<T>(op, o);
  }
}

// ---- attention mask bits: one warp per (b, q) row ------------------------------------------------
template <typename T>
__global__ void attn_mask_bits_kernel(const T* __restrict__ logits, uint32_t* __restrict__ bits,
                                      uint8_t* __restrict__ row_open, int rows, int P, int W32) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const T* lp = logits + (size_t)warp * P;
  int all_blocked = 1;
  for (int w = 0; w < W32; ++w) {
    const int p = w * 32 + lane;
    const bool valid = p < P;
    const bool blocked = valid && (to_f32<T>(lp[p]) < 0.f);
    const uint32_t word = __ballot_sync(0xffffffffu, blocked);
    const uint32_t vmask = __ballot_sync(0xffffffffu, valid);
    if (word != vmask) all_blocked = 0;
    if (lane == 0) bits[(size_t)warp * W32 + w] = word;
  }
  if (lane == 0) row_open[warp] = (uint8_t)all_blocked;
}

}  // namespace psalm

namespace psalm {
int mma_mask_proj(const void* me, const void* feats, long long feats_bstride, void* out, uint32_t* bits, uint8_t* row_open,
                  int B, int Q, int P, int dtype, cudaStream_t st);
static int g_mask_proj_impl = 0;   // 0 auto, 1 mma.sync, 2 wgmma GEMM where it applies
}

using namespace psalm;

extern "C" int psalm_set_mask_proj_impl(int impl) {
  PSALM_REQUIRE(impl >= 0 && impl <= 2, "set_mask_proj_impl: 0 (auto), 1 (mma.sync) or 2 (wgmma where P %% 256 == 0)");
  g_mask_proj_impl = impl;
  return PSALM_OK;
}

extern "C" int psalm_mask_bits_fused(const void* mask_embed, const void* feats, uint32_t* bits, uint8_t* row_open,
                                     int B, int Q, int P, int C, int dtype, void* stream) {
  return psalm_mask_bits_fused_strided(mask_embed, feats, (long long)P * C, bits, row_open, B, Q, P, C, dtype, stream);
}

extern "C" int psalm_mask_bits_fused_strided(const void* mask_embed, const void* feats, long long feats_batch_stride,
                                             uint32_t* bits, uint8_t* row_open, int B, int Q, int P, int C, int dtype,
                                             void* stream) {
  PSALM_REQUIRE(mask_embed && feats && bits && row_open, "mask_bits_fused: null pointer");
  PSALM_REQUIRE(feats_batch_stride >= 0 && feats_batch_stride % 8 == 0,
                "mask_bits_fused: feature batch stride %lld must be >= 0 and a multiple of 8", feats_batch_stride);
  if (dtype == PSALM_F32 || C != 256 || Q > 112) {
    set_error("mask_bits_fused: needs 16-bit storage, C == 256, Q <= 112 (got dtype %d, C %d, Q %d)", dtype, C, Q);
    return PSALM_E_UNSUPPORTED;
  }
  return mma_mask_proj(mask_embed, feats, feats_batch_stride, nullptr, bits, row_open, B, Q, P, dtype, (cudaStream_t)stream);
}

extern "C" int psalm_mask_logits(const void* mask_embed, const void* feats, void* out, int B, int Q, int P,
                                 int C, int dtype, int out_dtype, void* stream) {
  return psalm_mask_logits_strided(mask_embed, feats, (long long)P * C, out, B, Q, P, C, dtype, out_dtype, stream);
}

extern "C" int psalm_mask_logits_strided(const void* mask_embed, const void* feats, long long feats_batch_stride, void* out,
                                         int B, int Q, int P, int C, int dtype, int out_dtype, void* stream) {
  PSALM_REQUIRE(mask_embed && feats && out, "mask_logits: null pointer");
  PSALM_REQUIRE(out_dtype == dtype || out_dtype == PSALM_F32, "mask_logits: out dtype must be F32 or the input dtype");
  PSALM_REQUIRE(feats_batch_stride >= 0, "mask_logits: negative feature batch stride %lld", feats_batch_stride);
  // large maps: wgmma GEMMs out[b] = mask_embed[b] (Q x C, TMA zero-fills rows Q..127 of the tile) · feats[b]ᵀ (P x C),
  // both operands K-major as stored (csrc/gemm_wgmma.cu): one per image, or ONE with M = B * Q rows when every query set
  // reads the same feature map (stride 0: mask_embed [B, Q, C] is already [B * Q, C], out [B, Q, P] is [B * Q, P])
  if (dtype != PSALM_F32 && out_dtype == dtype && C == 256 && Q <= 128 && P % 256 == 0 &&
      (g_mask_proj_impl == 2 || (g_mask_proj_impl == 0 && P >= 8192))) {
    if (feats_batch_stride == 0)
      return psalm_linear_fused(mask_embed, C, feats, nullptr, out, (long long)B * Q, P, C, 0, 0, dtype, stream);
    const size_t es = dtype_size(dtype);
    for (int b = 0; b < B; ++b) {
      const int rc = psalm_linear_fused((const char*)mask_embed + (size_t)b * Q * C * es, C,
                                        (const char*)feats + (size_t)b * feats_batch_stride * es, nullptr,
                                        (char*)out + (size_t)b * Q * P * es, Q, P, C, 0, 0, dtype, stream);
      if (rc != PSALM_OK) return rc;
    }
    return PSALM_OK;
  }
  if (dtype != PSALM_F32 && out_dtype == dtype && C == 256 && Q <= 112 && P % 2 == 0 && feats_batch_stride % 8 == 0)
    return mma_mask_proj(mask_embed, feats, feats_batch_stride, out, nullptr, nullptr, B, Q, P, dtype, (cudaStream_t)stream);
  dim3 grid((P + 127) / 128, (Q + 31) / 32, B);
  cudaStream_t st = (cudaStream_t)stream;
#define ML(T, TO) mask_logits_kernel<T, TO><<<grid, 256, 0, st>>>((const T*)mask_embed, (const T*)feats, (TO*)out, Q, P, C, feats_batch_stride)
  if (dtype == PSALM_F32) ML(float, float);
  else if (dtype == PSALM_F16) { if (out_dtype == PSALM_F32) ML(__half, float); else ML(__half, __half); }
  else if (dtype == PSALM_BF16) { if (out_dtype == PSALM_F32) ML(__nv_bfloat16, float); else ML(__nv_bfloat16, __nv_bfloat16); }
  else { set_error("mask_logits: unknown dtype %d", dtype); return PSALM_E_ARG; }
#undef ML
  return check_launch("mask_logits_kernel");
}

extern "C" int psalm_bilinear_tokens(const void* in, void* out, int B, int Hi, int Wi, int Ho, int Wo, int C,
                                     int dtype, int out_dtype, int accumulate, void* stream) {
  PSALM_REQUIRE(in && out, "bilinear_tokens: null pointer");
  PSALM_REQUIRE(out_dtype == dtype || out_dtype == PSALM_F32, "bilinear_tokens: out dtype must be F32 or the input dtype");
  const long long n = (long long)B * Ho * Wo * C;
  const int blocks = (int)((n + 255) / 256 < 132 * 32 ? (n + 255) / 256 : 132 * 32);
  cudaStream_t st = (cudaStream_t)stream;
  if (out_dtype == dtype && C % (dtype == PSALM_F32 ? 4 : 8) == 0 && (reinterpret_cast<uintptr_t>(in) & 15) == 0 &&
      (reinterpret_cast<uintptr_t>(out) & 15) == 0) {
    const long long nv = n / (dtype == PSALM_F32 ? 4 : 8);
    const int vb = (int)((nv + 255) / 256 < 132 * 16 ? (nv + 255) / 256 : 132 * 16);
#define BLV(T) bilinear_tokens_vec_kernel<T><<<vb > 0 ? vb : 1, 256, 0, st>>>((const T*)in, (T*)out, B, Hi, Wi, Ho, Wo, C, accumulate)
    if (dtype == PSALM_F32) BLV(float);
    else if (dtype == PSALM_F16) BLV(__half);
    else if (dtype == PSALM_BF16) BLV(__nv_bfloat16);
    else { set_error("bilinear_tokens: unknown dtype %d", dtype); return PSALM_E_ARG; }
#undef BLV
    return check_launch("bilinear_tokens_vec_kernel");
  }
#define BL(T, TO) bilinear_tokens_kernel<T, TO><<<blocks > 0 ? blocks : 1, 256, 0, st>>>((const T*)in, (TO*)out, B, Hi, Wi, Ho, Wo, C, accumulate)
  if (dtype == PSALM_F32) BL(float, float);
  else if (dtype == PSALM_F16) { if (out_dtype == PSALM_F32) BL(__half, float); else BL(__half, __half); }
  else if (dtype == PSALM_BF16) { if (out_dtype == PSALM_F32) BL(__nv_bfloat16, float); else BL(__nv_bfloat16, __nv_bfloat16); }
  else { set_error("bilinear_tokens: unknown dtype %d", dtype); return PSALM_E_ARG; }
#undef BL
  return check_launch("bilinear_tokens_kernel");
}

extern "C" int psalm_attn_mask_bits(const void* logits, uint32_t* bits, uint8_t* row_open, int rows, int P,
                                    int dtype, void* stream) {
  PSALM_REQUIRE(logits && bits && row_open, "attn_mask_bits: null pointer");
  const int W32 = (P + 31) / 32;
  const int blocks = (rows * 32 + 255) / 256;
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == PSALM_F32) attn_mask_bits_kernel<float><<<blocks, 256, 0, st>>>((const float*)logits, bits, row_open, rows, P, W32);
  else if (dtype == PSALM_F16) attn_mask_bits_kernel<__half><<<blocks, 256, 0, st>>>((const __half*)logits, bits, row_open, rows, P, W32);
  else if (dtype == PSALM_BF16) attn_mask_bits_kernel<__nv_bfloat16><<<blocks, 256, 0, st>>>((const __nv_bfloat16*)logits, bits, row_open, rows, P, W32);
  else { set_error("attn_mask_bits: unknown dtype %d", dtype); return PSALM_E_ARG; }
  return check_launch("attn_mask_bits_kernel");
}
