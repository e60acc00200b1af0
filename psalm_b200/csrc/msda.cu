// Multi-scale deformable attention forward for sm_90a.
//
// Replaces ms_deformable_im2col_gpu_kernel (reference ops/src/cuda/ms_deform_im2col_cuda.cuh:243-304,
// one thread per output scalar, scalar loads, queries walked in linear order).  Design here:
//   * a (query, head) pair is owned by a group of G = D / (16 B / sizeof(T)) lanes; every corner
//     fetch is one 16-byte load per lane, i.e. one fully used 64/128-byte segment per group;
//   * a CTA owns ONE head and a 2-D PATCH of spatially adjacent queries of one level (encoder
//     self-attention: Lq == S), so the four bilinear corners of neighbouring queries hit the same
//     L1 lines; halo re-fetch comes out of L2 (value is 11-22 MB, L2 is 126 MB), never HBM;
//   * fp32 accumulation regardless of the storage type; zero padding by predication;
//   * the fused variant derives sampling locations and softmax weights in-kernel from the raw
//     Linear outputs, so `sampling_locations` / `attention_weights` never touch HBM.
#include "common.cuh"

namespace psalm {

constexpr int kMaxLevels = 8;
constexpr int kThreads = 256;

struct MsdaLevels {
  int H[kMaxLevels];
  int W[kMaxLevels];
  int start[kMaxLevels];
  int tile0[kMaxLevels + 1];  // first tile index of each level (patch mapping)
  int tiles_x[kMaxLevels];
  int L;
};

// -------------------------------------------------------------------------------------------
// one bilinear sample: acc += aw * bilinear(value, (x, y)); pointer arithmetic in elements.
// vbase points at (level origin, head, channel-lane); pix_stride = elements between pixels.
// -------------------------------------------------------------------------------------------
template <typename TV>
__device__ __forceinline__ void sample_accumulate(const TV* __restrict__ vbase, int H, int W,
                                                  int pix_stride, float x, float y, float aw,
                                                  float (&acc)[16 / sizeof(TV)]) {
  constexpr int CH = 16 / sizeof(TV);
  if (!(y > -1.f && x > -1.f && y < (float)H && x < (float)W)) return;
  const float yf = floorf(y), xf = floorf(x);
  const int y0 = (int)yf, x0 = (int)xf;
  const float ly = y - yf, lx = x - xf;
  const float hy = 1.f - ly, hx = 1.f - lx;
  const bool y0ok = y0 >= 0, y1ok = y0 + 1 <= H - 1;
  const bool x0ok = x0 >= 0, x1ok = x0 + 1 <= W - 1;
  const TV* p00 = vbase + ((long long)y0 * W + x0) * pix_stride;
  const TV* p10 = p00 + (long long)W * pix_stride;
  float f[CH];
  if (y0ok && x0ok) {
    load16_as_f32<TV>(p00, f);
    const float c = hy * hx * aw;
#pragma unroll
    for (int i = 0; i < CH; ++i) acc[i] = fmaf(c, f[i], acc[i]);
  }
  if (y0ok && x1ok) {
    load16_as_f32<TV>(p00 + pix_stride, f);
    const float c = hy * lx * aw;
#pragma unroll
    for (int i = 0; i < CH; ++i) acc[i] = fmaf(c, f[i], acc[i]);
  }
  if (y1ok && x0ok) {
    load16_as_f32<TV>(p10, f);
    const float c = ly * hx * aw;
#pragma unroll
    for (int i = 0; i < CH; ++i) acc[i] = fmaf(c, f[i], acc[i]);
  }
  if (y1ok && x1ok) {
    load16_as_f32<TV>(p10 + pix_stride, f);
    const float c = ly * lx * aw;
#pragma unroll
    for (int i = 0; i < CH; ++i) acc[i] = fmaf(c, f[i], acc[i]);
  }
}

// Resolve the query owned by group `g` of this CTA.  PATCH mapping: blockIdx.x enumerates 2-D
// tiles (TW x TH queries) level by level; linear mapping: NG consecutive queries.
template <int NG>
__device__ __forceinline__ bool resolve_query(const MsdaLevels& lv, bool patch, int g, int Lq,
                                              int& q, int& ql, int& qy, int& qx) {
  constexpr int TW = 8, TH = NG / 8;
  if (patch) {
    const int t = blockIdx.x;
    int l = 0;
#pragma unroll 1
    while (l + 1 < lv.L && t >= lv.tile0[l + 1]) ++l;
    const int tl = t - lv.tile0[l];
    const int ty = tl / lv.tiles_x[l], tx = tl - ty * lv.tiles_x[l];
    qy = ty * TH + g / TW;
    qx = tx * TW + g % TW;
    ql = l;
    q = lv.start[l] + qy * lv.W[l] + qx;
    return qy < lv.H[l] && qx < lv.W[l];
  }
  q = blockIdx.x * NG + g;
  ql = qy = qx = 0;
  return q < Lq;
}

// -------------------------------------------------------------------------------------------
// Vector kernel, op-boundary contract (loc / w tensors in memory).
//   grid = (tiles or ceil(Lq/NG), M, B), block = 256.
// -------------------------------------------------------------------------------------------
template <typename TV, typename TL, int G, int LT, int PT>
__global__ void __launch_bounds__(kThreads)
msda_vec_kernel(const TV* __restrict__ value, const TL* __restrict__ loc, const TL* __restrict__ w,
                TV* __restrict__ out, const int64_t* __restrict__ shapes_dev,
                const int64_t* __restrict__ starts_dev, MsdaLevels lv, int S, int M, int D,
                int rtL, int Lq, int rtP, int pix_stride, long long head_stride,
                long long batch_stride, int patch) {
  constexpr int CH = 16 / sizeof(TV);
  constexpr int NG = kThreads / G;
  const int L = LT ? LT : rtL;
  const int P = PT ? PT : rtP;
  const int g = threadIdx.x / G, cl = threadIdx.x % G;
  const int m = blockIdx.y, b = blockIdx.z;
  int q, ql, qy, qx;
  if (!resolve_query<NG>(lv, patch != 0, g, Lq, q, ql, qy, qx)) return;

  const size_t qm = ((size_t)b * Lq + q) * M + m;
  const TL* __restrict__ locp = loc + qm * (size_t)(L * P * 2);
  const TL* __restrict__ wp = w + qm * (size_t)(L * P);
  const TV* __restrict__ vb = value + (size_t)b * batch_stride + (size_t)m * head_stride + cl * CH;

  float acc[CH];
#pragma unroll
  for (int i = 0; i < CH; ++i) acc[i] = 0.f;

  // sampling locations / weights of this (query, head): 16-byte loads, every lane of the group
  // reads the same addresses (broadcast), 9 requests instead of 24 for (L,P) = (3,4)
  constexpr int LPT = LT * PT;
  constexpr bool kPreload = (LPT > 0) && (LPT % 4 == 0) && (sizeof(TL) == 4);
  float plx[kPreload ? LPT : 1], ply[kPreload ? LPT : 1], paw[kPreload ? LPT : 1];
  if constexpr (kPreload) {
    const float4* l4 = reinterpret_cast<const float4*>(locp);
    const float4* w4 = reinterpret_cast<const float4*>(wp);
#pragma unroll
    for (int i = 0; i < LPT / 2; ++i) {
      const float4 v = __ldg(l4 + i);
      plx[2 * i] = v.x; ply[2 * i] = v.y; plx[2 * i + 1] = v.z; ply[2 * i + 1] = v.w;
    }
#pragma unroll
    for (int i = 0; i < LPT / 4; ++i) {
      const float4 v = __ldg(w4 + i);
      paw[4 * i] = v.x; paw[4 * i + 1] = v.y; paw[4 * i + 2] = v.z; paw[4 * i + 3] = v.w;
    }
  }

#pragma unroll
  for (int l = 0; l < (LT ? LT : kMaxLevels); ++l) {
    if (!LT && l >= L) break;
    int H, W, st;
    if (shapes_dev) {
      H = (int)shapes_dev[2 * l];
      W = (int)shapes_dev[2 * l + 1];
      st = (int)starts_dev[l];
    } else {
      H = lv.H[l];
      W = lv.W[l];
      st = lv.start[l];
    }
    const TV* __restrict__ vl = vb + (size_t)st * pix_stride;
#pragma unroll
    for (int p = 0; p < (PT ? PT : 32); ++p) {
      if (!PT && p >= P) break;
      const int s = l * P + p;
      float lx, ly, aw;
      if constexpr (kPreload) {
        lx = plx[s]; ly = ply[s]; aw = paw[s];
      } else if constexpr (sizeof(TL) == 4) {
        const float2 xy = __ldg(reinterpret_cast<const float2*>(locp) + s);
        lx = xy.x;
        ly = xy.y;
        aw = __ldg(reinterpret_cast<const float*>(wp) + s);
      } else {
        lx = to_f32<TL>(locp[2 * s]);
        ly = to_f32<TL>(locp[2 * s + 1]);
        aw = to_f32<TL>(wp[s]);
      }
      sample_accumulate<TV>(vl, H, W, pix_stride, lx * (float)W - 0.5f, ly * (float)H - 0.5f, aw, acc);
    }
  }
  store16_from_f32<TV>(out + qm * (size_t)D + cl * CH, acc);
}

// -------------------------------------------------------------------------------------------
// Scalar kernel: any D / alignment (e.g. the reference's own test shapes D = 2).
// One thread per output scalar, like the reference, but with fp32 math for 16-bit types.
// -------------------------------------------------------------------------------------------
template <typename TV, typename TL>
__global__ void msda_scalar_kernel(const TV* __restrict__ value, const TL* __restrict__ loc,
                                   const TL* __restrict__ w, TV* __restrict__ out,
                                   const int64_t* __restrict__ shapes_dev,
                                   const int64_t* __restrict__ starts_dev, MsdaLevels lv, long long n,
                                   int S, int M, int D, int L, int Lq, int P, int pix_stride,
                                   long long head_stride, long long batch_stride) {
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < n;
       idx += (long long)gridDim.x * blockDim.x) {
    long long t = idx;
    const int c = (int)(t % D); t /= D;
    const int m = (int)(t % M); t /= M;
    const int q = (int)(t % Lq); t /= Lq;
    const int b = (int)t;
    const size_t qm = ((size_t)b * Lq + q) * M + m;
    const TL* locp = loc + qm * (size_t)(L * P * 2);
    const TL* wp = w + qm * (size_t)(L * P);
    const TV* vb = value + (size_t)b * batch_stride + (size_t)m * head_stride + c;
    float acc = 0.f;
    for (int l = 0; l < L; ++l) {
      int H, W, st;
      if (shapes_dev) {
        H = (int)shapes_dev[2 * l]; W = (int)shapes_dev[2 * l + 1]; st = (int)starts_dev[l];
      } else {
        H = lv.H[l]; W = lv.W[l]; st = lv.start[l];
      }
      const TV* vl = vb + (size_t)st * pix_stride;
      for (int p = 0; p < P; ++p) {
        const int s = l * P + p;
        const float x = to_f32<TL>(locp[2 * s]) * (float)W - 0.5f;
        const float y = to_f32<TL>(locp[2 * s + 1]) * (float)H - 0.5f;
        const float aw = to_f32<TL>(wp[s]);
        if (!(y > -1.f && x > -1.f && y < (float)H && x < (float)W)) continue;
        const float yf = floorf(y), xf = floorf(x);
        const int y0 = (int)yf, x0 = (int)xf;
        const float ly = y - yf, lx = x - xf, hy = 1.f - ly, hx = 1.f - lx;
        const TV* p00 = vl + ((long long)y0 * W + x0) * pix_stride;
        const TV* p10 = p00 + (long long)W * pix_stride;
        float v = 0.f;
        if (y0 >= 0 && x0 >= 0) v += hy * hx * to_f32<TV>(*p00);
        if (y0 >= 0 && x0 + 1 <= W - 1) v += hy * lx * to_f32<TV>(p00[pix_stride]);
        if (y0 + 1 <= H - 1 && x0 >= 0) v += ly * hx * to_f32<TV>(*p10);
        if (y0 + 1 <= H - 1 && x0 + 1 <= W - 1) v += ly * lx * to_f32<TV>(p10[pix_stride]);
        acc += v * aw;
      }
    }
    out[idx] = from_f32<TV>(acc);
  }
}

// -------------------------------------------------------------------------------------------
// Fused encoder kernel: raw offsets + logits -> softmax, reference points, sampling.
//   ow [B, Lq, M*L*P*2 + M*L*P]; value head-major [B, M, S, D]; Lq == S; patch mapping.
//
// The kernel is instruction-issue bound, not memory bound (ncu, profiles/r1_msda_fused_ncu.txt:
// issue slots 69 % busy, DRAM 6 %), so the per-sample scalar work is NOT replicated across the G
// lanes that share a (query, head): each lane derives the parameters of LP/G samples (softmax
// weight, clamped corner index, the four bilinear x attention weights with the zero-padding
// predicates folded in as zero weights) and the group exchanges them with warp shuffles — 5 SHFL per
// sample instead of ~90 ALU instructions per lane.  Corner loads are unconditional (clamped
// addresses), 16 bytes per lane.
// -------------------------------------------------------------------------------------------
template <typename TV, typename TO, int G, int LT, int PT>
__global__ void __launch_bounds__(kThreads, 4)   // <= 64 registers: 4 CTAs per SM (65 registers gave 3: occupancy 37.5 % -> 50 %)
msda_encoder_fused_kernel(const TV* __restrict__ value, const TO* __restrict__ ow,
                          TV* __restrict__ out, MsdaLevels lv, int S, int M, int D) {
  constexpr int CH = 16 / sizeof(TV);
  constexpr int NG = kThreads / G;
  constexpr int LP = LT * PT;
  constexpr int SPL = (LP + G - 1) / G;   // samples owned per lane
  const int g = threadIdx.x / G, cl = threadIdx.x % G;
  const int lane = threadIdx.x & 31;
  const int gbase = lane - cl;            // first lane of this group inside the warp
  const int m = blockIdx.y, b = blockIdx.z;
  int q, ql, qy, qx;
  const bool active = resolve_query<NG>(lv, true, g, S, q, ql, qy, qx);
  if (!active) {  // ragged tile edge: keep the lanes alive for the shuffles, on a valid dummy query
    q = lv.start[ql];
    qy = qx = 0;
  }
  const size_t row = ((size_t)b * S + q) * (size_t)(M * LP * 3);
  const TO* __restrict__ offp = ow + row + (size_t)m * LP * 2;
  const TO* __restrict__ lgp = ow + row + (size_t)M * LP * 2 + (size_t)m * LP;

  // ---- softmax over the L*P logits (F.softmax, ms_deform_attn.py:105), split across the group
  float lg[SPL];
  float mx = -INFINITY;
#pragma unroll
  for (int j = 0; j < SPL; ++j) {
    const int s = cl + j * G;
    lg[j] = s < LP ? to_f32<TO>(lgp[s]) : -INFINITY;
    mx = fmaxf(mx, lg[j]);
  }
#pragma unroll
  for (int o = 1; o < G; o <<= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
#pragma unroll
  for (int j = 0; j < SPL; ++j) {
    lg[j] = (cl + j * G) < LP ? expf(lg[j] - mx) : 0.f;
    sum += lg[j];
  }
#pragma unroll
  for (int o = 1; o < G; o <<= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float inv = 1.f / sum;

  // reference point = pixel centre of the query, normalised (msdeformattn.py:76-87)
  const float rx = ((float)qx + 0.5f) / (float)lv.W[ql];
  const float ry = ((float)qy + 0.5f) / (float)lv.H[ql];

  // ---- parameters of the samples this lane owns: four corner offsets (elements, relative to this
  //      head's value plane; 32-bit) and the four bilinear x attention weights
  constexpr int DC = G * CH;   // == D (checked on the host), compile-time for the address arithmetic
  uint32_t poff[SPL][4];
  float pw[SPL][4];
#pragma unroll
  for (int j = 0; j < SPL; ++j) {
    const int s = cl + j * G;
    poff[j][0] = poff[j][1] = poff[j][2] = poff[j][3] = 0u;
    pw[j][0] = pw[j][1] = pw[j][2] = pw[j][3] = 0.f;
    if (s < LP) {
      const int l = s / PT;
      const int H = lv.H[l], W = lv.W[l];
      float ox, oy;
      if constexpr (sizeof(TO) == 4) {
        const float2 o2 = __ldg(reinterpret_cast<const float2*>(offp) + s);
        ox = o2.x; oy = o2.y;
      } else {
        unpack2<TO>(__ldg(reinterpret_cast<const uint32_t*>(offp) + s), ox, oy);
      }
      // sampling_locations = ref + off / (W_l, H_l)  (ms_deform_attn.py:109-110), then the
      // kernel-side  w_im = loc_w * W - 0.5  (ms_deform_im2col_cuda.cuh:290-291)
      const float x = (rx + ox / (float)W) * (float)W - 0.5f;
      const float y = (ry + oy / (float)H) * (float)H - 0.5f;
      if (y > -1.f && x > -1.f && y < (float)H && x < (float)W) {
        const float yf = floorf(y), xf = floorf(x);
        const int y0 = (int)yf, x0 = (int)xf;
        const float ly = y - yf, lx = x - xf, hy = 1.f - ly, hx = 1.f - lx;
        const float aw = lg[j] * inv;
        const bool vy0 = y0 >= 0, vy1 = y0 + 1 <= H - 1, vx0 = x0 >= 0, vx1 = x0 + 1 <= W - 1;
        pw[j][0] = (vy0 && vx0) ? hy * hx * aw : 0.f;
        pw[j][1] = (vy0 && vx1) ? hy * lx * aw : 0.f;
        pw[j][2] = (vy1 && vx0) ? ly * hx * aw : 0.f;
        pw[j][3] = (vy1 && vx1) ? ly * lx * aw : 0.f;
        const int y0c = y0 < 0 ? 0 : y0, x0c = x0 < 0 ? 0 : x0;
        const int y1c = y0 + 1 > H - 1 ? H - 1 : y0 + 1, x1c = x0 + 1 > W - 1 ? W - 1 : x0 + 1;
        const int st = lv.start[l];
        poff[j][0] = (uint32_t)((st + y0c * W + x0c) * DC);
        poff[j][1] = (uint32_t)((st + y0c * W + x1c) * DC);
        poff[j][2] = (uint32_t)((st + y1c * W + x0c) * DC);
        poff[j][3] = (uint32_t)((st + y1c * W + x1c) * DC);
      }
    }
  }

  const TV* __restrict__ vb = value + ((size_t)b * M + m) * (size_t)S * DC + cl * CH;
  float2 acc2[CH / 2];   // accumulated with packed FFMA2: half the FMA issue slots of scalar FFMA
#pragma unroll
  for (int i = 0; i < CH / 2; ++i) acc2[i] = make_float2(0.f, 0.f);

#pragma unroll
  for (int s = 0; s < LP; ++s) {
    const int owner = gbase + (s % G), j = s / G;
    const uint32_t o00 = __shfl_sync(0xffffffffu, poff[j][0], owner);
    const uint32_t o01 = __shfl_sync(0xffffffffu, poff[j][1], owner);
    const uint32_t o10 = __shfl_sync(0xffffffffu, poff[j][2], owner);
    const uint32_t o11 = __shfl_sync(0xffffffffu, poff[j][3], owner);
    const float w00 = __shfl_sync(0xffffffffu, pw[j][0], owner);
    const float w01 = __shfl_sync(0xffffffffu, pw[j][1], owner);
    const float w10 = __shfl_sync(0xffffffffu, pw[j][2], owner);
    const float w11 = __shfl_sync(0xffffffffu, pw[j][3], owner);
    float2 f00[CH / 2], f01[CH / 2], f10[CH / 2], f11[CH / 2];
    load16_as_f32x2<TV>(vb + o00, f00);
    load16_as_f32x2<TV>(vb + o01, f01);
    load16_as_f32x2<TV>(vb + o10, f10);
    load16_as_f32x2<TV>(vb + o11, f11);
#pragma unroll
    for (int i = 0; i < CH / 2; ++i) {
      ffma2(acc2[i], f00[i], w00);
      ffma2(acc2[i], f01[i], w01);
      ffma2(acc2[i], f10[i], w10);
      ffma2(acc2[i], f11[i], w11);
    }
  }
  float acc[CH];
#pragma unroll
  for (int i = 0; i < CH / 2; ++i) {
    acc[2 * i] = acc2[i].x;
    acc[2 * i + 1] = acc2[i].y;
  }
  if (active) store16_from_f32<TV>(out + (((size_t)b * S + q) * M + m) * (size_t)DC + cl * CH, acc);
}

// -------------------------------------------------------------------------------------------
// host side
// -------------------------------------------------------------------------------------------
static int fill_levels(MsdaLevels& lv, const int64_t* shapes_host, const int64_t* starts_host, int L,
                       int NG, int& total_tiles, long long& sumHW) {
  lv.L = L;
  const int TW = 8, TH = NG / 8;
  int t = 0;
  sumHW = 0;
  for (int l = 0; l < kMaxLevels; ++l) {
    if (l < L) {
      lv.H[l] = (int)shapes_host[2 * l];
      lv.W[l] = (int)shapes_host[2 * l + 1];
      lv.start[l] = (int)starts_host[l];
      lv.tile0[l] = t;
      lv.tiles_x[l] = (lv.W[l] + TW - 1) / TW;
      t += lv.tiles_x[l] * ((lv.H[l] + TH - 1) / TH);
      sumHW += (long long)lv.H[l] * lv.W[l];
    } else {
      lv.H[l] = lv.W[l] = lv.start[l] = 0;
      lv.tile0[l] = t;
      lv.tiles_x[l] = 1;
    }
  }
  lv.tile0[kMaxLevels] = t;
  total_tiles = t;
  return 0;
}

template <typename TV, typename TL>
static int launch_msda(const void* value, const int64_t* shapes, const int64_t* starts, const void* loc,
                       const void* w, void* out, int B, int S, int M, int D, int L, int Lq, int P,
                       int value_layout, int shapes_on_host, cudaStream_t st) {
  constexpr int CH = 16 / sizeof(TV);
  const int pix_stride = value_layout == 0 ? M * D : D;
  const long long head_stride = value_layout == 0 ? D : (long long)S * D;
  const long long batch_stride = (long long)S * M * D;
  MsdaLevels lv;
  lv.L = L;
  const bool vec_ok = (D % CH == 0) && (D / CH <= 32) && ((D / CH) & (D / CH - 1)) == 0 &&
                      ((L * P * 2 * sizeof(TL)) % 8 == 0) &&
                      ((reinterpret_cast<uintptr_t>(value) | reinterpret_cast<uintptr_t>(out)) % 16 == 0) &&
                      (reinterpret_cast<uintptr_t>(loc) % 8 == 0) && (reinterpret_cast<uintptr_t>(w) % 4 == 0);
  const int G = vec_ok ? D / CH : 1;
  const int NG = kThreads / (G < 1 ? 1 : G);
  int tiles = 0;
  long long sumHW = 0;
  if (shapes_on_host) {
    fill_levels(lv, shapes, starts, L, NG >= 8 ? NG : 8, tiles, sumHW);
    PSALM_REQUIRE(sumHW == S, "msda: sum(H_l*W_l)=%lld != S=%d", sumHW, S);
  } else {
    for (int l = 0; l < kMaxLevels; ++l) lv.H[l] = lv.W[l] = lv.start[l] = lv.tiles_x[l] = lv.tile0[l] = 0;
    lv.tile0[kMaxLevels] = 0;
  }
  const int64_t* sdev = shapes_on_host ? nullptr : shapes;
  const int64_t* stdev = shapes_on_host ? nullptr : starts;

  if (!vec_ok) {
    const long long n = (long long)B * Lq * M * D;
    const int blocks = (int)((n + 255) / 256 < 132 * 32 ? (n + 255) / 256 : 132 * 32);
    msda_scalar_kernel<TV, TL><<<blocks > 0 ? blocks : 1, 256, 0, st>>>(
        (const TV*)value, (const TL*)loc, (const TL*)w, (TV*)out, sdev, stdev, lv, n, S, M, D, L, Lq, P,
        pix_stride, head_stride, batch_stride);
    return check_launch("msda_scalar_kernel");
  }
  // patch mapping only when the queries are the pixel grid itself and shapes are host-known
  const int patch = (shapes_on_host && Lq == S && NG >= 8) ? 1 : 0;
  dim3 grid(patch ? tiles : (Lq + NG - 1) / NG, M, B);
#define PSALM_MSDA_LAUNCH(GG, LT, PT)                                                                \
  msda_vec_kernel<TV, TL, GG, LT, PT><<<grid, kThreads, 0, st>>>(                                     \
      (const TV*)value, (const TL*)loc, (const TL*)w, (TV*)out, sdev, stdev, lv, S, M, D, L, Lq, P,   \
      pix_stride, head_stride, batch_stride, patch)
#define PSALM_MSDA_G(GG)                                      \
  do {                                                        \
    if (L == 3 && P == 4) PSALM_MSDA_LAUNCH(GG, 3, 4);        \
    else if (L == 4 && P == 4) PSALM_MSDA_LAUNCH(GG, 4, 4);   \
    else PSALM_MSDA_LAUNCH(GG, 0, 0);                         \
  } while (0)
  PSALM_REQUIRE(L <= kMaxLevels && P <= 32, "msda: L=%d (max %d) or P=%d (max 32) too large", L, kMaxLevels, P);
  switch (G) {
    case 1: PSALM_MSDA_G(1); break;
    case 2: PSALM_MSDA_G(2); break;
    case 4: PSALM_MSDA_G(4); break;
    case 8: PSALM_MSDA_G(8); break;
    case 16: PSALM_MSDA_G(16); break;
    case 32: PSALM_MSDA_G(32); break;
    default: set_error("msda: unsupported D=%d", D); return PSALM_E_UNSUPPORTED;
  }
#undef PSALM_MSDA_G
#undef PSALM_MSDA_LAUNCH
  return check_launch("msda_vec_kernel");
}


// -------------------------------------------------------------------------------------------
// Paired-column variant of the fused kernel: a (query, head) pair is owned by 2*G lanes.  Lanes 0..G-1 fetch the
// x0 column of every bilinear sample, lanes G..2G-1 the x1 column, so the two x-adjacent corners (adjacent
// 16*G-byte pixel records of the head-major value plane) are ONE 32*G-byte access per row instead of two separate
// instructions: a single L1 wavefront whenever x0 is even, i.e. ~25 % fewer wavefronts on the L1 gather path
// (DESIGN.md section 5).  Each half keeps partial sums; one xor-shuffle merges them at the end.
// Measured SLOWER than the single-group kernel (59.4 vs 53.4 us cold-cache at 1024^2, bf16): half as many queries
// per CTA and the softmax / sample arithmetic done twice cost more than the saved wavefronts.  Kept selectable
// (psalm_set_msda_impl(2)) and tested, not used by default.
// -------------------------------------------------------------------------------------------
template <typename TV, typename TO, int G, int LT, int PT>
__global__ void __launch_bounds__(kThreads)
msda_encoder_fused_pair_kernel(const TV* __restrict__ value, const TO* __restrict__ ow,
                               TV* __restrict__ out, MsdaLevels lv, int S, int M, int D) {
  constexpr int CH = 16 / sizeof(TV);
  constexpr int GG = 2 * G;
  constexpr int NG = kThreads / GG;
  constexpr int LP = LT * PT;
  constexpr int SPL = (LP + G - 1) / G;   // samples owned per lane (within its half)
  const int g = threadIdx.x / GG, cl = threadIdx.x % G, half = (threadIdx.x / G) & 1;
  const int lane = threadIdx.x & 31;
  const int hbase = lane - cl;            // first lane of this half-group inside the warp
  const int m = blockIdx.y, b = blockIdx.z;
  int q, ql, qy, qx;
  const bool active = resolve_query<NG>(lv, true, g, S, q, ql, qy, qx);
  if (!active) {
    q = lv.start[ql];
    qy = qx = 0;
  }
  const size_t row = ((size_t)b * S + q) * (size_t)(M * LP * 3);
  const TO* __restrict__ offp = ow + row + (size_t)m * LP * 2;
  const TO* __restrict__ lgp = ow + row + (size_t)M * LP * 2 + (size_t)m * LP;

  // softmax over the L*P logits, computed redundantly by both halves (G lanes each)
  float lg[SPL];
  float mx = -INFINITY;
#pragma unroll
  for (int j = 0; j < SPL; ++j) {
    const int s = cl + j * G;
    lg[j] = s < LP ? to_f32<TO>(lgp[s]) : -INFINITY;
    mx = fmaxf(mx, lg[j]);
  }
#pragma unroll
  for (int o = 1; o < G; o <<= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
#pragma unroll
  for (int j = 0; j < SPL; ++j) {
    lg[j] = (cl + j * G) < LP ? expf(lg[j] - mx) : 0.f;
    sum += lg[j];
  }
#pragma unroll
  for (int o = 1; o < G; o <<= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float inv = 1.f / sum;

  const float rx = ((float)qx + 0.5f) / (float)lv.W[ql];
  const float ry = ((float)qy + 0.5f) / (float)lv.H[ql];

  // parameters of the samples this lane owns, for ITS column: top / bottom corner offsets and weights
  constexpr int DC = G * CH;
  uint32_t poff[SPL][2];
  float pw[SPL][2];
#pragma unroll
  for (int j = 0; j < SPL; ++j) {
    const int s = cl + j * G;
    poff[j][0] = poff[j][1] = 0u;
    pw[j][0] = pw[j][1] = 0.f;
    if (s < LP) {
      const int l = s / PT;
      const int H = lv.H[l], W = lv.W[l];
      float ox, oy;
      if constexpr (sizeof(TO) == 4) {
        const float2 o2 = __ldg(reinterpret_cast<const float2*>(offp) + s);
        ox = o2.x; oy = o2.y;
      } else {
        unpack2<TO>(__ldg(reinterpret_cast<const uint32_t*>(offp) + s), ox, oy);
      }
      const float x = (rx + ox / (float)W) * (float)W - 0.5f;
      const float y = (ry + oy / (float)H) * (float)H - 0.5f;
      if (y > -1.f && x > -1.f && y < (float)H && x < (float)W) {
        const float yf = floorf(y), xf = floorf(x);
        const int y0 = (int)yf, x0 = (int)xf;
        const float ly = y - yf, lx = x - xf, hy = 1.f - ly, hx = 1.f - lx;
        const float aw = lg[j] * inv;
        const bool vy0 = y0 >= 0, vy1 = y0 + 1 <= H - 1;
        const bool vx = half ? (x0 + 1 <= W - 1) : (x0 >= 0);        // this half's column exists
        const float wx = (half ? lx : hx) * aw;
        pw[j][0] = (vy0 && vx) ? hy * wx : 0.f;
        pw[j][1] = (vy1 && vx) ? ly * wx : 0.f;
        const int y0c = y0 < 0 ? 0 : y0, y1c = y0 + 1 > H - 1 ? H - 1 : y0 + 1;
        int xc = x0 + half;
        xc = xc < 0 ? 0 : (xc > W - 1 ? W - 1 : xc);
        const int st = lv.start[l];
        poff[j][0] = (uint32_t)((st + y0c * W + xc) * DC);
        poff[j][1] = (uint32_t)((st + y1c * W + xc) * DC);
      }
    }
  }

  const TV* __restrict__ vb = value + ((size_t)b * M + m) * (size_t)S * DC + cl * CH;
  float2 acc2[CH / 2];
#pragma unroll
  for (int i = 0; i < CH / 2; ++i) acc2[i] = make_float2(0.f, 0.f);

#pragma unroll
  for (int s = 0; s < LP; ++s) {
    const int owner = hbase + (s % G), j = s / G;
    const uint32_t o0 = __shfl_sync(0xffffffffu, poff[j][0], owner);
    const uint32_t o1 = __shfl_sync(0xffffffffu, poff[j][1], owner);
    const float w0 = __shfl_sync(0xffffffffu, pw[j][0], owner);
    const float w1 = __shfl_sync(0xffffffffu, pw[j][1], owner);
    float2 f0[CH / 2], f1[CH / 2];
    load16_as_f32x2<TV>(vb + o0, f0);
    load16_as_f32x2<TV>(vb + o1, f1);
#pragma unroll
    for (int i = 0; i < CH / 2; ++i) {
      ffma2(acc2[i], f0[i], w0);
      ffma2(acc2[i], f1[i], w1);
    }
  }
  float acc[CH];
#pragma unroll
  for (int i = 0; i < CH / 2; ++i) {   // x0 column + x1 column
    acc[2 * i] = acc2[i].x + __shfl_xor_sync(0xffffffffu, acc2[i].x, G);
    acc[2 * i + 1] = acc2[i].y + __shfl_xor_sync(0xffffffffu, acc2[i].y, G);
  }
  if (active && half == 0) store16_from_f32<TV>(out + (((size_t)b * S + q) * M + m) * (size_t)DC + cl * CH, acc);
}

int g_msda_fused_impl = 0;   // 0 auto, 1 one lane group per (query, head), 2 paired columns, 3 TMA-staged tiles + mma (msda_smem.cu)

// TMA-staged shared-memory tiles + tensor-core contraction (msda_smem.cu): 16-bit storage, M = 8, D = 32, L = 3, P = 4
bool msda_smem_ok(int M, int D, int L, int P, int value_dtype, const int64_t* shapes_host);
int msda_smem_fused(const void* value, const void* ow, void* out, const int64_t* shapes_host, const int64_t* starts_host, int B,
                    int S, int value_dtype, int ow_dtype, cudaStream_t st);

template <typename TV, typename TO>
static int launch_fused(const void* value, const void* ow, void* out, const int64_t* shapes_host,
                        const int64_t* starts_host, int B, int S, int M, int D, int L, int P,
                        cudaStream_t st) {
  constexpr int CH = 16 / sizeof(TV);
  PSALM_REQUIRE(D % CH == 0, "msda_fused: D=%d not a multiple of %d", D, CH);
  const int G = D / CH;
  PSALM_REQUIRE(G == 4 || G == 8, "msda_fused: D=%d unsupported (need D/%d in {4,8})", D, CH);
  PSALM_REQUIRE((long long)S * D < (1ll << 31), "msda_fused: S*D=%lld exceeds the 32-bit corner offsets", (long long)S * D);
  PSALM_REQUIRE((L == 3 || L == 4) && P == 4, "msda_fused: (L,P)=(%d,%d) unsupported", L, P);
  const bool pair = g_msda_fused_impl == 2 && 2 * G <= 32;
  MsdaLevels lv;
  int tiles = 0;
  long long sumHW = 0;
  fill_levels(lv, shapes_host, starts_host, L, kThreads / (pair ? 2 * G : G), tiles, sumHW);
  PSALM_REQUIRE(sumHW == S, "msda_fused: sum(H_l*W_l)=%lld != S=%d", sumHW, S);
  dim3 grid(tiles, M, B);
#define PSALM_FUSED(KERN, GG, LT)                                                                   \
  KERN<TV, TO, GG, LT, 4><<<grid, kThreads, 0, st>>>((const TV*)value, (const TO*)ow, (TV*)out, lv, S, M, D)
  if (pair) {
    if (G == 4) { if (L == 3) PSALM_FUSED(msda_encoder_fused_pair_kernel, 4, 3); else PSALM_FUSED(msda_encoder_fused_pair_kernel, 4, 4); }
    else        { if (L == 3) PSALM_FUSED(msda_encoder_fused_pair_kernel, 8, 3); else PSALM_FUSED(msda_encoder_fused_pair_kernel, 8, 4); }
  } else {
    if (G == 4) { if (L == 3) PSALM_FUSED(msda_encoder_fused_kernel, 4, 3); else PSALM_FUSED(msda_encoder_fused_kernel, 4, 4); }
    else        { if (L == 3) PSALM_FUSED(msda_encoder_fused_kernel, 8, 3); else PSALM_FUSED(msda_encoder_fused_kernel, 8, 4); }
  }
#undef PSALM_FUSED
  return check_launch("msda_encoder_fused_kernel");
}

}  // namespace psalm

using namespace psalm;

extern "C" int psalm_msda_forward(const void* value, const int64_t* shapes, const int64_t* starts,
                                  const void* loc, const void* w, void* out, int B, int S, int M, int D,
                                  int L, int Lq, int P, int value_dtype, int loc_dtype, int value_layout,
                                  int shapes_on_host, void* stream) {
  PSALM_REQUIRE(value && shapes && starts && loc && w && out, "msda: null pointer argument");
  PSALM_REQUIRE(B > 0 && S > 0 && M > 0 && D > 0 && L > 0 && Lq > 0 && P > 0,
                "msda: non-positive dimension (B=%d S=%d M=%d D=%d L=%d Lq=%d P=%d)", B, S, M, D, L, Lq, P);
  PSALM_REQUIRE(value_layout == 0 || value_layout == 1, "msda: value_layout must be 0 or 1");
  PSALM_REQUIRE(M <= 65535 && B <= 65535, "msda: M or B exceeds grid limits");
  PSALM_REQUIRE(loc_dtype == PSALM_F32 || loc_dtype == value_dtype,
                "msda: loc dtype %d must be F32 or equal to the value dtype %d", loc_dtype, value_dtype);
  cudaStream_t st = (cudaStream_t)stream;
#define ARGS value, shapes, starts, loc, w, out, B, S, M, D, L, Lq, P, value_layout, shapes_on_host, st
  switch (value_dtype) {
    case PSALM_F32: return launch_msda<float, float>(ARGS);
    case PSALM_F16:
      return loc_dtype == PSALM_F32 ? launch_msda<__half, float>(ARGS) : launch_msda<__half, __half>(ARGS);
    case PSALM_BF16:
      return loc_dtype == PSALM_F32 ? launch_msda<__nv_bfloat16, float>(ARGS)
                                    : launch_msda<__nv_bfloat16, __nv_bfloat16>(ARGS);
  }
#undef ARGS
  set_error("msda: unknown value dtype %d", value_dtype);
  return PSALM_E_ARG;
}

extern "C" int psalm_set_msda_impl(int impl) {
  PSALM_REQUIRE(impl >= 0 && impl <= 3, "set_msda_impl: 0 (auto), 1 (one lane group per query-head), 2 (paired columns) or 3 (TMA tiles)");
  psalm::g_msda_fused_impl = impl;
  return PSALM_OK;
}

extern "C" int psalm_msda_encoder_fused(const void* value, const void* ow, void* out,
                                        const int64_t* shapes_host, const int64_t* starts_host, int B,
                                        int S, int M, int D, int L, int P, int value_dtype, int ow_dtype,
                                        void* stream) {
  PSALM_REQUIRE(value && ow && out && shapes_host && starts_host, "msda_fused: null pointer argument");
  PSALM_REQUIRE(B > 0 && S > 0 && M > 0 && D > 0, "msda_fused: non-positive dimension");
  cudaStream_t st = (cudaStream_t)stream;
  // auto = the L1-gather kernel: the TMA-tile + mma kernel (impl 3) is correct but measured slower at 1024^2
  // (84 us vs 53 us per layer-image: 53.7 M vs 39 M warp instructions, DESIGN.md section 5)
  if (g_msda_fused_impl == 3) {
    const bool ok = msda_smem_ok(M, D, L, P, value_dtype, shapes_host) && M <= 65535 && B <= 65535;
    if (ok) {
      long long sum = 0;
      for (int l = 0; l < L; ++l) sum += shapes_host[2 * l] * shapes_host[2 * l + 1];
      PSALM_REQUIRE(sum == S, "msda_fused: sum(H_l*W_l)=%lld != S=%d", sum, S);
      return msda_smem_fused(value, ow, out, shapes_host, starts_host, B, S, value_dtype, ow_dtype, st);
    }
    PSALM_REQUIRE(false, "msda_fused: the TMA-tile kernel needs 16-bit storage, M=8, D=32, L=3, P=4, levels coarse to fine");
  }
#define ARGS value, ow, out, shapes_host, starts_host, B, S, M, D, L, P, st
  if (value_dtype == PSALM_F32 && ow_dtype == PSALM_F32) return launch_fused<float, float>(ARGS);
  if (value_dtype == PSALM_F16 && ow_dtype == PSALM_F16) return launch_fused<__half, __half>(ARGS);
  if (value_dtype == PSALM_F16 && ow_dtype == PSALM_F32) return launch_fused<__half, float>(ARGS);
  if (value_dtype == PSALM_BF16 && ow_dtype == PSALM_BF16) return launch_fused<__nv_bfloat16, __nv_bfloat16>(ARGS);
  if (value_dtype == PSALM_BF16 && ow_dtype == PSALM_F32) return launch_fused<__nv_bfloat16, float>(ARGS);
#undef ARGS
  set_error("msda_fused: unsupported dtype combination value=%d ow=%d", value_dtype, ow_dtype);
  return PSALM_E_UNSUPPORTED;
}
