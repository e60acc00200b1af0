// Video object segmentation: the per-frame host loop of the reference's DAVIS evaluation (psalm/eval/eval_davis.py:
// 388-480) as three small kernels, so that a frame leaves the device as a uint8 label map plus a few hundred integers.
//
//   vos_pick_kernel      the per-object top-10 de-duplicating query pick (eval_davis.py:443-453) over the scores of
//                        region_inference (llava_phi.py:387-400), one warp;
//   vos_fuse_kernel      fuse_davis_mask (eval_davis.py:337-342) + the per-object areas and pairwise intersections of the
//                        memory check (:463-473), one bit per object per pixel;
//   vos_bits_kernel      detectron2's ResizeTransform.apply_segmentation (Pillow NEAREST) + FixedSizeCrop zero padding of
//   + vos_prefix_kernel  the kept masks (:406-408) as a bit mask at the network input size, with per-row set counts;
//   vp_pack_kernel       visual prompts (click, scribble, box, mask) at the original image size: enhance_with_circles
//   + vp_raster_kernel   (coco_instance_mapper.py:17-33) + the mapper's NEAREST resize and padding (:250), straight
//                        into the bit layout of vos_bits_kernel (the dilated mask is never built);
//   region_points_gather_kernel  "the i-th set pixel in nonzero() order" -> (y / H, x / W) for the host-drawn indices of
//                        sample_region_points (psalm_b200/region.py = context_cluster.py:31-40, :349-352).
#include "common.cuh"

namespace psalm {

constexpr int kVosMaxK = 32;
constexpr int kVosMaxQ = 128;
constexpr int kVosTopK = 10;   // eval_davis.py:446

// (score, query) order of the pick: larger score first, the lower query index on ties
__device__ __forceinline__ bool vos_before(float sa, int qa, float sb, int qb) {
  return sa > sb || (sa == sb && qa < qb);
}

template <typename T>
__global__ void __launch_bounds__(32) vos_pick_kernel(const T* __restrict__ logits, const float* __restrict__ stats,
                                                      int* __restrict__ pick, float* __restrict__ score, int K, int Q) {
  constexpr int PER = kVosMaxQ / 32;
  const int lane = threadIdx.x;
  float ms[PER];
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    const int q = lane + 32 * j;
    // query_mask_scores (llava_phi.py:441-443): sum(sigmoid * [x > 0]) / (count(x > 0) + 1e-6)
    ms[j] = q < Q ? stats[q * 5 + 1] / (stats[q * 5 + 0] + 1e-6f) : 0.f;
  }
  int prev_pick = 0;          // the reference's loop variables survive an object whose 10 candidates are all taken
  float prev_score = 0.f;
  int taken = -1;             // lane k holds the pick of object k once it is made (the reference's prev_idx list)
  for (int k = 0; k < K; ++k) {
    float s[PER];
#pragma unroll
    for (int j = 0; j < PER; ++j) {
      const int q = lane + 32 * j;
      const float x = q < Q ? to_f32<T>(logits[(size_t)k * Q + q]) : 0.f;
      s[j] = q < Q ? (1.f / (1.f + expf(-x))) * ms[j] : -INFINITY;
    }
    int cand[kVosTopK];
    float cscore[kVosTopK];
    unsigned used = 0;        // bit j: this lane's query lane + 32 j is already among the candidates
#pragma unroll
    for (int t = 0; t < kVosTopK; ++t) {
      float bs = -INFINITY;
      int bq = 0x7fffffff;
#pragma unroll
      for (int j = 0; j < PER; ++j) {
        const int q = lane + 32 * j;
        if (q < Q && !((used >> j) & 1u) && vos_before(s[j], q, bs, bq)) { bs = s[j]; bq = q; }
      }
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        const float os = __shfl_xor_sync(0xffffffffu, bs, off);
        const int oq = __shfl_xor_sync(0xffffffffu, bq, off);
        if (vos_before(os, oq, bs, bq)) { bs = os; bq = oq; }
      }
      cand[t] = bq;
      cscore[t] = bs;
      if ((bq & 31) == lane) used |= 1u << (bq >> 5);
    }
#pragma unroll
    for (int t = 0; t < kVosTopK; ++t) {
      const bool dup = __any_sync(0xffffffffu, lane < k && taken == cand[t]);
      if (!dup) {
        prev_pick = cand[t];
        prev_score = cscore[t];
        if (lane == k) taken = cand[t];
        break;
      }
    }
    if (lane == 0) {
      pick[k] = prev_pick;
      score[k] = prev_score;
    }
  }
}

// One thread per output pixel: the objects set at the pixel as one 32-bit word.  Label = fill of the highest set object
// (fuse_davis_mask assigns in object order, the later object wins).  Areas: one ballot + popc per object and warp;
// intersections: shared-memory atomics for the (rare) pixels where two or more objects are set.
__global__ void __launch_bounds__(256) vos_fuse_kernel(const float* __restrict__ masks, const int* __restrict__ fill,
                                                       uint8_t* __restrict__ labels, int* __restrict__ area,
                                                       int* __restrict__ inter, int K, long long HW) {
  __shared__ int s_area[kVosMaxK];
  __shared__ int s_inter[kVosMaxK * kVosMaxK];
  for (int i = threadIdx.x; i < kVosMaxK * kVosMaxK; i += blockDim.x) s_inter[i] = 0;
  if (threadIdx.x < kVosMaxK) s_area[threadIdx.x] = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long base = (long long)blockIdx.x * blockDim.x; base < HW; base += stride) {
    const long long p = base + threadIdx.x;
    unsigned b = 0;
    if (p < HW)
      for (int k = 0; k < K; ++k) b |= (masks[(size_t)k * HW + p] != 0.f ? 1u : 0u) << k;
    if (p < HW) labels[p] = b ? (uint8_t)fill[31 - __clz(b)] : (uint8_t)0;
    for (int k = 0; k < K; ++k) {
      const unsigned v = __ballot_sync(0xffffffffu, (b >> k) & 1u);
      if (lane == 0 && v) atomicAdd(&s_area[k], __popc(v));
    }
    if (__popc(b) > 1) {
      for (unsigned bi = b; bi; bi &= bi - 1) {
        const int i = __ffs(bi) - 1;
        for (unsigned bj = b & ~(1u << i); bj; bj &= bj - 1) atomicAdd(&s_inter[i * kVosMaxK + __ffs(bj) - 1], 1);
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < K * K; i += blockDim.x) {
    const int a = i / K, c = i % K;
    const int v = a == c ? s_area[a] : s_inter[a * kVosMaxK + c];
    if (v) atomicAdd(&inter[i], v);
  }
  if (threadIdx.x < K && s_area[threadIdx.x]) atomicAdd(&area[threadIdx.x], s_area[threadIdx.x]);
}

// One warp per (object, padded row): lane i of a 32-pixel step reads the source pixel of column x = 32 w + i through
// the Pillow index tables; the ballot is the bit word.  Lane 0 keeps the row's set count.
__global__ void __launch_bounds__(256) vos_bits_kernel(const float* __restrict__ masks, const int* __restrict__ src_row,
                                                       const int* __restrict__ src_col, uint32_t* __restrict__ bits,
                                                       int* __restrict__ row_prefix, int H, int W, int Hp, int Wp) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int y = blockIdx.x * (blockDim.x >> 5) + warp, k = blockIdx.y;
  if (y >= Hp) return;
  const int W32 = (Wp + 31) >> 5;
  const int sy = src_row[y];
  const float* row = masks + ((size_t)k * H + (sy < 0 ? 0 : sy)) * W;
  uint32_t* out = bits + ((size_t)k * Hp + y) * W32;
  int n = 0;
  for (int w = 0; w < W32; ++w) {
    const int x = (w << 5) + lane;
    const int sx = x < Wp ? src_col[x] : -1;
    const bool on = sy >= 0 && sx >= 0 && row[sx] != 0.f;
    const unsigned v = __ballot_sync(0xffffffffu, on);
    if (lane == 0) out[w] = v;
    n += __popc(v);
  }
  if (lane == 0) row_prefix[(size_t)k * (Hp + 1) + y + 1] = n;   // row counts; vos_prefix_kernel scans them in place
}

// One warp per object: exclusive prefix sum of the row counts (row_prefix[k, 0] = 0, row_prefix[k, Hp] = total).
__global__ void __launch_bounds__(32) vos_prefix_kernel(int* __restrict__ row_prefix, int* __restrict__ count, int Hp) {
  const int k = blockIdx.x, lane = threadIdx.x;
  int* rp = row_prefix + (size_t)k * (Hp + 1);
  const int per = (Hp + 31) / 32, lo = 1 + lane * per, hi = min(Hp + 1, lo + per);
  int local = 0;
  for (int i = lo; i < hi; ++i) local += rp[i];
  int incl = local;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, off);
    if (lane >= off) incl += v;
  }
  int run = incl - local;
  for (int i = lo; i < hi; ++i) {
    run += rp[i];
    rp[i] = run;
  }
  if (lane == 0) rp[0] = 0;
  if (lane == 31) count[k] = incl;
}

// Visual prompts (coco_instance_mapper.py:17-33, :233-251): enhance_with_circles (a disk of radius r around every
// source pixel equal to 1), then Pillow NEAREST + zero padding.  NEAREST reads one source pixel per output pixel, so the
// dilated mask is never built: output pixel (y, x) is set when a seed lies in the disk around (src_row[y], src_col[x]).
// draw_circle's float64 test sqrt(dx^2 + dy^2) <= r equals the integer test dx^2 + dy^2 <= r^2 for an integer r
// (sqrt is correctly rounded and r^2 is exact), so row dy of the disk is the span |dx| <= isqrt(r^2 - dy^2).

// One warp per (source row, region): the seeds as bits (== 1 for a dilated region, != 0 for r = 0, where the mask is
// resized as it is).
__global__ void __launch_bounds__(256) vp_pack_kernel(const uint8_t* __restrict__ src, const int* __restrict__ radius,
                                                      uint32_t* __restrict__ src_bits, int H0, int W0) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int y = blockIdx.x * (blockDim.x >> 5) + warp, k = blockIdx.y;
  if (y >= H0) return;
  const int S32 = (W0 + 31) >> 5;
  const bool ones_only = radius[k] > 0;
  const uint8_t* row = src + ((size_t)k * H0 + y) * W0;
  uint32_t* out = src_bits + ((size_t)k * H0 + y) * S32;
  for (int w = 0; w < S32; ++w) {
    const int x = (w << 5) + lane;
    const uint8_t v = x < W0 ? row[x] : 0;
    const unsigned b = __ballot_sync(0xffffffffu, ones_only ? v == 1 : v != 0);
    if (lane == 0) out[w] = b;
  }
}

__device__ __forceinline__ int isqrt_floor(int v) {
  int h = (int)sqrtf((float)v);
  while (h * h > v) --h;
  while ((h + 1) * (h + 1) <= v) ++h;
  return h;
}

// One warp per (padded row, region), lane i of a 32-pixel step tests output column 32 w + i: for every disk row dy the
// span [sx - h, sx + h] (clipped at the border) is tested word by word against the seed bits; the ballot is the output
// word.  Lane 0 keeps the row's set count for vos_prefix_kernel.
__global__ void __launch_bounds__(256) vp_raster_kernel(const uint32_t* __restrict__ src_bits, const int* __restrict__ radius,
                                                        const int* __restrict__ src_row, const int* __restrict__ src_col,
                                                        uint32_t* __restrict__ bits, int* __restrict__ row_prefix, int H0,
                                                        int W0, int Hp, int Wp) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int y = blockIdx.x * (blockDim.x >> 5) + warp, k = blockIdx.y;
  if (y >= Hp) return;
  const int W32 = (Wp + 31) >> 5, S32 = (W0 + 31) >> 5;
  const int r = radius[k], sy = src_row[y];
  const uint32_t* seeds = src_bits + (size_t)k * H0 * S32;
  uint32_t* out = bits + ((size_t)k * Hp + y) * W32;
  int n = 0;
  for (int w = 0; w < W32; ++w) {
    const int x = (w << 5) + lane;
    const int sx = x < Wp ? src_col[x] : -1;
    bool on = false;
    if (sy >= 0 && sx >= 0) {
      const int dy1 = min(r, H0 - 1 - sy);
      for (int dy = max(-r, -sy); dy <= dy1 && !on; ++dy) {
        const int h = isqrt_floor(r * r - dy * dy);
        const int lo = max(sx - h, 0), hi = min(sx + h, W0 - 1);
        const uint32_t* row = seeds + (size_t)(sy + dy) * S32;
        for (int wi = lo >> 5; wi <= (hi >> 5) && !on; ++wi) {
          const int b0 = max(lo - (wi << 5), 0), b1 = min(hi - (wi << 5), 31);
          on = (row[wi] & (0xffffffffu >> (31 - b1)) & (0xffffffffu << b0)) != 0u;
        }
      }
    }
    const unsigned v = __ballot_sync(0xffffffffu, on);
    if (lane == 0) out[w] = v;
    n += __popc(v);
  }
  if (lane == 0) row_prefix[(size_t)k * (Hp + 1) + y + 1] = n;
}

// One thread per (region, point): binary search of the row holding the sel-th set pixel, then the words of that row.
__global__ void __launch_bounds__(256) region_points_gather_kernel(const uint32_t* __restrict__ bits,
                                                                   const int* __restrict__ row_prefix,
                                                                   const int* __restrict__ sel,
                                                                   const int* __restrict__ mask_of_region,
                                                                   float* __restrict__ points, int R, int P, int Hp,
                                                                   int Wp) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R * P) return;
  const int m = mask_of_region[i / P];
  const int* rp = row_prefix + (size_t)m * (Hp + 1);
  const int target = sel[i];
  float y_out = 0.f, x_out = 0.f;
  if (target >= 0 && target < rp[Hp]) {
    int lo = 0, hi = Hp;                 // rp[lo] <= target < rp[hi]
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (rp[mid] <= target) lo = mid; else hi = mid;
    }
    const int W32 = (Wp + 31) >> 5;
    const uint32_t* row = bits + ((size_t)m * Hp + lo) * W32;
    int r = target - rp[lo];
    int x = 0;
    for (int w = 0; w < W32; ++w) {
      uint32_t v = row[w];
      const int c = __popc(v);
      if (r < c) {
        for (; r > 0; --r) v &= v - 1;   // drop the r lowest set bits
        x = (w << 5) + __ffs(v) - 1;
        break;
      }
      r -= c;
    }
    // m.nonzero() / torch.tensor([H, W]): int64 / int64 true division in fp32, round to nearest
    y_out = __fdiv_rn((float)lo, (float)Hp);
    x_out = __fdiv_rn((float)x, (float)Wp);
  }
  points[2 * (size_t)i] = y_out;
  points[2 * (size_t)i + 1] = x_out;
}

}  // namespace psalm

using namespace psalm;

extern "C" int psalm_vos_pick(const void* region_logits, const float* stats, int* pick, float* score, int K, int Q, int dtype,
                              void* stream) {
  PSALM_REQUIRE(region_logits && stats && pick && score, "vos_pick: null pointer");
  PSALM_REQUIRE(K > 0 && K <= kVosMaxK, "vos_pick: K=%d objects (1..%d)", K, kVosMaxK);
  PSALM_REQUIRE(Q >= kVosTopK && Q <= kVosMaxQ, "vos_pick: Q=%d queries (%d..%d)", Q, kVosTopK, kVosMaxQ);
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case PSALM_F32: vos_pick_kernel<float><<<1, 32, 0, st>>>((const float*)region_logits, stats, pick, score, K, Q); break;
    case PSALM_F16: vos_pick_kernel<__half><<<1, 32, 0, st>>>((const __half*)region_logits, stats, pick, score, K, Q); break;
    case PSALM_BF16:
      vos_pick_kernel<__nv_bfloat16><<<1, 32, 0, st>>>((const __nv_bfloat16*)region_logits, stats, pick, score, K, Q);
      break;
    default: set_error("vos_pick: unknown dtype %d", dtype); return PSALM_E_ARG;
  }
  return check_launch("vos_pick_kernel");
}

extern "C" int psalm_vos_fuse(const float* masks, const int* fill, const int* src_row, const int* src_col, uint8_t* labels,
                              int* area, int* inter, uint32_t* bits, int* row_prefix, int* count, int K, int H, int W, int Hp,
                              int Wp, void* stream) {
  PSALM_REQUIRE(masks && src_row && src_col && bits && row_prefix && count, "vos_fuse: null pointer");
  PSALM_REQUIRE(!labels || (fill && area && inter), "vos_fuse: labels need fill, area and inter");
  PSALM_REQUIRE(K > 0 && K <= kVosMaxK, "vos_fuse: K=%d objects (1..%d)", K, kVosMaxK);
  PSALM_REQUIRE(H > 0 && W > 0 && Hp > 0 && Wp > 0, "vos_fuse: bad shape");
  cudaStream_t st = (cudaStream_t)stream;
  if (labels) {
    if (cudaMemsetAsync(area, 0, sizeof(int) * K, st) != cudaSuccess ||
        cudaMemsetAsync(inter, 0, sizeof(int) * K * K, st) != cudaSuccess) {
      set_error("vos_fuse: cudaMemsetAsync failed");
      return PSALM_E_CUDA;
    }
    const long long HW = (long long)H * W;
    int sms = 132;
    int dev = 0;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const long long want = (HW + 255) / 256;
    const int blocks = (int)(want < 4LL * sms ? want : 4LL * sms);
    vos_fuse_kernel<<<blocks, 256, 0, st>>>(masks, fill, labels, area, inter, K, HW);
    if (int rc = check_launch("vos_fuse_kernel")) return rc;
  }
  vos_bits_kernel<<<dim3((Hp + 7) / 8, K), 256, 0, st>>>(masks, src_row, src_col, bits, row_prefix, H, W, Hp, Wp);
  if (int rc = check_launch("vos_bits_kernel")) return rc;
  vos_prefix_kernel<<<K, 32, 0, st>>>(row_prefix, count, Hp);
  return check_launch("vos_prefix_kernel");
}

extern "C" int psalm_visual_prompt_raster(const uint8_t* src, const int* radius, const int* src_row, const int* src_col,
                                          uint32_t* src_bits, uint32_t* bits, int* row_prefix, int* count, int K, int H0,
                                          int W0, int Hp, int Wp, void* stream) {
  PSALM_REQUIRE(src && radius && src_row && src_col && src_bits && bits && row_prefix && count,
                "visual_prompt_raster: null pointer");
  PSALM_REQUIRE(K > 0 && H0 > 0 && W0 > 0 && Hp > 0 && Wp > 0, "visual_prompt_raster: bad shape");
  cudaStream_t st = (cudaStream_t)stream;
  vp_pack_kernel<<<dim3((H0 + 7) / 8, K), 256, 0, st>>>(src, radius, src_bits, H0, W0);
  if (int rc = check_launch("vp_pack_kernel")) return rc;
  vp_raster_kernel<<<dim3((Hp + 7) / 8, K), 256, 0, st>>>(src_bits, radius, src_row, src_col, bits, row_prefix, H0, W0,
                                                          Hp, Wp);
  if (int rc = check_launch("vp_raster_kernel")) return rc;
  vos_prefix_kernel<<<K, 32, 0, st>>>(row_prefix, count, Hp);
  return check_launch("vos_prefix_kernel");
}

extern "C" int psalm_region_points_gather(const uint32_t* bits, const int* row_prefix, const int* sel,
                                          const int* mask_of_region, float* points, int R, int P, int Hp, int Wp,
                                          void* stream) {
  PSALM_REQUIRE(bits && row_prefix && sel && mask_of_region && points, "region_points_gather: null pointer");
  PSALM_REQUIRE(R > 0 && P > 0 && Hp > 0 && Wp > 0, "region_points_gather: bad shape");
  const int n = R * P;
  region_points_gather_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(bits, row_prefix, sel, mask_of_region,
                                                                                 points, R, P, Hp, Wp);
  return check_launch("region_points_gather_kernel");
}
