// COCO run-length encoding of binary masks on the device (the contract of pycocotools' maskApi.c: rleEncode,
// rleToString, rleFrString, rleDecode, rleArea, rleToBbox), restated for a batch of masks.
//
// Runs are taken in column-major pixel order j = x*H + y of a row-major [H,W] mask; the first run counts background.
// A "transition" is a pixel j whose value differs from pixel j-1 (pixel -1 counts as background); the end of run r is
// the (r+1)-th transition, and the last run ends at H*W.  Encoding is three entry points around two small
// device-to-host copies (the run total and the byte total, which size the outputs):
//   psalm_rle_count    dense masks -> per-column transition counts + a 1-bit column-major copy of the masks
//                      (the only read of the dense input), per-mask area / bbox, run offsets;
//   psalm_rle_runs     1-bit copy -> run ends; per-mask string lengths -> byte offsets;
//   psalm_rle_strings  run ends -> the compressed strings of rleToString.
#include <climits>

#include "common.cuh"

namespace {

constexpr int kScanThreads = 256;

int sm_count() {
  static psalm::PerDevice cache;
  const int d = psalm::PerDevice::dev();
  if (cache.first() || cache.v[d] == 0) cudaDeviceGetAttribute(&cache.v[d], cudaDevAttrMultiProcessorCount, d);
  return cache.v[d] > 0 ? cache.v[d] : 132;
}

// exclusive scan over a block of kScanThreads threads; *total receives the block sum
__device__ __forceinline__ long long block_excl_scan(long long v, long long* total) {
  __shared__ long long warp_sums[kScanThreads / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  long long incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) warp_sums[wid] = incl;
  __syncthreads();
  long long base = 0, sum = 0;
#pragma unroll
  for (int w = 0; w < kScanThreads / 32; ++w) {
    const long long s = warp_sums[w];
    if (w < wid) base += s;
    sum += s;
  }
  __syncthreads();   // warp_sums is reused by the next call
  *total = sum;
  return base + incl - v;
}

// number of 6-bit characters rleToString emits for one value
__device__ __forceinline__ int rle_chars(long long x) {
  int n = 0;
  bool more = true;
  while (more) {
    const int c = (int)(x & 0x1f);
    x >>= 5;   // arithmetic shift
    more = (c & 0x10) ? x != -1 : x != 0;
    ++n;
  }
  return n;
}

// value rleToString encodes for run r of a mask: cnt[r], minus cnt[r-2] for r > 2 (cnt[r] = ends[r] - ends[r-1])
__device__ __forceinline__ long long rle_value(const uint32_t* ends, long long r) {
  const long long c = (long long)ends[r] - (r > 0 ? (long long)ends[r - 1] : 0);
  if (r <= 2) return c;
  return c - ((long long)ends[r - 2] - (long long)ends[r - 3]);
}

template <typename T>
__device__ __forceinline__ bool fg(const T* p) { return __ldg(p) != T(0); }

// One warp per (mask, strip of 32 columns), one lane per column: each row of the strip is one coalesced load.  Per column:
// transitions (including the one into its top pixel from the bottom pixel of the previous column), foreground count,
// first / last foreground row; the column's bits go to `bits` [n, W, Hw] (column-major, 32 rows per word).
template <typename T>
__global__ void __launch_bounds__(256) rle_count_kernel(const T* __restrict__ masks, const unsigned long long* __restrict__ ptrs,
                                                        uint32_t* __restrict__ bits, int4* __restrict__ colstat, int n,
                                                        int H, int W) {
  const int lane = threadIdx.x & 31;
  const int strips = (W + 31) >> 5;
  const int Hw = (H + 31) >> 5;
  const long long tasks = (long long)n * strips;
  for (long long task = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; task < tasks;
       task += ((long long)gridDim.x * blockDim.x) >> 5) {
    const int i = (int)(task / strips);
    const int x0 = (int)(task % strips) * 32;
    const int x = x0 + lane;
    const bool live = x < W;
    const int xc = live ? x : W - 1;
    const T* m = ptrs ? reinterpret_cast<const T*>(ptrs[i]) : masks + (size_t)i * H * W;
    uint32_t* col = bits + ((size_t)i * W + xc) * Hw;
    int trans = 0, cnt = 0, ymin = H, ymax = -1;
    uint32_t word = 0;
    bool prev = false, top = false;
    int y = 0;
    for (; y + 8 <= H; y += 8) {   // eight independent row loads in flight per lane
      bool v[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] = fg(m + (size_t)(y + k) * W + xc);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int yy = y + k;
        if (yy == 0) top = v[k];
        else trans += v[k] != prev;
        prev = v[k];
        if (v[k]) { ++cnt; ymin = min(ymin, yy); ymax = yy; }
        word |= (uint32_t)v[k] << (yy & 31);
      }
      if (((y + 8) & 31) == 0) {
        if (live) col[(y + 7) >> 5] = word;
        word = 0;
      }
    }
    for (; y < H; ++y) {
      const bool v = fg(m + (size_t)y * W + xc);
      if (y == 0) top = v;
      else trans += v != prev;
      prev = v;
      if (v) { ++cnt; ymin = min(ymin, y); ymax = y; }
      word |= (uint32_t)v << (y & 31);
    }
    if ((H & 31) && live) col[Hw - 1] = word;
    // transition into the top pixel: compare with the bottom pixel of column x-1 (background before column 0)
    bool above = __shfl_up_sync(0xffffffffu, prev, 1);
    if (lane == 0) above = x0 > 0 ? fg(m + (size_t)(H - 1) * W + x0 - 1) : false;
    trans += top != above;
    if (live) colstat[(size_t)i * W + x] = make_int4(trans, cnt, ymin, ymax);
  }
}

// One block per mask: exclusive scan of the column transition counts (-> colstart), runs = transitions + 1,
// area = foreground pixels (rleArea), bbox = tight box of the foreground or zeros (rleToBbox).
__global__ void __launch_bounds__(kScanThreads) rle_mask_stats_kernel(const int4* __restrict__ colstat, int* __restrict__ colstart,
                                                                      long long* __restrict__ runs, long long* __restrict__ area,
                                                                      double* __restrict__ bbox, int W) {
  const int i = blockIdx.x;
  long long carry = 0, fgsum = 0;
  int xs = INT_MAX, xe = -1, ys = INT_MAX, ye = -1;
  for (int base = 0; base < W; base += kScanThreads) {
    const int x = base + threadIdx.x;
    const int4 s = x < W ? colstat[(size_t)i * W + x] : make_int4(0, 0, INT_MAX, -1);
    long long tot;
    const long long ex = block_excl_scan(s.x, &tot);
    if (x < W) colstart[(size_t)i * W + x] = (int)(carry + ex);
    carry += tot;
    fgsum += s.y;
    if (s.y > 0) { xs = min(xs, x); xe = max(xe, x); ys = min(ys, s.z); ye = max(ye, s.w); }
  }
  __shared__ long long red_sum[kScanThreads / 32];
  __shared__ int red[4][kScanThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    fgsum += __shfl_xor_sync(0xffffffffu, fgsum, o);
    xs = min(xs, __shfl_xor_sync(0xffffffffu, xs, o));
    ys = min(ys, __shfl_xor_sync(0xffffffffu, ys, o));
    xe = max(xe, __shfl_xor_sync(0xffffffffu, xe, o));
    ye = max(ye, __shfl_xor_sync(0xffffffffu, ye, o));
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) { red_sum[wid] = fgsum; red[0][wid] = xs; red[1][wid] = ys; red[2][wid] = xe; red[3][wid] = ye; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kScanThreads / 32; ++w) {
      fgsum = fgsum + red_sum[w];
      xs = min(xs, red[0][w]); ys = min(ys, red[1][w]); xe = max(xe, red[2][w]); ye = max(ye, red[3][w]);
    }
    runs[i] = carry + 1;
    area[i] = fgsum;
    double* bb = bbox + (size_t)i * 4;
    if (fgsum == 0) {
      bb[0] = bb[1] = bb[2] = bb[3] = 0.0;
    } else {
      bb[0] = xs; bb[1] = ys; bb[2] = xe - xs + 1; bb[3] = ye - ys + 1;
    }
  }
}

// in place: v[0..n-1] -> exclusive prefix sums v[0..n] (one block)
__global__ void __launch_bounds__(kScanThreads) rle_offsets_kernel(long long* __restrict__ v, int n) {
  long long carry = 0;
  for (int base = 0; base < n; base += kScanThreads) {
    const int k = base + threadIdx.x;
    const long long x = k < n ? v[k] : 0;
    long long tot;
    const long long ex = block_excl_scan(x, &tot);
    if (k < n) v[k] = carry + ex;
    carry += tot;
  }
  if (threadIdx.x == 0) v[n] = carry;
}

// One warp per (mask, strip), one lane per column: the linear index of every transition of the column, from the
// 1-bit copy, at the column's slot of the mask's run ends; the last column also writes the final end H*W.
__global__ void __launch_bounds__(256) rle_ends_kernel(const uint32_t* __restrict__ bits, const int* __restrict__ colstart,
                                                       const long long* __restrict__ run_off, uint32_t* __restrict__ ends,
                                                       int n, int H, int W) {
  const int lane = threadIdx.x & 31;
  const int strips = (W + 31) >> 5;
  const int Hw = (H + 31) >> 5;
  const uint32_t last_mask = (H & 31) ? (1u << (H & 31)) - 1u : 0xffffffffu;
  const long long tasks = (long long)n * strips;
  for (long long task = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; task < tasks;
       task += ((long long)gridDim.x * blockDim.x) >> 5) {
    const int i = (int)(task / strips);
    const int x0 = (int)(task % strips) * 32;
    const int x = x0 + lane;
    const bool live = x < W;
    const int xc = live ? x : W - 1;
    const uint32_t* col = bits + ((size_t)i * W + xc) * Hw;
    const uint32_t bottom = (col[Hw - 1] >> ((H - 1) & 31)) & 1u;
    uint32_t carry = __shfl_up_sync(0xffffffffu, bottom, 1);
    if (lane == 0) carry = x0 > 0 ? (bits[((size_t)i * W + x0 - 1) * Hw + Hw - 1] >> ((H - 1) & 31)) & 1u : 0u;
    if (!live) continue;
    uint32_t* out = ends + run_off[i] + colstart[(size_t)i * W + x];
    const uint32_t jbase = (uint32_t)x * (uint32_t)H;
    int t = 0;
    for (int k = 0; k < Hw; ++k) {
      const uint32_t w = col[k];
      uint32_t d = (w ^ ((w << 1) | carry)) & (k == Hw - 1 ? last_mask : 0xffffffffu);
      carry = w >> 31;
      while (d) {
        const int b = __ffs(d) - 1;
        d &= d - 1;
        out[t++] = jbase + (uint32_t)(k * 32 + b);
      }
    }
    if (x == W - 1) out[t] = (uint32_t)H * (uint32_t)W;
  }
}

// One block per mask: characters of the mask's string (sum over its runs of rle_chars) -> bytes[i]
__global__ void __launch_bounds__(kScanThreads) rle_string_len_kernel(const uint32_t* __restrict__ ends,
                                                                      const long long* __restrict__ run_off,
                                                                      long long* __restrict__ bytes) {
  const int i = blockIdx.x;
  const long long r0 = run_off[i], m = run_off[i + 1] - r0;
  const uint32_t* e = ends + r0;
  long long s = 0;
  for (long long r = threadIdx.x; r < m; r += kScanThreads) s += rle_chars(rle_value(e, r));
  long long tot;
  block_excl_scan(s, &tot);
  if (threadIdx.x == 0) bytes[i] = tot;
}

// One block per mask: rleToString.  Runs are taken in chunks of kScanThreads; a scan of the per-run character counts
// places every run's characters.
__global__ void __launch_bounds__(kScanThreads) rle_string_kernel(const uint32_t* __restrict__ ends,
                                                                  const long long* __restrict__ run_off,
                                                                  const long long* __restrict__ byte_off,
                                                                  uint8_t* __restrict__ chars) {
  const int i = blockIdx.x;
  const long long r0 = run_off[i], m = run_off[i + 1] - r0;
  const uint32_t* e = ends + r0;
  uint8_t* out = chars + byte_off[i];
  long long carry = 0;
  for (long long base = 0; base < m; base += kScanThreads) {
    const long long r = base + threadIdx.x;
    long long x = r < m ? rle_value(e, r) : 0;
    const int len = r < m ? rle_chars(x) : 0;
    long long tot;
    long long p = carry + block_excl_scan(len, &tot);
    for (int q = 0; q < len; ++q) {
      int c = (int)(x & 0x1f);
      x >>= 5;
      const bool more = (c & 0x10) ? x != -1 : x != 0;
      if (more) c |= 0x20;
      out[p++] = (uint8_t)(c + 48);
    }
    carry += tot;
  }
}

// rleFrString, one thread per mask: the string's values -> run ends (cumulative counts) at ends[byte_off[i]...]
// (a mask has at most as many runs as characters), and the run count.  Parsing stops at a NUL or the string's end.
__global__ void rle_parse_kernel(const uint8_t* __restrict__ chars, const long long* __restrict__ byte_off,
                                 uint32_t* __restrict__ ends, long long* __restrict__ nruns, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long b = byte_off[i], e = byte_off[i + 1];
  uint32_t* out = ends + b;
  long long p = b, m = 0;
  uint32_t c1 = 0, c2 = 0, acc = 0;   // cnt[m-1], cnt[m-2], running end
  while (p < e && chars[p]) {
    long long x = 0;
    int k = 0;
    bool more = true;
    while (more && p < e) {
      const int c = (int)chars[p] - 48;
      if (5 * k < 64) x |= (long long)(c & 0x1f) << (5 * k);
      more = (c & 0x20) != 0;
      ++p;
      ++k;
      if (!more && (c & 0x10) && 5 * k < 64) x |= -1LL << (5 * k);
    }
    if (m > 2) x += (long long)c2;
    const uint32_t cnt = (uint32_t)x;
    acc += cnt;
    out[m++] = acc;
    c2 = c1;
    c1 = cnt;
  }
  nruns[i] = m;
}

// rleDecode: out[i, y, x] = 1 when the run holding pixel j = x*H + y is odd (binary search in the run ends)
__global__ void __launch_bounds__(256) rle_paint_kernel(const uint32_t* __restrict__ ends, const long long* __restrict__ byte_off,
                                                        const long long* __restrict__ nruns, uint8_t* __restrict__ out,
                                                        int n, int H, int W) {
  const long long total = (long long)n * H * W;
  const long long hw = (long long)H * W;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(t / hw);
    const long long rem = t - (long long)i * hw;
    const int y = (int)(rem / W), x = (int)(rem - (long long)y * W);
    const uint32_t j = (uint32_t)x * (uint32_t)H + (uint32_t)y;
    const uint32_t* e = ends + byte_off[i];
    long long lo = 0, hi = nruns[i];   // first run whose end exceeds j
    while (lo < hi) {
      const long long mid = (lo + hi) >> 1;
      if (e[mid] > j) hi = mid;
      else lo = mid + 1;
    }
    out[t] = (uint8_t)(lo & 1);
  }
}

int grid_for(long long work_items, int threads) {
  const long long want = (work_items + threads - 1) / threads;
  const long long cap = (long long)sm_count() * 8;
  return (int)(want < 1 ? 1 : (want < cap ? want : cap));
}

int check_shape(int n, int H, int W) {
  PSALM_REQUIRE(n > 0 && H > 0 && W > 0, "rle: need n, H, W > 0 (got %d, %d, %d)", n, H, W);
  PSALM_REQUIRE((long long)H * W <= INT_MAX, "rle: H*W must fit int32 (got %d x %d)", H, W);
  return PSALM_OK;
}

}  // namespace

extern "C" size_t psalm_rle_workspace_bytes(int n, int H, int W) {
  const size_t cols = (size_t)n * W, Hw = (H + 31) / 32;
  return cols * Hw * 4 + cols * sizeof(int4) + cols * 4 + 16;
}

extern "C" int psalm_rle_count(const void* masks, const uint64_t* mask_ptrs, void* workspace, int64_t* run_off,
                               int64_t* area, double* bbox, int n, int H, int W, int dtype, void* stream) {
  if (int rc = check_shape(n, H, W)) return rc;
  PSALM_REQUIRE(masks || mask_ptrs, "psalm_rle_count: null masks");
  PSALM_REQUIRE(workspace && run_off && area && bbox, "psalm_rle_count: null output");
  PSALM_REQUIRE(dtype == PSALM_F32 || dtype == PSALM_U8, "psalm_rle_count: masks must be float32 or uint8 / bool");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t cols = (size_t)n * W, Hw = (H + 31) / 32;
  uint32_t* bits = (uint32_t*)workspace;
  int4* colstat = (int4*)(((uintptr_t)(bits + cols * Hw) + 15) & ~(uintptr_t)15);
  const long long warps = (long long)n * ((W + 31) / 32);
  const int grid = grid_for(warps * 32, 256);
  if (dtype == PSALM_F32)
    rle_count_kernel<float><<<grid, 256, 0, st>>>((const float*)masks, (const unsigned long long*)mask_ptrs, bits, colstat, n, H, W);
  else
    rle_count_kernel<uint8_t><<<grid, 256, 0, st>>>((const uint8_t*)masks, (const unsigned long long*)mask_ptrs, bits, colstat, n,
                                                   H, W);
  int* colstart = (int*)(colstat + cols);
  rle_mask_stats_kernel<<<n, kScanThreads, 0, st>>>(colstat, colstart, (long long*)run_off, (long long*)area, bbox, W);
  rle_offsets_kernel<<<1, kScanThreads, 0, st>>>((long long*)run_off, n);
  return psalm::check_launch("psalm_rle_count");
}

extern "C" int psalm_rle_runs(const void* workspace, const int64_t* run_off, uint32_t* ends, int64_t* byte_off, int n, int H,
                              int W, void* stream) {
  if (int rc = check_shape(n, H, W)) return rc;
  PSALM_REQUIRE(workspace && run_off && ends && byte_off, "psalm_rle_runs: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t cols = (size_t)n * W, Hw = (H + 31) / 32;
  const uint32_t* bits = (const uint32_t*)workspace;
  const int4* colstat = (const int4*)(((uintptr_t)(bits + cols * Hw) + 15) & ~(uintptr_t)15);
  const int* colstart = (const int*)(colstat + cols);
  const long long warps = (long long)n * ((W + 31) / 32);
  rle_ends_kernel<<<grid_for(warps * 32, 256), 256, 0, st>>>(bits, colstart, (const long long*)run_off, ends, n, H, W);
  rle_string_len_kernel<<<n, kScanThreads, 0, st>>>(ends, (const long long*)run_off, (long long*)byte_off);
  rle_offsets_kernel<<<1, kScanThreads, 0, st>>>((long long*)byte_off, n);
  return psalm::check_launch("psalm_rle_runs");
}

extern "C" int psalm_rle_strings(const uint32_t* ends, const int64_t* run_off, const int64_t* byte_off, uint8_t* chars, int n,
                                 void* stream) {
  PSALM_REQUIRE(n > 0, "psalm_rle_strings: n must be > 0");
  PSALM_REQUIRE(ends && run_off && byte_off && chars, "psalm_rle_strings: null pointer");
  rle_string_kernel<<<n, kScanThreads, 0, (cudaStream_t)stream>>>(ends, (const long long*)run_off, (const long long*)byte_off,
                                                                  chars);
  return psalm::check_launch("psalm_rle_strings");
}

extern "C" int psalm_rle_decode(const uint8_t* chars, const int64_t* byte_off, uint32_t* ends, int64_t* nruns, uint8_t* out,
                                int n, int H, int W, void* stream) {
  if (int rc = check_shape(n, H, W)) return rc;
  PSALM_REQUIRE(chars && byte_off && ends && nruns && out, "psalm_rle_decode: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  rle_parse_kernel<<<(n + 127) / 128, 128, 0, st>>>(chars, (const long long*)byte_off, ends, (long long*)nruns, n);
  rle_paint_kernel<<<grid_for((long long)n * H * W, 256), 256, 0, st>>>(ends, (const long long*)byte_off,
                                                                       (const long long*)nruns, out, n, H, W);
  return psalm::check_launch("psalm_rle_decode");
}
