// Tensor-core attention kernels for 16-bit storage (bf16 / fp16), fp32 accumulate and softmax.
//
//   flash_mma_kernel   FlashAttention-2 style: 64 query rows x 64-key tiles per CTA (4 warps), online
//                      softmax in registers, policies as in attn_simt.cu (causal prefill, masked
//                      cross-attention with packed bit masks + split-K, plain self-attention).
//   window_mma_kernel  one CTA per (Swin window, head): the whole 144 x 144 score tile lives in
//                      registers (9 warps x 16 rows), single-pass softmax, relative-position bias and
//                      the shift mask applied on the accumulators, window gather / zero padding / cyclic
//                      shift resolved once per CTA into a token table in shared memory.
// Both use warp-level mma.sync.m16n8k16 with ldmatrix operand fetch: these tiles are 144- or 64-wide with
// per-element bias / mask work in the accumulators (see DESIGN.md).
#include <type_traits>

#include <cooperative_groups.h>

#include "common.cuh"

namespace psalm {

struct AttnDims {
  int B, H, Lq, Lk, splits;
  float scale;
};

constexpr float kLog2e = 1.4426950408889634f;

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const void* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], const void* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
template <typename T>
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  if constexpr (sizeof(T) == 2 && std::is_same<T, __nv_bfloat16>::value) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  } else {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
}

// 16-byte async global->shared copy (LDGSTS); src_bytes = 0 zero-fills the destination
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, int src_bytes) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(a), "l"(gmem), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// 2^x on the SFU (MUFU.EX2), flush-to-zero: one instruction; exp2f() expands to range fix-ups around it.
// ex2.approx(-inf) = +0, which is what the masked / first-tile cases rely on.
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;\n" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ uint4 ldg16(const void* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }

// ------------------------------------------------------------------------------------------------
// policies (raw 16-byte loads = 8 elements; score(); paired stores)
// ------------------------------------------------------------------------------------------------
template <typename T>
struct CausalMma {
  const T* qkv;              // [B,T,3,nh,hd]
  const uint8_t* key_valid;  // [B,T] or null
  T* out;                    // [B,T,nh*hd]
  int T_, nh, hd;
  static constexpr bool kCausal = true;
  static constexpr bool kPrefix = false;
  __device__ __forceinline__ const T* ptr(int which, int b, int h, int n, int d0) const {
    return qkv + (((size_t)b * T_ + n) * 3 + which) * nh * hd + h * hd + d0;
  }
  __device__ __forceinline__ size_t row_stride() const { return (size_t)3 * nh * hd; }   // elements between keys
  __device__ __forceinline__ uint4 load8(int which, int b, int h, int n, int d0) const {
    return ldg16(ptr(which, b, h, n, d0));
  }
  // bit j set = key (kt*64 + j) is blocked for query row qi; kv = packed invalid-key bits of this tile
  __device__ __forceinline__ unsigned long long blocked(int b, int qi, int kt, unsigned long long kv) const {
    const int d = qi - kt * 64;   // keys with j > d are in the future
    const unsigned long long m = d >= 63 ? 0ull : (d < 0 ? ~0ull : (~0ull << (d + 1)));
    return m | kv;
  }
  __device__ __forceinline__ bool key_invalid(int b, int kj) const {
    return key_valid && !key_valid[(size_t)b * T_ + kj];
  }
  __device__ __forceinline__ void store2(int b, int h, int n, int d, float v0, float v1) const {
    *reinterpret_cast<uint32_t*>(out + ((size_t)b * T_ + n) * nh * hd + h * hd + d) = pack2<T>(v0, v1);
  }
  __device__ __forceinline__ void store(int b, int h, int n, int d, float v) const {
    out[((size_t)b * T_ + n) * nh * hd + h * hd + d] = from_f32<T>(v);
  }
};

template <typename T>
struct CrossMma {
  const T *q, *k, *v;
  const uint32_t* bits;
  const uint8_t* row_open;
  T* out;
  int Lq, Lk, nh, hd, W32;
  int kv_ld;   // elements between consecutive K (and V) rows: nh * hd, or more for views of a fused projection buffer
  long long kv_bstride;   // elements between the K (and V) rows of consecutive images: Lk * kv_ld, or 0 = one shared memory
  static constexpr bool kCausal = false;
  static constexpr bool kPrefix = false;
  __device__ __forceinline__ const T* ptr(int which, int b, int h, int n, int d0) const {
    if (which == 0) return q + ((size_t)b * Lq + n) * nh * hd + h * hd + d0;
    return (which == 1 ? k : v) + (size_t)b * kv_bstride + (size_t)n * kv_ld + h * hd + d0;
  }
  __device__ __forceinline__ size_t row_stride() const { return (size_t)kv_ld; }
  __device__ __forceinline__ uint4 load8(int which, int b, int h, int n, int d0) const {
    return ldg16(ptr(which, b, h, n, d0));
  }
  __device__ __forceinline__ unsigned long long blocked(int b, int qi, int kt, unsigned long long kv) const {
    if (!bits || qi >= Lq) return kv;
    const size_t row = (size_t)b * Lq + qi;
    if (row_open && row_open[row]) return kv;
    const uint32_t w0 = 2 * kt < W32 ? __ldg(bits + row * W32 + 2 * kt) : 0u;
    const uint32_t w1 = 2 * kt + 1 < W32 ? __ldg(bits + row * W32 + 2 * kt + 1) : 0u;
    return ((unsigned long long)w1 << 32 | w0) | kv;
  }
  __device__ __forceinline__ bool key_invalid(int b, int kj) const { return false; }
  __device__ __forceinline__ void store2(int b, int h, int n, int d, float v0, float v1) const {
    *reinterpret_cast<uint32_t*>(out + ((size_t)b * Lq + n) * nh * hd + h * hd + d) = pack2<T>(v0, v1);
  }
  __device__ __forceinline__ void store(int b, int h, int n, int d, float v) const {
    out[((size_t)b * Lq + n) * nh * hd + h * hd + d] = from_f32<T>(v);
  }
};

// Causal prefill of prompt suffixes behind a shared prefix: query t of sequence b attends the P prefix keys (head-major
// [nh, ld_rows, hd], the same for every b) and its own keys u <= t.  The virtual key axis is [prefix padded to Pt tiles
// of 64 | own keys], so that a 64-key tile is either all prefix (row stride hd) or all own keys (row stride 3 nh hd);
// keys in [P, 64 Pt) are invalid keys.
template <typename T>
struct PrefixCausalMma {
  const T* qkv;              // [B,T,3,nh,hd], rotary applied at positions P + t
  const T *pk, *pv;          // [nh, ld_rows, hd]
  const uint8_t* key_valid;  // [B,T] or null
  T* out;                    // [B,T,nh*hd]
  int T_, nh, hd, P, ld_rows, Pt;
  static constexpr bool kCausal = true;
  static constexpr bool kPrefix = true;   // the kernel's prefetch picks base and row stride per key tile
  __device__ __forceinline__ const T* ptr(int which, int b, int h, int n, int d0) const {
    return qkv + (((size_t)b * T_ + n) * 3 + which) * nh * hd + h * hd + d0;
  }
  __device__ __forceinline__ size_t row_stride() const { return (size_t)3 * nh * hd; }   // own keys
  __device__ __forceinline__ uint4 load8(int which, int b, int h, int n, int d0) const {
    return ldg16(ptr(which, b, h, n, d0));
  }
  __device__ __forceinline__ unsigned long long blocked(int b, int qi, int kt, unsigned long long kv) const {
    if (kt < Pt) return kv;
    const int d = qi - (kt - Pt) * 64;
    const unsigned long long m = d >= 63 ? 0ull : (d < 0 ? ~0ull : (~0ull << (d + 1)));
    return m | kv;
  }
  __device__ __forceinline__ bool key_invalid(int b, int kj) const {
    if (kj < Pt * 64) return kj >= P;
    return key_valid && !key_valid[(size_t)b * T_ + kj - Pt * 64];
  }
  __device__ __forceinline__ void store2(int b, int h, int n, int d, float v0, float v1) const {
    *reinterpret_cast<uint32_t*>(out + ((size_t)b * T_ + n) * nh * hd + h * hd + d) = pack2<T>(v0, v1);
  }
  __device__ __forceinline__ void store(int b, int h, int n, int d, float v) const {
    out[((size_t)b * T_ + n) * nh * hd + h * hd + d] = from_f32<T>(v);
  }
};

// ------------------------------------------------------------------------------------------------
// flash kernel: grid = (q_tiles * splits, H, B), block = 128 (4 warps x 16 query rows)
// ------------------------------------------------------------------------------------------------
// KG = key groups: the CTA has 4*KG warps; warp group `kg` walks the key tiles kt0+kg, kt0+kg+KG, ... with its
// own double-buffered K/V stages and named barrier, and the groups' (m, l, O) partials are merged through
// shared memory at the end (intra-CTA split-K).  At T ~ 900 / 100 queries the kernel is bound by the
// per-warp instruction latency of the longest CTA, so halving that CTA's tile count is what pays.
// CL = the `splits` CTAs of one (query tile, head, batch) form a thread-block cluster and reduce their (m, l, O)
// partials through distributed shared memory: no workspace round trip, no second launch.
template <typename T, int HD, typename Policy, int KG, bool CL = false>
__global__ void __launch_bounds__(128 * KG, KG == 2 ? 2 : 4) flash_mma_kernel(Policy pol, AttnDims dm, float* __restrict__ part) {
  constexpr int BQ = 64, BK = 64, LD = HD + 8;
  extern __shared__ __align__(16) unsigned char flash_smem[];
  T* Qs = reinterpret_cast<T*>(flash_smem);                                   // [BQ * LD]
  T* KVbase = Qs + BQ * LD;                                                   // [KG][2 stages][K|V][BK * LD]
  unsigned long long* kvbits = reinterpret_cast<unsigned long long*>(KVbase + KG * 4 * BK * LD);   // [128]
  const int kg = threadIdx.x >> 7;                 // key group of this warp
  const int tid = threadIdx.x & 127, warp = tid >> 5, lane = tid & 31;   // indices inside the group
  const int g = lane >> 2, t4 = lane & 3;
  // heavy (late, causal) query tiles first: better tail balance
  const int nqt = (dm.Lq + BQ - 1) / BQ;
  const int qt = nqt - 1 - (int)(blockIdx.x / dm.splits), sp = blockIdx.x % dm.splits;
  const int h = blockIdx.y, b = blockIdx.z;
  const int q0 = qt * BQ;
  const int ktiles = (dm.Lk + BK - 1) / BK;
  const int tps = (ktiles + dm.splits - 1) / dm.splits;
  const int kt0 = sp * tps;
  int kt1 = kt0 + tps < ktiles ? kt0 + tps : ktiles;
  if (Policy::kCausal) {
    int e = (q0 + BQ - 1) / BK + 1;
    if constexpr (Policy::kPrefix) e += pol.Pt;
    kt1 = e < kt1 ? e : kt1;
  }
  // ---- Q tile -> smem -> A fragments in registers
  for (int i = threadIdx.x; i < BQ * HD / 8; i += 128 * KG) {
    const int row = i / (HD / 8), d0 = (i % (HD / 8)) * 8;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (q0 + row < dm.Lq) v = pol.load8(0, b, h, q0 + row, d0);
    *reinterpret_cast<uint4*>(&Qs[row * LD + d0]) = v;
  }
  // invalid-key bits of every tile this CTA walks: one warp per tile, two keys per lane, two ballots
  for (int t = kt0 + (int)(threadIdx.x >> 5); t < kt1; t += 4 * KG) {
    const int k0 = t * BK + lane, k1 = k0 + 32;
    const uint32_t lo = __ballot_sync(0xffffffffu, k0 >= dm.Lk || pol.key_invalid(b, k0));
    const uint32_t hi = __ballot_sync(0xffffffffu, k1 >= dm.Lk || pol.key_invalid(b, k1));
    if (lane == 0) kvbits[t - kt0] = ((unsigned long long)hi << 32) | lo;
  }
  __syncthreads();
  uint32_t qa[HD / 16][4];
#pragma unroll
  for (int ks = 0; ks < HD / 16; ++ks)
    ldsm_x4(qa[ks], &Qs[(warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LD + ks * 16 + (lane >> 4) * 8]);

  float o[HD / 8][4];
#pragma unroll
  for (int i = 0; i < HD / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const int r0 = q0 + warp * 16 + g, r1 = r0 + 8;
  const float sc = dm.scale * kLog2e;   // scores are tracked in the log2 domain

  T* KVg = KVbase + (size_t)kg * 4 * BK * LD;    // this group's [2 stages][K|V] tiles
  auto group_sync = [&]() {
    if constexpr (KG == 1) __syncthreads();
    else asm volatile("bar.sync %0, 128;\n" ::"r"(1 + kg) : "memory");
  };
  // each thread owns NSLOT fixed (row, 16-byte chunk) slots of the K and V tiles: global pointers are formed
  // once and advanced by one tile stride per prefetch (no per-tile index arithmetic)
  constexpr int NSLOT = BK * HD / 8 / 128;
  const T* kbase = pol.ptr(1, b, h, 0, 0);
  const long long vdelta = pol.ptr(2, b, h, 0, 0) - kbase;      // V sits at a fixed element offset from K
  uint32_t goff[NSLOT];                                         // element offset of the slot inside a tile
#pragma unroll
  for (int j = 0; j < NSLOT; ++j) {
    const int i = tid + 128 * j;
    goff[j] = (uint32_t)((i / (HD / 8)) * (int)pol.row_stride() + (i % (HD / 8)) * 8);
  }
  const size_t tile_stride = (size_t)BK * pol.row_stride();
  auto prefetch = [&](int kt, int stage) {
    if constexpr (Policy::kPrefix) {
      // a prefix tile (shared head-major K / V, row stride HD) or a tile of the sequence's own keys (row stride 3 nh hd)
      const bool pre = kt < pol.Pt;
      const size_t rs = pre ? (size_t)HD : (size_t)3 * pol.nh * HD;
      const T* kb = pre ? pol.pk + ((size_t)h * pol.ld_rows + (size_t)kt * BK) * HD : pol.ptr(1, b, h, (kt - pol.Pt) * BK, 0);
      const T* vb = pre ? pol.pv + ((size_t)h * pol.ld_rows + (size_t)kt * BK) * HD : kb + (size_t)pol.nh * HD;
      const int left = pre ? pol.P - kt * BK : pol.T_ - (kt - pol.Pt) * BK;
#pragma unroll
      for (int j = 0; j < NSLOT; ++j) {
        const int i = tid + 128 * j;
        const int row = i / (HD / 8), c8 = (i % (HD / 8)) * 8;
        const int so = row * LD + c8;
        const bool ok = row < left;
        const size_t go = (size_t)row * rs + c8;
        cp_async16(&KVg[(stage * 2 + 0) * BK * LD + so], ok ? kb + go : pol.qkv, ok ? 16 : 0);
        cp_async16(&KVg[(stage * 2 + 1) * BK * LD + so], ok ? vb + go : pol.qkv, ok ? 16 : 0);
      }
      cp_async_commit();
      return;
    }
    const T* kt_base = kbase + (size_t)kt * tile_stride;
    const int left = dm.Lk - kt * BK;   // keys of this tile that exist
#pragma unroll
    for (int j = 0; j < NSLOT; ++j) {
      const int i = tid + 128 * j;
      const int row = i / (HD / 8);
      const int so = row * LD + (i % (HD / 8)) * 8;
      const bool ok = row < left;
      const T* src = ok ? kt_base + goff[j] : kbase;
      cp_async16(&KVg[(stage * 2 + 0) * BK * LD + so], src, ok ? 16 : 0);
      cp_async16(&KVg[(stage * 2 + 1) * BK * LD + so], src + vdelta, ok ? 16 : 0);
    }
    cp_async_commit();
  };
  const int ktg0 = kt0 + kg;
  if (ktg0 < kt1) prefetch(ktg0, 0);
  int itn = 0;
  for (int kt = ktg0; kt < kt1; kt += KG, ++itn) {
    const int stage = itn & 1;
    if (kt + KG < kt1) {
      prefetch(kt + KG, stage ^ 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    group_sync();
    const T* Ks = KVg + (stage * 2 + 0) * BK * LD;
    const T* Vs = KVg + (stage * 2 + 1) * BK * LD;
    float s[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < HD / 16; ++ks) {
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        uint32_t kb[4];
        const int mi = lane >> 3;
        ldsm_x4(kb, &Ks[(np * 16 + (lane & 7) + (mi >> 1) * 8) * LD + ks * 16 + (mi & 1) * 8]);
        mma16816<T>(s[2 * np], qa[ks], kb[0], kb[1]);
        mma16816<T>(s[2 * np + 1], qa[ks], kb[2], kb[3]);
      }
    }
    // ---- masks (bit tests against per-row 64-key masks; skipped when the whole tile is open),
    //      online softmax in the log2 domain
    const unsigned long long kv = kvbits[kt - kt0];
    const unsigned long long bm0 = pol.blocked(b, r0, kt, kv) >> (2 * t4);
    const unsigned long long bm1 = pol.blocked(b, r1, kt, kv) >> (2 * t4);
    const bool any_blocked = __any_sync(0xffffffffu, (bm0 | bm1) != 0ull);
    float tmax[2] = {-INFINITY, -INFINITY};
    if (!any_blocked) {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          s[nt][e] *= sc;
          tmax[e >> 1] = fmaxf(tmax[e >> 1], s[nt][e]);
        }
      }
    } else {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const unsigned long long bm = (e < 2) ? bm0 : bm1;
          const bool blk = (bm >> (nt * 8 + (e & 1))) & 1ull;
          s[nt][e] = blk ? -INFINITY : s[nt][e] * sc;
          tmax[e >> 1] = fmaxf(tmax[e >> 1], s[nt][e]);
        }
      }
    }
    float corr[2], msub[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      tmax[r] = fmaxf(tmax[r], __shfl_xor_sync(0xffffffffu, tmax[r], 1));
      tmax[r] = fmaxf(tmax[r], __shfl_xor_sync(0xffffffffu, tmax[r], 2));
      const float m_new = fmaxf(m_run[r], tmax[r]);
      corr[r] = (m_new == -INFINITY) ? 1.f : fast_exp2(m_run[r] - m_new);   // exp2f(-inf) = 0 for the first tile
      msub[r] = (m_new == -INFINITY) ? 0.f : m_new;                     // avoids (-inf) - (-inf)
      m_run[r] = m_new;
    }
    float psum[2] = {0.f, 0.f};
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float p = fast_exp2(s[nt][e] - msub[e >> 1]);   // blocked: 2^(-inf) = 0
        s[nt][e] = p;
        psum[e >> 1] += p;
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      psum[r] += __shfl_xor_sync(0xffffffffu, psum[r], 1);
      psum[r] += __shfl_xor_sync(0xffffffffu, psum[r], 2);
      l_run[r] = l_run[r] * corr[r] + psum[r];
    }
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) {
      o[i][0] *= corr[0]; o[i][1] *= corr[0];
      o[i][2] *= corr[1]; o[i][3] *= corr[1];
    }
    // ---- O += P V
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t pa[4];
      pa[0] = pack2<T>(s[2 * kk][0], s[2 * kk][1]);
      pa[1] = pack2<T>(s[2 * kk][2], s[2 * kk][3]);
      pa[2] = pack2<T>(s[2 * kk + 1][0], s[2 * kk + 1][1]);
      pa[3] = pack2<T>(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
      for (int dp = 0; dp < HD / 16; ++dp) {
        uint32_t vb[4];
        const int mi = lane >> 3;
        ldsm_x4_t(vb, &Vs[(kk * 16 + (lane & 7) + (mi & 1) * 8) * LD + dp * 16 + (mi >> 1) * 8]);
        mma16816<T>(o[2 * dp], pa, vb[0], vb[1]);
        mma16816<T>(o[2 * dp + 1], pa, vb[2], vb[3]);
      }
    }
    group_sync();   // every warp of the group is done with this stage before it is refilled
  }
  if constexpr (KG == 2) {
    // ---- merge the two key groups: group 1 parks (m, l, O) in shared memory, group 0 combines
    __syncthreads();
    float* xch = reinterpret_cast<float*>(KVbase) + (size_t)tid * (4 + HD / 2);
    if (kg == 1) {
      xch[0] = m_run[0]; xch[1] = m_run[1]; xch[2] = l_run[0]; xch[3] = l_run[1];
#pragma unroll
      for (int i = 0; i < HD / 8; ++i) {
        xch[4 + 4 * i] = o[i][0]; xch[5 + 4 * i] = o[i][1]; xch[6 + 4 * i] = o[i][2]; xch[7 + 4 * i] = o[i][3];
      }
    }
    __syncthreads();
    if (!CL && kg == 1) return;
    if (kg == 0) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float m1 = xch[r], l1 = xch[2 + r];
      const float mm = fmaxf(m_run[r], m1);
      const float c0 = (m_run[r] == -INFINITY) ? 0.f : exp2f(m_run[r] - mm);
      const float c1 = (m1 == -INFINITY) ? 0.f : exp2f(m1 - mm);
      l_run[r] = l_run[r] * c0 + l1 * c1;
      m_run[r] = mm;
#pragma unroll
      for (int i = 0; i < HD / 8; ++i) {
        o[i][2 * r] = o[i][2 * r] * c0 + xch[4 + 4 * i + 2 * r] * c1;
        o[i][2 * r + 1] = o[i][2 * r + 1] * c0 + xch[5 + 4 * i + 2 * r] * c1;
      }
    }
    }
  }
  // ---- epilogue
  if constexpr (CL) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    constexpr int RW = HD + 2;                         // row of the exchange buffer: O[HD], m, l
    float* red = reinterpret_cast<float*>(KVbase);     // [BQ][RW]; the K/V stages are dead by now
    __syncthreads();                                   // (KG == 2: group 0 has consumed xch)
    if (kg == 0) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        float* pr = red + (warp * 16 + g + 8 * r) * RW;
#pragma unroll
        for (int i = 0; i < HD / 8; ++i) {
          pr[i * 8 + 2 * t4] = o[i][2 * r];
          pr[i * 8 + 2 * t4 + 1] = o[i][2 * r + 1];
        }
        if (t4 == 0) {
          pr[HD] = m_run[r];
          pr[HD + 1] = l_run[r];
        }
      }
    }
    cluster.sync();
    // CTA `rank` finishes rows rank, rank + splits, ...: one thread per (row, channel)
    const int rank = (int)cluster.block_rank(), nr = (int)cluster.num_blocks();
    const int rows_mine = (BQ - rank + nr - 1) / nr;
    for (int idx = threadIdx.x; idx < rows_mine * HD; idx += 128 * KG) {
      const int row = rank + (idx / HD) * nr, d = idx % HD;
      const int qi = q0 + row;
      if (qi >= dm.Lq) continue;
      float M = -INFINITY;
      for (int s2 = 0; s2 < nr; ++s2) M = fmaxf(M, cluster.map_shared_rank(red, s2)[row * RW + HD]);
      float L = 0.f, O = 0.f;
      if (M != -INFINITY) {
        for (int s2 = 0; s2 < nr; ++s2) {
          const float* rr = cluster.map_shared_rank(red, s2) + row * RW;
          const float ms = rr[HD];
          const float e = (ms == -INFINITY) ? 0.f : exp2f(ms - M);
          L += rr[HD + 1] * e;
          O += rr[d] * e;
        }
      }
      pol.store(b, h, qi, d, L > 0.f ? O / L : 0.f);
    }
    cluster.sync();   // nobody leaves while its shared memory may still be read remotely
    return;
  }
  if (dm.splits == 1) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int qi = r ? r1 : r0;
      if (qi >= dm.Lq) continue;
      const float inv = l_run[r] > 0.f ? 1.f / l_run[r] : 0.f;
#pragma unroll
      for (int i = 0; i < HD / 8; ++i) pol.store2(b, h, qi, i * 8 + 2 * t4, o[i][2 * r] * inv, o[i][2 * r + 1] * inv);
    }
  } else {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int qi = r ? r1 : r0;
      if (qi >= dm.Lq) continue;
      float* pr = part + ((((size_t)b * dm.H + h) * dm.splits + sp) * dm.Lq + qi) * (HD + 2);
#pragma unroll
      for (int i = 0; i < HD / 8; ++i) {
        pr[i * 8 + 2 * t4] = o[i][2 * r];
        pr[i * 8 + 2 * t4 + 1] = o[i][2 * r + 1];
      }
      if (t4 == 0) {
        pr[HD] = m_run[r];      // log2 domain
        pr[HD + 1] = l_run[r];
      }
    }
  }
}

template <typename Policy, int HD>
__global__ void flash_combine_kernel(Policy pol, AttnDims dm, const float* __restrict__ part) {
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
        const float e = exp2f(ms - M);
        L += base[s * stride + HD + 1] * e;
        O += base[s * stride + d] * e;
      }
    }
    pol.store(b, h, qi, d, L > 0.f ? O / L : 0.f);
  }
}

// ------------------------------------------------------------------------------------------------
// Swin window kernel: grid = (B*nW, nh), block = 288 (9 warps), N = 144 tokens, head_dim 32
// ------------------------------------------------------------------------------------------------
// keys [16 NP0, 16 NP1) of one window for the 16 query rows of a warp: S = Q K^T, + bias (+ shift mask), running max /
// sum update, O = O * alpha + P V.  LD = 40 (32 + 8 padding), scores in the log2 domain.
template <typename T, int NP0, int NP1>
__device__ __forceinline__ void win_keys(const T* __restrict__ Ks, const T* __restrict__ Vs, const uint32_t (&qa)[2][4],
                                         const float* __restrict__ rc0, const float* __restrict__ rc1,
                                         const short* __restrict__ coff, const unsigned char* __restrict__ reg, int reg0,
                                         int reg1, bool wmask, float scl, int lane, int t4, float (&o)[4][4],
                                         float (&mrun)[2], float (&sum)[2]) {
  constexpr int LD = 40, NT = 2 * (NP1 - NP0);
  float s[NT][4];
#pragma unroll
  for (int i = 0; i < NT; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) {
#pragma unroll
    for (int np = NP0; np < NP1; ++np) {
      uint32_t kb[4];
      const int mi = lane >> 3;
      ldsm_x4(kb, &Ks[(np * 16 + (lane & 7) + (mi >> 1) * 8) * LD + ks * 16 + (mi & 1) * 8]);
      mma16816<T>(s[2 * (np - NP0)], qa[ks], kb[0], kb[1]);
      mma16816<T>(s[2 * (np - NP0) + 1], qa[ks], kb[2], kb[3]);
    }
  }
  float mx[2] = {mrun[0], mrun[1]};
  if (!wmask) {                    // window does not touch the wrapped border: no shift mask (warp-uniform)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const int kj = (2 * NP0 + nt) * 8 + 2 * t4;
      const int c2 = *reinterpret_cast<const int*>(&coff[kj]);   // column offsets of keys kj, kj + 1
      const int ca = (short)(c2 & 0xffff), cb = c2 >> 16;
      s[nt][0] = fmaf(s[nt][0], scl, rc0[ca]);
      s[nt][1] = fmaf(s[nt][1], scl, rc0[cb]);
      s[nt][2] = fmaf(s[nt][2], scl, rc1[ca]);
      s[nt][3] = fmaf(s[nt][3], scl, rc1[cb]);
      mx[0] = fmaxf(mx[0], fmaxf(s[nt][0], s[nt][1]));
      mx[1] = fmaxf(mx[1], fmaxf(s[nt][2], s[nt][3]));
    }
  } else {
    constexpr float kNeg = -100.f * kLog2e;   // the reference's additive -100 (swin_trans.py:232-240)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const int kj = (2 * NP0 + nt) * 8 + 2 * t4;
      const int c2 = *reinterpret_cast<const int*>(&coff[kj]);
      const int ca = (short)(c2 & 0xffff), cb = c2 >> 16;
      const int ra = reg[kj], rb = reg[kj + 1];
      s[nt][0] = fmaf(s[nt][0], scl, rc0[ca]) + (ra != reg0 ? kNeg : 0.f);
      s[nt][1] = fmaf(s[nt][1], scl, rc0[cb]) + (rb != reg0 ? kNeg : 0.f);
      s[nt][2] = fmaf(s[nt][2], scl, rc1[ca]) + (ra != reg1 ? kNeg : 0.f);
      s[nt][3] = fmaf(s[nt][3], scl, rc1[cb]) + (rb != reg1 ? kNeg : 0.f);
      mx[0] = fmaxf(mx[0], fmaxf(s[nt][0], s[nt][1]));
      mx[1] = fmaxf(mx[1], fmaxf(s[nt][2], s[nt][3]));
    }
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
  }
  if (NP0 > 0) {   // scores are finite (bias and the -100 mask are finite), so mx is finite from the first call on
    const float a0 = fast_exp2(mrun[0] - mx[0]), a1 = fast_exp2(mrun[1] - mx[1]);
    sum[0] *= a0;
    sum[1] *= a1;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      o[i][0] *= a0; o[i][1] *= a0;
      o[i][2] *= a1; o[i][3] *= a1;
    }
  }
  mrun[0] = mx[0];
  mrun[1] = mx[1];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    s[nt][0] = fast_exp2(s[nt][0] - mx[0]); s[nt][1] = fast_exp2(s[nt][1] - mx[0]);
    s[nt][2] = fast_exp2(s[nt][2] - mx[1]); s[nt][3] = fast_exp2(s[nt][3] - mx[1]);
    sum[0] += s[nt][0] + s[nt][1];
    sum[1] += s[nt][2] + s[nt][3];
  }
#pragma unroll
  for (int kk = NP0; kk < NP1; ++kk) {
    const int k2 = 2 * (kk - NP0);
    uint32_t pa[4];
    pa[0] = pack2<T>(s[k2][0], s[k2][1]);
    pa[1] = pack2<T>(s[k2][2], s[k2][3]);
    pa[2] = pack2<T>(s[k2 + 1][0], s[k2 + 1][1]);
    pa[3] = pack2<T>(s[k2 + 1][2], s[k2 + 1][3]);
#pragma unroll
    for (int dp = 0; dp < 2; ++dp) {
      uint32_t vb[4];
      const int mi = lane >> 3;
      ldsm_x4_t(vb, &Vs[(kk * 16 + (lane & 7) + (mi & 1) * 8) * LD + dp * 16 + (mi >> 1) * 8]);
      mma16816<T>(o[2 * dp], pa, vb[0], vb[1]);
      mma16816<T>(o[2 * dp + 1], pa, vb[2], vb[3]);
    }
  }
}

template <typename T, int HPC>
__global__ void __launch_bounds__(288, 3) window_mma_kernel(const T* __restrict__ qkv, const T* __restrict__ qkv_bias,
                                                            const float* __restrict__ rel, T* __restrict__ out,
                                                            int H, int W, int Hp, int Wp, int shift, int nh, int C,
                                                            int nWx, int nW) {
  // One CTA = one window x HPC consecutive heads; the Q/K/V tiles of head i+1 stream in with cp.async
  // while head i is computed (the un-pipelined version spent 30 % of its stall samples waiting on the
  // tile fill, profiles/r1c_window_mma_ncu_details.txt).
  constexpr int N = 144, WS = 12, HD = 32, LD = HD + 8;
  extern __shared__ __align__(16) unsigned char win_smem[];
  T* bufs = reinterpret_cast<T*>(win_smem);                     // [2 stages][3: q,k,v][N * LD]
  int* tok = reinterpret_cast<int*>(bufs + 2 * 3 * N * LD);     // [N]
  unsigned char* reg = reinterpret_cast<unsigned char*>(tok + N);  // [N]
  // The relative-position bias of a head has only (2 WS - 1)^2 = 529 distinct values (swin_trans.py:98-114 gathers
  // them into a dense [N, N] table: 83 KB of L2 traffic per (window, head), 11x the q/k/v bytes).  The ABI takes
  // the compact table; its 529 values are staged once per head into shared memory (pre-multiplied by log2e)
  // and indexed with (row base + column offset).
  constexpr int NREL = (2 * WS - 1) * (2 * WS - 1);
  float* relc = reinterpret_cast<float*>(reg + N);               // [2 stages][NREL + 3]
  short* coff = reinterpret_cast<short*>(relc + 2 * (NREL + 3)); // [N] column part of the compact index
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t4 = lane & 3;
  const int z = blockIdx.x, h0 = blockIdx.y * HPC;
  if (tid < N) {  // window gather: cyclic shift + zero padding resolved once (swin_trans.py:207-225)
    const int win = z % nW, bi = z / nW;
    const int wy = win / nWx, wx = win - wy * nWx;
    const int i = tid / WS, j = tid - i * WS;
    const int py = wy * WS + i, px = wx * WS + j;
    const int rh = py < Hp - WS ? 0 : (py < Hp - shift ? 1 : 2);
    const int rw = px < Wp - WS ? 0 : (px < Wp - shift ? 1 : 2);
    reg[tid] = (unsigned char)(rh * 3 + rw);
    int oy = py + shift, ox = px + shift;
    if (oy >= Hp) oy -= Hp;
    if (ox >= Wp) ox -= Wp;
    tok[tid] = (oy < H && ox < W) ? (bi * H + oy) * W + ox : -1;
    coff[tid] = (short)(-(i * (2 * WS - 1) + j));
  }
  // the -100 shift mask only exists in windows of the last window row / column (they hold several regions)
  const int win_ = z % nW;
  const bool wmask = shift > 0 && (win_ / nWx == nW / nWx - 1 || win_ % nWx == nWx - 1);
  __syncthreads();
  auto prefetch = [&](int h, int stage) {
    T* dst0 = bufs + (size_t)stage * 3 * N * LD;
    for (int i = tid; i < N * 3 * (HD / 8); i += 288) {
      const int which = i / (N * (HD / 8));
      const int rem = i - which * (N * (HD / 8));
      const int row = rem / (HD / 8), d0 = (rem % (HD / 8)) * 8;
      const int col = which * C + h * HD + d0;
      const int tk = tok[row];
      const T* src = tk >= 0 ? qkv + (size_t)tk * 3 * C + col : qkv_bias + col;
      cp_async16(dst0 + (size_t)which * N * LD + row * LD + d0, src, 16);
    }
    cp_async_commit();
  };
  auto load_rel = [&](int h, int stage) {   // compact bias table of head h ((2 WS - 1)^2 entries, index = swin_trans.py:93-103)
    for (int c = tid; c < NREL; c += 288)
      relc[stage * (NREL + 3) + c] = __ldg(rel + (size_t)h * NREL + c) * kLog2e;
  };
  prefetch(h0, 0);
  load_rel(h0, 0);
  const float sc = rsqrtf((float)HD);
  const int r0 = warp * 16 + g, r1 = r0 + 8;
  const int rb0 = (r0 / WS + WS - 1) * (2 * WS - 1) + (r0 % WS) + WS - 1;   // row part of the compact bias index
  const int rb1 = (r1 / WS + WS - 1) * (2 * WS - 1) + (r1 % WS) + WS - 1;
  const int reg0 = reg[r0], reg1 = reg[r1];
  const int tk0 = tok[r0], tk1 = tok[r1];
#pragma unroll 1
  for (int hi = 0; hi < HPC; ++hi) {
    const int h = h0 + hi, stage = hi & 1;
    if (hi + 1 < HPC) {
      prefetch(h + 1, stage ^ 1);
      load_rel(h + 1, stage ^ 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const T* Qs = bufs + (size_t)stage * 3 * N * LD;
    const T* Ks = Qs + N * LD;
    const T* Vs = Ks + N * LD;
    uint32_t qa[2][4];
#pragma unroll
    for (int ks = 0; ks < 2; ++ks)
      ldsm_x4(qa[ks], &Qs[(warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LD + ks * 16 + (lane >> 4) * 8]);
    // The 144 keys are processed as 80 + 64 with a running (max, sum) and one rescale of the output accumulators:
    // 40 score registers per thread instead of 72, which brings the kernel from 96 to <= 72 registers = 3 CTAs per SM
    // (27 warps instead of 18; the kernel is latency bound, profiles/r1m_window_mma_stage2_ncu_details.txt).
    const float* rc0 = relc + stage * (NREL + 3) + rb0;
    const float* rc1 = relc + stage * (NREL + 3) + rb1;
    const float scl = sc * kLog2e;   // scores go straight to the log2 domain: s * scale * log2e + bias * log2e
    float o[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    float mrun[2] = {-INFINITY, -INFINITY}, sum[2] = {0.f, 0.f};
    win_keys<T, 0, 5>(Ks, Vs, qa, rc0, rc1, coff, reg, reg0, reg1, wmask, scl, lane, t4, o, mrun, sum);
    win_keys<T, 5, 9>(Ks, Vs, qa, rc0, rc1, coff, reg, reg0, reg1, wmask, scl, lane, t4, o, mrun, sum);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], 1);
      sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], 2);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int tk = r ? tk1 : tk0;
      if (tk < 0) continue;  // padded token: cropped (swin_trans.py:244-245)
      const float inv = 1.f / sum[r];
#pragma unroll
      for (int i = 0; i < 4; ++i)
        *reinterpret_cast<uint32_t*>(out + (size_t)tk * C + h * HD + i * 8 + 2 * t4) =
            pack2<T>(o[i][2 * r] * inv, o[i][2 * r + 1] * inv);
    }
    __syncthreads();   // this stage is refilled two iterations later
  }
}

// ------------------------------------------------------------------------------------------------
// host launchers used by the C-ABI entry points in attn_simt.cu
// ------------------------------------------------------------------------------------------------
template <typename T, int HD, typename Policy, int KG>
static void launch_flash_kg(const Policy& pol, AttnDims dm, float* workspace, cudaStream_t st) {
  constexpr size_t smem = sizeof(T) * (64 * (HD + 8) + (size_t)KG * 4 * 64 * (HD + 8)) + sizeof(unsigned long long) * 128;
  static PerDevice once;   // per instantiation and per device
  if (once.first()) {
    cudaFuncSetAttribute(flash_mma_kernel<T, HD, Policy, KG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaFuncSetAttribute(flash_mma_kernel<T, HD, Policy, KG>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
  }
  dim3 grid(((dm.Lq + 63) / 64) * dm.splits, dm.H, dm.B);
  flash_mma_kernel<T, HD, Policy, KG><<<grid, 128 * KG, smem, st>>>(pol, dm, workspace);
}

// cluster split-K: cluster = the `splits` CTAs of one (query tile, head, batch); returns false if the launch
// configuration is not schedulable on this device (caller falls back to workspace + combine kernel)
template <typename T, int HD, typename Policy, int KG>
static bool launch_flash_cluster(const Policy& pol, AttnDims dm, cudaStream_t st) {
  constexpr size_t smem = sizeof(T) * (64 * (HD + 8) + (size_t)KG * 4 * 64 * (HD + 8)) + sizeof(unsigned long long) * 128;
  auto kern = flash_mma_kernel<T, HD, Policy, KG, true>;
  static PerDevice probe_state;   // per instantiation and device: largest cluster size proven schedulable
  const bool first_here = probe_state.first();
  int& max_cluster = probe_state.v[PerDevice::dev()];
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(((dm.Lq + 63) / 64) * dm.splits, dm.H, dm.B);
  cfg.blockDim = dim3(128 * KG);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = dm.splits;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  if (first_here) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    max_cluster = 0;
    for (int cs = 16; cs >= 2; cs >>= 1) {
      cudaLaunchConfig_t probe = cfg;
      cudaLaunchAttribute pa[1] = {at[0]};
      pa[0].val.clusterDim.x = cs;
      probe.gridDim = dim3(cs, 1, 1);
      probe.attrs = pa;
      int n = 0;
      if (cudaOccupancyMaxActiveClusters(&n, kern, &probe) == cudaSuccess && n > 0) {
        max_cluster = cs;
        break;
      }
    }
    cudaGetLastError();   // a failed probe is not an error of the call
  }
  if (dm.splits > max_cluster) return false;
  return cudaLaunchKernelEx(&cfg, kern, pol, dm, (float*)nullptr) == cudaSuccess;
}

// split-K reduction of the masked cross-attention: 0 = auto (thread-block cluster + DSMEM for <= 4 splits, where one
// launch beats two; workspace + combine kernel above that: large clusters schedule slowly), 1 = always workspace,
// 2 = always cluster (when schedulable).  Set through psalm_set_attention_impl.
int g_splitk_mode = 0;

template <typename T, typename Policy>
static int launch_flash(const Policy& pol, AttnDims dm, int hd, float* workspace, cudaStream_t st, const char* what) {
  PSALM_REQUIRE(dm.H <= 65535 && dm.B <= 65535, "%s: grid too large", what);
  PSALM_REQUIRE(dm.splits == 1 || workspace != nullptr, "%s: split-K needs a workspace", what);
  PSALM_REQUIRE(((dm.Lk + 63) / 64 + dm.splits - 1) / dm.splits <= 128,
                "%s: more than 128 key tiles per split (Lk=%d, splits=%d): raise splits", what, dm.Lk, dm.splits);
  // two key groups per CTA once a CTA would otherwise walk more than two key tiles
  const bool kg2 = ((dm.Lk + 63) / 64 + dm.splits - 1) / dm.splits > 2;
  if constexpr (!Policy::kCausal) {
    // masked cross-attention (head_dim 32), split-K: reduce inside a thread-block cluster when it can be scheduled
    if (hd == 32 && dm.splits > 1 && dm.splits <= 16 && (g_splitk_mode == 2 || (g_splitk_mode == 0 && dm.splits <= 4))) {
      const bool ok = kg2 ? launch_flash_cluster<T, 32, Policy, 2>(pol, dm, st) : launch_flash_cluster<T, 32, Policy, 1>(pol, dm, st);
      if (ok) return check_launch(what);
      cudaGetLastError();
    }
  }
  if (hd == 32) {
    if (kg2) launch_flash_kg<T, 32, Policy, 2>(pol, dm, workspace, st);
    else launch_flash_kg<T, 32, Policy, 1>(pol, dm, workspace, st);
    if (dm.splits > 1) flash_combine_kernel<Policy, 32><<<132 * 2, 256, 0, st>>>(pol, dm, workspace);
  } else if (hd == 64) {
    if (kg2) launch_flash_kg<T, 64, Policy, 2>(pol, dm, workspace, st);
    else launch_flash_kg<T, 64, Policy, 1>(pol, dm, workspace, st);
    if (dm.splits > 1) flash_combine_kernel<Policy, 64><<<132 * 2, 256, 0, st>>>(pol, dm, workspace);
  } else {
    set_error("%s: head_dim %d unsupported by the tensor-core path", what, hd);
    return PSALM_E_UNSUPPORTED;
  }
  return check_launch(what);
}

int mma_causal_attention(const void* qkv, const uint8_t* key_valid, void* out, int B, int T_, int nh, int hd,
                         int dtype, cudaStream_t st) {
  AttnDims dm{B, nh, T_, T_, 1, 1.0f / sqrtf((float)hd)};
  if (dtype == PSALM_BF16) {
    CausalMma<__nv_bfloat16> pol{(const __nv_bfloat16*)qkv, key_valid, (__nv_bfloat16*)out, T_, nh, hd};
    return launch_flash<__nv_bfloat16>(pol, dm, hd, nullptr, st, "causal_attention(mma)");
  }
  CausalMma<__half> pol{(const __half*)qkv, key_valid, (__half*)out, T_, nh, hd};
  return launch_flash<__half>(pol, dm, hd, nullptr, st, "causal_attention(mma)");
}

int mma_cross_attention(const void* q, const void* k, const void* v, const uint32_t* bits, const uint8_t* row_open,
                        void* out, float* workspace, int B, int Lq, int Lk, int nh, int hd, int splits, int dtype,
                        cudaStream_t st, int kv_ld, long long kv_bstride) {
  if (kv_ld <= 0) kv_ld = nh * hd;
  if (kv_bstride < 0) kv_bstride = (long long)Lk * kv_ld;
  AttnDims dm{B, nh, Lq, Lk, splits, 1.0f / sqrtf((float)hd)};
  if (dtype == PSALM_BF16) {
    using T = __nv_bfloat16;
    CrossMma<T> pol{(const T*)q, (const T*)k, (const T*)v, bits, row_open, (T*)out, Lq, Lk, nh, hd, (Lk + 31) / 32, kv_ld, kv_bstride};
    return launch_flash<T>(pol, dm, hd, workspace, st, "cross_attention(mma)");
  }
  using T = __half;
  CrossMma<T> pol{(const T*)q, (const T*)k, (const T*)v, bits, row_open, (T*)out, Lq, Lk, nh, hd, (Lk + 31) / 32, kv_ld, kv_bstride};
  return launch_flash<T>(pol, dm, hd, workspace, st, "cross_attention(mma)");
}

int mma_prefix_causal_attention(const void* qkv, const void* pk, const void* pv, int P, int ld_rows, const uint8_t* key_valid,
                                void* out, int B, int T_, int nh, int hd, int dtype, cudaStream_t st) {
  const int Pt = (P + 63) / 64;
  AttnDims dm{B, nh, T_, Pt * 64 + T_, 1, 1.0f / sqrtf((float)hd)};
  if (dtype == PSALM_BF16) {
    using T = __nv_bfloat16;
    PrefixCausalMma<T> pol{(const T*)qkv, (const T*)pk, (const T*)pv, key_valid, (T*)out, T_, nh, hd, P, ld_rows, Pt};
    return launch_flash<T>(pol, dm, hd, nullptr, st, "prefix_causal_attention(mma)");
  }
  using T = __half;
  PrefixCausalMma<T> pol{(const T*)qkv, (const T*)pk, (const T*)pv, key_valid, (T*)out, T_, nh, hd, P, ld_rows, Pt};
  return launch_flash<T>(pol, dm, hd, nullptr, st, "prefix_causal_attention(mma)");
}

template <typename T>
static int launch_window(const void* qkv, const void* qkv_bias, const float* rel, void* out, int B, int H, int W, int C,
                         int nh, int shift, cudaStream_t st) {
  const int ws = 12;
  const int Hp = (H + ws - 1) / ws * ws, Wp = (W + ws - 1) / ws * ws;
  const int nWx = Wp / ws, nW = nWx * (Hp / ws);
  constexpr size_t smem = sizeof(T) * 2 * 3 * 144 * 40 + sizeof(int) * 144 + 144 + sizeof(float) * 2 * (529 + 3) + sizeof(short) * 144;
#define WIN(HPC)                                                                                                  \
  do {                                                                                                            \
    static PerDevice once;                                                                                        \
    if (once.first()) {                                                                                           \
      cudaFuncSetAttribute(window_mma_kernel<T, HPC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);    \
      cudaFuncSetAttribute(window_mma_kernel<T, HPC>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);       \
    }                                                                                                             \
    dim3 grid(B * nW, nh / HPC);                                                                                  \
    window_mma_kernel<T, HPC><<<grid, 288, smem, st>>>((const T*)qkv, (const T*)qkv_bias, rel, (T*)out, H, W, Hp,   \
                                                      Wp, shift, nh, C, nWx, nW);                                 \
  } while (0)
  // enough CTAs for >= 2 waves of 132 SMs x 3 CTAs, otherwise prefer deeper per-CTA pipelining
  const long long windows = (long long)B * nW;
  if (nh % 4 == 0 && windows * (nh / 4) >= 600) WIN(4);
  else if (nh % 2 == 0 && windows * (nh / 2) >= 132) WIN(2);
  else WIN(1);
#undef WIN
  return check_launch("window_mma_kernel");
}

int mma_window_attention(const void* qkv, const void* qkv_bias, const float* rel, void* out, int B, int H, int W,
                         int C, int nh, int shift, int dtype, cudaStream_t st) {
  PSALM_REQUIRE(nh <= 65535, "window_attention: too many heads");
  if (dtype == PSALM_BF16) return launch_window<__nv_bfloat16>(qkv, qkv_bias, rel, out, B, H, W, C, nh, shift, st);
  return launch_window<__half>(qkv, qkv_bias, rel, out, B, H, W, C, nh, shift, st);
}

}  // namespace psalm
