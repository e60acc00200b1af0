// Masked cross-attention of the Mask2Former decoder (100 queries x HW keys, 8 heads x 32), flash-decoding style,
// fed by TMA.
//
// Replaces nn.MultiheadAttention with a float -inf mask of shape [B*8, 100, HW] and materialised probabilities
// (transformer_decoder/mask2former_transformer_decoder.py:93-105, :35-45 of CrossAttentionLayer.forward_post).
//
// Why a second kernel next to flash_mma_kernel<CrossMma> (attn_mma.cu): that one gives a CTA one head and 64 query
// rows, so at 100 queries the grid is B*8*2*splits CTAs of ~50 dependent key tiles each, every K/V row is fetched as
// a 64-byte fragment of a 512-byte row, the mask words are fetched per head, and it ran at 0.05-0.10 of the HBM
// roofline (profiles/r1j_cross_attention_16k_ncu_details.txt: 0.86 waves, 62 % of cycles without an eligible warp).
// Here:
//   * a CTA owns 4 heads of one key range of one image (two CTAs per SM): K/V rows are consumed in 256-byte
//     pieces, the packed mask words are fetched once per CTA and shared by its heads (the mask is head
//     independent, :754-759);
//   * K/V tiles [32 keys x 256 channels] arrive through TMA (cp.async.bulk.tensor.2d, SWIZZLE_128B boxes of
//     [32 x 64]) into a 4-stage mbarrier ring; one elected lane of warp 0 issues the 8 bulk copies of a tile three
//     steps ahead: no per-thread address arithmetic, no cp.async groups, conflict-free ldmatrix straight from the
//     swizzled image;
//   * two warps per head: rows 0-63 (4 m-tiles) and 64-111 (3 m-tiles, 112 >= 100 rows); a warp keeps the K
//     fragments of the stage in registers and sweeps its m-tiles over them; <= 128 registers per thread so that
//     16 warps (4 per SM sub-partition) hide the HMMA -> shuffle -> MUFU dependency chains of each other (the first
//     version, one warp per head x 7 m-tiles at 240 registers, issued 0.27 instructions per cycle per scheduler:
//     profiles/r2a_xattn_v1_ncu.txt);
//   * the softmax runs in the log2 domain on pre-scaled Q (q * scale * log2e folded into the Q staging); the score
//     accumulators start from minus the row's running reference, so exp2 applies to them directly; the reference is
//     raised (warp vote) only when a score exceeds it by 2^8; row sums stay lane-private until the epilogue;
//     (m-tile, key tile) pairs whose 16 x 32 mask block is fully blocked are skipped entirely;
//   * the grid is one wave: `splits` CTAs per image with B * splits <= SM count, partial (m, l, O) combined by a
//     small second kernel.
// Tensor work is warp-level mma.sync.m16n8k16: at head_dim 32 the contraction is 2 k-steps, the kernel is bound by
// the exp2 / mask ALU work on the score fragments (MUFU: 58.7 M exp2 at HW = 16384, B = 4 = 12.9 us of the SFU pipe),
// which larger tensor-core instructions would not remove (DESIGN.md section 4).
#include <cuda.h>

#include <type_traits>

#include "common.cuh"

namespace psalm {

namespace xa {
constexpr int NH = 8, HD = 32, C = 256, MT = 7, ROWS = MT * 16, KS = 32, STAGES = 4;
constexpr int HPC = 4;                             // heads per CTA: grid.y = NH / HPC head groups
constexpr int MT0 = 4;                             // m-tiles of the first warp of a head (rows 0..63); the second takes 3
constexpr int QLD = HD + 8;                        // padded Q row (elements): conflict-free ldmatrix
constexpr int BOX_BYTES = KS * 128;                // one [32 keys x 64 ch] box (two heads)
constexpr int KV_BYTES = (HPC / 2) * BOX_BYTES;    // K (or V) tile of a stage: 2 boxes = 8 KB
constexpr int STAGE_BYTES = 2 * KV_BYTES;          // 16 KB
constexpr int MAXSTEPS = 16;                       // key tiles per CTA (mask words of all of them are staged up front)
constexpr int THREADS = HPC * 2 * 32;              // 8 warps: warp = (head, m-half); 2 CTAs per SM = 4 warps per sub-partition
constexpr size_t SMEM = 1024 /*alignment slack*/ + (size_t)STAGES * STAGE_BYTES + (size_t)MAXSTEPS * ROWS * 4 +
                        (size_t)HPC * ROWS * QLD * 2 + 2 * STAGES * 8;
constexpr float kLog2e = 1.4426950408889634f;
}  // namespace xa

struct XaParams {
  const void* q;             // [B, Lq, 256]
  const uint32_t* bits;      // [B, Lq, W32] or null
  const uint8_t* row_open;   // [B, Lq] or null
  void* out;                 // [B, Lq, 256]
  float* part_o;             // [B, splits, 8, 112, 32]
  float* part_ml;            // [B, splits, 8, 112, 2]
  int B, Lq, Lk, W32, splits, steps_per_split;
  int kv_batch_rows;         // K / V rows between consecutive images in the tensor maps: Lk, or 0 = one shared memory
  float qscale;              // 1/sqrt(hd) * log2(e)
};

// ---- PTX helpers ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "XA_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra XA_DONE;\n"
      "bra XA_WAIT;\n"
      "XA_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];\n" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void xa_ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void xa_ldsm_x4_t(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
template <typename T>
__device__ __forceinline__ void xa_mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  if constexpr (std::is_same<T, __nv_bfloat16>::value) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  } else {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
}
// D = A B + C with D and C in different registers (the score accumulators start from -reference, shared by the n-tiles)
template <typename T>
__device__ __forceinline__ void xa_mma_c(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1, const float (&c)[4]) {
  if constexpr (std::is_same<T, __nv_bfloat16>::value) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%11,%12,%13};\n"
                 : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1), "f"(c[0]), "f"(c[1]), "f"(c[2]), "f"(c[3]));
  } else {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%11,%12,%13};\n"
                 : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1), "f"(c[0]), "f"(c[1]), "f"(c[2]), "f"(c[3]));
  }
}
__device__ __forceinline__ float xa_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;\n" : "=f"(y) : "f"(x));
  return y;
}

// ------------------------------------------------------------------------------------------------------------
// grid = (splits, NH / HPC, B), block = 256, 2 CTAs per SM
// ------------------------------------------------------------------------------------------------------------
template <typename T, int NMT>
struct XaWarpState {
  float o[NMT][4][4];
  float m_run[NMT][2], l_run[NMT][2];
};

// one key tile (32 keys) against NMT query m-tiles of one head; K fragments are shared by the m-tiles
template <typename T, int NMT>
__device__ __forceinline__ void xa_step(XaWarpState<T, NMT>& st, uint32_t sb, const uint32_t (&koff)[2][2],
                                        const uint32_t (&voff)[2][2], uint32_t q_addr, const uint32_t* mw, int g, int t4) {
  using namespace xa;
  uint32_t kf[2][2][4];
#pragma unroll
  for (int ks = 0; ks < 2; ++ks)
#pragma unroll
    for (int np = 0; np < 2; ++np) xa_ldsm_x4(kf[ks][np], sb + koff[ks][np]);
#pragma unroll
  for (int mt = 0; mt < NMT; ++mt) {
    const uint32_t w0 = mw[mt * 16 + g], w1 = mw[mt * 16 + g + 8];
    if (__all_sync(0xffffffffu, (w0 & w1) == 0xffffffffu)) continue;   // 16 rows x 32 keys all blocked
    uint32_t qa[2][4];
    xa_ldsm_x4(qa[0], q_addr + (uint32_t)(mt * 16 * QLD * 2));
    xa_ldsm_x4(qa[1], q_addr + (uint32_t)(mt * 16 * QLD * 2) + 32);
    // Scores are produced directly relative to the row's running reference m (log2 domain): the accumulators start
    // from -m, so the common path needs no subtraction, no exact row maximum and no quad shuffles.  The reference is
    // raised (and O, l rescaled) only when some score of the tile exceeds it by more than 2^8 - or on the row's first
    // open tile - which is exact: numerator and denominator share the reference.
    const float r0 = st.m_run[mt][0], r1 = st.m_run[mt][1];
    float cinit[4];
    cinit[0] = cinit[1] = (r0 == -INFINITY) ? 0.f : -r0;
    cinit[2] = cinit[3] = (r1 == -INFINITY) ? 0.f : -r1;
    float s[4][4];
#pragma unroll
    for (int np = 0; np < 2; ++np) {
      xa_mma_c<T>(s[2 * np], qa[0], kf[0][np][0], kf[0][np][1], cinit);
      xa_mma_c<T>(s[2 * np + 1], qa[0], kf[0][np][2], kf[0][np][3], cinit);
      xa_mma<T>(s[2 * np], qa[1], kf[1][np][0], kf[1][np][1]);
      xa_mma<T>(s[2 * np + 1], qa[1], kf[1][np][2], kf[1][np][3]);
    }
    // ---- mask (bit nt*8 + 2*t4 + (e&1) of the row word)
    const uint32_t b0 = w0 >> (2 * t4), b1 = w1 >> (2 * t4);
    float tmax0 = -INFINITY, tmax1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      s[nt][0] = ((b0 >> (nt * 8)) & 1u) ? -INFINITY : s[nt][0];
      s[nt][1] = ((b0 >> (nt * 8 + 1)) & 1u) ? -INFINITY : s[nt][1];
      s[nt][2] = ((b1 >> (nt * 8)) & 1u) ? -INFINITY : s[nt][2];
      s[nt][3] = ((b1 >> (nt * 8 + 1)) & 1u) ? -INFINITY : s[nt][3];
      tmax0 = fmaxf(tmax0, fmaxf(s[nt][0], s[nt][1]));
      tmax1 = fmaxf(tmax1, fmaxf(s[nt][2], s[nt][3]));
    }
    constexpr float kRaise = 8.f;
    const bool need0 = tmax0 > kRaise || (r0 == -INFINITY && tmax0 > -INFINITY);
    const bool need1 = tmax1 > kRaise || (r1 == -INFINITY && tmax1 > -INFINITY);
    if (__any_sync(0xffffffffu, need0 || need1)) {
      // exact row maxima (over the quad), new reference = old + delta, everything already accumulated scales by 2^-delta
      tmax0 = fmaxf(tmax0, __shfl_xor_sync(0xffffffffu, tmax0, 1));
      tmax1 = fmaxf(tmax1, __shfl_xor_sync(0xffffffffu, tmax1, 1));
      tmax0 = fmaxf(tmax0, __shfl_xor_sync(0xffffffffu, tmax0, 2));
      tmax1 = fmaxf(tmax1, __shfl_xor_sync(0xffffffffu, tmax1, 2));
      const bool up0 = tmax0 > kRaise || (r0 == -INFINITY && tmax0 > -INFINITY);   // row-uniform over the quad
      const bool up1 = tmax1 > kRaise || (r1 == -INFINITY && tmax1 > -INFINITY);
      const float d0 = up0 ? tmax0 : 0.f, d1 = up1 ? tmax1 : 0.f;
      // -d > 0 only on a row's first open tile, where l and O are still 0: the clamp keeps 2^-d finite there (a tile
      // maximum below -128 in the log2 domain would give inf, and 0 * inf = NaN in l and O); elsewhere -d <= 0
      const float c0 = xa_exp2(fminf(-d0, 64.f)), c1 = xa_exp2(fminf(-d1, 64.f));
      if (up0) st.m_run[mt][0] = (r0 == -INFINITY ? 0.f : r0) + d0;
      if (up1) st.m_run[mt][1] = (r1 == -INFINITY ? 0.f : r1) + d1;
      st.l_run[mt][0] *= c0;
      st.l_run[mt][1] *= c1;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        st.o[mt][i][0] *= c0; st.o[mt][i][1] *= c0;
        st.o[mt][i][2] *= c1; st.o[mt][i][3] *= c1;
        s[i][0] -= d0; s[i][1] -= d0;
        s[i][2] -= d1; s[i][3] -= d1;
      }
    }
    float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      s[nt][0] = xa_exp2(s[nt][0]);      // blocked: 2^(-inf) = 0
      s[nt][1] = xa_exp2(s[nt][1]);
      s[nt][2] = xa_exp2(s[nt][2]);
      s[nt][3] = xa_exp2(s[nt][3]);
      ps0 += s[nt][0] + s[nt][1];
      ps1 += s[nt][2] + s[nt][3];
    }
    st.l_run[mt][0] += ps0;     // lane-private partial row sums; reduced over the quad in the epilogue
    st.l_run[mt][1] += ps1;
    // ---- O += P V (V fragments fetched per m-tile: the shared-memory pipe is idle, registers are not)
#pragma unroll
    for (int kk = 0; kk < 2; ++kk) {
      uint32_t pa[4];
      pa[0] = pack2<T>(s[2 * kk][0], s[2 * kk][1]);
      pa[1] = pack2<T>(s[2 * kk][2], s[2 * kk][3]);
      pa[2] = pack2<T>(s[2 * kk + 1][0], s[2 * kk + 1][1]);
      pa[3] = pack2<T>(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
      for (int dp = 0; dp < 2; ++dp) {
        uint32_t vf[4];
        xa_ldsm_x4_t(vf, sb + voff[kk][dp]);
        xa_mma<T>(st.o[mt][2 * dp], pa, vf[0], vf[1]);
        xa_mma<T>(st.o[mt][2 * dp + 1], pa, vf[2], vf[3]);
      }
    }
  }
}

template <typename T, int NMT>
__device__ __forceinline__ void xa_epilogue(const XaWarpState<T, NMT>& st, const XaParams& p, int b, int sp, int h, int row0,
                                            int g, int t4) {
  using namespace xa;
#pragma unroll
  for (int mt = 0; mt < NMT; ++mt) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float l = st.l_run[mt][r];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      const int row = row0 + mt * 16 + g + 8 * r;
      if (p.splits == 1) {
        if (row < p.Lq) {
          const float inv = l > 0.f ? 1.f / l : 0.f;
          T* op = reinterpret_cast<T*>(p.out) + ((size_t)b * p.Lq + row) * C + h * HD + 2 * t4;
#pragma unroll
          for (int i = 0; i < 4; ++i)
            *reinterpret_cast<uint32_t*>(op + i * 8) = pack2<T>(st.o[mt][i][2 * r] * inv, st.o[mt][i][2 * r + 1] * inv);
        }
      } else {
        const size_t pr = (((size_t)b * p.splits + sp) * NH + h) * ROWS + row;
        float* po = p.part_o + pr * HD + 2 * t4;
#pragma unroll
        for (int i = 0; i < 4; ++i)
          *reinterpret_cast<float2*>(po + i * 8) = make_float2(st.o[mt][i][2 * r], st.o[mt][i][2 * r + 1]);
        if (t4 == 0) *reinterpret_cast<float2*>(p.part_ml + pr * 2) = make_float2(st.m_run[mt][r], l);
      }
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(xa::THREADS, 2)
xattn_tma_kernel(const __grid_constant__ CUtensorMap mapK, const __grid_constant__ CUtensorMap mapV, XaParams p) {
  using namespace xa;
  extern __shared__ unsigned char xa_smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(xa_smem_raw) + 1023) & ~(uintptr_t)1023);
  unsigned char* kv = smem;                                                    // [STAGES][K 8 KB | V 8 KB]
  uint32_t* maskw = reinterpret_cast<uint32_t*>(smem + (size_t)STAGES * STAGE_BYTES);   // [MAXSTEPS][ROWS]
  T* Qs = reinterpret_cast<T*>(maskw + MAXSTEPS * ROWS);                       // [HPC][ROWS][QLD]
  uint64_t* full = reinterpret_cast<uint64_t*>(Qs + (size_t)HPC * ROWS * QLD); // [STAGES]
  uint64_t* empty = full + STAGES;                                             // [STAGES]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int sp = blockIdx.x, hg = blockIdx.y, b = blockIdx.z;
  const int total_steps = (p.Lk + KS - 1) / KS;
  const int step0 = sp * p.steps_per_split;
  int nsteps = total_steps - step0;
  nsteps = nsteps < p.steps_per_split ? nsteps : p.steps_per_split;
  if (nsteps < 0) nsteps = 0;

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], THREADS / 32);
    }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();

  // ---- producer duty (one lane of warp 0, between its own compute steps): TMA of key tile `it` into its stage
  auto produce = [&](int it) {
    if (lane == 0) {
      const int stage = it % STAGES;
      if (it >= STAGES) mbar_wait(&empty[stage], ((it / STAGES) - 1) & 1);   // all 8 warps are done with the old tile
      mbar_arrive_expect_tx(&full[stage], (uint32_t)STAGE_BYTES);
      unsigned char* dst = kv + (size_t)stage * STAGE_BYTES;
      const int row0 = b * p.kv_batch_rows + (step0 + it) * KS;
#pragma unroll
      for (int bx = 0; bx < HPC / 2; ++bx) {
        tma_load_2d(dst + bx * BOX_BYTES, &mapK, (hg * (HPC / 2) + bx) * 64, row0, &full[stage]);
        tma_load_2d(dst + KV_BYTES + bx * BOX_BYTES, &mapV, (hg * (HPC / 2) + bx) * 64, row0, &full[stage]);
      }
    }
    __syncwarp();
  };
  if (warp == 0)   // the first tiles are in flight while the mask words and Q are staged
    for (int it = 0; it < STAGES - 1 && it < nsteps; ++it) produce(it);

  // ---- mask words of every key tile of this CTA, [step][row]: blocked bits, tail beyond Lk blocked, rows >= Lq fully
  //      blocked (never stored), open rows cleared (:647).  One round of global loads for the whole CTA, off the
  //      per-step critical path (the first version fetched them per step in the producer: +1.5 us of load latency per
  //      step on the warp every other warp waits for).
  {
    const bool has_bits = p.bits != nullptr;
    for (int i = tid; i < nsteps * ROWS; i += THREADS) {
      const int row = i / nsteps, j = i - row * nsteps;      // consecutive threads: consecutive words of a row
      const int kt = step0 + j;
      const int left = p.Lk - kt * KS;
      uint32_t w = 0xffffffffu;
      if (row < p.Lq) {
        const size_t r = (size_t)b * p.Lq + row;
        w = 0u;
        if (has_bits && !(p.row_open && p.row_open[r])) w = __ldg(p.bits + r * p.W32 + kt);
        if (left < 32) w |= 0xffffffffu << left;
      }
      maskw[j * ROWS + row] = w;
    }
  }

  // ---- Q of this head group -> shared memory, pre-scaled by scale * log2e (nn.MultiheadAttention scales q before
  //      the product too); all loads of a thread are issued before the first store
  {
    const T* qb = reinterpret_cast<const T*>(p.q) + (size_t)b * p.Lq * C + hg * HPC * HD;
    constexpr int CH = HPC * HD / 8;                 // 16-byte chunks per row of this head group
    constexpr int PER = (ROWS * CH + THREADS - 1) / THREADS;
    uint4 raw[PER];
#pragma unroll
    for (int j = 0; j < PER; ++j) {
      const int i = tid + j * THREADS;
      const int row = i / CH, c8 = i % CH;
      raw[j] = make_uint4(0, 0, 0, 0);
      if (i < ROWS * CH && row < p.Lq) raw[j] = __ldg(reinterpret_cast<const uint4*>(qb + (size_t)row * C + c8 * 8));
    }
#pragma unroll
    for (int j = 0; j < PER; ++j) {
      const int i = tid + j * THREADS;
      if (i >= ROWS * CH) break;
      const int row = i / CH, c8 = i % CH;
      float f[8];
      unpack2<T>(raw[j].x, f[0], f[1]);
      unpack2<T>(raw[j].y, f[2], f[3]);
      unpack2<T>(raw[j].z, f[4], f[5]);
      unpack2<T>(raw[j].w, f[6], f[7]);
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] *= p.qscale;
      const int hl = c8 >> 2, d0 = (c8 & 3) * 8;
      store16_from_f32<T>(Qs + ((size_t)hl * ROWS + row) * QLD + d0, f);
    }
  }
  __syncthreads();

  // ---- warp = (local head, m-half): rows [0, 64) or [64, 112) of the head
  const int hl = warp >> 1, half = warp & 1;
  const int h = hg * HPC + hl;
  const int g = lane >> 2, t4 = lane & 3;
  const int mi = lane >> 3, l7 = lane & 7;
  const uint32_t kv_base = smem_u32(kv);
  // byte offsets inside a stage of the ldmatrix rows this lane addresses (SWIZZLE_128B: 16-byte chunk ^= row & 7)
  const uint32_t box = (uint32_t)(hl >> 1) * BOX_BYTES;
  const uint32_t hc = (uint32_t)(hl & 1) * 4;      // first 16-byte chunk of this head inside the 128-byte row
  uint32_t koff[2][2], voff[2][2];
#pragma unroll
  for (int ks = 0; ks < 2; ++ks)
#pragma unroll
    for (int np = 0; np < 2; ++np) {
      const uint32_t r = np * 16 + l7 + (mi >> 1) * 8;
      const uint32_t ch = hc + ks * 2 + (mi & 1);
      koff[ks][np] = box + r * 128 + ((ch ^ (r & 7)) << 4);
    }
#pragma unroll
  for (int kk = 0; kk < 2; ++kk)
#pragma unroll
    for (int dp = 0; dp < 2; ++dp) {
      const uint32_t r = kk * 16 + l7 + (mi & 1) * 8;
      const uint32_t ch = hc + dp * 2 + (mi >> 1);
      voff[kk][dp] = KV_BYTES + box + r * 128 + ((ch ^ (r & 7)) << 4);
    }
  const int row0 = half * MT0 * 16;
  const uint32_t q_addr = smem_u32(Qs + ((size_t)hl * ROWS + row0) * QLD) +
                          (uint32_t)((l7 + ((lane >> 3) & 1) * 8) * QLD + (lane >> 4) * 8) * 2;

  auto run = [&](auto& st) {
    constexpr int NMT = sizeof(st.m_run) / (2 * sizeof(float));
#pragma unroll
    for (int mt = 0; mt < NMT; ++mt) {
#pragma unroll
      for (int i = 0; i < 4; ++i) st.o[mt][i][0] = st.o[mt][i][1] = st.o[mt][i][2] = st.o[mt][i][3] = 0.f;
      st.m_run[mt][0] = st.m_run[mt][1] = -INFINITY;
      st.l_run[mt][0] = st.l_run[mt][1] = 0.f;
    }
    for (int it = 0; it < nsteps; ++it) {
      const int stage = it % STAGES;
      if (warp == 0 && it + STAGES - 1 < nsteps) produce(it + STAGES - 1);   // refills the stage consumed at step it - 1
      mbar_wait(&full[stage], (it / STAGES) & 1);
      xa_step<T, NMT>(st, kv_base + (uint32_t)stage * STAGE_BYTES, koff, voff, q_addr, maskw + it * ROWS + row0, g, t4);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[stage]);
    }
    xa_epilogue<T, NMT>(st, p, b, sp, h, row0, g, t4);
  };
  if (half == 0) {
    XaWarpState<T, MT0> st;
    run(st);
  } else {
    XaWarpState<T, MT - MT0> st;
    run(st);
  }
}

// combine: one thread per (b, row, h, channel pair)
template <typename T>
__global__ void xattn_combine_kernel(XaParams p) {
  using namespace xa;
  const long long n = (long long)p.B * p.Lq * NH * (HD / 2);
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
    long long t = idx;
    const int d2 = (int)(t % (HD / 2)); t /= HD / 2;
    const int h = (int)(t % NH); t /= NH;
    const int row = (int)(t % p.Lq);
    const int b = (int)(t / p.Lq);
    float M = -INFINITY;
    for (int s = 0; s < p.splits; ++s)
      M = fmaxf(M, p.part_ml[((((size_t)b * p.splits + s) * NH + h) * ROWS + row) * 2]);
    float L = 0.f, O0 = 0.f, O1 = 0.f;
    if (M != -INFINITY) {
      for (int s = 0; s < p.splits; ++s) {
        const size_t pr = (((size_t)b * p.splits + s) * NH + h) * ROWS + row;
        const float2 ml = *reinterpret_cast<const float2*>(p.part_ml + pr * 2);
        if (ml.x == -INFINITY) continue;
        const float e = exp2f(ml.x - M);
        const float2 ov = *reinterpret_cast<const float2*>(p.part_o + pr * HD + 2 * d2);
        L += ml.y * e;
        O0 += ov.x * e;
        O1 += ov.y * e;
      }
    }
    const float inv = L > 0.f ? 1.f / L : 0.f;
    *reinterpret_cast<uint32_t*>(reinterpret_cast<T*>(p.out) + ((size_t)b * p.Lq + row) * C + h * HD + 2 * d2) =
        pack2<T>(O0 * inv, O1 * inv);
  }
}

// ---- host: tensor maps (driver entry point through the runtime, no link-time dependency on libcuda) ------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

static bool make_kv_map(CUtensorMap* map, const void* base, long long rows, long long row_stride_elems, int dtype) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return false;
  const cuuint64_t dims[2] = {(cuuint64_t)xa::C, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)row_stride_elems * 2};
  const cuuint32_t box[2] = {64, (cuuint32_t)xa::KS};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = fn(map, dtype == PSALM_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                        const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

static int xa_sm_count() {
  static PerDevice cache;
  const int d = PerDevice::dev();
  if (cache.first() || cache.v[d] == 0) cudaDeviceGetAttribute(&cache.v[d], cudaDevAttrMultiProcessorCount, d);
  return cache.v[d] > 0 ? cache.v[d] : 132;
}

static int xa_splits(int B, int Lk) {
  const int steps = (Lk + xa::KS - 1) / xa::KS;
  int s = 2 * xa_sm_count() / ((xa::NH / xa::HPC) * (B > 0 ? B : 1));   // one wave: 2 CTAs per SM
  const int cap = (steps + 3) / 4;                  // at least 4 key tiles (128 keys) per CTA
  if (s > cap) s = cap;
  if (s < 1) s = 1;
  const int need = (steps + xa::MAXSTEPS - 1) / xa::MAXSTEPS;   // a CTA stages the mask words of <= MAXSTEPS key tiles
  if (s < need) s = need;
  const int per = (steps + s - 1) / s;
  return (steps + per - 1) / per;                   // drop empty trailing splits
}

static int g_cross_impl = 0;   // 0 auto, 1 / 2 always the TMA-fed kernel of this file
// per-head flash kernel of attn_mma.cu (row-strided K / V views supported)
int mma_cross_attention(const void*, const void*, const void*, const uint32_t*, const uint8_t*, void*, float*, int, int, int, int,
                        int, int, int, cudaStream_t, int kv_ld, long long kv_bstride);
constexpr int kSmallLk = 2048;   // below this many keys the problem is launch / latency bound: the per-head kernel with
                                 // few key tiles per CTA wins (measured, tools/bench_cross.py)
static int small_splits(int B, int Lk) {
  const int ctas = B * 8 * 2;
  int want = (2 * 132 + ctas - 1) / ctas;
  const int cap = (Lk + 255) / 256;
  if (want > cap) want = cap;
  if (want > 16) want = 16;
  return want < 1 ? 1 : want;
}

}  // namespace psalm

extern "C" int psalm_set_cross_impl(int impl) {
  if (impl < 0 || impl > 2) {
    psalm::set_error("psalm_set_cross_impl: 0 (auto), 1 or 2 (TMA-fed mma.sync kernel at every key count)");
    return PSALM_E_ARG;
  }
  psalm::g_cross_impl = impl;
  return PSALM_OK;
}

extern "C" size_t psalm_masked_cross_attention_workspace_bytes(int B, int Lq, int Lk) {
  using namespace psalm;
  const int s = xa_splits(B, Lk);
  size_t a = s > 1 ? (size_t)B * s * xa::NH * xa::ROWS * (xa::HD + 2) * sizeof(float) : 0;
  const int ss = small_splits(B, Lk);
  const size_t u = ss > 1 ? (size_t)B * xa::NH * ss * Lq * (xa::HD + 2) * sizeof(float) : 0;
  return a > u ? a : u;      // any implementation may be selected at run time
}

extern "C" int psalm_masked_cross_attention(const void* q, const void* k, const void* v, long long kv_row_stride,
                                            const uint32_t* mask_bits, const uint8_t* row_open, void* out,
                                            float* workspace, size_t workspace_bytes, int B, int Lq, int Lk, int nh,
                                            int hd, int dtype, void* stream) {
  return psalm_masked_cross_attention_strided(q, k, v, kv_row_stride, (long long)Lk * kv_row_stride, mask_bits, row_open, out,
                                              workspace, workspace_bytes, B, Lq, Lk, nh, hd, dtype, stream);
}

extern "C" int psalm_masked_cross_attention_strided(const void* q, const void* k, const void* v, long long kv_row_stride,
                                                    long long kv_batch_stride, const uint32_t* mask_bits,
                                                    const uint8_t* row_open, void* out, float* workspace,
                                                    size_t workspace_bytes, int B, int Lq, int Lk, int nh, int hd, int dtype,
                                                    void* stream) {
  using namespace psalm;
  PSALM_REQUIRE(q && k && v && out, "masked_cross_attention: null pointer");
  PSALM_REQUIRE(nh == xa::NH && hd == xa::HD, "masked_cross_attention: needs 8 heads x 32 (got %d x %d)", nh, hd);
  PSALM_REQUIRE(dtype == PSALM_BF16 || dtype == PSALM_F16, "masked_cross_attention: 16-bit storage only");
  PSALM_REQUIRE(Lq >= 1 && Lq <= xa::ROWS, "masked_cross_attention: 1..%d queries (got %d)", xa::ROWS, Lq);
  PSALM_REQUIRE(B >= 1 && B <= 65535 && Lk >= 1, "masked_cross_attention: bad B / Lk");
  PSALM_REQUIRE(kv_row_stride >= xa::C && kv_row_stride % 8 == 0, "masked_cross_attention: K/V row stride %lld", kv_row_stride);
  PSALM_REQUIRE(kv_batch_stride >= 0 && kv_batch_stride % kv_row_stride == 0 &&
                    (long long)(B - 1) * (kv_batch_stride / kv_row_stride) + Lk < (1ll << 31),
                "masked_cross_attention: K/V batch stride %lld must be 0 or a multiple of the row stride %lld", kv_batch_stride,
                kv_row_stride);
  PSALM_REQUIRE(((uintptr_t)k & 15) == 0 && ((uintptr_t)v & 15) == 0 && ((uintptr_t)q & 15) == 0 && ((uintptr_t)out & 3) == 0,
                "masked_cross_attention: pointers must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  if (g_cross_impl == 0 && Lk < kSmallLk) {
    const int ss = small_splits(B, Lk);
    return mma_cross_attention(q, k, v, mask_bits, row_open, out, workspace, B, Lq, Lk, nh, hd, ss, dtype, st, (int)kv_row_stride,
                               kv_batch_stride);
  }
  const long long batch_rows = kv_batch_stride / kv_row_stride;
  XaParams p;
  p.q = q; p.bits = mask_bits; p.row_open = row_open; p.out = out;
  p.B = B; p.Lq = Lq; p.Lk = Lk; p.W32 = (Lk + 31) / 32;
  p.kv_batch_rows = (int)batch_rows;
  p.splits = xa_splits(B, Lk);
  const int steps = (Lk + xa::KS - 1) / xa::KS;
  p.steps_per_split = (steps + p.splits - 1) / p.splits;
  p.qscale = 1.0f / sqrtf((float)hd) * xa::kLog2e;
  p.part_o = p.part_ml = nullptr;
  if (p.splits > 1) {
    const size_t need = (size_t)B * p.splits * xa::NH * xa::ROWS * (xa::HD + 2) * sizeof(float);
    PSALM_REQUIRE(workspace && workspace_bytes >= need, "masked_cross_attention: workspace of %zu bytes needed", need);
    p.part_o = workspace;
    p.part_ml = workspace + (size_t)B * p.splits * xa::NH * xa::ROWS * xa::HD;
  }
  CUtensorMap mk, mv;
  const long long map_rows = (long long)(B - 1) * batch_rows + Lk;
  if (!make_kv_map(&mk, k, map_rows, kv_row_stride, dtype) || !make_kv_map(&mv, v, map_rows, kv_row_stride, dtype)) {
    set_error("masked_cross_attention: cuTensorMapEncodeTiled failed (driver without TMA support?)");
    return PSALM_E_CUDA;
  }
  dim3 grid(p.splits, xa::NH / xa::HPC, B);
  cudaError_t e;
  if (dtype == PSALM_BF16) {
    e = cudaFuncSetAttribute(xattn_tma_kernel<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)xa::SMEM);
    if (e == cudaSuccess) xattn_tma_kernel<__nv_bfloat16><<<grid, xa::THREADS, xa::SMEM, st>>>(mk, mv, p);
  } else {
    e = cudaFuncSetAttribute(xattn_tma_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)xa::SMEM);
    if (e == cudaSuccess) xattn_tma_kernel<__half><<<grid, xa::THREADS, xa::SMEM, st>>>(mk, mv, p);
  }
  if (e != cudaSuccess) {
    set_error("masked_cross_attention: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    return PSALM_E_CUDA;
  }
  if (p.splits > 1) {
    const long long n = (long long)B * Lq * xa::NH * (xa::HD / 2);
    const int blocks = (int)((n + 255) / 256);
    if (dtype == PSALM_BF16) xattn_combine_kernel<__nv_bfloat16><<<blocks, 256, 0, st>>>(p);
    else xattn_combine_kernel<__half><<<blocks, 256, 0, st>>>(p);
  }
  return check_launch("masked_cross_attention");
}
