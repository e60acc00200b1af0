// Linear layers with a fused epilogue on the Hopper tensor cores (wgmma): out = epilogue(A · Wᵀ + bias), 16-bit storage,
// fp32 accumulation in registers.
//
// Replaces, on the 16-bit path, the library GEMM + separate elementwise pass of
//   * Swin `Mlp.fc1` + exact-erf `nn.GELU` (swin_trans.py:37-44, 24 blocks): the stand-alone GELU pass re-reads and
//     re-writes the 4C-wide activation;
//   * MSDeformAttn `value_proj` + the [B,S,8,32] -> [B,8,S,32] head-major copy (ops/modules/ms_deform_attn.py:95-99
//     + our layout, DESIGN.md section 3): the epilogue stores each 32-column chunk (= one head) where the sampling
//     kernel wants it.
//
// Persistent CTA per SM, 128 x 256 output tiles, BK = 64 (one SWIZZLE_128B atom per row), three warpgroups:
//   warpgroup 0    TMA producer (one thread): A box [128 x 64] and W box [256 x 64] per k-block into a 3-stage ring
//                  (48 KB per stage); gives its registers to the consumers (setmaxnreg)
//   warpgroups 1-2 consumers: warpgroup c owns rows 64 c .. 64 c + 63 of the tile; per k-block 4 x wgmma m64n256k16
//                  from shared memory (both operands K-major, 128-byte swizzle), 128 fp32 accumulators per thread.  One
//                  k-block group stays in flight: the stage of k-block kb - 1 is handed back once kb is issued.
//                  Epilogue: + bias -> GELU -> 16-bit pack -> swizzled staging box in shared memory -> TMA stores
//                  ([64 rows x 128 B] boxes, or [32 x 64 B] head boxes) so that L2 sees whole lines.
//
// GELU: 0.5 x (1 + erf(x / sqrt 2)) = max(x, 0) - |x| E / 2 with E = erfc(|x| / sqrt 2); E / 2 = 2^q(t), q a degree-7
// polynomial fitted to log2(erfc(z) / 2) on z in [0, 5], t = sat(z / 5) (beyond z = 5, erfc < 2e-12).
// Relative error of the result < 2.5e-5 for |x| < 7, absolute < 1.5e-6 everywhere (checked against float64 erf) - two
// orders below the 16-bit rounding of the output - at one MUFU and 8 FMAs per element instead of libm's erff.
#include <cuda.h>

#include <type_traits>

#include "common.cuh"

namespace psalm {

namespace gw {
constexpr int BM = 128, BN = 256, BK = 64, NS = 3;
constexpr int A_BYTES = BM * BK * 2, W_BYTES = BN * BK * 2, STAGE = A_BYTES + W_BYTES;
constexpr int CONSUMERS = 2, THREADS = (CONSUMERS + 1) * 128;
constexpr int WG_ROWS = BM / CONSUMERS;                 // 64 rows per consumer warpgroup
constexpr int STG_WG = WG_ROWS * BN * 2;               // output staging of one consumer warpgroup: 32 KB
constexpr size_t SMEM = 1024 + (size_t)NS * STAGE + (size_t)CONSUMERS * STG_WG + 256;
static_assert(SMEM <= 227 * 1024, "H100: at most 227 KB of shared memory per block");
}  // namespace gw

struct GwParams {
  const void* bias;   // [N] storage dtype, or null
  int M, N, K;
  int S;              // rows per image (epilogue 2)
  int tiles_m, tiles_n;
};

__device__ __forceinline__ uint32_t gw_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// wgmma shared-memory descriptor: K-major, SWIZZLE_128B, 8-row groups 1024 B apart (stage bases are 1024-aligned)
__device__ __forceinline__ uint64_t gw_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3ffff) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
__device__ __forceinline__ void gw_mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(gw_u32(bar)), "r"(count));
}
#define gw_mbar_wait(bar, parity)                                                                       \
  do {                                                                                                  \
    uint32_t done_ = 0, spins_ = 0;                                                                     \
    while (!done_) {                                                                                    \
      asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"   \
                   "selp.u32 %0, 1, 0, p;\n\t}\n" : "=r"(done_) : "r"(gw_u32(bar)), "r"((uint32_t)(parity)) : "memory"); \
      if (++spins_ > (1u << 26)) __trap(); /* never hang the GPU on a protocol bug */                   \
    }                                                                                                   \
  } while (0)
__device__ __forceinline__ void gw_mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(gw_u32(bar)) : "memory");
}
__device__ __forceinline__ void gw_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(gw_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void gw_tma_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];\n" ::"r"(
          gw_u32(dst)),
      "l"(map), "r"(c0), "r"(c1), "r"(gw_u32(bar))
      : "memory");
}
__device__ __forceinline__ void gw_tma_store_2d(const CUtensorMap* map, int c0, int c1, const void* src) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%1, %2}], [%3];\n" ::"l"(map), "r"(c0), "r"(c1),
               "r"(gw_u32(src))
               : "memory");
}
__device__ __forceinline__ void gw_bar_wg(int id) { asm volatile("bar.sync %0, 128;\n" ::"r"(id) : "memory"); }

// d[128] += A(64 x 16) · B(16 x 256): thread (warp w, lane l) holds rows 16 w + l / 4 + 8 i, columns 8 j + 2 (l % 4) + h
// in d[4 j + 2 i + h]
template <typename T>
__device__ __forceinline__ void gw_wgmma(float (&d)[128], uint64_t da, uint64_t db, uint32_t accumulate);
template <>
__device__ __forceinline__ void gw_wgmma<__nv_bfloat16>(float (&d)[128], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, %128, %129, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "r"(accumulate));
}
template <>
__device__ __forceinline__ void gw_wgmma<__half>(float (&d)[128], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, %128, %129, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "r"(accumulate));
}

__device__ __forceinline__ float gw_gelu(float x) {   // see the header comment
  const float a = fabsf(x);
  const float t = __saturatef(a * (0.70710678f * 0.2f));
  float q = -1.401790814e+00f;
  q = fmaf(q, t, 7.022554923e+00f);
  q = fmaf(q, t, -1.563424726e+01f);
  q = fmaf(q, t, 2.078584664e+01f);
  q = fmaf(q, t, -1.893136839e+01f);
  q = fmaf(q, t, -2.294412836e+01f);
  q = fmaf(q, t, -8.139466606e+00f);
  q = fmaf(q, t, -1.000004739e+00f);
  float h;
  asm("ex2.approx.ftz.f32 %0, %1;\n" : "=f"(h) : "f"(q));
  return fmaf(-a, h, fmaxf(x, 0.f));
}

template <typename T, int EPI>
__global__ void __launch_bounds__(gw::THREADS, 1)
linear_wgmma_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapW,
                    const __grid_constant__ CUtensorMap mapO, GwParams p) {
  using namespace gw;
  extern __shared__ unsigned char gw_raw[];
  unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(gw_raw) + 1023) & ~(uintptr_t)1023);
  unsigned char* stg_all = base + (size_t)NS * STAGE;
  uint64_t* bars = reinterpret_cast<uint64_t*>(stg_all + (size_t)CONSUMERS * STG_WG);
  uint64_t* full = bars;               // [NS] TMA landed
  uint64_t* empty = bars + NS;         // [NS] the wgmmas reading the stage have retired (one arrival per consumer warp)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n_tiles = p.tiles_m * p.tiles_n;
  const int kblocks = p.K / BK;

  if (tid == 0) {
    for (int s = 0; s < NS; ++s) {
      gw_mbar_init(&full[s], 1);
      gw_mbar_init(&empty[s], CONSUMERS * 4);
    }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    // ------------------------------------------------ TMA producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (tid == 0) {
      uint32_t it = 0;
      for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const int tm = t / p.tiles_n, tn = t - tm * p.tiles_n;
        for (int kb = 0; kb < kblocks; ++kb, ++it) {
          const int s = it % NS;
          if (it >= NS) gw_mbar_wait(&empty[s], ((it / NS) - 1) & 1);
          unsigned char* st = base + (size_t)s * STAGE;
          gw_mbar_expect_tx(&full[s], STAGE);
          gw_tma_2d(st, &mapA, kb * BK, tm * BM, &full[s]);
          gw_tma_2d(st + A_BYTES, &mapW, kb * BK, tn * BN, &full[s]);
        }
      }
    }
    return;
  }
  // ------------------------------------------------ consumers
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
  const int wg = (warp >> 2) - 1, w4 = warp & 3, tw = tid & 127;
  unsigned char* stg = stg_all + (size_t)wg * STG_WG;
  const T* bias = reinterpret_cast<const T*>(p.bias);
  uint32_t it = 0, li = 0;
  float d[128];
  for (int t = blockIdx.x; t < n_tiles; t += gridDim.x, ++li) {
    const int tm = t / p.tiles_n, tn = t - tm * p.tiles_n;
    for (int kb = 0; kb < kblocks; ++kb, ++it) {
      const int s = it % NS;
      gw_mbar_wait(&full[s], (it / NS) & 1);
      const uint32_t sa = gw_u32(base + (size_t)s * STAGE) + wg * (WG_ROWS * 128), sw = gw_u32(base + (size_t)s * STAGE) + A_BYTES;
      asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory");
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) gw_wgmma<T>(d, gw_desc(sa + k * 32), gw_desc(sw + k * 32), (kb | k) ? 1u : 0u);
      asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory");
      if (kb > 0) {   // k-block kb - 1 has retired: its stage goes back to the producer
        asm volatile("wgmma.wait_group.sync.aligned 1;\n" ::: "memory");
        if (lane == 0) gw_mbar_arrive(&empty[(it - 1) % NS]);
      }
    }
    asm volatile("wgmma.wait_group.sync.aligned 0;\n" ::: "memory");
    if (lane == 0) gw_mbar_arrive(&empty[(it - 1) % NS]);

    // ---- epilogue: registers -> swizzled staging -> TMA store
    if (li > 0) {   // the previous tile's stores have finished reading the staging boxes
      if (tw == 0) asm volatile("cp.async.bulk.wait_group.read 0;\n" ::: "memory");
      gw_bar_wg(1 + wg);
    }
    const int col0 = tn * BN + 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      float b0 = 0.f, b1 = 0.f;
      if (bias) {
        const float2 bb = std::is_same<T, __nv_bfloat16>::value
                              ? __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(bias + col0 + 8 * j))
                              : __half22float2(*reinterpret_cast<const __half2*>(bias + col0 + 8 * j));
        b0 = bb.x;
        b1 = bb.y;
      }
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float x0 = d[4 * j + 2 * i] + b0, x1 = d[4 * j + 2 * i + 1] + b1;
        if (EPI == 1) {
          x0 = gw_gelu(x0);
          x1 = gw_gelu(x1);
        }
        const uint32_t v = pack2<T>(x0, x1);
        const int r = w4 * 16 + (lane >> 2) + 8 * i;   // row inside the warpgroup's 64
        uint32_t addr;
        if (EPI == 2) {   // box (r / 32, head j / 4) = [32 rows x 64 B], SWIZZLE_64B (16-byte chunk ^ bits 1-2 of the row)
          const int rr = r & 31;
          addr = gw_u32(stg) + ((r >> 5) * 8 + (j >> 2)) * 2048 + rr * 64 + ((((j & 3) ^ ((rr >> 1) & 3))) << 4) + (lane & 3) * 4;
        } else {          // box j / 8 = [64 rows x 128 B], SWIZZLE_128B (16-byte chunk ^ row % 8)
          addr = gw_u32(stg) + (j >> 3) * 8192 + r * 128 + (((j & 7) ^ (r & 7)) << 4) + (lane & 3) * 4;
        }
        asm volatile("st.shared.b32 [%0], %1;\n" ::"r"(addr), "r"(v) : "memory");
      }
    }
    asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
    gw_bar_wg(1 + wg);
    if (tw == 0) {
      const int row0 = tm * BM + wg * WG_ROWS;
      if (EPI == 2) {
#pragma unroll
        for (int rg = 0; rg < 2; ++rg) {
          const long long r0 = (long long)row0 + rg * 32;
          if (r0 >= p.M) break;
          const long long img = r0 / p.S, srow = r0 - img * p.S;
#pragma unroll
          for (int h = 0; h < 8; ++h) {
            const long long orow = (img * (p.N / 32) + (tn * 8 + h)) * p.S + srow;
            gw_tma_store_2d(&mapO, 0, (int)orow, stg + (rg * 8 + h) * 2048);
          }
        }
      } else if (row0 < p.M) {   // rows beyond M are clipped by the tensor map
#pragma unroll
        for (int b = 0; b < BN / 64; ++b) gw_tma_store_2d(&mapO, tn * BN + b * 64, row0, stg + b * 8192);
      }
      asm volatile("cp.async.bulk.commit_group;\n" ::: "memory");
    }
  }
  if (tw == 0) asm volatile("cp.async.bulk.wait_group 0;\n" ::: "memory");
}

// ---- host ------------------------------------------------------------------------------------------------------
typedef CUresult (*GwEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                               const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static GwEncodeFn gw_encode_fn() {
  static GwEncodeFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<GwEncodeFn>(p);
  }
  return fn;
}
static bool gw_make_map(CUtensorMap* map, const void* base, long long rows, long long cols, long long row_stride_elems,
                        int box_cols, int box_rows, CUtensorMapSwizzle swz, int dtype) {
  GwEncodeFn fn = gw_encode_fn();
  if (!fn) return false;
  const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)row_stride_elems * 2};
  const cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  return fn(map, dtype == PSALM_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
            const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
            CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
static int gw_sm_count() {
  static PerDevice cache;
  const int d = PerDevice::dev();
  if (cache.first() || cache.v[d] == 0) cudaDeviceGetAttribute(&cache.v[d], cudaDevAttrMultiProcessorCount, d);
  return cache.v[d] > 0 ? cache.v[d] : 132;
}

template <typename T, int EPI>
static cudaError_t gw_launch(const CUtensorMap& ma, const CUtensorMap& mw, const CUtensorMap& mo, const GwParams& p, int grid,
                             cudaStream_t st) {
  cudaError_t e = cudaFuncSetAttribute(linear_wgmma_kernel<T, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gw::SMEM);
  if (e != cudaSuccess) return e;
  linear_wgmma_kernel<T, EPI><<<grid, gw::THREADS, gw::SMEM, st>>>(ma, mw, mo, p);
  return cudaSuccess;
}

}  // namespace psalm

using namespace psalm;

extern "C" int psalm_linear_fused_supported(long long M, int N, int K, int epilogue, long long rows_per_image, int dtype) {
  if (dtype != PSALM_BF16 && dtype != PSALM_F16) return 0;
  if (M <= 0 || N <= 0 || K <= 0 || N % gw::BN || K % gw::BK || M > (1ll << 31) - gw::BM) return 0;
  if (epilogue < 0 || epilogue > 2) return 0;
  if (epilogue == 2 && (rows_per_image <= 0 || M % rows_per_image || rows_per_image % 32)) return 0;   // a 32-row box: one image
  return 1;
}

extern "C" int psalm_linear_fused(const void* a, long long a_row_stride, const void* w, const void* bias, void* out, long long M,
                                  int N, int K, int epilogue, long long rows_per_image, int dtype, void* stream) {
  PSALM_REQUIRE(a && w && out, "linear_fused: null pointer");
  PSALM_REQUIRE(psalm_linear_fused_supported(M, N, K, epilogue, rows_per_image, dtype),
                "linear_fused: unsupported shape M=%lld N=%d K=%d epilogue=%d (16-bit storage, N %% 256 == 0, K %% 64 == 0)", M, N, K,
                epilogue);
  PSALM_REQUIRE(a_row_stride >= K && a_row_stride % 8 == 0, "linear_fused: a_row_stride must be >= K and a multiple of 8 elements");
  PSALM_REQUIRE((reinterpret_cast<uintptr_t>(a) & 15) == 0 && (reinterpret_cast<uintptr_t>(w) & 15) == 0 &&
                    (reinterpret_cast<uintptr_t>(out) & 15) == 0 && (!bias || (reinterpret_cast<uintptr_t>(bias) & 15) == 0),
                "linear_fused: pointers must be 16-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  GwParams p;
  p.bias = bias; p.M = (int)M; p.N = N; p.K = K; p.S = (int)(epilogue == 2 ? rows_per_image : 1);
  p.tiles_m = (int)((M + gw::BM - 1) / gw::BM);
  p.tiles_n = N / gw::BN;
  CUtensorMap ma, mw, mo;
  const bool maps_ok =
      gw_make_map(&ma, a, M, K, a_row_stride, gw::BK, gw::BM, CU_TENSOR_MAP_SWIZZLE_128B, dtype) &&
      gw_make_map(&mw, w, N, K, K, gw::BK, gw::BN, CU_TENSOR_MAP_SWIZZLE_128B, dtype) &&
      (epilogue == 2 ? gw_make_map(&mo, out, M * (N / 32), 32, 32, 32, 32, CU_TENSOR_MAP_SWIZZLE_64B, dtype)
                     : gw_make_map(&mo, out, M, N, N, 64, gw::WG_ROWS, CU_TENSOR_MAP_SWIZZLE_128B, dtype));
  if (!maps_ok) {
    set_error("linear_fused: cuTensorMapEncodeTiled failed");
    return PSALM_E_CUDA;
  }
  const long long tiles = (long long)p.tiles_m * p.tiles_n;
  const int grid = (int)(tiles < gw_sm_count() ? tiles : gw_sm_count());
  cudaError_t e;
  const bool bf = dtype == PSALM_BF16;
  switch (epilogue) {
    case 0: e = bf ? gw_launch<__nv_bfloat16, 0>(ma, mw, mo, p, grid, st) : gw_launch<__half, 0>(ma, mw, mo, p, grid, st); break;
    case 1: e = bf ? gw_launch<__nv_bfloat16, 1>(ma, mw, mo, p, grid, st) : gw_launch<__half, 1>(ma, mw, mo, p, grid, st); break;
    default: e = bf ? gw_launch<__nv_bfloat16, 2>(ma, mw, mo, p, grid, st) : gw_launch<__half, 2>(ma, mw, mo, p, grid, st); break;
  }
  if (e != cudaSuccess) {
    set_error("linear_fused: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    return PSALM_E_CUDA;
  }
  return check_launch("linear_fused");
}
