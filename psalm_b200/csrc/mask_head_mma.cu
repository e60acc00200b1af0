// Tensor-core mask projection for 16-bit storage:  D[q, p] = sum_c mask_embed[q, c] * feats[p, c]
// (einsum "bqc,bchw->bqhw", mask2former_transformer_decoder.py:750, on token-major feats = both operands
// K-major).  One CTA = all (<= 112) queries x a tile of TP pixels, the whole K = 256 resident in shared
// memory (cp.async), mma.sync.m16n8k16 with fp32 accumulation.  Two epilogues:
//   kBits = true   the attention mask of the next decoder layer: bit = (D < 0) packed 32 pixels / word
//                  straight from the accumulators (quad OR-reduction) — the fp32 logits of the nine
//                  intermediate heads are never written (mask2former_transformer_decoder.py:754-759);
//   kBits = false  the final mask logits [B, Q, P] in the storage type.
#include <type_traits>

#include "common.cuh"

namespace psalm {

constexpr int MH_QP = 112, MH_C = 256, MH_LD = MH_C + 8;

__device__ __forceinline__ void mh_cp16(void* smem, const void* gmem, int bytes) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(a), "l"(gmem), "r"(bytes));
}
__device__ __forceinline__ void mh_ldsm(uint32_t (&r)[4], const void* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
template <typename T>
__device__ __forceinline__ void mh_mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
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

// grid = (ceil(P / TP), B), block = 128 (4 warps; warp w owns query m-tiles w and w + 4)
template <typename T, int TP, bool kBits>
__global__ void __launch_bounds__(128) mask_proj_mma_kernel(const T* __restrict__ me, const T* __restrict__ feats,
                                                            T* __restrict__ out, uint32_t* __restrict__ bits,
                                                            int Q, int P, int W32, long long fbs) {
  extern __shared__ __align__(16) unsigned char mh_smem[];
  T* As = reinterpret_cast<T*>(mh_smem);          // [MH_QP][MH_LD]  mask_embed
  T* Bs = As + MH_QP * MH_LD;                     // [TP][MH_LD]     feats tile
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b = blockIdx.y, p0 = blockIdx.x * TP;
  const T* meb = me + (size_t)b * Q * MH_C;
  const T* fb = feats + (size_t)b * fbs;   // fbs = P * C, or 0: one feature map for every query set
  for (int i = tid; i < MH_QP * (MH_C / 8); i += 128) {
    const int row = i / (MH_C / 8), c8 = (i % (MH_C / 8)) * 8;
    const bool ok = row < Q;
    mh_cp16(&As[row * MH_LD + c8], meb + (size_t)(ok ? row : 0) * MH_C + c8, ok ? 16 : 0);
  }
  for (int i = tid; i < TP * (MH_C / 8); i += 128) {
    const int row = i / (MH_C / 8), c8 = (i % (MH_C / 8)) * 8;
    const bool ok = p0 + row < P;
    mh_cp16(&Bs[row * MH_LD + c8], fb + (size_t)(ok ? p0 + row : 0) * MH_C + c8, ok ? 16 : 0);
  }
  asm volatile("cp.async.commit_group;\n" ::);
  asm volatile("cp.async.wait_group 0;\n" ::);
  __syncthreads();

  constexpr int NT = TP / 8;
  float acc[2][NT][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < NT; ++j) acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.f;
  const int mi = lane >> 3;
  const bool two = warp + 4 < MH_QP / 16;   // warps 0..2 own two m-tiles, warp 3 one
#pragma unroll 4
  for (int ks = 0; ks < MH_C / 16; ++ks) {
    uint32_t a0[4], a1[4];
    mh_ldsm(a0, &As[(warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * MH_LD + ks * 16 + (lane >> 4) * 8]);
    if (two) mh_ldsm(a1, &As[((warp + 4) * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * MH_LD + ks * 16 + (lane >> 4) * 8]);
#pragma unroll
    for (int np = 0; np < NT / 2; ++np) {
      uint32_t bf[4];
      mh_ldsm(bf, &Bs[(np * 16 + (lane & 7) + (mi >> 1) * 8) * MH_LD + ks * 16 + (mi & 1) * 8]);
      mh_mma<T>(acc[0][2 * np], a0, bf[0], bf[1]);
      mh_mma<T>(acc[0][2 * np + 1], a0, bf[2], bf[3]);
      if (two) {
        mh_mma<T>(acc[1][2 * np], a1, bf[0], bf[1]);
        mh_mma<T>(acc[1][2 * np + 1], a1, bf[2], bf[3]);
      }
    }
  }
  const int g = lane >> 2, t4 = lane & 3;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt) {
    if (mt == 1 && !two) break;
    const int qbase = (warp + 4 * mt) * 16;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int q = qbase + g + 8 * r;
      if constexpr (kBits) {
#pragma unroll
        for (int wd = 0; wd < TP / 32; ++wd) {
          uint32_t word = 0;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int nt = wd * 4 + j;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int pl = nt * 8 + 2 * t4 + e;   // pixel within the tile
              if (p0 + pl < P && acc[mt][nt][2 * r + e] < 0.f) word |= 1u << (pl & 31);
            }
          }
          word |= __shfl_xor_sync(0xffffffffu, word, 1);
          word |= __shfl_xor_sync(0xffffffffu, word, 2);
          if (t4 == 0 && q < Q && (p0 / 32 + wd) < W32) bits[((size_t)b * Q + q) * W32 + p0 / 32 + wd] = word;
        }
      } else {
        if (q < Q) {
#pragma unroll
          for (int nt = 0; nt < NT; ++nt) {
            const int pp = p0 + nt * 8 + 2 * t4;
            T* dst = out + ((size_t)b * Q + q) * P + pp;
            if (pp + 1 < P && (((size_t)dst) & 3) == 0) *reinterpret_cast<uint32_t*>(dst) = pack2<T>(acc[mt][nt][2 * r], acc[mt][nt][2 * r + 1]);
            else {
              if (pp < P) dst[0] = from_f32<T>(acc[mt][nt][2 * r]);
              if (pp + 1 < P) dst[1] = from_f32<T>(acc[mt][nt][2 * r + 1]);
            }
          }
        }
      }
    }
  }
}

// row_open[row] = every valid key of the row is blocked (mask2former_transformer_decoder.py:647)
__global__ void row_open_kernel(const uint32_t* __restrict__ bits, uint8_t* __restrict__ row_open, int rows, int P,
                                int W32) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows) return;
  bool all = true;
  for (int w = lane; w < W32; w += 32) {
    const int valid = P - w * 32;
    const uint32_t vm = valid >= 32 ? 0xffffffffu : ((1u << valid) - 1u);
    if ((bits[(size_t)warp * W32 + w] & vm) != vm) all = false;
  }
  all = __all_sync(0xffffffffu, all);
  if (lane == 0) row_open[warp] = all ? 1 : 0;
}

template <typename T>
static int launch_mask_proj(const void* me, const void* feats, void* out, uint32_t* bits, uint8_t* row_open, int B,
                            int Q, int P, long long fbs, cudaStream_t st) {
  const int W32 = (P + 31) / 32;
  cudaError_t e;
  if (bits) {
    constexpr int TP = 32;
    const size_t smem = sizeof(T) * (MH_QP + TP) * MH_LD;
    e = cudaFuncSetAttribute(mask_proj_mma_kernel<T, TP, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("mask_proj: %s", cudaGetErrorString(e)); return PSALM_E_CUDA; }
    dim3 grid((P + TP - 1) / TP, B);
    mask_proj_mma_kernel<T, TP, true><<<grid, 128, smem, st>>>((const T*)me, (const T*)feats, nullptr, bits, Q, P, W32, fbs);
    row_open_kernel<<<(B * Q * 32 + 255) / 256, 256, 0, st>>>(bits, row_open, B * Q, P, W32);
  } else {
    constexpr int TP = 64;
    const size_t smem = sizeof(T) * (MH_QP + TP) * MH_LD;
    e = cudaFuncSetAttribute(mask_proj_mma_kernel<T, TP, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("mask_proj: %s", cudaGetErrorString(e)); return PSALM_E_CUDA; }
    dim3 grid((P + TP - 1) / TP, B);
    mask_proj_mma_kernel<T, TP, false><<<grid, 128, smem, st>>>((const T*)me, (const T*)feats, (T*)out, nullptr, Q, P, W32, fbs);
  }
  return check_launch("mask_proj_mma_kernel");
}

int mma_mask_proj(const void* me, const void* feats, long long feats_bstride, void* out, uint32_t* bits, uint8_t* row_open,
                  int B, int Q, int P, int dtype, cudaStream_t st) {
  if (dtype == PSALM_BF16) return launch_mask_proj<__nv_bfloat16>(me, feats, out, bits, row_open, B, Q, P, feats_bstride, st);
  return launch_mask_proj<__half>(me, feats, out, bits, row_open, B, Q, P, feats_bstride, st);
}

}  // namespace psalm
