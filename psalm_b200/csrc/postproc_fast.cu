// Tensor-core formulation of the fused eval_seg post-processing (reference language_model/llava_phi.py:1399-1406
// up-sampling + the task heads :325-447) for 16-bit logits and power-of-two up-sampling (the x4 the model uses).
//
// Bilinear x4 up-sampling of a tile of 8 x 16 output pixels touches at most 4 x 6 source taps, so for ALL queries
// at once it is a small GEMM   X[pixel, query] = Wt[pixel, tap] . Src[tap, query]   (K = 4 x 8 tap slots): the
// weights are multiples of 1/64 (exact in bf16 / fp16), the logits are already 16-bit, products are exact and the
// sum is fp32.
// Each warp owns one 16-pixel row of the tile; the accumulator fragment of that GEMM (rows = pixels, columns =
// queries) is, after the sigmoid, exactly the A-operand fragment of the semantic GEMM
//   sem[pixel, class] = S[pixel, query] . P[query, class]   (fp16 x fp16 -> fp32)
// so the [Q, H, W] logits / sigmoid tensors never exist, not even in shared memory.  Thresholds (x > 0, x >= 0)
// leave the warp as ballots; counts are popc over ballots; sum(sigmoid * [x > 0]) is accumulated in 2^-22 fixed
// point per thread (integer adds: order-independent, deterministic); the panoptic arg-max is an in-thread scan
// plus a 4-lane butterfly.  CTAs are persistent (2 per SM) and walk tiles with a software-prefetched source
// window, so the class-probability operand and all statistics stay on chip for the whole launch.
#include "common.cuh"

namespace psalm {

constexpr int PF_TH = 8, PF_TW = 16;   // output tile: one 16-pixel row per warp
constexpr int PF_QP = 112;            // queries padded to 14 n-tiles
constexpr int PF_CP = 144;            // classes padded to 18 n-tiles
constexpr int PF_TR = 4, PF_TC = 8;   // source window slots per tile (rows x columns)
constexpr int PF_TAPS = PF_TR * PF_TC;   // K of the up-sampling GEMM (tap = row * 8 + column)
constexpr int PF_SLD = PF_TAPS + 8;   // source row stride (elements): 80 B rows, conflict-free ldmatrix
constexpr int PF_NLD = 7;             // 4-byte source pieces staged per thread
constexpr int PF_ALD = PF_QP + 8;     // class-probability row stride (halfs)
constexpr int PF_NV = 56;             // accumulator values per thread (14 n-tiles x 4)
constexpr int PF_KMAX = 256;          // instance slots kept in shared memory
constexpr int PF_THREADS = 256;

struct PostprocFastArgs {
  const void* logits;      // [Q, H4, W4] 16-bit
  const __half* probsT;    // [PF_CP, PF_QP] fp16 class-major, zero padded, or null
  const float* wq;         // [Q] or null
  const float* negq;       // [Q]
  const int* slot_query;   // [K] or null
  float* sem_seg;          // [ncls, H, W]
  float* inst_masks;       // [K, H, W]
  int* ids;                // [H, W]
  unsigned char* in_mask;  // [H, W]
  float* partials;         // [gridDim.x, Q, 5]
  int Q, H4, W4, H, W, ncls, K;
  int tiles_x, ntiles;
};

template <typename T> struct PfMma;
template <> struct PfMma<__half> {
  static __device__ __forceinline__ void mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
};
template <> struct PfMma<__nv_bfloat16> {
  static __device__ __forceinline__ void mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
};

__device__ __forceinline__ void pf_ldsm_x4(uint32_t (&r)[4], const void* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}

// ATen area_pixel_compute_source_index, align_corners = false (UpSample.h), clamped at 0
__device__ __host__ __forceinline__ float pf_srcf(float scale, int d) {
  const float s = scale * ((float)d + 0.5f) - 0.5f;
  return s < 0.f ? 0.f : s;
}

struct PfTile {
  int ty0, tx0, sy0, sx0, SR, SC;
};

__device__ __forceinline__ PfTile pf_tile(const PostprocFastArgs& a, int tile, float sh, float sw) {
  PfTile t;
  const int tyi = tile / a.tiles_x, txi = tile - tyi * a.tiles_x;
  t.ty0 = tyi * PF_TH;
  t.tx0 = txi * PF_TW;
  const int ylast = min(t.ty0 + PF_TH, a.H) - 1, xlast = min(t.tx0 + PF_TW, a.W) - 1;
  t.sy0 = (int)pf_srcf(sh, t.ty0);
  t.sx0 = (int)pf_srcf(sw, t.tx0) & ~1;   // even start: the window is staged in aligned 4-byte pieces
  const int sy1 = min((int)pf_srcf(sh, ylast) + 1, a.H4 - 1), sx1 = min((int)pf_srcf(sw, xlast) + 1, a.W4 - 1);
  t.SR = sy1 - t.sy0 + 1;
  t.SC = sx1 - t.sx0 + 1;
  return t;
}

// source taps of one tile -> shared memory ([query][tap slot], the [n][k] storage of the B operand), asynchronously:
// thread -> (tap slots 2 (tid & 15), +1; queries (tid >> 4) + 16 k), one 4-byte cp.async each (zero-filled where the
// slot lies outside the window or the query does not exist)
template <typename T>
__device__ __forceinline__ void pf_stage_src(const PostprocFastArgs& a, const PfTile& t, int tid, T* dst) {
  const int tp = tid & 15, q0 = tid >> 4;
  const int ty = tp >> 2, tx = (tp & 3) * 2;
  const int nb = ty < t.SR ? (tx + 1 < t.SC ? 4 : (tx < t.SC ? 2 : 0)) : 0;   // bytes of this piece that exist
  const size_t plane = (size_t)a.H4 * a.W4;
  const T* p = reinterpret_cast<const T*>(a.logits) + (size_t)q0 * plane + (size_t)(t.sy0 + ty) * a.W4 + (t.sx0 + tx);
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(dst + q0 * PF_SLD + 2 * tp);
#pragma unroll
  for (int k = 0; k < PF_NLD; ++k) {
    const int n = (q0 + 16 * k < a.Q) ? nb : 0;
    const T* src = n ? p + (size_t)k * 16 * plane : reinterpret_cast<const T*>(a.logits);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(d + (uint32_t)(k * 16 * PF_SLD * sizeof(T))), "l"(src), "r"(n));
  }
  asm volatile("cp.async.commit_group;\n" ::);
}

// sigmoid on the SFU: ex2 + rcp (2 ulp), no range fix-ups (x is a finite logit)
__device__ __forceinline__ float pf_sigmoid(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.f + e));
  return r;
}

template <typename T>
__global__ void __launch_bounds__(PF_THREADS, 2) postproc_fast_kernel(PostprocFastArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __half* As = reinterpret_cast<__half*>(smem_raw);                                  // [PF_CP][PF_ALD]
  T* srcs2 = reinterpret_cast<T*>(As + PF_CP * PF_ALD);                              // [2 stages][PF_QP][PF_SLD]
  uint32_t* bal_pos = reinterpret_cast<uint32_t*>(srcs2 + 2 * PF_QP * PF_SLD);       // [8 warps][PF_NV]
  uint32_t* bal_ge = bal_pos + 8 * PF_NV;                                            // [8][PF_NV]
  int* ps_acc = reinterpret_cast<int*>(bal_ge + 8 * PF_NV);                          // [28][256] fixed-point partial sums
  float* wqs = reinterpret_cast<float*>(ps_acc + 28 * PF_THREADS);                   // [PF_QP]
  float* nqs = wqs + PF_QP;                                                          // [PF_QP]
  int* area_s = reinterpret_cast<int*>(nqs + PF_QP);                                 // [PF_QP]
  int* inter_s = area_s + PF_QP;                                                     // [PF_QP]
  int* slots = inter_s + PF_QP;                                                      // [PF_KMAX] packed ballot coordinates
  int* zflag = slots + PF_KMAX;                                                      // [8] warp saw an exact zero logit

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t4 = lane & 3;
  const int Q = a.Q;
  const bool pan = a.wq != nullptr, sem = a.probsT != nullptr, inst = a.slot_query != nullptr;
  const float sh = (float)a.H4 / (float)a.H, sw = (float)a.W4 / (float)a.W;

  // ---- once per CTA: operands and accumulators that live for the whole launch
  if (sem)
    for (int i = tid; i < PF_CP * PF_QP / 8; i += PF_THREADS) {
      const int row = i / (PF_QP / 8), c8 = (i % (PF_QP / 8)) * 8;
      *reinterpret_cast<uint4*>(&As[row * PF_ALD + c8]) = __ldg(reinterpret_cast<const uint4*>(a.probsT + row * PF_QP + c8));
    }
  for (int i = tid; i < PF_QP; i += PF_THREADS) {
    wqs[i] = (pan && i < Q) ? a.wq[i] : 0.f;
    nqs[i] = (pan && i < Q) ? a.negq[i] : -1.f;
    area_s[i] = 0;
    inter_s[i] = 0;
  }
  for (int i = tid; i < PF_KMAX; i += PF_THREADS) {
    // query -> where its bits sit in a warp's ballots: word (q >> 3) * 4 + (q & 1) (+ 2 for pixels 8..15), lane column (q & 7) >> 1
    const int q = (inst && i < a.K) ? a.slot_query[i] : -1;
    slots[i] = q < 0 ? -1 : (((q >> 3) * 4 + (q & 1)) | (((q & 7) >> 1) << 8));
  }
#pragma unroll
  for (int i = 0; i < 28; ++i) ps_acc[i * PF_THREADS + tid] = 0;
  int cnt_tot = 0, ge_tot = 0;   // thread q < Q: running count(x > 0), count(x >= 0)

  int tile = blockIdx.x, it = 0;
  PfTile tl = pf_tile(a, tile < a.ntiles ? tile : 0, sh, sw);
  if (tile < a.ntiles) pf_stage_src<T>(a, tl, tid, srcs2);

  for (; tile < a.ntiles; tile += gridDim.x, ++it) {
    const T* srcs = srcs2 + (it & 1) * PF_QP * PF_SLD;
    asm volatile("cp.async.wait_all;\n" ::);
    __syncthreads();   // this tile's window has landed; every warp is done with the previous tile's buffers
    const PfTile cur = tl;
    if (tile + (int)gridDim.x < a.ntiles) {   // next tile's window streams in behind this tile's math
      tl = pf_tile(a, tile + gridDim.x, sh, sw);
      pf_stage_src<T>(a, tl, tid, srcs2 + ((it + 1) & 1) * PF_QP * PF_SLD);
    }

    // ---- A operand: bilinear weights of this warp's 16 pixels (tile row `warp`) over the 16 taps
    const int py = cur.ty0 + warp;
    const int px0 = cur.tx0 + g, px1 = px0 + 8;
    const bool rowok = py < a.H;
    const bool inb0 = rowok && px0 < a.W, inb1 = rowok && px1 < a.W;
    uint32_t aw[2][4];   // [k-step][fragment register]; tap = ty * 8 + tx -> ty = 2 kstep + (i >> 1), tx = 2 t4 + (i & 1)
    {
      const float fy = pf_srcf(sh, rowok ? py : a.H - 1);
      const int y0 = (int)fy, y1 = y0 + (y0 < a.H4 - 1 ? 1 : 0);
      const float ly = fy - (float)y0, hy = 1.f - ly;
      const int r0 = y0 - cur.sy0, r1 = y1 - cur.sy0;
      float wy[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) wy[r] = (r == r0 ? hy : 0.f) + (r == r1 ? ly : 0.f);
      float wx[2][2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int px = h ? px1 : px0;
        const float fx = pf_srcf(sw, px < a.W ? px : a.W - 1);
        const int x0 = (int)fx, x1 = x0 + (x0 < a.W4 - 1 ? 1 : 0);
        const float lx = fx - (float)x0, hx = 1.f - lx;
        const int c0 = x0 - cur.sx0, c1 = x1 - cur.sx0;
#pragma unroll
        for (int b = 0; b < 2; ++b) wx[h][b] = ((2 * t4 + b) == c0 ? hx : 0.f) + ((2 * t4 + b) == c1 ? lx : 0.f);
      }
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {
        aw[ks][0] = pack2<T>(wy[2 * ks] * wx[0][0], wy[2 * ks] * wx[0][1]);           // row g,     taps row 2ks
        aw[ks][1] = pack2<T>(wy[2 * ks] * wx[1][0], wy[2 * ks] * wx[1][1]);           // row g + 8
        aw[ks][2] = pack2<T>(wy[2 * ks + 1] * wx[0][0], wy[2 * ks + 1] * wx[0][1]);   // row g,     taps row 2ks + 1
        aw[ks][3] = pack2<T>(wy[2 * ks + 1] * wx[1][0], wy[2 * ks + 1] * wx[1][1]);
      }
    }

    // ---- X[pixel, query] = Wt . Src : xs[j][c] -> pixel g + 8 (c >> 1), query 8 j + 2 t4 + (c & 1)
    float xs[14][4];
#pragma unroll
    for (int j = 0; j < 14; ++j) xs[j][0] = xs[j][1] = xs[j][2] = xs[j][3] = 0.f;
#pragma unroll
    for (int jp = 0; jp < 7; ++jp) {
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {
        uint32_t r[4];
        pf_ldsm_x4(r, &srcs[((2 * jp + (lane >> 4)) * 8 + (lane & 7)) * PF_SLD + ks * 16 + ((lane >> 3) & 1) * 8]);
        PfMma<T>::mma(xs[2 * jp], aw[ks], r[0], r[1]);
        PfMma<T>::mma(xs[2 * jp + 1], aw[ks], r[2], r[3]);
      }
    }

    // x == 0 exactly is the only case where (x >= 0) and (x > 0) differ: detect it once per warp
    float mn = 1.f;
#pragma unroll
    for (int j = 0; j < 14; ++j) {
      if (8 * j + 8 <= Q) {   // whole n-tile holds real queries (warp-uniform)
        mn = fminf(fminf(mn, fabsf(xs[j][0])), fminf(fabsf(xs[j][1]), fminf(fabsf(xs[j][2]), fabsf(xs[j][3]))));
      } else {
#pragma unroll
        for (int c = 0; c < 4; ++c) mn = (8 * j + 2 * t4 + (c & 1) < Q) ? fminf(mn, fabsf(xs[j][c])) : mn;
      }
    }
    const bool has_zero = __any_sync(0xffffffffu, mn == 0.f);
    if (lane == 0) zflag[warp] = has_zero;
    if (has_zero) {   // rare: (x >= 0) ballots differ from the (x > 0) ones
#pragma unroll
      for (int j = 0; j < 14; ++j)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const uint32_t bg = __ballot_sync(0xffffffffu, ((c < 2) ? inb0 : inb1) && xs[j][c] >= 0.f);
          if (lane == 0) bal_ge[warp * PF_NV + j * 4 + c] = bg;
        }
    }
    const uint32_t* bal_gew = has_zero ? bal_ge : bal_pos;   // this warp's (x >= 0) ballots

    float bv0 = -2.f, bv1 = -2.f;
    int bq0 = 0, bq1 = 0;
#pragma unroll
    for (int j = 0; j < 14; ++j) {
      float2 w2 = make_float2(0.f, 0.f), n2 = make_float2(0.f, 0.f);
      if (pan) {
        w2 = *reinterpret_cast<const float2*>(&wqs[8 * j + 2 * t4]);
        n2 = *reinterpret_cast<const float2*>(&nqs[8 * j + 2 * t4]);
      }
      int fix[4];
      uint32_t bp[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const float x = xs[j][c];
        const float s = pf_sigmoid(x);
        const bool pos = ((c < 2) ? inb0 : inb1) && x > 0.f;
        bp[c] = __ballot_sync(0xffffffffu, pos);
        // (pos ? s : 0) + 2 lies in [2, 3]: its bit pattern is 0x40000000 + round(s * 2^22)
        fix[c] = __float_as_int((pos ? s : 0.f) + 2.0f);
        if (pan) {
          const float v = fmaf((c & 1) ? w2.y : w2.x, s, (c & 1) ? n2.y : n2.x);
          const int q = 8 * j + 2 * t4 + (c & 1);
          if (c < 2) { if (v > bv0) { bv0 = v; bq0 = q; } }     // ascending q, strict >: first maximum wins
          else       { if (v > bv1) { bv1 = v; bq1 = q; } }
        }
        xs[j][c] = s;
      }
      if (lane == 0) *reinterpret_cast<uint4*>(&bal_pos[warp * PF_NV + j * 4]) = make_uint4(bp[0], bp[1], bp[2], bp[3]);
      // own slot, wrapping integer add: exact and order-independent.  Every add carries 2 * 0x40000000 = 2^31 of
      // exponent bits, removed at the end from the number of tiles; the payload is at most 2^23 per tile.
      atomicAdd(reinterpret_cast<unsigned int*>(&ps_acc[(2 * j) * PF_THREADS + tid]), (unsigned int)fix[0] + (unsigned int)fix[2]);
      atomicAdd(reinterpret_cast<unsigned int*>(&ps_acc[(2 * j + 1) * PF_THREADS + tid]), (unsigned int)fix[1] + (unsigned int)fix[3]);
    }
    __syncwarp();

    // ---- panoptic arg-max: merge the 4 lanes of a quad (they hold the other queries of the same pixels)
    if (pan) {
#pragma unroll
      for (int off = 1; off <= 2; off <<= 1) {
        const float ov0 = __shfl_xor_sync(0xffffffffu, bv0, off), ov1 = __shfl_xor_sync(0xffffffffu, bv1, off);
        const int oq0 = __shfl_xor_sync(0xffffffffu, bq0, off), oq1 = __shfl_xor_sync(0xffffffffu, bq1, off);
        if (ov0 > bv0 || (ov0 == bv0 && oq0 < bq0)) { bv0 = ov0; bq0 = oq0; }
        if (ov1 > bv1 || (ov1 == bv1 && oq1 < bq1)) { bv1 = ov1; bq1 = oq1; }
      }
      if (t4 < 2) {   // lane t4 == 0 commits pixel g, lane t4 == 1 commits pixel g + 8
        const int h = t4;
        const int qb = h ? bq1 : bq0;
        const bool ib = h ? inb1 : inb0;
        if (ib) {
          const uint32_t word = bal_gew[warp * PF_NV + (qb >> 3) * 4 + (qb & 1) + 2 * h];
          const bool im = (word >> (g * 4 + ((qb & 7) >> 1))) & 1u;
          const size_t o = (size_t)py * a.W + (h ? px1 : px0);
          a.ids[o] = qb;
          a.in_mask[o] = im ? 1 : 0;
          atomicAdd(&area_s[qb], 1);
          if (im) atomicAdd(&inter_s[qb], 1);
        }
      }
    }

    // ---- semantic map: sem[pixel, class] = S[pixel, q] . P[q, class]; S fragments come straight from xs
    if (sem) {
      uint32_t sa[7][4];
#pragma unroll
      for (int ks = 0; ks < 7; ++ks) {
        sa[ks][0] = pack2<__half>(xs[2 * ks][0], xs[2 * ks][1]);
        sa[ks][1] = pack2<__half>(xs[2 * ks][2], xs[2 * ks][3]);
        sa[ks][2] = pack2<__half>(xs[2 * ks + 1][0], xs[2 * ks + 1][1]);
        sa[ks][3] = pack2<__half>(xs[2 * ks + 1][2], xs[2 * ks + 1][3]);
      }
      const size_t cs = (size_t)a.H * a.W;
      float* p0 = a.sem_seg + (size_t)(2 * t4) * cs + (size_t)py * a.W + px0;   // class 8 nt + 2 t4
      float* p1 = p0 + cs;                                                      // class 8 nt + 2 t4 + 1
#pragma unroll
      for (int n3 = 0; n3 < PF_CP / 48; ++n3) {   // 3 x 16 classes at a time: six independent accumulator chains
        if (n3 * 48 >= a.ncls) break;
        float acc[6][4];
#pragma unroll
        for (int i = 0; i < 6; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
#pragma unroll
        for (int ks = 0; ks < 7; ++ks) {
#pragma unroll
          for (int u = 0; u < 3; ++u) {
            uint32_t r[4];
            pf_ldsm_x4(r, &As[((2 * (3 * n3 + u) + (lane >> 4)) * 8 + (lane & 7)) * PF_ALD + ks * 16 + ((lane >> 3) & 1) * 8]);
            PfMma<__half>::mma(acc[2 * u], sa[ks], r[0], r[1]);
            PfMma<__half>::mma(acc[2 * u + 1], sa[ks], r[2], r[3]);
          }
        }
#pragma unroll
        for (int i = 0; i < 6; ++i) {
          const int c0 = (6 * n3 + i) * 8 + 2 * t4;
          if (c0 < a.ncls) {
            if (inb0) p0[0] = acc[i][0];
            if (inb1) p0[8] = acc[i][2];
          }
          if (c0 + 1 < a.ncls) {
            if (inb0) p1[0] = acc[i][1];
            if (inb1) p1[8] = acc[i][3];
          }
          p0 += 8 * cs;
          p1 += 8 * cs;
        }
      }
    }
    __syncthreads();   // ballots of every warp are visible

    // ---- per-query counts of this tile: popc over the ballots of the 8 warps
    if (tid < Q) {
      const int q = tid, vi = (q >> 3) * 4 + (q & 1);
      const uint32_t m = 0x11111111u << ((q & 7) >> 1);
      int c = 0, cg = 0;
#pragma unroll
      for (int w = 0; w < 8; ++w) {
        const uint32_t* bg = zflag[w] ? bal_ge : bal_pos;
        c += __popc(bal_pos[w * PF_NV + vi] & m) + __popc(bal_pos[w * PF_NV + vi + 2] & m);
        cg += __popc(bg[w * PF_NV + vi] & m) + __popc(bg[w * PF_NV + vi + 2] & m);
      }
      cnt_tot += c;
      ge_tot += cg;
    }

    // ---- instance masks in slot order: one warp per slot, one lane per run of 4 pixels
    if (inst) {
      const int r = lane >> 2, xo = (lane & 3) * 4;        // tile row, x offset of the run
      const int yy = cur.ty0 + r, xx = cur.tx0 + xo;
      if (yy < a.H && xx < a.W) {
        const uint32_t* brow = bal_pos + r * PF_NV + 2 * (xo >> 3);   // ballots of the warp that owns row r
        const int sh0 = (xo & 7) * 4;
        const bool vec = (xx + 3 < a.W) && ((a.W & 3) == 0);
        const size_t cs = (size_t)a.H * a.W;
        float* dst = a.inst_masks + (size_t)warp * cs + (size_t)yy * a.W + xx;
        for (int k = warp; k < a.K; k += 32, dst += 32 * cs) {   // 4 slots in flight
          int info[4];
          uint32_t wd[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) info[u] = (k + 8 * u < a.K) ? slots[k + 8 * u] : -1;
#pragma unroll
          for (int u = 0; u < 4; ++u) wd[u] = brow[info[u] < 0 ? 0 : (info[u] & 0xff)];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            if (info[u] < 0) continue;
            const uint32_t b = wd[u] >> (sh0 + (info[u] >> 8));
            // bit -> 0.0f / 1.0f: (bit at position p) * (0x3f800000 >> p)
            const float f0 = __uint_as_float((b & 0x1u) * 0x3f800000u), f1 = __uint_as_float((b & 0x10u) * 0x03f80000u);
            const float f2 = __uint_as_float((b & 0x100u) * 0x003f8000u), f3 = __uint_as_float((b & 0x1000u) * 0x0003f800u);
            float* d = dst + (size_t)(8 * u) * cs;
            if (vec) {
              *reinterpret_cast<float4*>(d) = make_float4(f0, f1, f2, f3);
            } else {
              d[0] = f0;
              if (xx + 1 < a.W) d[1] = f1;
              if (xx + 2 < a.W) d[2] = f2;
              if (xx + 3 < a.W) d[3] = f3;
            }
          }
        }
      }
    }
  }

  // ---- per-CTA partial statistics
  __syncthreads();
  if (tid < Q) {
    const int q = tid;
    // sum(sigmoid * [x > 0]): slot 2 (q >> 3) + (q & 1) of the 64 threads with t4 == (q & 7) >> 1
    unsigned long long tot = 0;
    const int slot = 2 * (q >> 3) + (q & 1), tq = (q & 7) >> 1;
    const unsigned int carry = (unsigned int)it << 31;   // it adds of 2^31 per slot (mod 2^32)
    for (int w = 0; w < 8; ++w)
      for (int gg = 0; gg < 8; ++gg) tot += (unsigned int)ps_acc[slot * PF_THREADS + w * 32 + gg * 4 + tq] - carry;
    float* part = a.partials + ((size_t)blockIdx.x * Q + q) * 5;
    part[0] = (float)cnt_tot;
    part[1] = (float)((double)tot * (1.0 / 4194304.0));
    part[2] = (float)ge_tot;
    part[3] = (float)area_s[q];
    part[4] = (float)inter_s[q];
  }
}

constexpr size_t pf_smem_bytes(size_t tsize) {
  return sizeof(__half) * PF_CP * PF_ALD + tsize * 2 * PF_QP * PF_SLD + sizeof(uint32_t) * 2 * 8 * PF_NV + sizeof(int) * 8 +
         sizeof(int) * 28 * PF_THREADS + sizeof(float) * 2 * PF_QP + sizeof(int) * 2 * PF_QP + sizeof(int) * PF_KMAX;
}

static int pf_sm_count() {
  static int sms = 0;
  if (!sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  }
  return sms;
}

int postproc_fast_ctas(int H, int W);

// power-of-two up-sampling whose per-tile source window fits the 16-tap GEMM
bool postproc_fast_ok(int Q, int H4, int W4, int H, int W, int ncls, int K, int dtype) {
  if (dtype != PSALM_F16 && dtype != PSALM_BF16) return false;
  if (Q <= 0 || Q > PF_QP || ncls > PF_CP || H4 <= 0 || W4 <= 0) return false;
  if (H % H4 || W % W4 || (W4 & 1) || K > PF_KMAX) return false;   // (even rows: 4-byte aligned source pieces)
  const int fy = H / H4, fx = W / W4;
  auto pow2 = [](int v) { return v >= 1 && v <= 8 && (v & (v - 1)) == 0; };
  if (!pow2(fy) || !pow2(fx)) return false;
  const float sh = (float)H4 / (float)H, sw = (float)W4 / (float)W;
  int SR = 0, SC = 0;
  for (int ty0 = 0; ty0 < H; ty0 += PF_TH) {
    const int yl = (ty0 + PF_TH < H ? ty0 + PF_TH : H) - 1;
    int s1 = (int)pf_srcf(sh, yl) + 1;
    if (s1 > H4 - 1) s1 = H4 - 1;
    const int n = s1 - (int)pf_srcf(sh, ty0) + 1;
    SR = n > SR ? n : SR;
  }
  for (int tx0 = 0; tx0 < W; tx0 += PF_TW) {
    const int xl = (tx0 + PF_TW < W ? tx0 + PF_TW : W) - 1;
    int s1 = (int)pf_srcf(sw, xl) + 1;
    if (s1 > W4 - 1) s1 = W4 - 1;
    const int n = s1 - ((int)pf_srcf(sw, tx0) & ~1) + 1;
    SC = n > SC ? n : SC;
  }
  const int tiles = ((W + PF_TW - 1) / PF_TW) * ((H + PF_TH - 1) / PF_TH);
  const int ctas = postproc_fast_ctas(H, W);
  if ((tiles + ctas - 1) / ctas > 255) return false;   // 32-bit fixed-point accumulators
  return SR <= PF_TR && SC <= PF_TC;
}

int postproc_fast_ctas(int H, int W) {
  const int tiles = ((W + PF_TW - 1) / PF_TW) * ((H + PF_TH - 1) / PF_TH);
  const int want = 2 * pf_sm_count();
  return tiles < want ? tiles : want;
}

int postproc_fast_launch(const void* logits, const void* probsT_f16, const float* wq, const float* negq,
                         const int* slot_query, float* sem_seg, float* inst_masks, int* ids, unsigned char* in_mask,
                         float* partials, int Q, int H4, int W4, int H, int W, int ncls, int K, int dtype,
                         cudaStream_t st) {
  PostprocFastArgs a{logits, (const __half*)probsT_f16, wq, negq, slot_query, sem_seg, inst_masks, ids, in_mask, partials,
                     Q, H4, W4, H, W, ncls, K, (W + PF_TW - 1) / PF_TW, 0};
  a.ntiles = a.tiles_x * ((H + PF_TH - 1) / PF_TH);
  const int grid = postproc_fast_ctas(H, W);
  const size_t smem = pf_smem_bytes(2);
  cudaError_t e;
  if (dtype == PSALM_F16) {
    e = cudaFuncSetAttribute(postproc_fast_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) postproc_fast_kernel<__half><<<grid, PF_THREADS, smem, st>>>(a);
  } else {
    e = cudaFuncSetAttribute(postproc_fast_kernel<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) postproc_fast_kernel<__nv_bfloat16><<<grid, PF_THREADS, smem, st>>>(a);
  }
  if (e != cudaSuccess) {
    set_error("postproc_fused: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    return PSALM_E_CUDA;
  }
  return check_launch("postproc_fast_kernel");
}

}  // namespace psalm
