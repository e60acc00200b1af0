// Autoregressive decode of the LLM (SURVEY.md section 8 f4): paged KV cache + single-token causal attention.
//
// Replaces, for the chat path (psalm/serve/cli.py:89-96 -> PSALM.generate -> PhiAttention with past_key_values,
// language_model/llava_phi.py:773-778 single-token branch), the `torch.cat((past_key, key), dim=2)` growth of HF's
// DynamicCache (a full copy of the cache per layer per token) and the eager [B, 32, 1, T] score / softmax / matmul
// chain, by
//   psalm_kv_cache_write      K / V rows of new tokens -> fixed-size pages through a block table (nothing is ever moved)
//   psalm_paged_decode_attention  one CTA per (head, sequence): every lane owns whole keys (no per-key shuffles), an
//                             online softmax per lane, ONE warp-shuffle butterfly + a 4-warp shared-memory merge at the
//                             end.  HBM-bound: K and V of the sequence are read exactly once, 128 B per (key, head).
// Page layout: [num_pages, n_heads, page_size, head_dim] (head-major inside a page, so the keys of one head are
// contiguous 128-byte rows).  Block table [B, max_pages] int32, sequence lengths [B] int32.
#include "common.cuh"

namespace psalm {

template <typename T>
__global__ void kv_cache_write_kernel(const T* __restrict__ qkv, T* __restrict__ kc, T* __restrict__ vc,
                                      const int* __restrict__ block_table, const int* __restrict__ start_pos, int B, int Tn,
                                      int nh, int hd, int ps, int max_pages) {
  constexpr int CH = 16 / sizeof(T);
  const int chunks = hd / CH;
  const long long n = (long long)B * Tn * 2 * nh * chunks;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    long long r = i;
    const int c = (int)(r % chunks); r /= chunks;
    const int h = (int)(r % nh); r /= nh;
    const int which = (int)(r % 2); r /= 2;
    const int t = (int)(r % Tn);
    const int b = (int)(r / Tn);
    const int pos = start_pos[b] + t;
    const int page = block_table[b * max_pages + pos / ps], slot = pos % ps;
    const uint4 v = *reinterpret_cast<const uint4*>(qkv + ((((size_t)b * Tn + t) * 3 + 1 + which) * nh + h) * hd + c * CH);
    T* dst = (which ? vc : kc) + (((size_t)page * nh + h) * ps + slot) * hd + c * CH;
    *reinterpret_cast<uint4*>(dst) = v;
  }
}

// grid = (nh, B), block = 128.  q [B, nh, hd] with batch stride q_stride (elements); out [B, nh * hd].
template <typename T, int HD>
__global__ void __launch_bounds__(128) paged_decode_kernel(const T* __restrict__ q, long long q_stride, const T* __restrict__ kc,
                                                          const T* __restrict__ vc, const int* __restrict__ block_table,
                                                          const int* __restrict__ seq_lens, T* __restrict__ out, int nh, int ps,
                                                          int max_pages, float scale_log2e) {
  constexpr int CH = 16 / sizeof(T);
  __shared__ float qs[HD];
  __shared__ float red[4][HD + 2];
  const int h = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid < HD) qs[tid] = to_f32<T>(q[(size_t)b * q_stride + (size_t)h * HD + tid]) * scale_log2e;
  __syncthreads();
  const int len = seq_lens[b];
  float m = -INFINITY, l = 0.f, acc[HD];
#pragma unroll
  for (int d = 0; d < HD; ++d) acc[d] = 0.f;
  for (int k = tid; k < len; k += 128) {   // this lane owns key k
    const int page = block_table[b * max_pages + k / ps], slot = k % ps;
    const size_t row = (((size_t)page * nh + h) * ps + slot) * HD;
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < HD / CH; ++c) {
      float f[CH];
      load16_as_f32<T>(kc + row + c * CH, f);
#pragma unroll
      for (int e = 0; e < CH; ++e) s = fmaf(f[e], qs[c * CH + e], s);
    }
    const float mn = fmaxf(m, s);
    const float corr = exp2f(m - mn), p = exp2f(s - mn);   // exp2f(-inf) = 0 on the first key
    l = l * corr + p;
#pragma unroll
    for (int c = 0; c < HD / CH; ++c) {
      float f[CH];
      load16_as_f32<T>(vc + row + c * CH, f);
#pragma unroll
      for (int e = 0; e < CH; ++e) acc[c * CH + e] = fmaf(p, f[e], acc[c * CH + e] * corr);
    }
    m = mn;
  }
  // ---- merge the 32 lanes (butterfly), then the 4 warps
  float M = m;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) M = fmaxf(M, __shfl_xor_sync(0xffffffffu, M, o));
  const float sc = (m == -INFINITY) ? 0.f : exp2f(m - M);
  l *= sc;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
#pragma unroll
  for (int d = 0; d < HD; ++d) {
    float a = acc[d] * sc;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) red[warp][d] = a;
  }
  if (lane == 0) {
    red[warp][HD] = M;
    red[warp][HD + 1] = l;
  }
  __syncthreads();
  if (tid < HD) {
    float MM = fmaxf(fmaxf(red[0][HD], red[1][HD]), fmaxf(red[2][HD], red[3][HD]));
    float L = 0.f, O = 0.f;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const float e = (red[w][HD] == -INFINITY) ? 0.f : exp2f(red[w][HD] - MM);
      L += red[w][HD + 1] * e;
      O += red[w][tid] * e;
    }
    out[((size_t)b * nh + h) * HD + tid] = from_f32<T>(L > 0.f ? O / L : 0.f);
  }
}

}  // namespace psalm

using namespace psalm;

extern "C" int psalm_kv_cache_write(const void* qkv, void* kcache, void* vcache, const int* block_table, const int* start_pos,
                                    int B, int T_, int nh, int hd, int page_size, int max_pages, int dtype, void* stream) {
  PSALM_REQUIRE(qkv && kcache && vcache && block_table && start_pos, "kv_cache_write: null pointer");
  PSALM_REQUIRE(B > 0 && T_ > 0 && nh > 0 && page_size > 0 && max_pages > 0, "kv_cache_write: bad dimension");
  PSALM_REQUIRE(hd % (16 / (int)dtype_size(dtype)) == 0, "kv_cache_write: head_dim %d not a multiple of 16 bytes", hd);
  cudaStream_t st = (cudaStream_t)stream;
  const long long n = (long long)B * T_ * 2 * nh * (hd / (16 / (int)dtype_size(dtype)));
  const int blocks = (int)((n + 255) / 256 < 132 * 8 ? (n + 255) / 256 : 132 * 8);
  if (dtype == PSALM_F32) kv_cache_write_kernel<float><<<blocks, 256, 0, st>>>((const float*)qkv, (float*)kcache, (float*)vcache, block_table, start_pos, B, T_, nh, hd, page_size, max_pages);
  else if (dtype == PSALM_F16) kv_cache_write_kernel<__half><<<blocks, 256, 0, st>>>((const __half*)qkv, (__half*)kcache, (__half*)vcache, block_table, start_pos, B, T_, nh, hd, page_size, max_pages);
  else if (dtype == PSALM_BF16) kv_cache_write_kernel<__nv_bfloat16><<<blocks, 256, 0, st>>>((const __nv_bfloat16*)qkv, (__nv_bfloat16*)kcache, (__nv_bfloat16*)vcache, block_table, start_pos, B, T_, nh, hd, page_size, max_pages);
  else { set_error("kv_cache_write: bad dtype %d", dtype); return PSALM_E_ARG; }
  return check_launch("kv_cache_write_kernel");
}

extern "C" int psalm_paged_decode_attention(const void* q, long long q_batch_stride, const void* kcache, const void* vcache,
                                            const int* block_table, const int* seq_lens, void* out, int B, int nh, int hd,
                                            int page_size, int max_pages, int dtype, void* stream) {
  PSALM_REQUIRE(q && kcache && vcache && block_table && seq_lens && out, "paged_decode_attention: null pointer");
  PSALM_REQUIRE(B > 0 && B <= 65535 && nh > 0 && page_size > 0 && max_pages > 0, "paged_decode_attention: bad dimension");
  PSALM_REQUIRE(hd == 64 || hd == 32, "paged_decode_attention: head_dim %d unsupported (32 or 64)", hd);
  cudaStream_t st = (cudaStream_t)stream;
  const float sc = 1.0f / sqrtf((float)hd) * 1.4426950408889634f;
  dim3 grid(nh, B);
#define PD(TT, HH) paged_decode_kernel<TT, HH><<<grid, 128, 0, st>>>((const TT*)q, q_batch_stride, (const TT*)kcache, (const TT*)vcache, \
                                                                     block_table, seq_lens, (TT*)out, nh, page_size, max_pages, sc)
  if (dtype == PSALM_F32) { if (hd == 64) PD(float, 64); else PD(float, 32); }
  else if (dtype == PSALM_F16) { if (hd == 64) PD(__half, 64); else PD(__half, 32); }
  else if (dtype == PSALM_BF16) { if (hd == 64) PD(__nv_bfloat16, 64); else PD(__nv_bfloat16, 32); }
  else { set_error("paged_decode_attention: bad dtype %d", dtype); return PSALM_E_ARG; }
#undef PD
  return check_launch("paged_decode_kernel");
}
