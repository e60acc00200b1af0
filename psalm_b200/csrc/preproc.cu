// Input pipeline on the device: pixel normalisation + zero padding to the patch grid + unfold into the
// patch-embedding GEMM operand, one pass.
//
// Replaces (reference): the mapper's `(image - pixel_mean) / pixel_std` on the HOST in fp32
// (datasets_mapper/coco_panoptic_mapper.py:161 — the image then crosses PCIe as 12 bytes per pixel instead of 3),
// PatchEmbed's F.pad to a multiple of the patch size and the memory shuffle inside its stride-4 convolution
// (multimodal_encoder/swin_trans.py:427-441).  HBM-bound byte shuffling: one thread moves the 4 horizontally
// adjacent pixels of one (patch row, channel) — a 4-byte (u8) or 16-byte (fp32) load and an 8 / 16-byte store
// that is contiguous across the threads of a patch.
#include "common.cuh"

namespace psalm {

template <typename TI>
__device__ __forceinline__ float pix(const TI* p);
template <> __device__ __forceinline__ float pix<uint8_t>(const uint8_t* p) { return (float)*p; }
template <> __device__ __forceinline__ float pix<float>(const float* p) { return *p; }
template <> __device__ __forceinline__ float pix<__half>(const __half* p) { return __half2float(*p); }
template <> __device__ __forceinline__ float pix<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }

// out [B, Wh*Ww, Cin*PS*PS], element (c, i, j) of patch (py, px) = norm(img[b, c, py*PS + i, px*PS + j]),
// 0 outside the image (the reference pads the NORMALISED tensor with zeros).
template <typename TI, typename TO, int PS>
__global__ void __launch_bounds__(256) patchify_kernel(const TI* __restrict__ img, TO* __restrict__ out,
                                                       const float* __restrict__ mean, const float* __restrict__ stdv,
                                                       int B, int Cin, int H, int W, int Wh, int Ww) {
  const long long n = (long long)B * Wh * Ww * Cin * PS;   // one thread per (b, py, px, c, i): PS pixels
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    long long r = t;
    const int i = (int)(r % PS); r /= PS;
    const int c = (int)(r % Cin); r /= Cin;
    const int px = (int)(r % Ww); r /= Ww;
    const int py = (int)(r % Wh);
    const int b = (int)(r / Wh);
    const int y = py * PS + i, x0 = px * PS;
    float v[PS];
    const bool norm = mean != nullptr;
    const float m = norm ? mean[c] : 0.f, s = norm ? stdv[c] : 1.f;
    const TI* row = img + (((size_t)b * Cin + c) * H + y) * (size_t)W + x0;
#pragma unroll
    for (int j = 0; j < PS; ++j) {
      float f = 0.f;
      if (y < H && x0 + j < W) {
        f = pix<TI>(row + j);
        if (norm) f = (f - m) / s;   // same two fp32 operations, in the same order, as the mapper
      }
      v[j] = f;
    }
    TO* dst = out + t * PS;
#pragma unroll
    for (int j = 0; j < PS; ++j) dst[j] = from_f32<TO>(v[j]);
  }
}

template <typename TI>
static int launch_patchify(const void* img, void* out, const float* mean, const float* stdv, int B, int Cin, int H,
                           int W, int ps, int out_dtype, cudaStream_t st) {
  const int Wh = (H + ps - 1) / ps, Ww = (W + ps - 1) / ps;
  const long long n = (long long)B * Wh * Ww * Cin * ps;
  const int blocks = (int)((n + 255) / 256 < 132 * 16 ? (n + 255) / 256 : 132 * 16);
#define PSALM_PATCHIFY(TO)                                                                                       \
  patchify_kernel<TI, TO, 4><<<blocks, 256, 0, st>>>((const TI*)img, (TO*)out, mean, stdv, B, Cin, H, W, Wh, Ww)
  if (out_dtype == PSALM_F32) PSALM_PATCHIFY(float);
  else if (out_dtype == PSALM_F16) PSALM_PATCHIFY(__half);
  else PSALM_PATCHIFY(__nv_bfloat16);
#undef PSALM_PATCHIFY
  return check_launch("psalm_patchify");
}

}  // namespace psalm

extern "C" int psalm_patchify(const void* images, void* patches, const float* mean, const float* stdv, int B, int Cin,
                              int H, int W, int patch, int in_dtype, int out_dtype, void* stream) {
  using namespace psalm;
  PSALM_REQUIRE(images && patches, "patchify: null pointer");
  PSALM_REQUIRE((mean == nullptr) == (stdv == nullptr), "patchify: mean and std come together");
  PSALM_REQUIRE(patch == 4, "patchify: patch size %d unsupported (Swin uses 4)", patch);
  PSALM_REQUIRE(B > 0 && Cin > 0 && H > 0 && W > 0, "patchify: bad shape");
  PSALM_REQUIRE(out_dtype == PSALM_F32 || out_dtype == PSALM_F16 || out_dtype == PSALM_BF16, "patchify: bad out dtype");
  cudaStream_t st = (cudaStream_t)stream;
  switch (in_dtype) {
    case PSALM_U8: return launch_patchify<uint8_t>(images, patches, mean, stdv, B, Cin, H, W, patch, out_dtype, st);
    case PSALM_F32: return launch_patchify<float>(images, patches, mean, stdv, B, Cin, H, W, patch, out_dtype, st);
    case PSALM_F16: return launch_patchify<__half>(images, patches, mean, stdv, B, Cin, H, W, patch, out_dtype, st);
    case PSALM_BF16: return launch_patchify<__nv_bfloat16>(images, patches, mean, stdv, B, Cin, H, W, patch, out_dtype, st);
  }
  set_error("patchify: unsupported input dtype %d", in_dtype);
  return PSALM_E_UNSUPPORTED;
}
