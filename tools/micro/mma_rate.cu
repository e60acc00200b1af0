// Micro-benchmark: issue rate of warp-level mma.sync.m16n8k16 (bf16 -> fp32) and MUFU.EX2 on sm_90a (H100), per SM.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/micro/mma_rate tools/micro/mma_rate.cu
#include <cstdio>
#include <cuda_runtime.h>

template <int CHAINS>
__global__ void mma_kernel(float* out, int iters) {
  float d[CHAINS][4];
#pragma unroll
  for (int c = 0; c < CHAINS; ++c) d[c][0] = d[c][1] = d[c][2] = d[c][3] = 0.f;
  unsigned a0 = threadIdx.x, a1 = a0 * 3, a2 = a0 * 5, a3 = a0 * 7, b0 = a0 * 11, b1 = a0 * 13;
  for (int i = 0; i < iters; ++i) {
#pragma unroll
    for (int c = 0; c < CHAINS; ++c)
      asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                   : "+f"(d[c][0]), "+f"(d[c][1]), "+f"(d[c][2]), "+f"(d[c][3])
                   : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
  }
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < CHAINS; ++c) s += d[c][0] + d[c][1] + d[c][2] + d[c][3];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int CHAINS>
__global__ void ex2_kernel(float* out, int iters) {
  float x[CHAINS];
#pragma unroll
  for (int c = 0; c < CHAINS; ++c) x[c] = -0.001f * (threadIdx.x + c);
  for (int i = 0; i < iters; ++i) {
#pragma unroll
    for (int c = 0; c < CHAINS; ++c) asm volatile("ex2.approx.ftz.f32 %0, %0;\n" : "+f"(x[c]));
  }
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < CHAINS; ++c) s += x[c];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

int main() {
  float* out;
  cudaMalloc(&out, 148 * 1024 * sizeof(float) * 4);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  int clk_khz = 0;
  cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
  const int iters = 20000;
  for (int warps = 4; warps <= 32; warps *= 2) {
    for (int rep = 0; rep < 2; ++rep) {
      cudaEventRecord(e0);
      mma_kernel<8><<<148, warps * 32>>>(out, iters);
      cudaEventRecord(e1);
      cudaEventSynchronize(e1);
    }
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    const double n = (double)iters * 8 * warps;   // mma per SM
    printf("mma.sync m16n8k16 bf16: %2d warps/SM: %.2f mma/us/SM -> %.1f clk per mma per SM at %d MHz (%.1f dense TFLOP/s chip)\n",
           warps, n / (ms * 1e3), ms * 1e-3 * clk_khz * 1e3 / n, clk_khz / 1000, n * 148 * 4096 / (ms * 1e-3) / 1e12);
  }
  for (int warps = 4; warps <= 32; warps *= 2) {
    for (int rep = 0; rep < 2; ++rep) {
      cudaEventRecord(e0);
      ex2_kernel<8><<<148, warps * 32>>>(out, iters);
      cudaEventRecord(e1);
      cudaEventSynchronize(e1);
    }
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    const double n = (double)iters * 8 * warps * 32;   // ex2 per SM
    printf("ex2.approx: %2d warps/SM: %.1f ex2/clk/SM\n", warps, n / (ms * 1e-3 * clk_khz * 1e3));
  }
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
