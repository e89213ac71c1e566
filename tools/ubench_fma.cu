// ubench_fma.cu — issue rate of FFMA vs the mixed-precision FHFMA.BF16 (fma.rn.f32.bf16) on one SM partition, to read
// the GEMV_MIXED_FMA experiment (DESIGN.md section 9): if FHFMA runs at the FFMA rate the batch-1 projection loop sheds
// 43 % of its instructions, at half rate it gains nothing.   build: nvcc -arch=sm_90a -O3 -o tools/bin/ubench_fma tools/ubench_fma.cu
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

template <int MODE>
__global__ void k(float* out, const uint32_t* in, int iters, long long* cyc) {
  float a[8];
  uint32_t w = in[threadIdx.x], x = in[threadIdx.x + 1024];
  for (int i = 0; i < 8; ++i) a[i] = (float)i;
  const float fw = __uint_as_float(w & 0xffff0000u), fx = __uint_as_float(x << 16);
  __syncthreads();
  const long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (MODE == 0) {
        a[i] = fmaf(fw, fx, a[i]);
      } else if (MODE == 1) {
        asm volatile("{\n\t.reg .b16 wl, wh, xl, xh;\n\tmov.b32 {wl, wh}, %1;\n\tmov.b32 {xl, xh}, %2;\n\tfma.rn.f32.bf16 %0, wl, xl, %0;\n\t}" : "+f"(a[i]) : "r"(w), "r"(x));
      } else {  // unpack + FFMA, as the default loop does per element
        float fl = __uint_as_float(w << 16), fh = __uint_as_float(x & 0xffff0000u);
        a[i] = fmaf(fl, fh, a[i]);
        w = w * 3u + 1u;
      }
    }
  }
  const long long t1 = clock64();
  float s = 0;
  for (int i = 0; i < 8; ++i) s += a[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}

int main() {
  float* out;
  uint32_t* in;
  long long* cyc;
  cudaMalloc(&out, 1 << 20);
  cudaMalloc(&in, 1 << 16);
  cudaMemset(in, 0x3f, 1 << 16);
  cudaMallocManaged(&cyc, 8);
  const int iters = 4096;
  for (int threads : {128, 256, 512, 1024}) {
    long long c[3];
    for (int mode = 0; mode < 3; ++mode) {
      for (int rep = 0; rep < 2; ++rep) {
        if (mode == 0) k<0><<<1, threads>>>(out, in, iters, cyc);
        if (mode == 1) k<1><<<1, threads>>>(out, in, iters, cyc);
        if (mode == 2) k<2><<<1, threads>>>(out, in, iters, cyc);
        cudaDeviceSynchronize();
      }
      c[mode] = *cyc;
    }
    const double n = (double)iters * 8 * threads / 32;  // warp-level FMA instructions issued by the CTA
    printf("threads %4d: FFMA %.2f warp-inst/clk/SM, FHFMA.BF16 %.2f, unpack+FFMA %.2f (FMAs only counted)\n", threads, n / c[0], n / c[1], n / c[2]);
  }
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
