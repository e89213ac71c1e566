// dequant.cu — GGUF block dequantisation on load ("dequant-on-load -> bf16", BASELINE config 3).
//
// Block semantics follow llama.cpp's gguf-py (site-packages/gguf/quants.py, the first-party definition):
//   Q4_0  quants.py:241-253   32 elems: fp16 d | 16 B nibbles;  w = d * (q - 8); elems 0..15 = low nibbles, 16..31 = high
//   Q8_0  quants.py:396-401   32 elems: fp16 d | 32 x int8;      w = d * q
//   Q4_K  quants.py:478-522   256 elems: fp16 d, fp16 dmin, 12 B packed 6-bit (scale,min) x 8, 128 B nibbles;
//                             w = (d*sc) * q - (dmin*m)
//   Q6_K  quants.py:554-572   256 elems: 128 B ql, 64 B qh, 16 x int8 scales, fp16 d;  w = (d*scale) * (q6 - 32)
// fp32 arithmetic with the same operation order as the numpy code (no FMA contraction), then one RNE rounding to bf16.
// HBM-bound, load-time only.
#include <cuda_fp16.h>

#include "common.cuh"
#include "kernels.h"
#include "loader.h"

namespace {

__device__ __forceinline__ float half_at(const uint8_t* p) {
  const unsigned short u = (unsigned short)p[0] | ((unsigned short)p[1] << 8);
  return __half2float(__ushort_as_half(u));
}

__device__ __forceinline__ float deq_q4_0(const uint8_t* base, int64_t e) {
  const uint8_t* b = base + (e >> 5) * 18;
  const int j = (int)(e & 31);
  const int q = j < 16 ? (b[2 + j] & 0xF) : (b[2 + j - 16] >> 4);
  return __fmul_rn(half_at(b), (float)(q - 8));
}

__device__ __forceinline__ float deq_q8_0(const uint8_t* base, int64_t e) {
  const uint8_t* b = base + (e >> 5) * 34;
  return __fmul_rn((float)(int8_t)b[2 + (e & 31)], half_at(b));
}

__device__ __forceinline__ float deq_q4_k(const uint8_t* base, int64_t e) {
  const uint8_t* b = base + (e >> 8) * 144;
  const int i = (int)(e & 255);
  const int is = i >> 5;  // sub-block 0..7
  const uint8_t* sc = b + 4;
  int s, m;
  if (is < 4) {
    s = sc[is] & 63;
    m = sc[is + 4] & 63;
  } else {
    s = (sc[is + 4] & 0xF) | ((sc[is - 4] >> 6) << 4);
    m = (sc[is + 4] >> 4) | ((sc[is] >> 6) << 4);
  }
  const uint8_t byte = b[16 + (is >> 1) * 32 + (i & 31)];
  const int q = (is & 1) ? (byte >> 4) : (byte & 0xF);
  const float d = __fmul_rn(half_at(b), (float)s);
  const float dm = __fmul_rn(half_at(b + 2), (float)m);
  return __fsub_rn(__fmul_rn(d, (float)q), dm);
}

__device__ __forceinline__ float deq_q6_k(const uint8_t* base, int64_t e) {
  const uint8_t* b = base + (e >> 8) * 210;
  const int i = (int)(e & 255);
  const int r = i >> 5, c = i & 31;  // row of 32 in the (8, 32) view of quants.py:565-569
  const int ql = (b[(r >> 2) * 64 + (r & 1) * 32 + c] >> (4 * ((r & 3) >> 1))) & 0xF;
  const int qh = (b[128 + (r >> 2) * 32 + c] >> (2 * (r & 3))) & 3;
  const int q = (int)(int8_t)(ql | (qh << 4)) - 32;
  const float d = __fmul_rn(half_at(b + 208), (float)(int8_t)b[192 + (i >> 4)]);
  return __fmul_rn(d, (float)q);
}

__global__ void dequant_kernel(const uint8_t* __restrict__ src, int dtype, int64_t n, bf16* __restrict__ dst) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    float v;
    switch (dtype) {
      case ssb::DT_Q4_0: v = deq_q4_0(src, e); break;
      case ssb::DT_Q8_0: v = deq_q8_0(src, e); break;
      case ssb::DT_Q4_K: v = deq_q4_k(src, e); break;
      case ssb::DT_Q6_K: v = deq_q6_k(src, e); break;
      case ssb::DT_F16: v = __half2float(reinterpret_cast<const __half*>(src)[e]); break;
      case ssb::DT_F32: v = reinterpret_cast<const float*>(src)[e]; break;
      default: v = __bfloat162float(reinterpret_cast<const bf16*>(src)[e]); break;
    }
    dst[e] = __float2bfloat16_rn(v);
  }
}

}  // namespace

// src: raw GGUF tensor bytes on the device; dst: n bf16 values (row-major, GGUF element order)
cudaError_t launch_dequant(const void* src, int dtype, int64_t n, bf16* dst, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  const int64_t blocks = (n + 255) / 256;
  dequant_kernel<<<(unsigned)(blocks > 132 * 32 ? 132 * 32 : blocks), 256, 0, s>>>((const uint8_t*)src, dtype, n, dst);
  return cudaGetLastError();
}
