// gemv_core.cuh — the tensor-pipe consumer loop shared by proj_rows_kernel (kernels.cu) and decode_mega_kernel (mega.cu):
// a stage holds 16 weight rows x 1024 k with rows padded to GEMV_RS elements (the eight rows of an 8 x 8 ldmatrix tile then
// fall into different bank groups); warp w multiplies ALL 16 rows by the k slice [128 w, 128 w + 128) of the chunk: 8 k-steps
// of mma.sync m16n8k16 with A = ldmatrix.x4 of the stage and B = the staged activations (batch row n = column n of the 8).
// c[4] is the warp's 16 x 8 fp32 fragment, accumulated over the chunks of a pass.  k beyond `len` contributes nothing: whole
// k-steps are skipped and the activation fragment is zero there (callers zero-fill the ring at kernel start so stale weights
// are finite).
#pragma once
#include "common.cuh"

constexpr int GEMV_RS = 1024 + 8;  // stage row stride in elements
SSB_DEVINL void ldmatrix_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, uint32_t saddr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(saddr));
}
SSB_DEVINL void mma_bf16_16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
// stage = first element of the 16-row stage in shared memory; xs = [BT][K] activations; k0/len = this chunk
template <int BT>
SSB_DEVINL void mma_chunk(const bf16* stage, const bf16* xs, int K, int k0, int len, int warp, int lane, float (&c)[4]) {
  const int kw0 = warp * 128;
  const int lrow = (lane & 7) + ((lane >> 3) & 1) * 8, lko = (lane >> 4) * 8;  // ldmatrix source row / k offset of this lane
  const int bn = lane >> 2, bk = (lane & 3) * 2;                               // B fragment: batch row, k pair
  const uint32_t st = smem_u32(stage) + (uint32_t)(lrow * GEMV_RS + kw0 + lko) * 2u;
  const bf16* xrow = xs + (size_t)(bn < BT ? bn : 0) * K + k0 + kw0 + bk;
  if (len == 1024) {
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      uint32_t a0, a1, a2, a3, b0 = 0u, b1 = 0u;
      ldmatrix_x4(a0, a1, a2, a3, st + (uint32_t)ks * 32u);
      if (bn < BT) {
        b0 = *reinterpret_cast<const uint32_t*>(xrow + ks * 16);
        b1 = *reinterpret_cast<const uint32_t*>(xrow + ks * 16 + 8);
      }
      mma_bf16_16816(c, a0, a1, a2, a3, b0, b1);
    }
  } else {
    for (int ks = 0; ks < 8; ++ks) {
      const int kk = kw0 + ks * 16;
      if (kk >= len) break;  // warp-uniform
      uint32_t a0, a1, a2, a3, b0 = 0u, b1 = 0u;
      ldmatrix_x4(a0, a1, a2, a3, st + (uint32_t)ks * 32u);
      if (bn < BT) {
        if (kk + bk < len) b0 = *reinterpret_cast<const uint32_t*>(xrow + ks * 16);
        if (kk + bk + 8 < len) b1 = *reinterpret_cast<const uint32_t*>(xrow + ks * 16 + 8);
      }
      mma_bf16_16816(c, a0, a1, a2, a3, b0, b1);
    }
  }
}
// fragment element (row, col) lives in lane 4 * (row % 8) + col / 2, register (row / 8) * 2 + col % 2: every warp writes its
// k-slice sums to rs[warp][16][4]
template <int BT>
SSB_DEVINL void mma_store_partial(float* rs_warp, int lane, const float (&c)[4]) {
  const int col = (lane & 3) * 2, row = lane >> 2;
  if (col < BT) {
    rs_warp[row * 4 + col] = c[0];
    rs_warp[(row + 8) * 4 + col] = c[2];
  }
  if (col + 1 < BT) {
    rs_warp[row * 4 + col + 1] = c[1];
    rs_warp[(row + 8) * 4 + col + 1] = c[3];
  }
}
