// gemv_core.cuh — the consumer inner loop shared by proj_rows_kernel (kernels.cu) and decode_mega_kernel (mega.cu):
// one warp, two weight rows (w0, w1) of one K-chunk staged in shared memory, BT activation rows in shared memory.
// Full chunks (1024 elements) take a fully unrolled path: all 8+4*BT 128-bit shared loads are issued before the first
// FMA, and every (row, 256-element sub-chunk) has its own accumulator so no FMA chain is longer than 8 (a rolled loop with
// two 32-deep chains is latency-bound).
#pragma once
#include "common.cuh"

// GEMV_MIXED_FMA=1 (compile-time experiment, variant library "fhfma"; never run on hardware): the mixed-precision
// FMA `fma.rn.f32.bf16` (SASS FHFMA.BF16 with .H0/.H1 operand halves) takes the packed bf16 weights and activations as
// they sit in the registers, so the 24 shift/mask unpack instructions per 8 weights x 2 rows disappear and the loop is
// FMAs and shared loads only.  bf16 x bf16 is exact in fp32 and the accumulation order below is the same, so the
// results are bit-identical to the fmaf path.
#ifndef GEMV_MIXED_FMA
#define GEMV_MIXED_FMA 0
#endif
// acc += lo(w)*lo(x); acc += hi(w)*hi(x)   (in this order)
SSB_DEVINL float fma2_bf16(uint32_t w, uint32_t x, float acc) {
  asm("{\n\t.reg .b16 wl, wh, xl, xh;\n\tmov.b32 {wl, wh}, %1;\n\tmov.b32 {xl, xh}, %2;\n\t"
      "fma.rn.f32.bf16 %0, wl, xl, %0;\n\tfma.rn.f32.bf16 %0, wh, xh, %0;\n\t}"
      : "+f"(acc)
      : "r"(w), "r"(x));
  return acc;
}
// Which loop a tile height uses: at 1 row the loop is not issue-bound and the unpack costs little; from 2 rows on the
// x-operand unpack is paid per row, which the mixed FMA removes.  Both are bit-identical.
template <int BT>
struct GemvMixed {
  static constexpr bool value = GEMV_MIXED_FMA != 0 || BT >= 2;
};

template <int BT>
SSB_DEVINL void gemv_chunk(const bf16* __restrict__ w0, const bf16* __restrict__ w1, const bf16* __restrict__ xs, int K, int k0, int len,
                           int lane, float (&acc0)[BT], float (&acc1)[BT]) {
  if (len == 1024) {
    uint4 a0[4], a1[4];
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      a0[it] = *reinterpret_cast<const uint4*>(w0 + lane * 8 + it * 256);
      a1[it] = *reinterpret_cast<const uint4*>(w1 + lane * 8 + it * 256);
    }
#pragma unroll
    for (int b = 0; b < BT; ++b) {
      uint4 xv[4];
#pragma unroll
      for (int it = 0; it < 4; ++it) xv[it] = *reinterpret_cast<const uint4*>(xs + (size_t)b * K + k0 + lane * 8 + it * 256);
      float p0[4], p1[4];
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        const uint32_t u0[4] = {a0[it].x, a0[it].y, a0[it].z, a0[it].w};
        const uint32_t u1[4] = {a1[it].x, a1[it].y, a1[it].z, a1[it].w};
        const uint32_t xu[4] = {xv[it].x, xv[it].y, xv[it].z, xv[it].w};
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          if constexpr (GemvMixed<BT>::value) {
            s0 = fma2_bf16(u0[i], xu[i], s0);
            s1 = fma2_bf16(u1[i], xu[i], s1);
          } else {
            const float xl = bf_lo(xu[i]), xh = bf_hi(xu[i]);
            s0 = fmaf(bf_lo(u0[i]), xl, s0);
            s0 = fmaf(bf_hi(u0[i]), xh, s0);
            s1 = fmaf(bf_lo(u1[i]), xl, s1);
            s1 = fmaf(bf_hi(u1[i]), xh, s1);
          }
        }
        p0[it] = s0;
        p1[it] = s1;
      }
      acc0[b] += (p0[0] + p0[1]) + (p0[2] + p0[3]);
      acc1[b] += (p1[0] + p1[1]) + (p1[2] + p1[3]);
    }
  } else {
    for (int c = lane * 8; c < len; c += 256) {
      const uint4 a0 = *reinterpret_cast<const uint4*>(w0 + c);
      const uint4 a1 = *reinterpret_cast<const uint4*>(w1 + c);
      const uint32_t u0[4] = {a0.x, a0.y, a0.z, a0.w};
      const uint32_t u1[4] = {a1.x, a1.y, a1.z, a1.w};
#pragma unroll
      for (int b = 0; b < BT; ++b) {
        const uint4 xv = *reinterpret_cast<const uint4*>(xs + (size_t)b * K + k0 + c);
        const uint32_t xu[4] = {xv.x, xv.y, xv.z, xv.w};
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          if constexpr (GemvMixed<BT>::value) {
            s0 = fma2_bf16(u0[i], xu[i], s0);
            s1 = fma2_bf16(u1[i], xu[i], s1);
          } else {
            const float xl = bf_lo(xu[i]), xh = bf_hi(xu[i]);
            s0 = fmaf(bf_lo(u0[i]), xl, s0);
            s0 = fmaf(bf_hi(u0[i]), xh, s0);
            s1 = fmaf(bf_lo(u1[i]), xl, s1);
            s1 = fmaf(bf_hi(u1[i]), xh, s1);
          }
        }
        acc0[b] += s0;
        acc1[b] += s1;
      }
    }
  }
}


// ---------------------------------------------------------------------------------------------------------------------
// Tensor-pipe form of the consumer loop (used by decode_mega_kernel and proj_rows_kernel): a stage holds 16 weight
// rows x 1024 k with rows padded to GEMV_RS elements (the eight rows of an 8 x 8 ldmatrix tile then fall into different bank
// groups); warp w multiplies ALL 16 rows by the k slice [128 w, 128 w + 128) of the chunk: 8 k-steps of mma.sync m16n8k16 with
// A = ldmatrix.x4 of the stage and B = the staged activations (batch row n = column n of the 8).  c[4] is the warp's 16 x 8
// fp32 fragment, accumulated over the chunks of a pass.  k beyond `len` contributes nothing: whole k-steps are skipped and the
// activation fragment is zero there (callers zero-fill the ring at kernel start so stale weights are finite).
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
