// tc_gemm.cu — dense projections on the Hopper tensor cores (wgmma + TMA + mbarrier), sm_90a.
//
//   Y[M_tok, N] = X[M_tok, K] * W[N, K]^T          (HF nn.Linear, HF:models/llama/modeling_llama.py:238-249,177-183)
//
// computed transposed so the WEIGHT rows are the wgmma M dimension:  D[128 weight rows, TN tokens] += A * B^T with
//   A = W tile  [128 x 64]  (K-major, TMA 128B-swizzled)      -> two wgmma m64 halves, one per consumer warpgroup
//   B = X tile  [TN  x 64]  (K-major, TMA 128B-swizzled)      -> wgmma N = TN (16..256)
// Tokens are the wgmma N dimension, so the same kernel serves prefill (TN = 128 / 256, tensor-pipe bound) and batched
// decode (TN = 16/32, HBM bound: weights stream HBM -> TMA -> smem -> tensor core without touching registers).
// Warp roles (384 threads): warps 0..7 = two consumer warpgroups (warpgroup g issues the wgmmas of weight rows
// [64 g, 64 g + 64) and keeps that 64 x TN accumulator in registers), warps 8..11 = producer warpgroup (one thread issues
// the TMA loads).  setmaxnreg moves registers from the producer to the consumers: a 64 x 256 accumulator is 128 per thread.  The producer keeps the
// shared-memory ring full while the consumers run the fused epilogue (RoPE/KV-append | SwiGLU | residual, same math as
// gemv_epilogue), so the weight stream of the next tile overlaps the epilogue of this one.
#include <cuda.h>

#include "common.cuh"
#include "kernels.h"
#include "sk_partition.h"
#include "tc_gemm.h"

#include "epilogue.cuh"

constexpr int TC_BM = 128;   // weight rows per tile (two wgmma m64 halves)
constexpr int TC_BK = 64;    // K elements per stage = one 128-byte swizzle span of bf16
constexpr int TC_CONSUMERS = 256;  // two warpgroups
constexpr int TC_THREADS = TC_CONSUMERS + 128;  // + the producer warpgroup (one thread issues the TMA loads)
constexpr int TC_EPI_TOK = 32;     // tokens per epilogue pass
constexpr int TC_STG_LD = 68;      // staging row pitch in floats: fragment stores hit 32 distinct banks

SSB_DEVINL void tma_load_2d(void* dst_smem, const CUtensorMap* tm, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(dst_smem)),
      "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
SSB_DEVINL void prefetch_tmap(const CUtensorMap* tm) { asm volatile("prefetch.tensormap [%0];" ::"l"(tm) : "memory"); }

// wgmma shared-memory descriptor, K-major, SWIZZLE_128B: 8-row groups of 128 B rows, groups 1024 B apart
// (start>>4 [0,14) | LBO>>4 [16,30) (unused for swizzled K-major) | SBO>>4 [32,46) | layout [62,64): 1 = 128B swizzle)
SSB_DEVINL uint64_t wgmma_desc_k_sw128(uint32_t smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
template <int R>
SSB_DEVINL void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
SSB_DEVINL void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
constexpr int TC_PRODUCER_REGS = 40, TC_CONSUMER_REGS = 232;  // 128 x 40 + 256 x 232 <= 64 K registers
SSB_DEVINL void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
SSB_DEVINL void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
SSB_DEVINL void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma window
template <int R>
SSB_DEVINL void acc_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, both operands K-major in shared memory; fp32 accumulators, N / 2 per thread
SSB_DEVINL void wgmma_bf16(float (&d)[8], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
SSB_DEVINL void wgmma_bf16(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
SSB_DEVINL void wgmma_bf16(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
SSB_DEVINL void wgmma_bf16(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

template <int TN>
struct TcCfg {
  static constexpr int A_BYTES = TC_BM * TC_BK * 2;                       // 16 KiB
  static constexpr int B_BYTES = TN * TC_BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + ((B_BYTES + 1023) / 1024) * 1024;
  static constexpr int BUDGET = 200 * 1024;  // of the 227 KiB a block may use; the rest is barriers, positions, staging
  static constexpr int STAGES = BUDGET / STAGE_BYTES > 8 ? 8 : BUDGET / STAGE_BYTES;
  static constexpr int ACC = TN / 2;                                      // fp32 accumulators per consumer thread
  static constexpr int PASS = TN < TC_EPI_TOK ? TN : TC_EPI_TOK;          // tokens per epilogue pass
  static constexpr int STG_FLOATS = TC_EPI_TOK * TC_STG_LD;               // staging of one warpgroup's 64 rows x PASS tokens
  static constexpr int BAR_BYTES = 256;
  static constexpr size_t SMEM = (size_t)STAGES * STAGE_BYTES + 1024 /*align slack*/ + BAR_BYTES + 2 * TN * 4 /*per-token pos / KV block*/ +
                                 2 * STG_FLOATS * 4;
  static_assert(2 * STAGES * 8 <= BAR_BYTES, "barrier area");
};

// Epilogue inputs of CG consecutive tokens of one row pair — residual words (EPI_RESID) or packed RoPE cos|sin
// (EPI_QKV_ROPE, positions staged in shared memory).  They do not depend on the accumulator, so they are requested
// before the pass's accumulators are staged; `on` = this thread runs the epilogue of a real row pair.
template <int EPI, int CG>
SSB_DEVINL void tc_epi_inputs(const GemvArgs& a, int pair, int m0, const int* __restrict__ s_pos, bool on, uint32_t (&w)[CG]) {
  if constexpr (EPI == EPI_RESID) {
#pragma unroll
    for (int j = 0; j < CG; ++j)
      w[j] = (on && m0 + j < a.M) ? __ldcg(reinterpret_cast<const uint32_t*>(a.resid + (size_t)(m0 + j) * a.ld_out + 2 * pair)) : 0u;
  } else if constexpr (EPI == EPI_QKV_ROPE) {
    const int half = a.head_dim >> 1, q_pairs = a.q_rows >> 1, qk_pairs = (a.q_rows + a.kv_rows) >> 1;
    const int pp = pair < q_pairs ? pair : pair - q_pairs;
    const int jj = pp % half;
#pragma unroll
    for (int j = 0; j < CG; ++j) w[j] = (on && pair < qk_pairs && m0 + j < a.M) ? a.rope_cs[(size_t)s_pos[j] * half + jj] : 0u;
  }
}
// eight tokens of one row pair with their inputs already loaded (w = the eight words tc_epi_inputs produced for them)
template <int EPI>
SSB_DEVINL void tc_epi_store8(const GemvArgs& a, int pair, int m0, const int* __restrict__ s_pos, const int* __restrict__ s_blk,
                              const uint32_t* w, const float (&v0)[8], const float (&v1)[8]) {
  if constexpr (EPI == EPI_RESID) {
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (m0 + j < a.M)
        *reinterpret_cast<uint32_t*>(a.out_bf16 + (size_t)(m0 + j) * a.ld_out + 2 * pair) =
            pack_bf16(bf16r(v0[j]) + bf_lo(w[j]), bf16r(v1[j]) + bf_hi(w[j]));
  } else if constexpr (EPI == EPI_QKV_ROPE) {
    tc_epilogue8_qkv_cs(a, pair, m0, s_pos, s_blk, w, v0, v1);
  } else {
    tc_epilogue8<EPI>(a, pair, m0, v0, v1);
  }
}

// Fused epilogue of one consumer warpgroup: its 64 weight rows x TN tokens, accumulators in the wgmma fragment layout
// (register i of thread t: row 16 (t / 32) + (t % 32) / 4 + 8 ((i / 2) % 2), token 8 (i / 4) + 2 (t % 4) + i % 2).
// In passes of PASS tokens the fragment goes through shared memory (stg, [token][row] with pitch TC_STG_LD), and each
// thread then finishes eight consecutive tokens of one row PAIR (2 p, 2 p + 1) — the pair the engine's weight layout puts
// together (RoPE partners, gate / up).  m_base = first token of the tile; row0 = first weight row of this warpgroup.
template <int TN, int EPI>
SSB_DEVINL void wg_epilogue(const GemvArgs& a, float (&acc)[TN / 2], int row0, int m_base, const int* __restrict__ s_pos,
                            const int* __restrict__ s_blk, float* stg, int wg, int t) {
  using Cfg = TcCfg<TN>;
  constexpr int P = Cfg::PASS;
  const int warp = t >> 5, lane = t & 31;
  const int frow = 16 * warp + (lane >> 2), fcol = 2 * (lane & 3);
  const int lp = t & 31, chunk = t >> 5;  // epilogue item: local pair, 8-token chunk of the pass
  const int pair = (row0 >> 1) + lp;
  const bool on = chunk * 8 < P && 2 * pair < a.N;
#pragma unroll
  for (int g0 = 0; g0 < TN; g0 += P) {
    if (m_base + g0 >= a.M) break;  // warpgroup-uniform
    const int m0 = m_base + g0 + 8 * chunk;
    uint32_t w[8];
    tc_epi_inputs<EPI, 8>(a, pair, m0, s_pos + g0 + 8 * chunk, on, w);
    named_bar_sync(2 + wg, 128);  // the previous pass has read the staging buffer
#pragma unroll
    for (int j = g0 / 8; j < (g0 + P) / 8; ++j)
#pragma unroll
      for (int r = 0; r < 4; ++r) stg[(8 * j - g0 + fcol + (r & 1)) * TC_STG_LD + frow + 8 * (r >> 1)] = acc[4 * j + r];
    named_bar_sync(2 + wg, 128);
    if (on && m0 < a.M) {
      float v0[8], v1[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 v = *reinterpret_cast<const float2*>(stg + (8 * chunk + j) * TC_STG_LD + 2 * lp);
        v0[j] = v.x;
        v1[j] = v.y;
      }
      tc_epi_store8<EPI>(a, pair, m0, s_pos + g0 + 8 * chunk, s_blk + g0 + 8 * chunk, w, v0, v1);
    }
  }
}

// Consumer mainloop over k-blocks [kb0, kb1) of one weight tile.  Each 64-element k-block is multiplied into a fresh
// partial (four k16 wgmmas, at most 128 token columns at a time) that is then added to the accumulator with an ordinary
// fp32 add.  Chaining every k-block inside the tensor core instead loses precision over long K on Hopper: at Llama-2-7B,
// 32 layers, the logits' error against the fp32 oracle grew from 6.5e-2 to 7.4e-2 (CPU bf16 oracle: 7.3e-2; measured on
// an H100 80GB HBM3, tests/test_fullwidth_gpu.py::test_full_depth_7b_vs_fp32_oracle).
// A stage goes back to the producer as soon as its wgmmas have retired.
template <int TN>
SSB_DEVINL void wg_mainloop(float (&acc)[TN / 2], uint8_t* smem, uint64_t* full, uint64_t* empty, int& stage, uint32_t& phase,
                            int kb0, int kb1, int wg, int t) {
  using Cfg = TcCfg<TN>;
  constexpr int NC = TN < 128 ? TN : 128;  // token columns per wgmma
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(&full[stage], phase);
    const uint32_t sa = smem_u32(smem + (size_t)stage * Cfg::STAGE_BYTES);
#pragma unroll
    for (int c = 0; c < TN / NC; ++c) {
      float part[NC / 2];
      const uint64_t ad = wgmma_desc_k_sw128(sa + wg * (64 * 128));
      const uint64_t bd = wgmma_desc_k_sw128(sa + Cfg::A_BYTES + c * NC * 128);  // B rows are 128 B: NC rows = NC * 128 B
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < TC_BK / 16; ++k)  // k16 = 32 B: advance the start address inside the swizzle span
        wgmma_bf16(part, ad + (uint64_t)(k * 2), bd + (uint64_t)(k * 2), k != 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(part);
#pragma unroll
      for (int i = 0; i < NC / 2; ++i) acc[c * (NC / 2) + i] = kb > kb0 ? acc[c * (NC / 2) + i] + part[i] : part[i];
    }
    if (t == 0) mbar_arrive(&empty[stage]);
    if (++stage == Cfg::STAGES) {
      stage = 0;
      phase ^= 1;
    }
  }
}

template <int TN, int EPI>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemvArgs a) {
  using Cfg = TcCfg<TN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)Cfg::STAGES * Cfg::STAGE_BYTES);
  uint64_t* full = bars;
  uint64_t* empty = bars + Cfg::STAGES;
  [[maybe_unused]] int* s_pos = reinterpret_cast<int*>(reinterpret_cast<uint8_t*>(bars) + Cfg::BAR_BYTES);  // [TN] position of each token of the current tile (QKV epilogue)
  [[maybe_unused]] int* s_blk = s_pos + TN;                                                               // [TN] KV block holding that position
  float* stg = reinterpret_cast<float*>(s_blk + TN);                                                      // [2][PASS tokens][TC_STG_LD]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_ntiles = (a.N + TC_BM - 1) / TC_BM;
  const int n_mtiles = (a.M + TN - 1) / TN;
  const int n_tiles = n_ntiles * n_mtiles;
  const int nkb = (a.K + TC_BK - 1) / TC_BK;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    for (int s = 0; s < Cfg::STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 2);  // one arrive per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();  // activations (B operand, residual) come from the previous kernel

  if (warp >= TC_CONSUMERS / 32) {
    // ---------------------------------------------------------------- TMA producer
    setmaxnreg_dec<TC_PRODUCER_REGS>();
    if (warp == TC_CONSUMERS / 32 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int mt = tile % n_mtiles, nt = tile / n_mtiles;  // token tiles fastest: CTAs running together share a weight tile (one HBM read)
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          uint8_t* sa = smem + (size_t)stage * Cfg::STAGE_BYTES;
          mbar_expect_tx(&full[stage], Cfg::A_BYTES + Cfg::B_BYTES);
          tma_load_2d(sa, &tmA, kb * TC_BK, nt * TC_BM, &full[stage]);
          tma_load_2d(sa + Cfg::A_BYTES, &tmB, kb * TC_BK, mt * TN, &full[stage]);
          if (++stage == Cfg::STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ---------------------------------------------------------------- consumer warpgroups: wgmma, then the fused epilogue
    setmaxnreg_inc<TC_CONSUMER_REGS>();
    const int wg = warp >> 2, t = threadIdx.x & 127;
    int stage = 0;
    uint32_t phase = 0;
    float acc[Cfg::ACC];
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      const int mt = tile % n_mtiles, nt = tile / n_mtiles;
      if constexpr (EPI == EPI_QKV_ROPE) {
        // stage the tile's per-token position and KV block (two dependent loads, once per token)
        named_bar_sync(1, TC_CONSUMERS);  // the previous tile's epilogue no longer reads s_pos / s_blk
        for (int i = threadIdx.x; i < TN; i += TC_CONSUMERS) {
          const int m = mt * TN + i;
          int pos = 0, blk = 0;
          if (m < a.M) {
            pos = __ldcg(a.row_pos + m);
            blk = a.block_table[(size_t)a.row_slot[m] * a.bt_stride + pos / a.block_size];
          }
          s_pos[i] = pos;
          s_blk[i] = blk;
        }
      }
      wg_mainloop<TN>(acc, smem, full, empty, stage, phase, 0, nkb, wg, t);
      if constexpr (EPI == EPI_QKV_ROPE) named_bar_sync(1, TC_CONSUMERS);
      wg_epilogue<TN, EPI>(a, acc, nt * TC_BM + 64 * wg, mt * TN, s_pos, s_blk, stg + wg * Cfg::STG_FLOATS, wg, t);
    }
  }
}

// ====================================================================================================================
// stream-K variant for ONE token tile (batched decode, M <= TN <= 64): the (weight tile, k-block) units of the whole
// matrix are laid end to end and every CTA streams an equal contiguous share, so all SMs pull the same number of weight
// bytes no matter how many 128-row tiles N has (a 4096-row matrix is only 32 tiles for 132 SMs).  A tile whose k-range
// is split over several CTAs is reduced through a small fp32 workspace: the parts that do not start at k = 0 are
// written out ("contributors"), the CTA holding the k = 0 part ("owner" — it reaches that part LAST in its own range,
// when the others are already done) adds them to its register accumulators and runs the fused epilogue.
// Dependencies only point from higher to lower CTA index ranges that are processed earlier, so there is no cycle.
// ====================================================================================================================
struct SkWs {
  float* part;      // [slots][TN * 128] fp32, in the consumers' fragment order
  unsigned* flags;  // [slots], zero on entry and on exit
  unsigned long long* prof;  // [grid][8] globaltimer stamps (TC_SK_PROF builds), may be null
};
#ifndef TC_SK_PROF
#define TC_SK_PROF 0
#endif
// phase stamps of one stream-K launch, per CTA: 0 entry, 1 setup done (barriers), 2 first weight tile landed,
// 3 last wgmma retired, 4 (unused), 5 epilogue done, 6 exit, 7 = number of segments
SSB_DEVINL void sk_stamp(const SkWs& ws, int i) {
#if TC_SK_PROF
  if (ws.prof) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    ws.prof[(size_t)blockIdx.x * 8 + i] = t;
  }
#endif
}

#ifndef TC_SK_PREFETCH_RING
#define TC_SK_PREFETCH_RING 0
#endif
template <int TN, int EPI>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_gemm_sk_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemvArgs a, const SkWs ws) {
  using Cfg = TcCfg<TN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)Cfg::STAGES * Cfg::STAGE_BYTES);
  uint64_t* full = bars;
  uint64_t* empty = bars + Cfg::STAGES;
  [[maybe_unused]] int* s_pos = reinterpret_cast<int*>(reinterpret_cast<uint8_t*>(bars) + Cfg::BAR_BYTES);  // [TN] position of each token (QKV epilogue), staged once
  [[maybe_unused]] int* s_blk = s_pos + TN;                                                               // [TN] KV block holding that position
  float* stg = reinterpret_cast<float*>(s_blk + TN);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_ntiles = (a.N + TC_BM - 1) / TC_BM;
  const int nkb = (a.K + TC_BK - 1) / TC_BK;
  // 32-bit unit arithmetic (the launcher checks U * grid < 2^31): 64-bit divisions are software routines on the
  // critical path of every segment and of the owner's contributor search
  const int U = n_ntiles * nkb;
  const int G = (int)gridDim.x;
  const int u0 = sk_begin(blockIdx.x, U, G), u1 = sk_begin(blockIdx.x + 1, U, G);  // sk_partition.h (checked exhaustively on the host)

  if (threadIdx.x == 0) {
    sk_stamp(ws, 0);
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    for (int s = 0; s < Cfg::STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 2);
    }
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) sk_stamp(ws, 1);
  pdl_launch_dependents();

  if (warp >= TC_CONSUMERS / 32) {
    // ---------------------------------------------------------------- TMA producer.  The weight (A) stream does not
    // depend on the previous kernel: it starts before griddepcontrol.wait; the activation (B) loads wait for it.
    setmaxnreg_dec<TC_PRODUCER_REGS>();
    if (warp == TC_CONSUMERS / 32 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      bool waited = false;
      int ustart = u0;
#if TC_SK_PREFETCH_RING
      // compile-time experiment (not measured): put the weight tiles of the first ring-full of units in flight before
      // the dependency wait instead of only the first one, so the HBM stream of this projection ramps up while the
      // previous kernel drains; the activation tiles follow after the wait on the same barriers.
      {
        const int upre = min(u1, u0 + Cfg::STAGES);
        int st = 0;
        for (int u = u0; u < upre; ++u, ++st) {  // the ring starts empty: no empty-wait in the first pass
          mbar_expect_tx(&full[st], Cfg::A_BYTES + Cfg::B_BYTES);
          tma_load_2d(smem + (size_t)st * Cfg::STAGE_BYTES, &tmA, (int)(u % nkb) * TC_BK, (int)(u / nkb) * TC_BM, &full[st]);
        }
        pdl_wait();
        waited = true;
        st = 0;
        for (int u = u0; u < upre; ++u, ++st)
          tma_load_2d(smem + (size_t)st * Cfg::STAGE_BYTES + Cfg::A_BYTES, &tmB, (int)(u % nkb) * TC_BK, 0, &full[st]);
        const int n = (int)(upre - u0);
        stage = n % Cfg::STAGES;
        phase = n == Cfg::STAGES ? 1u : 0u;
        ustart = upre;
      }
#endif
      for (int u = ustart; u < u1; ++u) {
        const int nt = u / nkb, kb = u - nt * nkb;
        mbar_wait(&empty[stage], phase ^ 1);
        uint8_t* sa = smem + (size_t)stage * Cfg::STAGE_BYTES;
        mbar_expect_tx(&full[stage], Cfg::A_BYTES + Cfg::B_BYTES);
        tma_load_2d(sa, &tmA, kb * TC_BK, nt * TC_BM, &full[stage]);
        if (!waited) {
          pdl_wait();
          waited = true;
        }
        tma_load_2d(sa + Cfg::A_BYTES, &tmB, kb * TC_BK, 0, &full[stage]);
        if (++stage == Cfg::STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
  } else {
    // ---------------------------------------------------------------- consumer warpgroups
    setmaxnreg_inc<TC_CONSUMER_REGS>();
    pdl_wait();  // residuals / positions written by the previous kernel; the workspace flags of the previous launch
    const int wg = warp >> 2, t = threadIdx.x & 127;
    if constexpr (EPI == EPI_QKV_ROPE) {
      // per-token position and KV block, once per CTA (two dependent loads)
      for (int i = threadIdx.x; i < TN; i += TC_CONSUMERS) {
        int pos = 0, blk = 0;
        if (i < a.M) {
          pos = __ldcg(a.row_pos + i);
          blk = a.block_table[(size_t)a.row_slot[i] * a.bt_stride + pos / a.block_size];
        }
        s_pos[i] = pos;
        s_blk[i] = blk;
      }
      named_bar_sync(1, TC_CONSUMERS);
    }
    int stage = 0;
    uint32_t phase = 0;
    int it = 0;
    float acc[Cfg::ACC];
    for (int u = u0; u < u1; ++it) {
      const int nt = u / nkb, kb0 = u - nt * nkb;
      const int kb1 = min(nkb, kb0 + (u1 - u));
      const bool is_first_seg = (u == u0);
      if (TC_SK_PROF && threadIdx.x == 0 && is_first_seg) {
        mbar_wait(&full[0], 0);
        sk_stamp(ws, 2);
      }
      wg_mainloop<TN>(acc, smem, full, empty, stage, phase, kb0, kb1, wg, t);
      if (TC_SK_PROF && threadIdx.x == 0 && u + (kb1 - kb0) >= u1) sk_stamp(ws, 3);
      // this thread's accumulators in fragment order: index i * 256 + threadIdx.x of a slot
      if (kb0 != 0) {
        // contributor: dump the partial accumulator to this CTA's slot (slot 0 = first segment of the range, else 1)
        const int slot = blockIdx.x * 2 + (is_first_seg ? 0 : 1);
        float* dst = ws.part + (size_t)slot * (TN * 128) + threadIdx.x;
#pragma unroll
        for (int i = 0; i < Cfg::ACC; ++i) dst[(size_t)i * TC_CONSUMERS] = acc[i];
        // the barrier orders the 256 threads' stores before thread 0's release store (release is cumulative at gpu scope)
        named_bar_sync(1, TC_CONSUMERS);
        if (threadIdx.x == 0) asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(ws.flags + slot), "r"(1u) : "memory");
      } else {
        // owner: the part starting at k = 0.  Contributors = the CTAs whose ranges cover the rest of this tile: the next
        // n_contrib CTAs (every CTA has a non-empty range: grid <= U), each with its FIRST segment.  All flags are read
        // in one batch (they are normally up long before the owner gets here).
        const int t_end = (nt + 1) * nkb;  // first unit after this tile
        const int n_contrib = sk_contributors(blockIdx.x, U, G, u + (kb1 - kb0), t_end);
        const int slot0 = (blockIdx.x + 1) * 2;  // contributor i dumped into slot0 + 2 i
        for (;;) {
          unsigned ok = 1u;
#pragma unroll
          for (int i = 0; i < SK_MAX_CONTRIB; ++i) {
            unsigned f = 1u;
            if (i < n_contrib) asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(f) : "l"(ws.flags + slot0 + 2 * i) : "memory");
            ok &= (f != 0u) ? 1u : 0u;
          }
          if (ok) break;
        }
        asm volatile("fence.acq_rel.gpu;" ::: "memory");  // acquire: the contributors' partials are visible to this thread
        const float* src = ws.part + (size_t)slot0 * (TN * 128) + threadIdx.x;
#pragma unroll 1
        for (int i = 0; i < n_contrib; ++i) {  // contributor order: i, then i + 1
          const float* p = src + (size_t)(2 * i) * (TN * 128);
#pragma unroll
          for (int r = 0; r < Cfg::ACC; ++r) acc[r] += __ldcg(p + (size_t)r * TC_CONSUMERS);
        }
        wg_epilogue<TN, EPI>(a, acc, nt * TC_BM + 64 * wg, 0, s_pos, s_blk, stg + wg * Cfg::STG_FLOATS, wg, t);
        named_bar_sync(1, TC_CONSUMERS);  // every consumer thread has read the partials
        if (threadIdx.x < n_contrib) ws.flags[slot0 + 2 * threadIdx.x] = 0;  // clean for the next launch
      }
      u += kb1 - kb0;
    }
    if (TC_SK_PROF && threadIdx.x == 0) {
      sk_stamp(ws, 5);
      if (ws.prof) ws.prof[(size_t)blockIdx.x * 8 + 7] = (unsigned long long)it;
    }
  }
  if (TC_SK_PROF) {
    __syncthreads();
    if (threadIdx.x == 0) sk_stamp(ws, 6);
  }
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

// 2-D K-major bf16 tensor map: global [rows, cols] with row pitch ld elements, box [box_rows, 64 cols], 128B swizzle
cudaError_t tc_make_tmap(TcTensorMap* out, const bf16* ptr, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return cudaErrorNotSupported;
  static_assert(sizeof(TcTensorMap) == sizeof(CUtensorMap), "tensor map size");
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)TC_BK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(reinterpret_cast<CUtensorMap*>(out), CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<bf16*>(ptr), dims, strides, box,
                   estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

// Token-tile width (wgmma N).  Decode-sized forwards: the smallest tile that holds the batch (stream-K kernel).
int tc_pick_tn(int M) { return M <= 16 ? 16 : M <= 32 ? 32 : M <= 64 ? 64 : 128; }
// Prefill-sized forwards choose per projection between 128- and 256-token tiles.  A 128 x 256 tile ingests 48 KiB of
// operands per k-block for twice the FLOPs of a 128 x 128 tile's 32 KiB (87 vs 64 FLOP per byte through the L2 -> SM path)
// and halves the re-reads of a
// weight tile (one read per token tile) — but it also halves the tile count, and the persistent grid runs whole waves:
// pick the width with the smaller  waves x per-tile cost  (cost 1.0 vs 1.7: the operand bytes and a longer epilogue), 128 on a tie.
int tc_pick_tn_prefill(int M, int N, int n_sm) {
  if (M <= 128) return tc_pick_tn(M);
  const long long nt = (N + TC_BM - 1) / TC_BM;
  const long long t128 = nt * ((M + 127) / 128), t256 = nt * ((M + 255) / 256);
  const long long w128 = (t128 + n_sm - 1) / n_sm, w256 = (t256 + n_sm - 1) / n_sm;
  return 17 * w256 < 10 * w128 ? 256 : 128;
}
int tc_weight_box_rows() { return TC_BM; }

template <int TN, int EPI>
static cudaError_t launch_tc_t(const TcTensorMap& tmA, const TcTensorMap& tmB, const GemvArgs& a, const LaunchCfg& lc) {
  using Cfg = TcCfg<TN>;
  static std::atomic<unsigned long long> attr_mask{0};  // per instantiation, per device
  if (first_launch_on_device(attr_mask)) {
    cudaError_t e = cudaFuncSetAttribute(tc_gemm_kernel<TN, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM);
    if (e != cudaSuccess) return e;
  }
  const int n_tiles = ((a.N + TC_BM - 1) / TC_BM) * ((a.M + TN - 1) / TN);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(n_tiles < lc.n_sm ? n_tiles : lc.n_sm);
  cfg.blockDim = dim3(TC_THREADS);
  cfg.dynamicSmemBytes = Cfg::SMEM;
  cfg.stream = lc.stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = lc.pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, tc_gemm_kernel<TN, EPI>, *reinterpret_cast<const CUtensorMap*>(&tmA),
                            *reinterpret_cast<const CUtensorMap*>(&tmB), a);
}

template <int EPI>
static cudaError_t launch_tc_e(int tn, const TcTensorMap& tmA, const TcTensorMap& tmB, const GemvArgs& a, const LaunchCfg& lc) {
  switch (tn) {
    case 16: return launch_tc_t<16, EPI>(tmA, tmB, a, lc);
    case 32: return launch_tc_t<32, EPI>(tmA, tmB, a, lc);
    case 64: return launch_tc_t<64, EPI>(tmA, tmB, a, lc);
    case 128: return launch_tc_t<128, EPI>(tmA, tmB, a, lc);
    case 256: return launch_tc_t<256, EPI>(tmA, tmB, a, lc);
  }
  return cudaErrorInvalidValue;
}

template <int TN, int EPI>
static cudaError_t launch_sk_t(const TcTensorMap& tmA, const TcTensorMap& tmB, const GemvArgs& a, const LaunchCfg& lc) {
  using Cfg = TcCfg<TN>;
  static std::atomic<unsigned long long> attr_mask{0};  // per instantiation, per device
  if (first_launch_on_device(attr_mask)) {
    cudaError_t e = cudaFuncSetAttribute(tc_gemm_sk_kernel<TN, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM);
    if (e != cudaSuccess) return e;
  }
  const int nkb = (a.K + TC_BK - 1) / TC_BK;
  const long long U = (long long)((a.N + TC_BM - 1) / TC_BM) * nkb;
  const int grid = sk_grid(U, nkb, lc.n_sm);  // >= nkb/8 units per CTA: a tile spans at most 8 full + 2 partial ranges
  if (grid * 2 > lc.sk_slots || !sk_fits(U, grid)) return cudaErrorInvalidValue;
  const SkWs ws = {lc.sk_part, lc.sk_flags, lc.sk_prof};
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(TC_THREADS);
  cfg.dynamicSmemBytes = Cfg::SMEM;
  cfg.stream = lc.stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = lc.pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, tc_gemm_sk_kernel<TN, EPI>, *reinterpret_cast<const CUtensorMap*>(&tmA),
                            *reinterpret_cast<const CUtensorMap*>(&tmB), a, ws);
}

template <int EPI>
static cudaError_t launch_sk_e(int tn, const TcTensorMap& tmA, const TcTensorMap& tmB, const GemvArgs& a, const LaunchCfg& lc) {
  switch (tn) {
    case 16: return launch_sk_t<16, EPI>(tmA, tmB, a, lc);
    case 32: return launch_sk_t<32, EPI>(tmA, tmB, a, lc);
    case 64: return launch_sk_t<64, EPI>(tmA, tmB, a, lc);
  }
  return cudaErrorInvalidValue;
}

static cudaError_t launch_tc_streamk(const TcTensorMap& tmA, const TcTensorMap& tmB, int tn, const GemvArgs& a, int epi, const LaunchCfg& lc) {
  switch (epi) {
    case EPI_QKV_ROPE: return launch_sk_e<EPI_QKV_ROPE>(tn, tmA, tmB, a, lc);
    case EPI_SWIGLU: return launch_sk_e<EPI_SWIGLU>(tn, tmA, tmB, a, lc);
    case EPI_RESID: return launch_sk_e<EPI_RESID>(tn, tmA, tmB, a, lc);
    case EPI_BF16: return launch_sk_e<EPI_BF16>(tn, tmA, tmB, a, lc);
    case EPI_F32: return launch_sk_e<EPI_F32>(tn, tmA, tmB, a, lc);
    case EPI_GELU: return launch_sk_e<EPI_GELU>(tn, tmA, tmB, a, lc);
    case EPI_RESID2: return launch_sk_e<EPI_RESID2>(tn, tmA, tmB, a, lc);
    case EPI_F32_BF16R: return launch_sk_e<EPI_F32_BF16R>(tn, tmA, tmB, a, lc);
  }
  return cudaErrorInvalidValue;
}

// tmB must have been built with box_rows == tn
cudaError_t launch_tc_gemm(const TcTensorMap& tmA, const TcTensorMap& tmB, int tn, const GemvArgs& a, int epi, const LaunchCfg& lc) {
  if ((a.N & 1) || (a.K & 7)) return cudaErrorInvalidValue;
  if (a.M <= tn && tn <= 64 && lc.sk_part && !a.row_map) return launch_tc_streamk(tmA, tmB, tn, a, epi, lc);  // batched decode
  switch (epi) {
    case EPI_QKV_ROPE: return launch_tc_e<EPI_QKV_ROPE>(tn, tmA, tmB, a, lc);
    case EPI_SWIGLU: return launch_tc_e<EPI_SWIGLU>(tn, tmA, tmB, a, lc);
    case EPI_RESID: return launch_tc_e<EPI_RESID>(tn, tmA, tmB, a, lc);
    case EPI_BF16: return launch_tc_e<EPI_BF16>(tn, tmA, tmB, a, lc);
    case EPI_F32: return launch_tc_e<EPI_F32>(tn, tmA, tmB, a, lc);
    case EPI_GELU: return launch_tc_e<EPI_GELU>(tn, tmA, tmB, a, lc);
    case EPI_RESID2: return launch_tc_e<EPI_RESID2>(tn, tmA, tmB, a, lc);
    case EPI_F32_BF16R: return launch_tc_e<EPI_F32_BF16R>(tn, tmA, tmB, a, lc);
  }
  return cudaErrorInvalidValue;
}

// LayerNorm (prefill): y = bf16((x - mean) * rstd * w + b), fp32 statistics   HF:models/falcon/modeling_falcon.py:572-576
__global__ void __launch_bounds__(256) layernorm_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w, const bf16* __restrict__ b,
                                                        bf16* __restrict__ out, int K, float eps) {
  __shared__ float red[8];
  pdl_wait();
  pdl_launch_dependents();
  const int m = blockIdx.x, tid = threadIdx.x;
  const bf16* src = x + (size_t)m * K;
  float sm = 0.f;
  for (int k = tid * 8; k < K; k += 256 * 8) {
    const uint4 v = *reinterpret_cast<const uint4*>(src + k);
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) sm += bf_lo(u[i]) + bf_hi(u[i]);
  }
  sm = warp_sum(sm);
  if ((tid & 31) == 0) red[tid >> 5] = sm;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) tot += red[i];
  __syncthreads();
  const float mean = tot / (float)K;
  float sq = 0.f;
  for (int k = tid * 8; k < K; k += 256 * 8) {
    const uint4 v = *reinterpret_cast<const uint4*>(src + k);
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float lo = bf_lo(u[i]) - mean, hi = bf_hi(u[i]) - mean;
      sq += lo * lo + hi * hi;
    }
  }
  sq = warp_sum(sq);
  if ((tid & 31) == 0) red[tid >> 5] = sq;
  __syncthreads();
  tot = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) tot += red[i];
  const float rstd = rsqrtf(tot / (float)K + eps);
  for (int k = tid * 8; k < K; k += 256 * 8) {
    const uint4 v = *reinterpret_cast<const uint4*>(src + k);
    const uint4 wv = ldg128(w + k);
    const uint4 bv = ldg128(b + k);
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
    const uint32_t wu[4] = {wv.x, wv.y, wv.z, wv.w};
    const uint32_t bu[4] = {bv.x, bv.y, bv.z, bv.w};
    uint32_t o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
      o[i] = pack_bf16((bf_lo(u[i]) - mean) * rstd * bf_lo(wu[i]) + bf_lo(bu[i]), (bf_hi(u[i]) - mean) * rstd * bf_hi(wu[i]) + bf_hi(bu[i]));
    *reinterpret_cast<uint4*>(out + (size_t)m * K + k) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

cudaError_t launch_layernorm(const bf16* x, const bf16* w, const bf16* b, bf16* out, int M, int K, float eps, const LaunchCfg& lc) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(M);
  cfg.blockDim = dim3(256);
  cfg.stream = lc.stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = lc.pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, layernorm_kernel, x, w, b, out, K, eps);
}

// ------------------------------------------------------------------------------------------------ RMSNorm (prefill)
// xn[m][:] = w * bf16(x[m][:] * rsqrt(mean(x^2) + eps))     HF:models/llama/modeling_llama.py:62-67
__global__ void __launch_bounds__(256) rmsnorm_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w, bf16* __restrict__ out,
                                                      int K, float eps) {
  __shared__ float red[8];
  pdl_wait();
  pdl_launch_dependents();
  const int m = blockIdx.x, tid = threadIdx.x;
  const bf16* src = x + (size_t)m * K;
  float ss = 0.f;
  for (int k = tid * 8; k < K; k += 256 * 8) {
    const uint4 v = *reinterpret_cast<const uint4*>(src + k);
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float lo = bf_lo(u[i]), hi = bf_hi(u[i]);
      ss += lo * lo + hi * hi;
    }
  }
  ss = warp_sum(ss);
  if ((tid & 31) == 0) red[tid >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) tot += red[i];
  const float rstd = rsqrtf(tot / (float)K + eps);
  for (int k = tid * 8; k < K; k += 256 * 8) {
    const uint4 v = *reinterpret_cast<const uint4*>(src + k);
    const uint4 wv = ldg128(w + k);
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
    const uint32_t wu[4] = {wv.x, wv.y, wv.z, wv.w};
    uint32_t o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
      o[i] = pack_bf16(bf16r(bf_lo(u[i]) * rstd) * bf_lo(wu[i]), bf16r(bf_hi(u[i]) * rstd) * bf_hi(wu[i]));
    *reinterpret_cast<uint4*>(out + (size_t)m * K + k) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

cudaError_t launch_rmsnorm(const bf16* x, const bf16* w, bf16* out, int M, int K, float eps, const LaunchCfg& lc) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(M);
  cfg.blockDim = dim3(256);
  cfg.stream = lc.stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = lc.pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, rmsnorm_kernel, x, w, out, K, eps);
}
