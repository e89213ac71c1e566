// epilogue.cuh — fused projection epilogues shared by the CUDA-core GEMV (kernels.cu) and the wgmma GEMM
// (tc_gemm.cu).  Both kernels hand over the fp32 dot products of one PAIR of physical weight rows (2*pair, 2*pair+1)
// for token row m; the engine lays weights out so that the pair is (RoPE partner j, j+d/2) for q/k and
// (gate_i, up_i) for the MLP (DESIGN.md "weight layout").  Rounding points follow HF bf16 tensor ops
// (HF:models/llama/modeling_llama.py:138-168 RoPE, :177-183 SwiGLU, :325,:331 residual adds).
#pragma once
#include "common.cuh"
#include "kernels.h"

template <int BT, int EPI>
SSB_DEVINL void gemv_epilogue(const GemvArgs& a, int pair, int m, float v0, float v1) {
  // v0/v1: fp32 dot products of physical rows (2*pair, 2*pair+1) for tile row m (global row index)
  if constexpr (EPI == EPI_F32) {
    const size_t o = (size_t)m * a.ld_out + 2 * pair;
    if (a.f32_add) {
      const float2 ad = __ldcg(reinterpret_cast<const float2*>(a.f32_add + o));
      v0 += ad.x;
      v1 += ad.y;
    }
    a.out_f32[o] = v0;
    a.out_f32[o + 1] = v1;
  } else if constexpr (EPI == EPI_GELU) {
    // nn.GELU() (erf form) on the bf16 Linear output, result bf16   HF:models/falcon/modeling_falcon.py:539-541
    const float g0 = bf16r(v0), g1 = bf16r(v1);
    const float y0 = 0.5f * g0 * (1.0f + erff(g0 * 0.70710678118654752440f));
    const float y1 = 0.5f * g1 * (1.0f + erff(g1 * 0.70710678118654752440f));
    *reinterpret_cast<uint32_t*>(a.out_bf16 + (size_t)m * a.ld_out + 2 * pair) = pack_bf16(y0, y1);
  } else if constexpr (EPI == EPI_RESID2) {
    // mlp_output += attention_output; output = mlp_output + residual   (bf16 adds)  HF:...modeling_falcon.py:628-636
    const size_t o = (size_t)m * a.ld_out + 2 * pair;
    const uint32_t r2 = __ldcg(reinterpret_cast<const uint32_t*>(a.resid2 + o));
    const uint32_t r = __ldcg(reinterpret_cast<const uint32_t*>(a.resid + o));
    const float t0 = bf16r(bf16r(v0) + bf_lo(r2)), t1 = bf16r(bf16r(v1) + bf_hi(r2));
    *reinterpret_cast<uint32_t*>(a.out_bf16 + o) = pack_bf16(t0 + bf_lo(r), t1 + bf_hi(r));
  } else if constexpr (EPI == EPI_F32_PUSH) {
    const long long o = a.push_off + (long long)m * a.ld_out + 2 * pair;
    const float2 v = make_float2(v0, v1);
    for (int r = 0; r < a.push_n; ++r) *reinterpret_cast<float2*>(a.push_dst[r] + o) = v;  // posted remote stores
  } else if constexpr (EPI == EPI_F32_BF16R) {
    a.out_f32[(size_t)m * a.ld_out + 2 * pair] = bf16r(v0);
    a.out_f32[(size_t)m * a.ld_out + 2 * pair + 1] = bf16r(v1);
  } else if constexpr (EPI == EPI_BF16) {
    *reinterpret_cast<uint32_t*>(a.out_bf16 + (size_t)m * a.ld_out + 2 * pair) = pack_bf16(v0, v1);
  } else if constexpr (EPI == EPI_RESID) {
    size_t o = (size_t)m * a.ld_out + 2 * pair;
    uint32_t r = __ldcg(reinterpret_cast<const uint32_t*>(a.resid + o));  // L2: other CTAs/phases write h
    *reinterpret_cast<uint32_t*>(a.out_bf16 + o) = pack_bf16(bf16r(v0) + bf_lo(r), bf16r(v1) + bf_hi(r));
  } else if constexpr (EPI == EPI_SWIGLU) {
    float g = bf16r(v0), u = bf16r(v1);
    float s = bf16r(g / (1.0f + expf(-g)));
    a.out_bf16[(size_t)m * a.ld_out + pair] = __float2bfloat16_rn(s * u);
  } else if constexpr (EPI == EPI_QKV_ROPE) {
    const int hd = a.head_dim, half = hd >> 1;
    const int q_pairs = a.q_rows >> 1, k_pairs = a.kv_rows >> 1;
    const int pos = __ldcg(a.row_pos + m);
    if (pair < q_pairs + k_pairs) {
      const bool is_q = pair < q_pairs;
      const int pp = is_q ? pair : pair - q_pairs;
      const int head = pp / half, j = pp - head * half;
      const uint32_t cs = a.rope_cs[(size_t)pos * half + j];
      const float c = bf_lo(cs), s = bf_hi(cs);
      const float x0 = bf16r(v0), x1 = bf16r(v1);  // Linear outputs are bf16
      // (q*cos) + (rotate_half(q)*sin), every op rounded to bf16 like the HF bf16 tensor ops
      const float y0 = bf16r(bf16r(x0 * c) + bf16r(-x1 * s));
      const float y1 = bf16r(bf16r(x1 * c) + bf16r(x0 * s));
      if (is_q) {
        bf16* q = a.q_out + (size_t)m * a.q_rows + head * hd + j;
        q[0] = __float2bfloat16_rn(y0);
        q[half] = __float2bfloat16_rn(y1);
      } else {
        const int slot = a.row_slot[m];
        const int blk = a.block_table[(size_t)slot * a.bt_stride + pos / a.block_size];
        bf16* k = a.kcache + (((size_t)blk * a.kvh + head) * a.block_size + (pos % a.block_size)) * hd + j;
        k[0] = __float2bfloat16_rn(y0);
        k[half] = __float2bfloat16_rn(y1);
      }
    } else {
      const int e = 2 * (pair - q_pairs - k_pairs);
      const int head = e / hd, j = e - head * hd;
      const int slot = a.row_slot[m];
      const int blk = a.block_table[(size_t)slot * a.bt_stride + pos / a.block_size];
      bf16* v = a.vcache + (((size_t)blk * a.kvh + head) * a.block_size + (pos % a.block_size)) * hd + j;
      *reinterpret_cast<uint32_t*>(v) = pack_bf16(v0, v1);
    }
  }
}


// ---------------------------------------------------------------------------------------------------------------------
// Epilogue inputs fetched at the START of a row-pair pass (GEMV kernels).  The residual / position / RoPE-table / block-table
// reads are one or two DEPENDENT L2 round trips; done after the K loop they sit on the critical path of every
// pass of every consumer warp (a QKV pass of the persistent kernel is a short stretch of streaming).  They depend on nothing the
// pass computes, so the lane that will run the epilogue for row m issues them before the first weight chunk and the K loop
// hides them.  Safe with out == resid: a pair's residual element is written by this pair's own epilogue only.
struct EpiPre {
  uint32_t r;    // EPI_RESID: residual word (2 x bf16)
  int pos, blk;  // EPI_QKV_ROPE: position of the row, KV block of that position
  uint32_t cs;   // EPI_QKV_ROPE: packed cos | sin of (pos, j)
};
template <int EPI>
SSB_DEVINL EpiPre epi_prefetch(const GemvArgs& a, int pair, int m) {
  EpiPre p = {0u, 0, 0, 0u};
  if constexpr (EPI == EPI_RESID) {
    p.r = __ldcg(reinterpret_cast<const uint32_t*>(a.resid + (size_t)m * a.ld_out + 2 * pair));
  } else if constexpr (EPI == EPI_QKV_ROPE) {
    const int half = a.head_dim >> 1;
    const int q_pairs = a.q_rows >> 1, k_pairs = a.kv_rows >> 1;
    p.pos = __ldcg(a.row_pos + m);
    if (pair < q_pairs + k_pairs) {
      const int pp = pair < q_pairs ? pair : pair - q_pairs;
      p.cs = a.rope_cs[(size_t)p.pos * half + (pp % half)];
    }
    if (pair >= q_pairs) p.blk = a.block_table[(size_t)a.row_slot[m] * a.bt_stride + p.pos / a.block_size];
  }
  return p;
}
// same math and rounding points as gemv_epilogue for the two epilogues that have prefetched inputs
template <int BT, int EPI>
SSB_DEVINL void gemv_epilogue_pre(const GemvArgs& a, int pair, int m, float v0, float v1, const EpiPre& pre) {
  if constexpr (EPI == EPI_RESID) {
    const size_t o = (size_t)m * a.ld_out + 2 * pair;
    *reinterpret_cast<uint32_t*>(a.out_bf16 + o) = pack_bf16(bf16r(v0) + bf_lo(pre.r), bf16r(v1) + bf_hi(pre.r));
  } else if constexpr (EPI == EPI_QKV_ROPE) {
    const int hd = a.head_dim, half = hd >> 1;
    const int q_pairs = a.q_rows >> 1, k_pairs = a.kv_rows >> 1;
    const int pos = pre.pos;
    if (pair < q_pairs + k_pairs) {
      const bool is_q = pair < q_pairs;
      const int pp = is_q ? pair : pair - q_pairs;
      const int head = pp / half, j = pp - head * half;
      const float c = bf_lo(pre.cs), s = bf_hi(pre.cs);
      const float x0 = bf16r(v0), x1 = bf16r(v1);
      const float y0 = bf16r(bf16r(x0 * c) + bf16r(-x1 * s));
      const float y1 = bf16r(bf16r(x1 * c) + bf16r(x0 * s));
      if (is_q) {
        bf16* q = a.q_out + (size_t)m * a.q_rows + head * hd + j;
        q[0] = __float2bfloat16_rn(y0);
        q[half] = __float2bfloat16_rn(y1);
      } else {
        bf16* k = a.kcache + (((size_t)pre.blk * a.kvh + head) * a.block_size + (pos % a.block_size)) * hd + j;
        k[0] = __float2bfloat16_rn(y0);
        k[half] = __float2bfloat16_rn(y1);
      }
    } else {
      const int e = 2 * (pair - q_pairs - k_pairs);
      const int head = e / hd, j = e - head * hd;
      bf16* v = a.vcache + (((size_t)pre.blk * a.kvh + head) * a.block_size + (pos % a.block_size)) * hd + j;
      *reinterpret_cast<uint32_t*>(v) = pack_bf16(v0, v1);
    }
  } else {
    gemv_epilogue<BT, EPI>(a, pair, m, v0, v1);
  }
}

// Eight tokens at once for one row pair (tensor-core kernels: a thread owns a weight row across the token tile).
// The per-token epilogue above does dependent global loads (residual, position, rope table, block table) followed by a
// store; out_bf16 may alias resid, so the compiler cannot hoist the next token's loads above the previous store and
// the tile epilogue degenerates into ~TN serialized L2 round trips .  Here all loads of
// the eight tokens are issued first.
// QKV + RoPE + KV-append for eight tokens of one row pair with the token-dependent inputs (position, KV block of that
// position) already staged in shared memory by the caller (tc_gemm_kernel stages them once per token tile while the MMAs of
// the tile run).  The generic form below re-reads row_pos -> {rope table, row_slot -> block_table} per thread: three
// dependent L2 round trips per eight tokens, which can make the prefill QKV GEMM take longer than gate/up for a
// fraction of its FLOPs.  Here only the rope-table read remains, all eight issued at once.
SSB_DEVINL void tc_epilogue8_qkv_cs(const GemvArgs& a, int pair, int m0, const int* __restrict__ s_pos, const int* __restrict__ s_blk,
                                    const uint32_t* cs, const float (&v0)[8], const float (&v1)[8]) {
  // cs[j] = packed cos | sin of (token m0 + j, this pair), already loaded by the caller (unused for V rows)
  const int hd = a.head_dim, half = hd >> 1;
  const int q_pairs = a.q_rows >> 1, k_pairs = a.kv_rows >> 1;
  const bool is_q = pair < q_pairs, is_k = !is_q && pair < q_pairs + k_pairs;
  if (is_q || is_k) {
    const int pp = is_q ? pair : pair - q_pairs;
    const int head = pp / half, jj = pp - head * half;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (m0 + j >= a.M) continue;
      const float c = bf_lo(cs[j]), s = bf_hi(cs[j]);
      const float x0 = bf16r(v0[j]), x1 = bf16r(v1[j]);
      const float y0 = bf16r(bf16r(x0 * c) + bf16r(-x1 * s));
      const float y1 = bf16r(bf16r(x1 * c) + bf16r(x0 * s));
      bf16* dst = is_q ? a.q_out + (size_t)(m0 + j) * a.q_rows + head * hd + jj
                       : a.kcache + (((size_t)s_blk[j] * a.kvh + head) * a.block_size + (s_pos[j] % a.block_size)) * hd + jj;
      dst[0] = __float2bfloat16_rn(y0);
      dst[half] = __float2bfloat16_rn(y1);
    }
  } else {
    const int e = 2 * (pair - q_pairs - k_pairs);
    const int head = e / hd, jj = e - head * hd;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (m0 + j >= a.M) continue;
      bf16* v = a.vcache + (((size_t)s_blk[j] * a.kvh + head) * a.block_size + (s_pos[j] % a.block_size)) * hd + jj;
      *reinterpret_cast<uint32_t*>(v) = pack_bf16(v0[j], v1[j]);
    }
  }
}
SSB_DEVINL void tc_epilogue8_qkv_staged(const GemvArgs& a, int pair, int m0, const int* __restrict__ s_pos, const int* __restrict__ s_blk,
                                        const float (&v0)[8], const float (&v1)[8]) {
  const int half = a.head_dim >> 1;
  const int q_pairs = a.q_rows >> 1, k_pairs = a.kv_rows >> 1;
  uint32_t cs[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
  if (pair < q_pairs + k_pairs) {
    const int pp = pair < q_pairs ? pair : pair - q_pairs;
    const int jj = pp % half;
#pragma unroll
    for (int j = 0; j < 8; ++j) cs[j] = (m0 + j < a.M) ? a.rope_cs[(size_t)s_pos[j] * half + jj] : 0u;
  }
  tc_epilogue8_qkv_cs(a, pair, m0, s_pos, s_blk, cs, v0, v1);
}

template <int EPI>
SSB_DEVINL void tc_epilogue8(const GemvArgs& a, int pair, int m0, const float (&v0)[8], const float (&v1)[8]) {
  if constexpr (EPI == EPI_RESID || EPI == EPI_RESID2) {
    uint32_t r[8], r2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      r[j] = r2[j] = 0;
      if (m0 + j < a.M) {
        const size_t o = (size_t)(m0 + j) * a.ld_out + 2 * pair;
        r[j] = __ldcg(reinterpret_cast<const uint32_t*>(a.resid + o));
        if constexpr (EPI == EPI_RESID2) r2[j] = __ldcg(reinterpret_cast<const uint32_t*>(a.resid2 + o));
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (m0 + j < a.M) {
        const size_t o = (size_t)(m0 + j) * a.ld_out + 2 * pair;
        float t0 = bf16r(v0[j]), t1 = bf16r(v1[j]);
        if constexpr (EPI == EPI_RESID2) {
          t0 = bf16r(t0 + bf_lo(r2[j]));
          t1 = bf16r(t1 + bf_hi(r2[j]));
        }
        *reinterpret_cast<uint32_t*>(a.out_bf16 + o) = pack_bf16(t0 + bf_lo(r[j]), t1 + bf_hi(r[j]));
      }
    }
  } else if constexpr (EPI == EPI_QKV_ROPE) {
    const int hd = a.head_dim, half = hd >> 1;
    const int q_pairs = a.q_rows >> 1, k_pairs = a.kv_rows >> 1;
    int pos[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) pos[j] = (m0 + j < a.M) ? __ldcg(a.row_pos + m0 + j) : 0;
    const bool is_q = pair < q_pairs, is_k = !is_q && pair < q_pairs + k_pairs;
    int blk[8];
    if (!is_q) {
      int slot[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) slot[j] = (m0 + j < a.M) ? a.row_slot[m0 + j] : 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) blk[j] = (m0 + j < a.M) ? a.block_table[(size_t)slot[j] * a.bt_stride + pos[j] / a.block_size] : 0;
    }
    if (is_q || is_k) {
      const int pp = is_q ? pair : pair - q_pairs;
      const int head = pp / half, jj = pp - head * half;
      uint32_t cs[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) cs[j] = a.rope_cs[(size_t)pos[j] * half + jj];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (m0 + j >= a.M) continue;
        const float c = bf_lo(cs[j]), s = bf_hi(cs[j]);
        const float x0 = bf16r(v0[j]), x1 = bf16r(v1[j]);
        const float y0 = bf16r(bf16r(x0 * c) + bf16r(-x1 * s));
        const float y1 = bf16r(bf16r(x1 * c) + bf16r(x0 * s));
        bf16* dst = is_q ? a.q_out + (size_t)(m0 + j) * a.q_rows + head * hd + jj
                         : a.kcache + (((size_t)blk[j] * a.kvh + head) * a.block_size + (pos[j] % a.block_size)) * hd + jj;
        dst[0] = __float2bfloat16_rn(y0);
        dst[half] = __float2bfloat16_rn(y1);
      }
    } else {
      const int e = 2 * (pair - q_pairs - k_pairs);
      const int head = e / hd, jj = e - head * hd;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (m0 + j >= a.M) continue;
        bf16* v = a.vcache + (((size_t)blk[j] * a.kvh + head) * a.block_size + (pos[j] % a.block_size)) * hd + jj;
        *reinterpret_cast<uint32_t*>(v) = pack_bf16(v0[j], v1[j]);
      }
    }
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (m0 + j < a.M) gemv_epilogue<1, EPI>(a, pair, m0 + j, v0[j], v1[j]);
  }
}
