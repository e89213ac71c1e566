// kernels.cu — hand-written sm_90a kernels of the decode loop (small-batch path).
//
// Math follows the HF-transformers Llama forward the reference's serving image wraps
// (SURVEY.md §8a K1-K9; HF = site-packages/transformers):
//   RMSNorm      HF:models/llama/modeling_llama.py:62-67   (fp32 stats, cast to bf16 BEFORE the weight multiply)
//   q/k/v/o/mlp  HF:models/llama/modeling_llama.py:177-183,238-288 (bf16 Linear, fp32 accumulate, bf16 output)
//   RoPE         HF:models/llama/modeling_llama.py:124-168 (bf16 cos/sin, half-split pairing (j, j+d/2))
//   attention    HF:models/llama/modeling_llama.py:199-221 (scores rounded to bf16, * d^-1/2 in bf16, fp32 softmax)
//   greedy pick  HF:generation/utils.py:2762,2793 (logits.float(), argmax)
//
// The dominant kernel is proj_rows_kernel: y[M<=4, N] = x * W^T with W streamed from HBM exactly once through a
// TMA-engine (cp.async.bulk) -> shared-memory mbarrier ring, consumed by 8 warps with fp32 FMAs and warp-shuffle
// reductions; norm prologue and RoPE/KV-append/SwiGLU/residual epilogues are fused.  It is HBM-bound (SURVEY §8d):
// algorithmic bytes per launch = 2*N*K.
#include "common.cuh"
#include "kernels.h"
#include <cstring>

#include "gemv_core.cuh"

// =====================================================================================================================
// proj_rows_kernel
// =====================================================================================================================
constexpr int GV_CW = 8;                        // consumer warps
constexpr int GV_PW = 4;                        // producer warps: the compiler lowers per-lane cp.async.bulk to a serial
                                                // ELECT loop (~70 cycles per copy), so one warp tops out near 29 B/clk/SM
constexpr int GV_THREADS = (GV_CW + GV_PW) * 32;
constexpr int GV_ROWS = 2 * GV_CW;              // weight rows per stage (each consumer warp owns one row pair)
constexpr int GV_KC = 1024;                     // K elements per stage
constexpr int GV_MAX_STAGES = 6;                // up to 6 x 32 KiB in flight per SM (as many as fit beside the staged activations)
constexpr int GV_RS = GEMV_RS;                  // stage row stride (padded for ldmatrix, gemv_core.cuh)
constexpr int GV_STAGE_ELEMS = GV_ROWS * GV_RS;
constexpr int GV_RED_FLOATS = 2 * GV_CW * 16 * 4;  // cross-warp sum of the k slices, double-buffered by pass

int gemv_pick_bt(int M, int K);
static size_t gemv_smem_bytes(int bt, int K, int stages) {
  return (size_t)stages * GV_STAGE_ELEMS * 2 + (size_t)bt * K * 2 + 2 * (size_t)stages * 8 + 128 + (size_t)GV_RED_FLOATS * 4;
}
static int gemv_pick_stages(int bt, int K) {
  int s = GV_MAX_STAGES;
  while (s > 2 && gemv_smem_bytes(bt, K, s) > 225 * 1024) --s;
  return s;
}

int gemv_grid_ctas(int M, int N, int K, int n_sm) {
  const int bt = gemv_pick_bt(M, K), P = N / 2;
  return (n_sm < P ? n_sm : P) * ((M + bt - 1) / bt);
}

int gemv_pick_bt(int M, int K) {
  int bt = M >= 3 ? 4 : (M >= 2 ? 2 : 1);  // 3 rows ride a 4-row tile: two passes of a 2-row tile would stream the weights twice
  while (bt > 1 && gemv_smem_bytes(bt, K, 2) > 225 * 1024) bt >>= 1;
  return bt;
}

#include "epilogue.cuh"

template <int BT, int EPI, int NORM>
__global__ void __launch_bounds__(GV_THREADS, 1) proj_rows_kernel(const GemvArgs a) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const int n_stages = a.n_stages;
  bf16* tiles = reinterpret_cast<bf16*>(smem_raw);            // [n_stages][ROWS][RS]
  bf16* xs = tiles + (size_t)n_stages * GV_STAGE_ELEMS;       // [BT][K]
  uint64_t* full = reinterpret_cast<uint64_t*>(xs + (size_t)BT * a.K);
  uint64_t* empty = full + n_stages;
  float* red = reinterpret_cast<float*>(empty + n_stages);    // [32]
  float* red_s = red + 32;                                    // [2][GV_CW][16][4] k-slice partial sums

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int K = a.K;
  const int P = a.N >> 1;  // row pairs
  const int p0 = (int)(((long long)blockIdx.x * P) / gridDim.x);
  const int p1 = (int)(((long long)(blockIdx.x + 1) * P) / gridDim.x);
  const int m0 = blockIdx.y * BT;
  const int nk = (K + GV_KC - 1) / GV_KC;

  for (size_t i = tid; i < (size_t)n_stages * GV_STAGE_ELEMS / 8; i += GV_THREADS)
    reinterpret_cast<uint4*>(tiles)[i] = make_uint4(0, 0, 0, 0);  // k tails multiply stale ring contents by zero: keep them finite
  if (tid == 0) {
    for (int s = 0; s < n_stages; ++s) {
      mbar_init(&full[s], GV_PW);
      mbar_init(&empty[s], GV_CW);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();

  if (warp >= GV_CW) {
    // ------------------------------------------------------------ producer: weights never depend on the previous
    // kernel, so the stream from HBM starts before griddepcontrol.wait (PDL prologue overlap).
    const uint64_t pol = policy_evict_first();
    int stage = 0;
    uint32_t phase = 0;
    for (int ps = p0; ps < p1; ps += GV_CW) {
      const int nr = 2 * min(GV_CW, p1 - ps);
      for (int kc = 0; kc < nk; ++kc) {
        const int k0 = kc * GV_KC;
        const int len = min(GV_KC, K - k0);
        mbar_wait(&empty[stage], phase ^ 1);
        // producer warp pw owns rows [pw*RPP, (pw+1)*RPP) of the stage
        constexpr int RPP = GV_ROWS / GV_PW;
        const int r0 = (warp - GV_CW) * RPP;
        const int mine = max(0, min(RPP, nr - r0));
        if (lane == 0) mbar_expect_tx(&full[stage], (uint32_t)(mine * len * 2));
        __syncwarp();
        if (lane < mine)
          bulk_g2s_hint(tiles + ((size_t)stage * GV_ROWS + r0 + lane) * GV_RS, a.W + (size_t)(2 * ps + r0 + lane) * K + k0,
                        (uint32_t)(len * 2), &full[stage], pol);
        if (++stage == n_stages) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
  } else {
    // ------------------------------------------------------------ consumers
    pdl_wait();  // activations of the previous kernel are now visible
    const int ctid = tid;  // 0..255
#pragma unroll
    for (int b = 0; b < BT; ++b) {
      const int m = m0 + b;
      bf16* xrow = xs + (size_t)b * K;
      if (m >= a.M) {
        for (int k = ctid * 8; k < K; k += GV_CW * 32 * 8) *reinterpret_cast<uint4*>(xrow + k) = make_uint4(0, 0, 0, 0);
        continue;
      }
      const bf16* src = a.x + (size_t)(a.row_map ? a.row_map[m] : m) * a.ldx;
      if constexpr (NORM == NORM_RMS) {
        float ss = 0.f;
        for (int k = ctid * 8; k < K; k += GV_CW * 32 * 8) {
          uint4 v = *reinterpret_cast<const uint4*>(src + k);
          const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            float lo = bf_lo(u[i]), hi = bf_hi(u[i]);
            ss += lo * lo + hi * hi;
          }
        }
        ss = warp_sum(ss);
        if (lane == 0) red[warp] = ss;
        named_bar_sync(1, GV_CW * 32);
        float tot = 0.f;
#pragma unroll
        for (int w = 0; w < GV_CW; ++w) tot += red[w];
        named_bar_sync(1, GV_CW * 32);  // red[] reused by the next tile row
        const float rstd = rsqrtf(tot / (float)K + a.eps);
        for (int k = ctid * 8; k < K; k += GV_CW * 32 * 8) {
          uint4 v = *reinterpret_cast<const uint4*>(src + k);
          uint4 w = ldg128(a.norm_w + k);
          const uint32_t u[4] = {v.x, v.y, v.z, v.w};
          const uint32_t wu[4] = {w.x, w.y, w.z, w.w};
          uint32_t o[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            // w * bf16(x * rstd): normalised value is cast to bf16 BEFORE the (bf16) weight multiply
            float lo = bf16r(bf_lo(u[i]) * rstd) * bf_lo(wu[i]);
            float hi = bf16r(bf_hi(u[i]) * rstd) * bf_hi(wu[i]);
            o[i] = pack_bf16(lo, hi);
          }
          *reinterpret_cast<uint4*>(xrow + k) = make_uint4(o[0], o[1], o[2], o[3]);
        }
      } else if constexpr (NORM == NORM_LN) {
        // torch.nn.LayerNorm on bf16: fp32 statistics, y = (x - mean) * rstd * w + b in fp32, ONE rounding to bf16
        // (HF:models/falcon/modeling_falcon.py:572-576,594-596 ln_attn / ln_mlp / ln_f)
        float sm = 0.f;
        for (int k = ctid * 8; k < K; k += GV_CW * 32 * 8) {
          const uint4 v = *reinterpret_cast<const uint4*>(src + k);
          const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int i = 0; i < 4; ++i) sm += bf_lo(u[i]) + bf_hi(u[i]);
        }
        sm = warp_sum(sm);
        if (lane == 0) red[warp] = sm;
        named_bar_sync(1, GV_CW * 32);
        float tot = 0.f;
#pragma unroll
        for (int w = 0; w < GV_CW; ++w) tot += red[w];
        named_bar_sync(1, GV_CW * 32);
        const float mean = tot / (float)K;
        float sq = 0.f;
        for (int k = ctid * 8; k < K; k += GV_CW * 32 * 8) {
          const uint4 v = *reinterpret_cast<const uint4*>(src + k);
          const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float lo = bf_lo(u[i]) - mean, hi = bf_hi(u[i]) - mean;
            sq += lo * lo + hi * hi;
          }
        }
        sq = warp_sum(sq);
        if (lane == 0) red[warp] = sq;
        named_bar_sync(1, GV_CW * 32);
        tot = 0.f;
#pragma unroll
        for (int w = 0; w < GV_CW; ++w) tot += red[w];
        named_bar_sync(1, GV_CW * 32);
        const float rstd = rsqrtf(tot / (float)K + a.eps);
        for (int k = ctid * 8; k < K; k += GV_CW * 32 * 8) {
          const uint4 v = *reinterpret_cast<const uint4*>(src + k);
          const uint4 w = ldg128(a.norm_w + k);
          const uint4 bb = ldg128(a.norm_b + k);
          const uint32_t u[4] = {v.x, v.y, v.z, v.w};
          const uint32_t wu[4] = {w.x, w.y, w.z, w.w};
          const uint32_t bu[4] = {bb.x, bb.y, bb.z, bb.w};
          uint32_t o[4];
#pragma unroll
          for (int i = 0; i < 4; ++i)
            o[i] = pack_bf16((bf_lo(u[i]) - mean) * rstd * bf_lo(wu[i]) + bf_lo(bu[i]),
                             (bf_hi(u[i]) - mean) * rstd * bf_hi(wu[i]) + bf_hi(bu[i]));
          *reinterpret_cast<uint4*>(xrow + k) = make_uint4(o[0], o[1], o[2], o[3]);
        }
      } else {
        for (int k = ctid * 8; k < K; k += GV_CW * 32 * 8)
          *reinterpret_cast<uint4*>(xrow + k) = *reinterpret_cast<const uint4*>(src + k);
      }
    }
    named_bar_sync(1, GV_CW * 32);

    // tensor-pipe consumers (gemv_core.cuh: mma_chunk): warp w multiplies all 16 rows of a stage by its 128-wide k slice; the 8
    // slices are summed through shared memory per pass and warp w runs the epilogue of pair ps + w, lane b = batch row m0 + b
    int stage = 0;
    uint32_t phase = 0;
    int pass = 0;
    for (int ps = p0; ps < p1; ps += GV_CW, ++pass) {
      const int pair = ps + warp;
      const bool valid = pair < p1;
      float c[4] = {0.f, 0.f, 0.f, 0.f};
      // the epilogue's dependent global reads, issued now and hidden by the K loop (epilogue.cuh: EpiPre)
      [[maybe_unused]] EpiPre pre = {0u, 0, 0, 0u};
      if constexpr (EPI == EPI_RESID || EPI == EPI_QKV_ROPE) {
        if (valid && lane < BT && m0 + lane < a.M) pre = epi_prefetch<EPI>(a, pair, m0 + lane);
      }
      for (int kc = 0; kc < nk; ++kc) {
        const int k0 = kc * GV_KC;
        const int len = min(GV_KC, K - k0);
        mbar_wait(&full[stage], phase);
        mma_chunk<BT>(tiles + (size_t)stage * GV_STAGE_ELEMS, xs, K, k0, len, warp, lane, c);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[stage]);
        if (++stage == n_stages) {
          stage = 0;
          phase ^= 1;
        }
      }
      float* rb = red_s + (size_t)(pass & 1) * (GV_CW * 64);
      mma_store_partial<BT>(rb + warp * 64, lane, c);
      named_bar_sync(1, GV_CW * 32);
      if (valid && lane < BT && m0 + lane < a.M) {
        float v0 = 0.f, v1 = 0.f;
#pragma unroll
        for (int w = 0; w < GV_CW; ++w) {  // fixed order: deterministic
          v0 += rb[w * 64 + (2 * warp) * 4 + lane];
          v1 += rb[w * 64 + (2 * warp + 1) * 4 + lane];
        }
        if constexpr (EPI == EPI_RESID || EPI == EPI_QKV_ROPE) {
          gemv_epilogue_pre<BT, EPI>(a, pair, m0 + lane, v0, v1, pre);
        } else {
          gemv_epilogue<BT, EPI>(a, pair, m0 + lane, v0, v1);
        }
      }
    }
    if constexpr (EPI == EPI_F32_PUSH) {
      // all pushes of this CTA are issued: make them visible system-wide, then count this CTA in at every rank
      named_bar_sync(1, GV_CW * 32);
      if (tid == 0) {
        __threadfence_system();
        for (int r = 0; r < a.push_n; ++r)
          asm volatile("red.release.sys.global.add.u64 [%0], %1;" ::"l"(a.push_flags[r] + a.push_rank), "l"(1ull) : "memory");
      }
    }
  }
}

template <typename KernelT, typename... Args>
static cudaError_t launch_ex(KernelT kernel, dim3 grid, dim3 block, size_t smem, const LaunchCfg& lc, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = lc.stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = lc.pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, args...);
}

template <int BT, int EPI, int NORM>
static cudaError_t launch_gemv_t(const GemvArgs& a_in, const LaunchCfg& lc) {
  GemvArgs a = a_in;
  a.n_stages = gemv_pick_stages(BT, a.K);
  const size_t smem = gemv_smem_bytes(BT, a.K, a.n_stages);
  static std::atomic<unsigned long long> attr_mask{0};  // per instantiation, per device
  if (first_launch_on_device(attr_mask)) {
    cudaError_t e = cudaFuncSetAttribute(proj_rows_kernel<BT, EPI, NORM>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return e;
  }
  const int P = a.N / 2;
  int gx = lc.n_sm < P ? lc.n_sm : P;
  dim3 grid(gx, (a.M + BT - 1) / BT);
  return launch_ex(proj_rows_kernel<BT, EPI, NORM>, grid, dim3(GV_THREADS), smem, lc, a);
}

template <int EPI, int NORM>
static cudaError_t launch_gemv_bt(const GemvArgs& a, const LaunchCfg& lc) {
  switch (gemv_pick_bt(a.M, a.K)) {
    case 4: return launch_gemv_t<4, EPI, NORM>(a, lc);
    case 2: return launch_gemv_t<2, EPI, NORM>(a, lc);
    default: return launch_gemv_t<1, EPI, NORM>(a, lc);
  }
}

cudaError_t launch_gemv(const GemvArgs& a, int epi, int norm, const LaunchCfg& lc) {
  if ((a.N & 1) || (a.K & 7)) return cudaErrorInvalidValue;
  if (norm == NORM_RMS) {
    switch (epi) {
      case EPI_QKV_ROPE: return launch_gemv_bt<EPI_QKV_ROPE, NORM_RMS>(a, lc);
      case EPI_SWIGLU: return launch_gemv_bt<EPI_SWIGLU, NORM_RMS>(a, lc);
      case EPI_F32_BF16R: return launch_gemv_bt<EPI_F32_BF16R, NORM_RMS>(a, lc);
      default: return cudaErrorInvalidValue;
    }
  }
  if (norm == NORM_LN) {
    switch (epi) {
      case EPI_QKV_ROPE: return launch_gemv_bt<EPI_QKV_ROPE, NORM_LN>(a, lc);
      case EPI_GELU: return launch_gemv_bt<EPI_GELU, NORM_LN>(a, lc);
      case EPI_F32_BF16R: return launch_gemv_bt<EPI_F32_BF16R, NORM_LN>(a, lc);
      default: return cudaErrorInvalidValue;
    }
  }
  switch (epi) {
    case EPI_RESID2: return launch_gemv_bt<EPI_RESID2, NORM_NONE>(a, lc);
    case EPI_RESID: return launch_gemv_bt<EPI_RESID, NORM_NONE>(a, lc);
    case EPI_F32: return launch_gemv_bt<EPI_F32, NORM_NONE>(a, lc);
    case EPI_F32_PUSH: return launch_gemv_bt<EPI_F32_PUSH, NORM_NONE>(a, lc);
    case EPI_BF16: return launch_gemv_bt<EPI_BF16, NORM_NONE>(a, lc);
    default: return cudaErrorInvalidValue;
  }
}

// =====================================================================================================================
// paged-KV decode attention, split over the context, flash-style merge, last-arriving CTA combines the splits
// =====================================================================================================================
constexpr int AT_WARPS = 4;
constexpr int AT_THREADS = AT_WARPS * 32;

template <int D, int G>
__global__ void __launch_bounds__(AT_THREADS) attn_decode_kernel(const AttnArgs a) {
  constexpr int LPR = D / 8;        // lanes per K/V row (16 B each)
  constexpr int RPW = 32 / LPR;     // rows per warp iteration
  constexpr int NSUB = AT_WARPS * RPW;
  __shared__ float sm_m[NSUB][G];
  __shared__ float sm_l[NSUB][G];
  __shared__ float sm_o[NSUB][G][D];
  __shared__ int sm_last;

  pdl_wait();
  pdl_launch_dependents();

  const int split = blockIdx.x, row = blockIdx.z;
  const int kvh = blockIdx.y / (a.group / G);   // G = query heads handled by this CTA (all share one KV head)
  const int head0 = blockIdx.y * G;             // heads are kv-major: head = kvh*group + g
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int sub = lane / LPR, li = lane % LPR;
  const int slot = a.row_slot[row];
  const int ctx = a.row_pos[row] + 1;
  const int BS = a.block_size;
  int chunk = (ctx + a.n_splits - 1) / a.n_splits;
  chunk = ((chunk + BS - 1) / BS) * BS;
  const int n_active = (ctx + chunk - 1) / chunk;
  if (split >= n_active) return;
  const int t_begin = split * chunk;
  const int t_end = min(ctx, t_begin + chunk);
  const int HD = a.n_heads * D;  // q/out row stride

  // ATTN_LITE=1 (compile-time experiment, variant library "attnlite" = with GEMV_MIXED_FMA; never run on hardware): the
  // split-context decode attention is instruction-bound at batch 32 (~85 instructions per 2 x 512 B of K/V per warp).
  // q and K stay packed and q.k runs on the mixed-precision FMA (same products, same order: bit-identical), and the
  // accumulator rescale is skipped while the running maximum does not move (corr = exp(0) = 1 exactly: bit-identical).
#ifndef ATTN_LITE
#define ATTN_LITE 0
#endif
#if ATTN_LITE
  uint32_t qp[G][4];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const uint4 v = *reinterpret_cast<const uint4*>(a.q + (size_t)row * HD + (head0 + g) * D + li * 8);
    qp[g][0] = v.x;
    qp[g][1] = v.y;
    qp[g][2] = v.z;
    qp[g][3] = v.w;
  }
#else
  float q[G][8];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const uint4 v = *reinterpret_cast<const uint4*>(a.q + (size_t)row * HD + (head0 + g) * D + li * 8);
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      q[g][2 * i] = bf_lo(u[i]);
      q[g][2 * i + 1] = bf_hi(u[i]);
    }
  }
#endif
  float m[G], l[G], acc[G][8];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    m[g] = -1e30f;
    l[g] = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[g][i] = 0.f;
  }
  const int* bt = a.block_table + (size_t)slot * a.bt_stride;
  // Latency-bound at small batch: issue the K/V loads of UNR token groups before consuming any (2*UNR 16-byte loads in
  // flight per lane).  The trip count is warp-uniform; the shuffles use the full mask, so every lane executes them even
  // when its own token is past the end (a half-warp leaving early would deadlock the warp).
  constexpr int UNR = (G <= 2) ? 4 : 2;
  constexpr int TSTEP = AT_WARPS * RPW;
  for (int tb = t_begin + warp * RPW; tb < t_end; tb += TSTEP * UNR) {
    uint4 kq[UNR], vq[UNR];
    bool tvq[UNR];
#pragma unroll
    for (int u = 0; u < UNR; ++u) {
      const int t = tb + u * TSTEP + sub;
      tvq[u] = t < t_end;
      kq[u] = make_uint4(0, 0, 0, 0);
      vq[u] = make_uint4(0, 0, 0, 0);
      if (tvq[u]) {
        const int blk = bt[t / BS];
        const size_t off = (((size_t)blk * a.kvh + kvh) * BS + (t % BS)) * D + li * 8;
        kq[u] = *reinterpret_cast<const uint4*>(a.kcache + off);
        vq[u] = *reinterpret_cast<const uint4*>(a.vcache + off);
      }
    }
#pragma unroll
    for (int u = 0; u < UNR; ++u) {
      if (tb + u * TSTEP >= t_end) break;  // warp-uniform
      const bool tv = tvq[u];
      const uint32_t ku[4] = {kq[u].x, kq[u].y, kq[u].z, kq[u].w};
      const uint32_t vu[4] = {vq[u].x, vq[u].y, vq[u].z, vq[u].w};
      float vf[8];
#if !ATTN_LITE
      float kf[8];
#endif
#pragma unroll
      for (int i = 0; i < 4; ++i) {
#if !ATTN_LITE
        kf[2 * i] = bf_lo(ku[i]);
        kf[2 * i + 1] = bf_hi(ku[i]);
#endif
        vf[2 * i] = bf_lo(vu[i]);
        vf[2 * i + 1] = bf_hi(vu[i]);
      }
#pragma unroll
      for (int g = 0; g < G; ++g) {
        float d = 0.f;
#if ATTN_LITE
#pragma unroll
        for (int i = 0; i < 4; ++i) d = fma2_bf16(qp[g][i], ku[i], d);  // d += q[2i] k[2i]; d += q[2i+1] k[2i+1]
#else
#pragma unroll
        for (int i = 0; i < 8; ++i) d = fmaf(q[g][i], kf[i], d);
#endif
#pragma unroll
        for (int o = LPR / 2; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
        if (!tv) continue;
        const float s = bf16r(bf16r(d) * a.scale);  // matmul output is bf16, then "* scaling" in bf16
        const float mn = fmaxf(m[g], s);
#if ATTN_LITE
        const float p = __expf(s - mn);
        if (mn != m[g]) {  // the running maximum moved: rescale (otherwise corr == 1 exactly)
          const float corr = __expf(m[g] - mn);
          m[g] = mn;
          l[g] *= corr;
#pragma unroll
          for (int i = 0; i < 8; ++i) acc[g][i] *= corr;
        }
        l[g] += p;
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[g][i] = fmaf(p, vf[i], acc[g][i]);
#else
        const float corr = __expf(m[g] - mn);
        const float p = __expf(s - mn);
        m[g] = mn;
        l[g] = l[g] * corr + p;
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[g][i] = fmaf(p, vf[i], acc[g][i] * corr);
#endif
      }
    }
  }
  const int sidx = warp * RPW + sub;
#pragma unroll
  for (int g = 0; g < G; ++g) {
    if (li == 0) {
      sm_m[sidx][g] = m[g];
      sm_l[sidx][g] = l[g];
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) sm_o[sidx][g][li * 8 + i] = acc[g][i];
  }
  __syncthreads();
  const size_t pbase = ((size_t)row * gridDim.y + blockIdx.y) * a.n_splits;
  for (int idx = tid; idx < G * D; idx += AT_THREADS) {
    const int g = idx / D, dd = idx % D;
    float mm = -1e30f;
#pragma unroll
    for (int s = 0; s < NSUB; ++s) mm = fmaxf(mm, sm_m[s][g]);
    float ll = 0.f, oo = 0.f;
#pragma unroll
    for (int s = 0; s < NSUB; ++s) {
      const float w = __expf(sm_m[s][g] - mm);
      ll += sm_l[s][g] * w;
      oo += sm_o[s][g][dd] * w;
    }
    if (n_active == 1) {
      a.out[(size_t)row * HD + (head0 + g) * D + dd] = __float2bfloat16_rn(oo / ll);
    } else {
      a.part_o[(pbase + split) * (G * D) + idx] = oo;
      if (dd == 0) {
        a.part_ml[(pbase + split) * (2 * G) + g] = mm;
        a.part_ml[(pbase + split) * (2 * G) + G + g] = ll;
      }
    }
  }
  if (n_active == 1) return;
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const int old = atomicAdd(&a.counters[row * gridDim.y + blockIdx.y], 1);
    sm_last = (old == n_active - 1);
  }
  __syncthreads();
  if (!sm_last) return;
  __threadfence();
  for (int idx = tid; idx < G * D; idx += AT_THREADS) {
    const int g = idx / D, dd = idx % D;
    float mm = -1e30f;
    for (int s = 0; s < n_active; ++s) mm = fmaxf(mm, __ldcg(&a.part_ml[(pbase + s) * (2 * G) + g]));
    float ll = 0.f, oo = 0.f;
    for (int s = 0; s < n_active; ++s) {
      const float w = __expf(__ldcg(&a.part_ml[(pbase + s) * (2 * G) + g]) - mm);
      ll += __ldcg(&a.part_ml[(pbase + s) * (2 * G) + G + g]) * w;
      oo += __ldcg(&a.part_o[(pbase + s) * (G * D) + idx]) * w;
    }
    a.out[(size_t)row * HD + (head0 + g) * D + dd] = __float2bfloat16_rn(oo / ll);
  }
  if (tid == 0) a.counters[row * gridDim.y + blockIdx.y] = 0;
}

template <int D, int G>
static cudaError_t launch_attn_t(const AttnArgs& a, const LaunchCfg& lc) {
  dim3 grid(a.n_splits, a.kvh * (a.group / G), a.M);
  return launch_ex(attn_decode_kernel<D, G>, grid, dim3(AT_THREADS), 0, lc, a);
}

cudaError_t launch_attn_gqa(const AttnArgs& a, int gc, const LaunchCfg& lc);  // attn_gqa.cu

cudaError_t launch_attn_decode(const AttnArgs& a, const LaunchCfg& lc) {
  const int gc = (a.group % 8 == 0) ? 8 : (a.group % 4 == 0) ? 4 : (a.group % 2 == 0) ? 2 : 1;
  if (gc >= 4) return launch_attn_gqa(a, gc, lc);  // grouped-query models: K/V staged once in smem, warp per q head
  if (a.head_dim == 128) {
    switch (gc) {
      case 1: return launch_attn_t<128, 1>(a, lc);
      case 2: return launch_attn_t<128, 2>(a, lc);
      case 4: return launch_attn_t<128, 4>(a, lc);
      case 8: return launch_attn_t<128, 8>(a, lc);
    }
  } else if (a.head_dim == 64) {
    switch (gc) {
      case 1: return launch_attn_t<64, 1>(a, lc);
      case 2: return launch_attn_t<64, 2>(a, lc);
      case 4: return launch_attn_t<64, 4>(a, lc);
      case 8: return launch_attn_t<64, 8>(a, lc);
    }
  }
  return cudaErrorInvalidValue;
}

// =====================================================================================================================
// embedding gather, greedy argmax
// =====================================================================================================================
__global__ void __launch_bounds__(128) embed_kernel(const bf16* __restrict__ embed, const int* __restrict__ row_tok,
                                                    bf16* __restrict__ h, int hidden, int* step_counter, int* fwd_counter, int* push_counter) {
  pdl_wait();
  pdl_launch_dependents();
  const int m = blockIdx.x;
  if (m == 0 && threadIdx.x == 0) {
    if (step_counter) *step_counter += 1;
    if (fwd_counter) *fwd_counter += 1;
    if (push_counter) *push_counter += 1;
  }
  const bf16* src = embed + (size_t)row_tok[m] * hidden;
  bf16* dst = h + (size_t)m * hidden;
  for (int k = threadIdx.x * 8; k < hidden; k += 128 * 8)
    *reinterpret_cast<uint4*>(dst + k) = *reinterpret_cast<const uint4*>(src + k);
}

cudaError_t launch_embed(const bf16* embed, const int* row_tok, bf16* h, int M, int hidden, int* step_counter,
                         int* fwd_counter, int* push_counter, const LaunchCfg& lc) {
  return launch_ex(embed_kernel, dim3(M), dim3(128), 0, lc, embed, row_tok, h, hidden, step_counter, fwd_counter, push_counter);
}

__global__ void __launch_bounds__(1024) argmax_kernel(const float* __restrict__ logits, int V, int n_rows,
                                                      int* __restrict__ tok_out, int* __restrict__ hist,
                                                      const int* __restrict__ step, int* __restrict__ pos_inc) {
  __shared__ float sv[32];
  __shared__ int si[32];
  pdl_wait();
  pdl_launch_dependents();
  const int r = blockIdx.x;
  const float* lg = logits + (size_t)r * V;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int i = threadIdx.x; i < V; i += 1024) {
    const float v = lg[i];
    if (v > best || (v == best && i < bi)) {
      best = v;
      bi = i;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) {
      best = ov;
      bi = oi;
    }
  }
  if ((threadIdx.x & 31) == 0) {
    sv[threadIdx.x >> 5] = best;
    si[threadIdx.x >> 5] = bi;
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    best = sv[threadIdx.x];
    bi = si[threadIdx.x];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) {
        best = ov;
        bi = oi;
      }
    }
    if (threadIdx.x == 0) {
      tok_out[r] = bi;
      if (hist) hist[(size_t)(*step) * n_rows + r] = bi;
      if (pos_inc) pos_inc[r] += 1;
    }
  }
}

cudaError_t launch_argmax(const float* logits, int V, int n_rows, int* tok_out, int* hist, const int* step,
                          int* pos_inc, const LaunchCfg& lc) {
  return launch_ex(argmax_kernel, dim3(n_rows), dim3(1024), 0, lc, logits, V, n_rows, tok_out, hist, step, pos_inc);
}

// =====================================================================================================================
// load-time kernels: row gather + dtype convert, synthetic weights
// =====================================================================================================================
template <typename T>
__device__ __forceinline__ float to_f32(T v);
template <>
__device__ __forceinline__ float to_f32<bf16>(bf16 v) { return __bfloat162float(v); }
template <>
__device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }
template <>
__device__ __forceinline__ float to_f32<float>(float v) { return v; }

template <typename T>
__global__ void gather_rows_kernel(bf16* __restrict__ dst, int64_t dst_ld, const T* __restrict__ src, int64_t src_ld,
                                   const int* __restrict__ row_idx, int rows, int col0, int cols) {
  const int r = blockIdx.y;
  const int64_t sr = row_idx ? row_idx[r] : r;
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < cols; c += gridDim.x * blockDim.x)
    dst[(size_t)r * dst_ld + c] = __float2bfloat16_rn(to_f32<T>(src[sr * src_ld + col0 + c]));
}

cudaError_t launch_gather_rows(bf16* dst, int64_t dst_ld, const void* src, int src_dtype, int64_t src_ld,
                               const int* row_idx, int rows, int col0, int cols, cudaStream_t s) {
  if (rows == 0 || cols == 0) return cudaSuccess;
  dim3 grid((cols + 255) / 256 > 64 ? 64 : (cols + 255) / 256, rows);
  if (src_dtype == 0)
    gather_rows_kernel<bf16><<<grid, 256, 0, s>>>(dst, dst_ld, (const bf16*)src, src_ld, row_idx, rows, col0, cols);
  else if (src_dtype == 1)
    gather_rows_kernel<__half><<<grid, 256, 0, s>>>(dst, dst_ld, (const __half*)src, src_ld, row_idx, rows, col0, cols);
  else if (src_dtype == 2)
    gather_rows_kernel<float><<<grid, 256, 0, s>>>(dst, dst_ld, (const float*)src, src_ld, row_idx, rows, col0, cols);
  else
    return cudaErrorInvalidValue;
  return cudaGetLastError();
}

// twin of oracle/synth.py::synth_f32 + f32_to_bf16_bits (bit-exact; no FMA contraction)
__host__ __device__ inline uint16_t synth_value(uint64_t seed, uint32_t tid, uint64_t idx, float amp, float base) {
  uint64_t z = idx + (uint64_t)tid * 0x9E3779B97F4A7C15ull + seed * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z = z ^ (z >> 31);
  const float u = ((float)(uint32_t)(z >> 41) - 4194304.0f + 0.5f) * 2.384185791015625e-07f;  // 2^-22
#ifdef __CUDA_ARCH__
  const float v = __fadd_rn(base, __fmul_rn(u, amp));
  return __bfloat16_as_ushort(__float2bfloat16_rn(v));
#else
  volatile float prod = u * amp;
  volatile float v = base + prod;
  uint32_t b;
  float vv = v;
  memcpy(&b, &vv, 4);
  const uint32_t rnd = ((b >> 16) & 1u) + 0x7FFFu;
  return (uint16_t)((b + rnd) >> 16);
#endif
}

__global__ void synth_fill_kernel(bf16* __restrict__ dst, int64_t dst_ld, const int* __restrict__ row_idx, int rows, int col0, int cols,
                                  int64_t full_cols, uint64_t seed, uint32_t tid, float amp, float base) {
  const int r = blockIdx.y;
  const int64_t lr = row_idx ? row_idx[r] : r;
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < cols; c += gridDim.x * blockDim.x)
    dst[(size_t)r * dst_ld + c] = __ushort_as_bfloat16(synth_value(seed, tid, (uint64_t)(lr * full_cols + col0 + c), amp, base));
}

cudaError_t launch_synth_fill(bf16* dst, int64_t dst_ld, const int* row_idx, int rows, int col0, int cols, int64_t full_cols,
                              uint64_t seed, uint32_t tid, float amp, float base, cudaStream_t s) {
  if (rows == 0 || cols == 0) return cudaSuccess;
  dim3 grid((cols + 255) / 256 > 64 ? 64 : (cols + 255) / 256, rows);
  synth_fill_kernel<<<grid, 256, 0, s>>>(dst, dst_ld, row_idx, rows, col0, cols, full_cols, seed, tid, amp, base);
  return cudaGetLastError();
}

void synth_fill_host(uint64_t seed, uint32_t tid, int64_t start, int64_t n, float amp, float base, uint16_t* dst) {
  for (int64_t i = 0; i < n; ++i) dst[i] = synth_value(seed, tid, (uint64_t)(start + i), amp, base);
}

__global__ void bf16_to_f32_kernel(const bf16* __restrict__ src, float* __restrict__ dst, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    dst[i] = __bfloat162float(src[i]);
}
cudaError_t launch_bf16_to_f32(const bf16* src, float* dst, int64_t n, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  bf16_to_f32_kernel<<<(int)((n + 255) / 256 > 4096 ? 4096 : (n + 255) / 256), 256, 0, s>>>(src, dst, n);
  return cudaGetLastError();
}

// =====================================================================================================================
// tensor-parallel one-shot allreduce + residual: h = bf16(bf16(sum_r partial_r) + h)
// Every rank pushes a flag to every peer (release, system scope), polls its own flags (acquire), then reads the peers'
// fp32 partials straight over NVLink (peer-mapped pointers) and sums them in rank order, so all ranks produce the
// same bits.  Partials are double-buffered by allreduce parity: a buffer is rewritten two allreduces later, after a
// barrier every peer passed only once it had finished reading (program order), so no second barrier is needed.
// HF semantics: o_proj/down_proj output is bf16(sum over the full K) then "+ residual" in bf16
// (HF:models/llama/modeling_llama.py:325,331); the fp32 cross-rank sum is the same sum in a different order.
// =====================================================================================================================
SSB_DEVINL void st_release_sys(uint32_t* p, uint32_t v) { asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
SSB_DEVINL uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
SSB_DEVINL float4 ld_relaxed_sys_f4(const float* p) {
  float4 v;
  asm volatile("ld.relaxed.sys.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}

constexpr int TP_MAX = 8;
constexpr int TP_THREADS = 256;

SSB_DEVINL uint32_t ld_relaxed_sys_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__global__ void __launch_bounds__(TP_THREADS) tp_allreduce_resid_kernel(const TpArgs a) {
  pdl_wait();  // this rank's partials (previous kernel) are complete and visible
  pdl_launch_dependents();
  const uint32_t epoch = (uint32_t)(*a.tp_step) * (uint32_t)a.n_per_step + (uint32_t)a.seq_in_step + 1u;
  const int parity = a.seq_in_step & 1;
  const int total4 = a.M * a.hidden / 4;
  const size_t poff = (size_t)parity * a.parity_stride;
  const bool push = a.variant & 4;
  if (push) {
    // push model: copy this rank's partial into slot [parity][rank] of every peer (posted stores), then flag.
    // slots live in the upper part of the partial buffers: (8 + parity*8 + src) * M * hidden  (M <= 4)
    const size_t slot = (size_t)(8 + parity * 8 + a.rank) * a.M * a.hidden;
    if (blockIdx.x == 0) {
      for (int i = threadIdx.x; i < total4; i += TP_THREADS) {
        const float4 v = reinterpret_cast<const float4*>(a.peer_partials[a.rank] + poff)[i];
        for (int r = 0; r < a.size; ++r) reinterpret_cast<float4*>(a.peer_partials[r] + slot)[i] = v;
      }
      __syncthreads();
    }
  }
  if (blockIdx.x == 0 && threadIdx.x < a.size && threadIdx.x != a.rank) {
    if (!(a.variant & 1) || push) __threadfence_system();
    st_release_sys(a.peer_flags[threadIdx.x] + a.rank, epoch);  // "rank's partials for `epoch` are ready"
  }
  if (threadIdx.x < a.size && threadIdx.x != a.rank) {
    const uint32_t* f = a.peer_flags[a.rank] + threadIdx.x;
    SpinGuard sg;
    if (a.variant & 2) {
      while ((int32_t)(ld_relaxed_sys_u32(f) - epoch) < 0) sg.poll();
      __threadfence_system();
    } else {
      while ((int32_t)(ld_acquire_sys(f) - epoch) < 0) sg.poll();
    }
  }
  __syncthreads();
  for (int i = blockIdx.x * TP_THREADS + threadIdx.x; i < total4; i += gridDim.x * TP_THREADS) {
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int r = 0; r < TP_MAX; ++r) {
      if (r < a.size) {
        float4 v;
        if (push)
          v = __ldcg(reinterpret_cast<const float4*>(a.peer_partials[a.rank] + (size_t)(8 + parity * 8 + r) * a.M * a.hidden) + i);
        else
          v = ld_relaxed_sys_f4(a.peer_partials[r] + poff + (size_t)i * 4);
        s.x += v.x;
        s.y += v.y;
        s.z += v.z;
        s.w += v.w;
      }
    }
    const uint2 rv = *reinterpret_cast<const uint2*>(a.resid + (size_t)i * 4);
    uint2 o;
    o.x = pack_bf16(bf16r(s.x) + bf_lo(rv.x), bf16r(s.y) + bf_hi(rv.x));
    o.y = pack_bf16(bf16r(s.z) + bf_lo(rv.y), bf16r(s.w) + bf_hi(rv.y));
    *reinterpret_cast<uint2*>(a.out + (size_t)i * 4) = o;
  }
}

__global__ void __launch_bounds__(TP_THREADS) tp_reduce_push_kernel(const TpPushArgs a) {
  // no griddepcontrol.wait on purpose: the data dependency is carried by the arrival counters (every producing CTA of
  // every rank, including this one, counts itself in after its pushes), so this kernel may start while the GEMV runs
  pdl_launch_dependents();
  // arrival counters accumulate: allreduces completed before this one = (push forwards before this one) * n_per_step
  // + seq_in_step (the forward counter was already incremented for the current forward, hence the -1)
  const unsigned long long target =
      ((unsigned long long)((unsigned)(*a.tp_step) - 1u) * (unsigned)a.n_per_step + (unsigned)a.seq_in_step + 1ull) * a.arrivals_per_epoch;
  if (threadIdx.x < a.size) {
    const unsigned long long* f = a.flags + threadIdx.x;
    unsigned long long v;
    SpinGuard sg;
    do {
      sg.poll();
      asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(f) : "memory");
    } while (v < target);
  }
  __syncthreads();
  const int parity = a.seq_in_step & 1;
  const float* base = a.recv + (long long)parity * a.parity_stride;
  const int total4 = a.M * a.hidden / 4;
  for (int i = blockIdx.x * TP_THREADS + threadIdx.x; i < total4; i += gridDim.x * TP_THREADS) {
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int r = 0; r < TP_MAX; ++r) {
      if (r < a.size) {
        const float4 v = __ldcg(reinterpret_cast<const float4*>(base + (long long)r * a.src_stride) + i);
        s.x += v.x;
        s.y += v.y;
        s.z += v.z;
        s.w += v.w;
      }
    }
    const uint2 rv = __ldcg(reinterpret_cast<const uint2*>(a.resid) + i);
    uint2 o;
    o.x = pack_bf16(bf16r(s.x) + bf_lo(rv.x), bf16r(s.y) + bf_hi(rv.x));
    o.y = pack_bf16(bf16r(s.z) + bf_lo(rv.y), bf16r(s.w) + bf_hi(rv.y));
    reinterpret_cast<uint2*>(a.out)[i] = o;
  }
}

// LL push allreduce for decode-sized forwards of the multi-kernel path (Falcon, "use_mega": 0, "tp_mega": 0): thread =
// one (row, pair).  It reads its fp32 partial pair (this rank's projection output), stores {v0, epoch, v1, epoch} into slot
// [parity][rank][row][pair] of EVERY rank (own included) with one 16-byte store each, then polls its own slots of all source
// ranks until both epoch halves match, sums in rank order (bit-identical on every rank), adds the residual.  No flag, no
// fence, no remote read: one NVLink one-way latency.  Slot reuse: parity double-buffering + stream order (a rank launches
// allreduce k+2 after its k+1 completed, which needed every peer's k+1 pushes, issued after that peer finished reading k).
SSB_DEVINL void st_relaxed_sys_v4(uint4* p, const uint4& v) {
  asm volatile("st.relaxed.sys.global.v4.b32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
SSB_DEVINL uint4 ld_relaxed_sys_v4(const uint4* p) {
  uint4 v;
  asm volatile("ld.relaxed.sys.global.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__global__ void __launch_bounds__(TP_THREADS) tp_allreduce_ll_kernel(const TpArgs a, const TpLlArgs l) {
  pdl_wait();  // this rank's partials (previous kernel) are complete and visible
  pdl_launch_dependents();
  const uint32_t epoch = (uint32_t)(*a.tp_step) * (uint32_t)a.n_per_step + (uint32_t)a.seq_in_step + 1u;
  const int parity = a.seq_in_step & 1;
  const int P = a.hidden >> 1;
  const int total = a.M * P;
  const float* mine = a.peer_partials[a.rank] + (size_t)parity * a.parity_stride;
  const size_t base = (size_t)parity * (size_t)l.parity_stride;
  SpinGuard sg;
  for (int i = blockIdx.x * TP_THREADS + threadIdx.x; i < total; i += gridDim.x * TP_THREADS) {
    const int m = i / P, p = i - m * P;
    const float2 v = *reinterpret_cast<const float2*>(mine + (size_t)m * a.hidden + 2 * p);
    const uint4 w = make_uint4(__float_as_uint(v.x), epoch, __float_as_uint(v.y), epoch);
    const size_t o = base + (size_t)a.rank * (size_t)l.src_stride + (size_t)m * P + p;
#pragma unroll
    for (int r = 0; r < TP_MAX; ++r)
      if (r < a.size) st_relaxed_sys_v4(l.peer_ll[r] + o, w);
    float2 s = make_float2(0.f, 0.f);
#pragma unroll
    for (int r = 0; r < TP_MAX; ++r) {
      if (r < a.size) {
        const uint4* slot = l.peer_ll[a.rank] + base + (size_t)r * (size_t)l.src_stride + (size_t)m * P + p;
        uint4 x = ld_relaxed_sys_v4(slot);
        while (x.y != epoch || x.w != epoch) {
          sg.poll();
          x = ld_relaxed_sys_v4(slot);
        }
        s.x += __uint_as_float(x.x);
        s.y += __uint_as_float(x.z);
      }
    }
    const size_t ho = (size_t)m * a.hidden + 2 * (size_t)p;
    const uint32_t rv = *reinterpret_cast<const uint32_t*>(a.resid + ho);
    *reinterpret_cast<uint32_t*>(a.out + ho) = pack_bf16(bf16r(s.x) + bf_lo(rv), bf16r(s.y) + bf_hi(rv));
  }
}

cudaError_t launch_tp_allreduce_ll(const TpArgs& a, const TpLlArgs& l, const LaunchCfg& lc) {
  if (a.size > TP_MAX || (a.hidden & 1) || a.M > 4 || !l.peer_ll) return cudaErrorInvalidValue;
  const int total = a.M * (a.hidden >> 1);
  int grid = (total + TP_THREADS - 1) / TP_THREADS;  // every thread spins: all CTAs must be co-resident (<= 64 CTAs of 256 threads)
  grid = grid < 1 ? 1 : (grid > 64 ? 64 : grid);
  return launch_ex(tp_allreduce_ll_kernel, dim3(grid), dim3(TP_THREADS), 0, lc, a, l);
}

cudaError_t launch_tp_reduce_push(const TpPushArgs& a, const LaunchCfg& lc) {
  if (a.size > TP_MAX || (a.hidden & 3)) return cudaErrorInvalidValue;
  const int total4 = a.M * a.hidden / 4;
  int grid = (total4 + TP_THREADS - 1) / TP_THREADS;
  grid = grid < 1 ? 1 : (grid > 32 ? 32 : grid);
  return launch_ex(tp_reduce_push_kernel, dim3(grid), dim3(TP_THREADS), 0, lc, a);
}

cudaError_t launch_tp_allreduce_resid(const TpArgs& a, const LaunchCfg& lc) {
  if (a.size > TP_MAX || (a.hidden & 3)) return cudaErrorInvalidValue;
  const int total4 = a.M * a.hidden / 4;
  int grid = (total4 + TP_THREADS * 2 - 1) / (TP_THREADS * 2);
  grid = grid < 1 ? 1 : (grid > 64 ? 64 : grid);
  return launch_ex(tp_allreduce_resid_kernel, dim3(grid), dim3(TP_THREADS), 0, lc, a);
}
