// mega.cu — the whole small-batch decode step as ONE persistent kernel (one CTA per SM).
//
// Why: at batch <= 4 every projection is a GEMV whose weights stream from HBM exactly once; with one kernel per
// projection the HBM stream stops at every kernel boundary (drain + launch + refill, 5 kernels x L layers).  Here a producer warp per SM streams the weights of ALL phases of the step back to back
// through one mbarrier ring (cp.async.bulk, up to 6 x 32 KiB in flight per SM) and never waits for a phase boundary;
// the 8 consumer warps follow it through the phases
//     embed | per layer: RMSNorm+QKV+RoPE+KV-append | paged attention | O+residual | RMSNorm+gate/up+SwiGLU |
//     down+residual | final RMSNorm + lm_head | greedy pick
// separated by grid-wide barriers (atomic counter in L2).  While consumers sit in a barrier or in the attention phase
// the producer keeps the ring full, so HBM stays busy.  Math and rounding points are identical to proj_rows_kernel /
// attn_decode_kernel (HF:models/llama/modeling_llama.py:62-67,138-221,292-332; HF:generation/utils.py:2762,2793).
#include "common.cuh"
#include "epilogue.cuh"
#include "gemv_core.cuh"
#include "kernels.h"
#include "mega.h"

constexpr int MG_CW = 8;                      // consumer warps
constexpr int MG_PW = 4;                      // producer warps (one warp issues ~1 bulk copy / 70 cycles: see kernels.cu)
constexpr int MG_THREADS = (MG_CW + MG_PW) * 32;
constexpr int MG_ROWS = 2 * MG_CW;
constexpr int MG_KC = 1024;
// The consumers multiply on the tensor pipe (mma.sync m16n8k16, the batch rows as the N = 8 columns), even at batch 1.
// One ldmatrix.x4 + one HMMA retire a 16 x 16 weight tile (512 B) where an unpack + FFMA loop on the CUDA cores needs
// ~25 instructions: such consumers barely outrun an SM's HBM share, so a stall is never caught up, and at 4 rows they are
// the bottleneck outright.  Stage rows are padded to GEMV_RS = 1032 elements so that the eight rows of an 8 x 8 ldmatrix
// tile fall into different bank groups (gemv_core.cuh).
constexpr int MG_STAGE_ELEMS = MG_ROWS * GEMV_RS;      // 32 KiB of bf16 + 256 B of padding
constexpr int MG_RED_FLOATS = 2 * MG_CW * 16 * 4;      // cross-warp reduction of the K slices, double-buffered by pass

struct Ring {
  int stage;
  uint32_t phase;
};

// ---------------------------------------------------------------- distribution of a projection's rows over the CTAs
// The unit of work is one PASS: up to MG_CW row pairs (one ring stage of rows) x all of K, what the consumers accumulate
// before their cross-warp reduction.
//
// Single GPU: passes are claimed at run time.  A fixed per-CTA share makes every weight phase end when the slowest SM has
// streamed its share (SMs differ in HBM rate by a few percent, and the 6-stage ring absorbs only ~8 us of that), while the
// fast SMs' producers stall on a full ring.  Here the producer claims the next pass with an atomicAdd on the counter of the
// matrix (MegaArgs::grid_bar + MEGA_CLAIM_OFF + 4 * layer + {0 wqkv, 1 wo, 2 wgu, 3 wdown}; 4 * n_layers = lm_head) once a
// ring stage is free, and tells its consumers which pass the stage starts through s_pass / s_pend[stage].  A claimed index
// past the last pass ends the matrix for this CTA: the producer publishes s_pass = -1 through the `full` barrier with no
// bytes.  A phase still ends up to one pass after its first CTA is done, so the last 2 x MG_TAIL_PAIRS x gridDim.x pairs
// (claim_range) go out in passes of MG_TAIL_PAIRS: half the tail at half the stage fill.  The per-row arithmetic (k-slice order, warp-order sum, epilogue) does not depend on which CTA runs a pass, so results are
// bit-identical to any other distribution.
//
// Tensor parallel: every CTA keeps the fixed range [p0, p1) of part_range.  The row-parallel exchange (tp_reduce_cta,
// tp_reduce_ll) relies on CTA c of every rank owning the same pair range.
SSB_DEVINL void part_range(int P, int& p0, int& p1) {
  p0 = (int)(((long long)blockIdx.x * P) / gridDim.x);
  p1 = (int)(((long long)(blockIdx.x + 1) * P) / gridDim.x);
}
constexpr int MG_TAIL_PAIRS = MG_CW / 2;
// row pairs [ps, pe) of claim c of a matrix of P pairs (ps >= P: none left)
SSB_DEVINL void claim_range(int c, int P, int& ps, int& pe) {
  const int full_pairs = max(0, P - 2 * MG_TAIL_PAIRS * (int)gridDim.x) / MG_CW * MG_CW;
  const int n_full = full_pairs / MG_CW;
  ps = c < n_full ? c * MG_CW : full_pairs + (c - n_full) * MG_TAIL_PAIRS;
  pe = min(P, ps + (c < n_full ? MG_CW : MG_TAIL_PAIRS));
}
constexpr int MG_MAX_STAGES = 8;
__shared__ int s_pass[MG_MAX_STAGES];  // first row pair of the pass that starts at ring stage s, -1 = end of the matrix
__shared__ int s_pend[MG_MAX_STAGES];  // its end
__shared__ int s_claim[2];             // a claim, from the claiming lane to the other producer warps (double-buffered)

SSB_DEVINL uint4 ldcg128(const void* p) { return __ldcg(reinterpret_cast<const uint4*>(p)); }
SSB_DEVINL unsigned ld_acquire_gpu(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

SSB_DEVINL unsigned long long gtimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#define MG_STAMP()                                                                                                  \
  do {                                                                                                              \
    if (a.prof && (blockIdx.x == 0 || a.prof_all) && tid == 0 && n_prof < 1023)                                     \
      a.prof[(a.prof_all ? (size_t)blockIdx.x * 1024 : 0) + n_prof++] = gtimer();                                   \
  } while (0)

// grid-wide barrier among the consumer threads of all CTAs (the producer warp does not take part)
// Arrive with ONE release-reduction instead of fence.sc + atomic, leave through the acquire load alone.  The CTA barrier
// before it makes the other consumer threads' writes visible to thread 0, whose gpu-scope release is cumulative; the
// CTA barrier after the acquire hands the observed writes on to them.  There are 160 barriers per 7B token, so the cost of
// one barrier matters (tools/ubench_gridbar times the flavours).
SSB_DEVINL void grid_sync(unsigned* bar, unsigned& n_done, unsigned n_ctas) {
  named_bar_sync(1, MG_CW * 32);
  ++n_done;
  if (threadIdx.x == 0) {
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(bar) : "memory");
    const unsigned target = n_done * n_ctas;
    while (ld_acquire_gpu(bar) < target) {
    }
  }
  named_bar_sync(1, MG_CW * 32);
}

// ---------------------------------------------------------------- producer: stream this CTA's passes of one matrix
// DYN: passes claimed on `claim` (see part_range above); n_claims counts this CTA's claims over the launch and picks the
// s_claim buffer.  !DYN: the fixed range of part_range.
template <bool DYN>
SSB_DEVINL void produce(const bf16* W, int N, int K, bf16* tiles, uint64_t* full, uint64_t* empty, int n_stages, Ring& r,
                        uint64_t pol, int lane, int pw, [[maybe_unused]] unsigned* claim, [[maybe_unused]] unsigned& n_claims) {
  const int P = N >> 1;
  int p0 = 0, p1 = P;
  if constexpr (!DYN) part_range(P, p0, p1);
  const int nk = (K + MG_KC - 1) / MG_KC;
  for (int ps = p0;; ps += MG_CW) {
    if constexpr (DYN) {
      // claim only once the pass's first stage is free, so that a claimed pass never queues behind this CTA's ring
      mbar_wait(&empty[r.stage], r.phase ^ 1);
      int* slot = s_claim + (n_claims++ & 1);  // rewritten two claims later, after every producer warp has read it
      if (pw == 0 && lane == 0) *slot = (int)atomicAdd(claim, 1u);
      named_bar_sync(2, MG_PW * 32);  // all four producer warps copy rows of the claimed pass
      claim_range(*slot, P, ps, p1);
      if (pw == 0 && lane == 0) {  // published by this lane's arrive on full[stage]
        s_pass[r.stage] = ps < P ? ps : -1;
        s_pend[r.stage] = p1;
      }
      if (ps >= P) {  // matrix exhausted: the end marker completes full[stage] with no bytes
        if (lane == 0) mbar_arrive(&full[r.stage]);
        if (++r.stage == n_stages) {
          r.stage = 0;
          r.phase ^= 1;
        }
        return;
      }
    } else if (ps >= p1) {
      return;
    }
    const int nr = 2 * min(MG_CW, p1 - ps);
    for (int kc = 0; kc < nk; ++kc) {
      const int k0 = kc * MG_KC;
      const int len = min(MG_KC, K - k0);
      mbar_wait(&empty[r.stage], r.phase ^ 1);
      constexpr int RPP = MG_ROWS / MG_PW;
      const int r0 = pw * RPP;
      const int mine = max(0, min(RPP, nr - r0));
      if (lane == 0) mbar_expect_tx(&full[r.stage], (uint32_t)(mine * len * 2));
      __syncwarp();
      if (lane < mine)
        bulk_g2s_hint(tiles + ((size_t)r.stage * MG_ROWS + r0 + lane) * GEMV_RS, W + (size_t)(2 * ps + r0 + lane) * K + k0,
                      (uint32_t)(len * 2), &full[r.stage], pol);
      if (++r.stage == n_stages) {
        r.stage = 0;
        r.phase ^= 1;
      }
    }
  }
}

// ---------------------------------------------------------------- consumers: stage x (optionally RMS-normalised)
template <int BT, int NORM>
SSB_DEVINL void stage_x(const bf16* x, int ldx, int M, int K, const bf16* norm_w, float eps, bf16* xs, float* red, int tid, int warp,
                        int lane) {
#pragma unroll
  for (int b = 0; b < BT; ++b) {
    bf16* xrow = xs + (size_t)b * K;
    if (b >= M) {
      for (int k = tid * 8; k < K; k += MG_CW * 32 * 8) *reinterpret_cast<uint4*>(xrow + k) = make_uint4(0, 0, 0, 0);
      continue;
    }
    const bf16* src = x + (size_t)b * ldx;
    if constexpr (NORM == NORM_RMS) {
      float ss = 0.f;
      for (int k = tid * 8; k < K; k += MG_CW * 32 * 8) {
        const uint4 v = ldcg128(src + k);
        *reinterpret_cast<uint4*>(xrow + k) = v;  // raw copy first, normalised in place below
        const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float lo = bf_lo(u[i]), hi = bf_hi(u[i]);
          ss += lo * lo + hi * hi;
        }
      }
      ss = warp_sum(ss);
      if (lane == 0) red[warp] = ss;
      named_bar_sync(1, MG_CW * 32);
      float tot = 0.f;
#pragma unroll
      for (int w = 0; w < MG_CW; ++w) tot += red[w];
      named_bar_sync(1, MG_CW * 32);
      const float rstd = rsqrtf(tot / (float)K + eps);
      for (int k = tid * 8; k < K; k += MG_CW * 32 * 8) {  // same thread -> same elements as the copy above
        const uint4 v = *reinterpret_cast<const uint4*>(xrow + k);
        const uint4 w = ldg128(norm_w + k);
        const uint32_t u[4] = {v.x, v.y, v.z, v.w};
        const uint32_t wu[4] = {w.x, w.y, w.z, w.w};
        uint32_t o[4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
          o[i] = pack_bf16(bf16r(bf_lo(u[i]) * rstd) * bf_lo(wu[i]), bf16r(bf_hi(u[i]) * rstd) * bf_hi(wu[i]));
        *reinterpret_cast<uint4*>(xrow + k) = make_uint4(o[0], o[1], o[2], o[3]);
      }
    } else {
      for (int k = tid * 8; k < K; k += MG_CW * 32 * 8) *reinterpret_cast<uint4*>(xrow + k) = ldcg128(src + k);
    }
  }
  named_bar_sync(1, MG_CW * 32);
}

// ---------------------------------------------------------------- consumers: one projection (same loop as proj_rows_kernel)
constexpr int EPI_LL = 100;  // mega-only epilogue: "tp_mega": 3 push exchange (see mega.h)
struct LlCtx {
  const MegaArgs* ma;
  uint32_t epoch;
  size_t off;  // parity + source-rank offset (uint4 units) into every receive buffer
};
SSB_DEVINL void st_relaxed_sys_v4(uint4* p, const uint4& v) {
  asm volatile("st.relaxed.sys.global.v4.b32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
SSB_DEVINL uint4 ld_relaxed_sys_v4(const uint4* p) {
  uint4 v;
  asm volatile("ld.relaxed.sys.global.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}

// claimed passes: wait for the stage that starts the next pass and read its first row pair.  At the end marker the stage
// is handed back and false returned.  The wait is repeated by the pass's first chunk, which then returns at once.
SSB_DEVINL bool next_pass(uint64_t* full, uint64_t* empty, int n_stages, Ring& r, int lane, int& ps, int& pe) {
  mbar_wait(&full[r.stage], r.phase);
  ps = s_pass[r.stage];
  pe = s_pend[r.stage];
  if (ps >= 0) return true;
  __syncwarp();  // every lane has read s_pass before the producer may rewrite it
  if (lane == 0) mbar_arrive(&empty[r.stage]);
  if (++r.stage == n_stages) {
    r.stage = 0;
    r.phase ^= 1;
  }
  return false;
}

// One projection on the tensor pipe.  A stage = 16 weight rows x 1024 k; warp w multiplies ALL 16 rows by the k slice
// [128 w, 128 w + 128) of the chunk (8 k-steps of m16n8k16: A = ldmatrix.x4 of the padded stage, B = the staged activations,
// batch row n = column n of the 8), accumulating its slice over the chunks of the pass in one 16 x 8 fp32 fragment.  At the
// end of the pass the 8 slices are summed through shared memory in warp order and warp w runs the epilogue of pair w, lane
// b = batch row b.  k beyond the chunk length contributes nothing: whole k-steps are skipped and the activation fragment is
// zero there (the ring is zero-filled at kernel start, so stale weights are finite).
template <int BT, int EPI, bool DYN>
SSB_DEVINL void consume(const GemvArgs& a, const bf16* tiles, const bf16* xs, uint64_t* full, uint64_t* empty, int n_stages, Ring& r,
                        int warp, int lane, float* red_s, [[maybe_unused]] const LlCtx* ll = nullptr) {
  static_assert(MG_CW == 8 && MG_KC == 1024, "8 k slices of 128");
  const int K = a.K;
  const int P = a.N >> 1;
  int p0 = 0, p1 = P;
  if constexpr (!DYN) part_range(P, p0, p1);
  const int nk = (K + MG_KC - 1) / MG_KC;
  int pass = 0;
  for (int ps = p0;; ps += MG_CW, ++pass) {
    if constexpr (DYN) {
      if (!next_pass(full, empty, n_stages, r, lane, ps, p1)) break;
    } else if (ps >= p1) {
      break;
    }
    const int pair = ps + warp;
    const bool valid = pair < p1;
    float c[4] = {0.f, 0.f, 0.f, 0.f};
    [[maybe_unused]] EpiPre pre = {0u, 0, 0, 0u};
    if constexpr (EPI == EPI_RESID || EPI == EPI_QKV_ROPE) {
      if (valid && lane < BT && lane < a.M) pre = epi_prefetch<EPI>(a, pair, lane);
    }
    for (int kc = 0; kc < nk; ++kc) {
      const int k0 = kc * MG_KC;
      const int len = min(MG_KC, K - k0);
      mbar_wait(&full[r.stage], r.phase);
      mma_chunk<BT>(tiles + (size_t)r.stage * MG_STAGE_ELEMS, xs, K, k0, len, warp, lane, c);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[r.stage]);
      if (++r.stage == n_stages) {
        r.stage = 0;
        r.phase ^= 1;
      }
    }
    // ---- sum the 8 k slices: fragment element (row, col) lives in lane 4*(row % 8) + col/2, register (row/8)*2 + col%2
    mma_store_partial<BT>(red_s + (size_t)(pass & 1) * (MG_CW * 16 * 4) + (size_t)warp * 64, lane, c);
    named_bar_sync(1, MG_CW * 32);
    if (valid && lane < BT && lane < a.M) {
      const float* rb = red_s + (size_t)(pass & 1) * (MG_CW * 16 * 4);
      float v0 = 0.f, v1 = 0.f;
#pragma unroll
      for (int w = 0; w < MG_CW; ++w) {  // fixed order: deterministic
        v0 += rb[w * 64 + (2 * warp) * 4 + lane];
        v1 += rb[w * 64 + (2 * warp + 1) * 4 + lane];
      }
      if constexpr (EPI == EPI_LL) {
        const MegaArgs& ma = *ll->ma;
        const uint4 w = make_uint4(__float_as_uint(v0), ll->epoch, __float_as_uint(v1), ll->epoch);
        const size_t o = ll->off + (size_t)lane * (size_t)(ma.hidden >> 1) + (size_t)pair;
#pragma unroll
        for (int rk = 0; rk < 8; ++rk)
          if (rk < ma.tp_size) st_relaxed_sys_v4(ma.peer_ll[rk] + o, w);  // own slot included: the reduce reads all ranks alike
      } else if constexpr (EPI == EPI_RESID || EPI == EPI_QKV_ROPE) {
        gemv_epilogue_pre<BT, EPI>(a, pair, lane, v0, v1, pre);
      } else {
        gemv_epilogue<BT, EPI>(a, pair, lane, v0, v1);
      }
    }
  }
}

// ---------------------------------------------------------------- consumers: paged attention, one (row, head unit, 16-token
// chunk) per warp; all K/V loads of the chunk are issued before any is consumed; the last-arriving warp of a
// (row, head unit) merges the chunk partials.
template <int D, int G>
SSB_DEVINL void attention_phase(const MegaArgs& a, const bf16* kcache, const bf16* vcache, int warp, int lane) {
  constexpr int LPR = D / 8, RPW = 32 / LPR;
  constexpr int UNR = (G <= 2) ? 8 : 2;
  constexpr int CH = RPW * UNR;  // tokens per unit
  const int HU = a.n_heads / G;  // head units per row
  const int sub = lane / LPR, li = lane % LPR;
  const int HD = a.n_heads * D;
  const int BS = a.block_size;
  const int gw = blockIdx.x * MG_CW + warp, nw = gridDim.x * MG_CW;
  // units are enumerated row-major: (m, hu, chunk); chunk counts differ per row (ragged contexts)
  int base = 0;
  for (int m = 0; m < a.M; ++m) {
    const int ctx = __ldcg(a.row_pos + m) + 1;
    const int n_chunks = (ctx + CH - 1) / CH;
    const int n_units = HU * n_chunks;
    const int slot = a.row_slot[m];
    const int* bt = a.block_table + (size_t)slot * a.bt_stride;
    // first unit index of this row owned by this warp
    int u = ((gw - base) % nw + nw) % nw;
    for (; u < n_units; u += nw) {
      const int hu = u / n_chunks, ck = u - hu * n_chunks;
      const int kvh = (hu * G) / a.group;
      const int t0 = ck * CH;
      float q[G][8];
#pragma unroll
      for (int g = 0; g < G; ++g) {
        const uint4 v = ldcg128(a.q + (size_t)m * HD + (hu * G + g) * D + li * 8);
        const uint32_t uu[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          q[g][2 * i] = bf_lo(uu[i]);
          q[g][2 * i + 1] = bf_hi(uu[i]);
        }
      }
      uint4 kq[UNR], vq[UNR];
      bool tvq[UNR];
#pragma unroll
      for (int x = 0; x < UNR; ++x) {
        const int t = t0 + x * RPW + sub;
        tvq[x] = t < ctx;
        kq[x] = make_uint4(0, 0, 0, 0);
        vq[x] = make_uint4(0, 0, 0, 0);
        if (tvq[x]) {
          const int blk = bt[t / BS];
          const size_t off = (((size_t)blk * a.kvh + kvh) * BS + (t % BS)) * D + li * 8;
          kq[x] = ldcg128(kcache + off);
          vq[x] = ldcg128(vcache + off);
        }
      }
      float mx[G], l[G], acc[G][8];
#pragma unroll
      for (int g = 0; g < G; ++g) {
        mx[g] = -1e30f;
        l[g] = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[g][i] = 0.f;
      }
#pragma unroll
      for (int x = 0; x < UNR; ++x) {
        const uint32_t ku[4] = {kq[x].x, kq[x].y, kq[x].z, kq[x].w};
        const uint32_t vu[4] = {vq[x].x, vq[x].y, vq[x].z, vq[x].w};
        float kf[8], vf[8];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          kf[2 * i] = bf_lo(ku[i]);
          kf[2 * i + 1] = bf_hi(ku[i]);
          vf[2 * i] = bf_lo(vu[i]);
          vf[2 * i + 1] = bf_hi(vu[i]);
        }
#pragma unroll
        for (int g = 0; g < G; ++g) {
          float d = 0.f;
#pragma unroll
          for (int i = 0; i < 8; ++i) d = fmaf(q[g][i], kf[i], d);
#pragma unroll
          for (int o = LPR / 2; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
          if (!tvq[x]) continue;
          const float s = bf16r(bf16r(d) * a.scale);
          const float mn = fmaxf(mx[g], s);
          const float corr = __expf(mx[g] - mn);
          const float p = __expf(s - mn);
          mx[g] = mn;
          l[g] = l[g] * corr + p;
#pragma unroll
          for (int i = 0; i < 8; ++i) acc[g][i] = fmaf(p, vf[i], acc[g][i] * corr);
        }
      }
      // merge the RPW sub-groups of the warp (lanes li + k*LPR hold the same dims of different tokens)
#pragma unroll
      for (int g = 0; g < G; ++g) {
#pragma unroll
        for (int o = LPR; o < 32; o <<= 1) {
          const float om = __shfl_xor_sync(0xffffffffu, mx[g], o);
          const float ol = __shfl_xor_sync(0xffffffffu, l[g], o);
          const float mn = fmaxf(mx[g], om);
          const float wa = __expf(mx[g] - mn), wb = __expf(om - mn);
          l[g] = l[g] * wa + ol * wb;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float oa = __shfl_xor_sync(0xffffffffu, acc[g][i], o);
            acc[g][i] = acc[g][i] * wa + oa * wb;
          }
          mx[g] = mn;
        }
      }
      const size_t pidx = ((size_t)m * HU + hu) * a.max_chunks + ck;
      if (n_chunks == 1) {
        if (sub == 0) {
#pragma unroll
          for (int g = 0; g < G; ++g) {
            const float inv = 1.0f / l[g];
            uint32_t o[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) o[i] = pack_bf16(acc[g][2 * i] * inv, acc[g][2 * i + 1] * inv);
            *reinterpret_cast<uint4*>(a.attn + (size_t)m * HD + (hu * G + g) * D + li * 8) = make_uint4(o[0], o[1], o[2], o[3]);
          }
        }
        continue;
      }
      if (sub == 0) {
#pragma unroll
        for (int g = 0; g < G; ++g) {
          float* po = a.part_o + (pidx * G + g) * D + li * 8;
          *reinterpret_cast<float4*>(po) = make_float4(acc[g][0], acc[g][1], acc[g][2], acc[g][3]);
          *reinterpret_cast<float4*>(po + 4) = make_float4(acc[g][4], acc[g][5], acc[g][6], acc[g][7]);
          if (li == 0) {
            a.part_ml[(pidx * G + g) * 2] = mx[g];
            a.part_ml[(pidx * G + g) * 2 + 1] = l[g];
          }
        }
      }
      __threadfence();
      __syncwarp();
      int last = 0;
      if (lane == 0) last = (atomicAdd(&a.counters[m * HU + hu], 1) == n_chunks - 1);
      last = __shfl_sync(0xffffffffu, last, 0);
      if (!last) continue;
      __threadfence();
      // this warp merges all chunks of (m, hu): lane handles 4 consecutive dims of head g = lane / (D/4) (+ stride)
      const size_t pb = ((size_t)m * HU + hu) * a.max_chunks;
      for (int e = lane * 4; e < G * D; e += 128) {
        const int g = e / D, dd = e % D;
        float M2 = -1e30f;
        for (int c = 0; c < n_chunks; ++c) M2 = fmaxf(M2, __ldcg(&a.part_ml[((pb + c) * G + g) * 2]));
        float L2 = 0.f;
        float4 O = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int c = 0; c < n_chunks; ++c) {
          const float w = __expf(__ldcg(&a.part_ml[((pb + c) * G + g) * 2]) - M2);
          L2 += __ldcg(&a.part_ml[((pb + c) * G + g) * 2 + 1]) * w;
          const float4 o = __ldcg(reinterpret_cast<const float4*>(a.part_o + ((pb + c) * G + g) * D + dd));
          O.x += o.x * w;
          O.y += o.y * w;
          O.z += o.z * w;
          O.w += o.w * w;
        }
        const float inv = 1.0f / L2;
        uint2 o;
        o.x = pack_bf16(O.x * inv, O.y * inv);
        o.y = pack_bf16(O.z * inv, O.w * inv);
        *reinterpret_cast<uint2*>(a.attn + (size_t)m * HD + (hu * G + g) * D + dd) = o;
      }
      if (lane == 0) a.counters[m * HU + hu] = 0;
    }
    base = (base + n_units) % nw;
  }
}

// ---------------------------------------------------------------- consumers: paged attention, CTA-cooperative form for small
// groups (G = 1, 2, 4 query heads per unit; Llama-2-7B / 13B are G = 1).  One (row, head unit, context split) per CTA: the
// 8 consumer warps take consecutive token slices of the split, keep the per-warp online softmax of attention_phase, and
// combine their 8 partial states through shared memory (the activation staging area is free in this phase).  Only ONE
// partial per CTA reaches global memory and a (row, head unit) has at most 8 of them, merged by the last-arriving CTA with
// 128 threads in parallel.  The per-warp form above leaves 36 partials per head at ctx 576 for ONE warp to merge serially, a
// tail the barrier behind the attention phase waits for.
template <int D, int G>
SSB_DEVINL void attention_phase_coop(const MegaArgs& a, const bf16* kcache, const bf16* vcache, float* sm, int* sm_flag, int tid, int warp,
                                     int lane) {
  constexpr int LPR = D / 8, RPW = 32 / LPR;
  // load batch of a warp: 20 tokens at G = 1 / D = 128, so that a 512..640-token context cut into 4 splits x 8 warps
  // (18-20 tokens per warp) is ONE batch of loads, i.e. one memory latency
  constexpr int UNR = (G == 1) ? 10 : (G == 2) ? 4 : 2;
  constexpr int TB = RPW * UNR;  // tokens per load batch of a warp
  constexpr int GD = G * D;
  const int HU = a.n_heads / G;
  const int sub = lane / LPR, li = lane % LPR;
  const int HD = a.n_heads * D;
  const int BS = a.block_size;
  const int n_ctas = gridDim.x;
  float* sm_ml = sm;                   // [MG_CW][G][2]
  float* sm_o = sm + MG_CW * G * 2;    // [MG_CW][G*D]
  int want = n_ctas / max(1, a.M * HU);  // context splits per (row, head unit): fill the grid, at most 8 partials to merge
  want = max(1, min(want, min(8, a.max_chunks)));
  int base = 0;
  for (int m = 0; m < a.M; ++m) {
    const int ctx = __ldcg(a.row_pos + m) + 1;
    int slen = (ctx + want - 1) / want;                        // tokens per split ...
    slen = ((slen + MG_CW * RPW - 1) / (MG_CW * RPW)) * (MG_CW * RPW);  // ... a whole number of RPW-token groups per warp
    const int n_active = (ctx + slen - 1) / slen;
    const int wlen = slen / MG_CW;                             // tokens per warp
    const int n_units = HU * n_active;
    const int slot = a.row_slot[m];
    const int* bt = a.block_table + (size_t)slot * a.bt_stride;
    for (int u = (((int)blockIdx.x - base) % n_ctas + n_ctas) % n_ctas; u < n_units; u += n_ctas) {
      const int hu = u / n_active, sp = u - hu * n_active;
      const int kvh = (hu * G) / a.group;
      const int t_begin = sp * slen + warp * wlen;
      const int t_end = min(ctx, t_begin + wlen);
      float q[G][8];
#pragma unroll
      for (int g = 0; g < G; ++g) {
        const uint4 v = ldcg128(a.q + (size_t)m * HD + (hu * G + g) * D + li * 8);
        const uint32_t uu[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          q[g][2 * i] = bf_lo(uu[i]);
          q[g][2 * i + 1] = bf_hi(uu[i]);
        }
      }
      float mx[G], l[G], acc[G][8];
#pragma unroll
      for (int g = 0; g < G; ++g) {
        mx[g] = -1e30f;
        l[g] = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[g][i] = 0.f;
      }
      for (int tb = t_begin; tb < t_end; tb += TB) {  // warp-uniform bounds
        uint4 kq[UNR], vq[UNR];
        bool tvq[UNR];
#pragma unroll
        for (int x = 0; x < UNR; ++x) {
          const int t = tb + x * RPW + sub;
          tvq[x] = t < t_end;
          kq[x] = make_uint4(0, 0, 0, 0);
          vq[x] = make_uint4(0, 0, 0, 0);
          if (tvq[x]) {
            const int blk = bt[t / BS];
            const size_t off = (((size_t)blk * a.kvh + kvh) * BS + (t % BS)) * D + li * 8;
            kq[x] = ldcg128(kcache + off);
            vq[x] = ldcg128(vcache + off);
          }
        }
#pragma unroll
        for (int x = 0; x < UNR; ++x) {
          if (tb + x * RPW >= t_end) break;  // warp-uniform
          const uint32_t ku[4] = {kq[x].x, kq[x].y, kq[x].z, kq[x].w};
          const uint32_t vu[4] = {vq[x].x, vq[x].y, vq[x].z, vq[x].w};
          float kf[8], vf[8];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            kf[2 * i] = bf_lo(ku[i]);
            kf[2 * i + 1] = bf_hi(ku[i]);
            vf[2 * i] = bf_lo(vu[i]);
            vf[2 * i + 1] = bf_hi(vu[i]);
          }
#pragma unroll
          for (int g = 0; g < G; ++g) {
            float d = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) d = fmaf(q[g][i], kf[i], d);
#pragma unroll
            for (int o = LPR / 2; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
            if (!tvq[x]) continue;
            const float sc = bf16r(bf16r(d) * a.scale);
            const float mn = fmaxf(mx[g], sc);
            const float corr = __expf(mx[g] - mn);
            const float pw = __expf(sc - mn);
            mx[g] = mn;
            l[g] = l[g] * corr + pw;
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[g][i] = fmaf(pw, vf[i], acc[g][i] * corr);
          }
        }
      }
      // merge the RPW token sub-groups of the warp (lanes li + k*LPR hold the same dims of different tokens)
#pragma unroll
      for (int g = 0; g < G; ++g) {
#pragma unroll
        for (int o = LPR; o < 32; o <<= 1) {
          const float om = __shfl_xor_sync(0xffffffffu, mx[g], o);
          const float ol = __shfl_xor_sync(0xffffffffu, l[g], o);
          const float mn = fmaxf(mx[g], om);
          const float wa = __expf(mx[g] - mn), wb = __expf(om - mn);
          l[g] = l[g] * wa + ol * wb;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float oa = __shfl_xor_sync(0xffffffffu, acc[g][i], o);
            acc[g][i] = acc[g][i] * wa + oa * wb;
          }
          mx[g] = mn;
        }
      }
      // ---- combine the 8 warps through shared memory (a warp whose slice is empty contributes m = -1e30, l = 0)
      named_bar_sync(1, MG_CW * 32);  // previous unit's readers are done with sm_*
      if (sub == 0) {
#pragma unroll
        for (int g = 0; g < G; ++g) {
          float* po = sm_o + (size_t)warp * GD + g * D + li * 8;
          *reinterpret_cast<float4*>(po) = make_float4(acc[g][0], acc[g][1], acc[g][2], acc[g][3]);
          *reinterpret_cast<float4*>(po + 4) = make_float4(acc[g][4], acc[g][5], acc[g][6], acc[g][7]);
          if (li == 0) {
            sm_ml[(warp * G + g) * 2] = mx[g];
            sm_ml[(warp * G + g) * 2 + 1] = l[g];
          }
        }
      }
      named_bar_sync(1, MG_CW * 32);
      const size_t pidx = ((size_t)m * HU + hu) * a.max_chunks + sp;
      for (int e = tid; e < GD; e += MG_CW * 32) {  // thread e owns output dim e of the unit
        const int g = e / D;
        float M2 = -1e30f;
#pragma unroll
        for (int w = 0; w < MG_CW; ++w) M2 = fmaxf(M2, sm_ml[(w * G + g) * 2]);
        float L2 = 0.f, O = 0.f;
#pragma unroll
        for (int w = 0; w < MG_CW; ++w) {
          const float wt = __expf(sm_ml[(w * G + g) * 2] - M2);
          L2 += sm_ml[(w * G + g) * 2 + 1] * wt;
          O += sm_o[(size_t)w * GD + e] * wt;
        }
        if (n_active == 1) {
          a.attn[(size_t)m * HD + (size_t)hu * GD + e] = __float2bfloat16_rn(O / L2);
        } else {
          a.part_o[pidx * GD + e] = O;
          if (e % D == 0) {
            a.part_ml[(pidx * G + g) * 2] = M2;
            a.part_ml[(pidx * G + g) * 2 + 1] = L2;
          }
        }
      }
      if (n_active == 1) continue;
      __threadfence();
      named_bar_sync(1, MG_CW * 32);
      if (tid == 0) *sm_flag = (atomicAdd(&a.counters[m * HU + hu], 1) == n_active - 1);
      named_bar_sync(1, MG_CW * 32);
      if (!*sm_flag) continue;
      __threadfence();
      const size_t pb = ((size_t)m * HU + hu) * a.max_chunks;
      for (int e = tid; e < GD; e += MG_CW * 32) {
        const int g = e / D;
        float M2 = -1e30f;
        for (int c = 0; c < n_active; ++c) M2 = fmaxf(M2, __ldcg(&a.part_ml[((pb + c) * G + g) * 2]));
        float L2 = 0.f, O = 0.f;
        for (int c = 0; c < n_active; ++c) {
          const float wt = __expf(__ldcg(&a.part_ml[((pb + c) * G + g) * 2]) - M2);
          L2 += __ldcg(&a.part_ml[((pb + c) * G + g) * 2 + 1]) * wt;
          O += __ldcg(&a.part_o[(pb + c) * GD + e]) * wt;
        }
        a.attn[(size_t)m * HD + (size_t)hu * GD + e] = __float2bfloat16_rn(O / L2);
      }
      if (tid == 0) a.counters[m * HU + hu] = 0;
    }
    base = (base + n_units) % n_ctas;
  }
}

// ---------------------------------------------------------------- consumers: paged attention for GQA groups of 8 (Llama-2-70B
// 64/8, Falcon-40B 128/8): one (row, KV head, context split) per CTA.  The K/V rows of the split are staged ONCE in shared
// memory (the activation staging area is free during this phase) and consumer warp g computes query head g against the
// tile — the scheme of attn_gqa_kernel (attn_gqa.cu).  The per-warp variant above gives a G = 8 unit only 4 tokens
// (register budget), i.e. 144 context chunks at ctx 576 whose partials ONE warp then merges serially.  Here the context is cut into about gridDim.x / (rows * KV heads) splits (18 of 32 tokens
// at 70B), so the last-arriving CTA merges 18 partials with one warp per head.
constexpr int MG_ATT_TILE = 32;  // tokens staged per pass: 2 x 32 x D bf16 = 16 KiB at D = 128
template <int D>
SSB_DEVINL void attention_phase_cta(const MegaArgs& a, const bf16* kcache, const bf16* vcache, bf16* tile, int* sm_flag, int tid, int warp,
                                    int lane) {
  constexpr int G = 8, LPR = D / 8, RPW = 32 / LPR, T = MG_ATT_TILE;
  static_assert(MG_CW == G, "one consumer warp per query head of the group");
  bf16(*sK)[D] = reinterpret_cast<bf16(*)[D]>(tile);
  bf16(*sV)[D] = reinterpret_cast<bf16(*)[D]>(tile + (size_t)T * D);
  const int HU = a.n_heads / G;
  const int sub = lane / LPR, li = lane % LPR;
  const int HD = a.n_heads * D;
  const int BS = a.block_size;
  const int n_ctas = gridDim.x;
  int want = n_ctas / max(1, a.M * HU);  // context splits per (row, KV head) so that the units about fill the grid
  want = max(1, min(want, a.max_chunks));
  int base = 0;
  for (int m = 0; m < a.M; ++m) {
    const int ctx = __ldcg(a.row_pos + m) + 1;
    int chunk = (ctx + want - 1) / want;
    chunk = ((chunk + T - 1) / T) * T;
    const int n_active = (ctx + chunk - 1) / chunk;
    const int n_units = HU * n_active;
    const int slot = a.row_slot[m];
    const int* bt = a.block_table + (size_t)slot * a.bt_stride;
    for (int u = (((int)blockIdx.x - base) % n_ctas + n_ctas) % n_ctas; u < n_units; u += n_ctas) {
      const int hu = u / n_active, sp = u - hu * n_active;
      const int kvh = (hu * G) / a.group;
      const int t_begin = sp * chunk, t_end = min(ctx, t_begin + chunk);
      const bool head_on = warp < G;
      float q[8];
      {
        const uint4 v = ldcg128(a.q + (size_t)m * HD + (hu * G + (head_on ? warp : 0)) * D + li * 8);
        const uint32_t uu[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          q[2 * i] = bf_lo(uu[i]);
          q[2 * i + 1] = bf_hi(uu[i]);
        }
      }
      float mx = -1e30f, l = 0.f, acc[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = 0.f;
      for (int p0 = t_begin; p0 < t_end; p0 += T) {
        const int np = min(T, t_end - p0);
        named_bar_sync(1, MG_CW * 32);  // previous tile (or previous unit / phase) fully consumed
        for (int i = tid; i < np * LPR; i += MG_CW * 32) {
          const int tt = i / LPR, c = i - tt * LPR;
          const int t = p0 + tt;
          const size_t off = (((size_t)bt[t / BS] * a.kvh + kvh) * BS + (t % BS)) * D + c * 8;
          const uint4 kq = ldcg128(kcache + off), vq = ldcg128(vcache + off);
          *reinterpret_cast<uint4*>(&sK[tt][c * 8]) = kq;
          *reinterpret_cast<uint4*>(&sV[tt][c * 8]) = vq;
        }
        named_bar_sync(1, MG_CW * 32);
        if (head_on) {
          for (int tb = 0; tb < np; tb += RPW) {  // warp-uniform trip count (full-mask shuffles below)
            const int tt = tb + sub;
            const bool tv = tt < np;
            uint4 kv = make_uint4(0, 0, 0, 0), vv = make_uint4(0, 0, 0, 0);
            if (tv) {
              kv = *reinterpret_cast<const uint4*>(&sK[tt][li * 8]);
              vv = *reinterpret_cast<const uint4*>(&sV[tt][li * 8]);
            }
            const uint32_t ku[4] = {kv.x, kv.y, kv.z, kv.w};
            const uint32_t vu[4] = {vv.x, vv.y, vv.z, vv.w};
            float d = 0.f;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              d = fmaf(q[2 * i], bf_lo(ku[i]), d);
              d = fmaf(q[2 * i + 1], bf_hi(ku[i]), d);
            }
#pragma unroll
            for (int o = LPR / 2; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
            if (!tv) continue;
            const float sc = bf16r(bf16r(d) * a.scale);
            const float mn = fmaxf(mx, sc);
            const float corr = __expf(mx - mn), pw = __expf(sc - mn);
            mx = mn;
            l = l * corr + pw;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              acc[2 * i] = fmaf(pw, bf_lo(vu[i]), acc[2 * i] * corr);
              acc[2 * i + 1] = fmaf(pw, bf_hi(vu[i]), acc[2 * i + 1] * corr);
            }
          }
        }
      }
      // merge the RPW token sub-groups of the warp
#pragma unroll
      for (int o = LPR; o < 32; o <<= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, mx, o);
        const float ol = __shfl_xor_sync(0xffffffffu, l, o);
        const float mn = fmaxf(mx, om);
        const float wa = __expf(mx - mn), wb = __expf(om - mn);
        l = l * wa + ol * wb;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float oa = __shfl_xor_sync(0xffffffffu, acc[i], o);
          acc[i] = acc[i] * wa + oa * wb;
        }
        mx = mn;
      }
      const size_t pidx = ((size_t)m * HU + hu) * a.max_chunks + sp;
      if (n_active == 1) {
        if (head_on && sub == 0) {
          const float inv = 1.0f / l;
          uint32_t o[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) o[i] = pack_bf16(acc[2 * i] * inv, acc[2 * i + 1] * inv);
          *reinterpret_cast<uint4*>(a.attn + (size_t)m * HD + (hu * G + warp) * D + li * 8) = make_uint4(o[0], o[1], o[2], o[3]);
        }
        continue;
      }
      if (head_on && sub == 0) {
        float* po = a.part_o + (pidx * G + warp) * D + li * 8;
        *reinterpret_cast<float4*>(po) = make_float4(acc[0], acc[1], acc[2], acc[3]);
        *reinterpret_cast<float4*>(po + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
        if (li == 0) {
          a.part_ml[(pidx * G + warp) * 2] = mx;
          a.part_ml[(pidx * G + warp) * 2 + 1] = l;
        }
      }
      __threadfence();
      named_bar_sync(1, MG_CW * 32);
      if (tid == 0) *sm_flag = (atomicAdd(&a.counters[m * HU + hu], 1) == n_active - 1);
      named_bar_sync(1, MG_CW * 32);
      if (!*sm_flag) continue;
      __threadfence();
      if (head_on) {  // warp g merges head g over the splits; a lane owns 4 dims
        const size_t pb = ((size_t)m * HU + hu) * a.max_chunks;
        for (int dd = lane * 4; dd < D; dd += 128) {
          float M2 = -1e30f;
          for (int c = 0; c < n_active; ++c) M2 = fmaxf(M2, __ldcg(&a.part_ml[((pb + c) * G + warp) * 2]));
          float L2 = 0.f;
          float4 O = make_float4(0.f, 0.f, 0.f, 0.f);
          for (int c = 0; c < n_active; ++c) {
            const float w = __expf(__ldcg(&a.part_ml[((pb + c) * G + warp) * 2]) - M2);
            L2 += __ldcg(&a.part_ml[((pb + c) * G + warp) * 2 + 1]) * w;
            const float4 o = __ldcg(reinterpret_cast<const float4*>(a.part_o + ((pb + c) * G + warp) * D + dd));
            O.x += o.x * w;
            O.y += o.y * w;
            O.z += o.z * w;
            O.w += o.w * w;
          }
          const float inv = 1.0f / L2;
          uint2 o;
          o.x = pack_bf16(O.x * inv, O.y * inv);
          o.y = pack_bf16(O.z * inv, O.w * inv);
          *reinterpret_cast<uint2*>(a.attn + (size_t)m * HD + (hu * G + warp) * D + dd) = o;
        }
      }
      if (tid == 0) a.counters[m * HU + hu] = 0;
    }
    base = (base + n_units) % n_ctas;
  }
}

// system-scope accessors for the cross-GPU exchange (same PTX as the allreduce kernel in kernels.cu)
constexpr int TP_MAX = 8;
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

// ---------------------------------------------------------------- consumers: allreduce(sum) + residual under tensor
// parallelism, between two grid barriers (see mega.h).  `seq` = index of this allreduce inside the forward.
SSB_DEVINL void tp_reduce_phase(const MegaArgs& a, int seq, int tid) {
  const uint32_t epoch = (uint32_t)ld_acquire_gpu(reinterpret_cast<const unsigned*>(a.fwd_counter)) * (uint32_t)(2 * a.n_layers) +
                         (uint32_t)seq + 1u;
  const size_t poff = (size_t)(seq & 1) * (size_t)a.parity_stride;
  if (blockIdx.x == 0 && tid < a.tp_size && tid != a.tp_rank) {
    __threadfence_system();  // the partials of ALL local CTAs (observed through the grid barrier) before the flag
    st_release_sys(a.peer_flags[tid] + a.tp_rank, epoch);
  }
  if (tid < a.tp_size && tid != a.tp_rank) {
    const uint32_t* f = a.peer_flags[a.tp_rank] + tid;
    SpinGuard sg;
    while ((int32_t)(ld_acquire_sys(f) - epoch) < 0) sg.poll();
  }
  named_bar_sync(1, MG_CW * 32);
  const int total4 = a.M * a.hidden / 4;
  for (int i = blockIdx.x * (MG_CW * 32) + tid; i < total4; i += gridDim.x * MG_CW * 32) {
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int r = 0; r < TP_MAX; ++r) {  // rank order: every rank computes bit-identical sums
      if (r < a.tp_size) {
        const float4 v = ld_relaxed_sys_f4(a.peer_partials[r] + poff + (size_t)i * 4);
        s.x += v.x;
        s.y += v.y;
        s.z += v.z;
        s.w += v.w;
      }
    }
    const uint2 rv = __ldcg(reinterpret_cast<const uint2*>(a.h) + i);
    uint2 o;
    o.x = pack_bf16(bf16r(s.x) + bf_lo(rv.x), bf16r(s.y) + bf_hi(rv.x));
    o.y = pack_bf16(bf16r(s.z) + bf_lo(rv.y), bf16r(s.w) + bf_hi(rv.y));
    reinterpret_cast<uint2*>(a.h)[i] = o;
  }
}

SSB_DEVINL float2 ld_relaxed_sys_f2(const float* p) {
  float2 v;
  asm volatile("ld.relaxed.sys.global.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(p) : "memory");
  return v;
}

// "tp_mega": 2 (mega.h): exchange between the CTAs with the same index on every rank, called right after the row-parallel
// projection WITHOUT a grid barrier in between.  Buffer reuse: this CTA rewrites its range of the parity buffer two
// allreduces later, after it received the peers' CTA-c flag of the allreduce in between, which they store only after
// their loads of this one have returned (program order + release).
constexpr int MG_CTA_FLAG_STRIDE = 256;
SSB_DEVINL void tp_reduce_cta(const MegaArgs& a, int seq, int tid) {
  const uint32_t epoch = (uint32_t)ld_acquire_gpu(reinterpret_cast<const unsigned*>(a.fwd_counter)) * (uint32_t)(2 * a.n_layers) +
                         (uint32_t)seq + 1u;
  const size_t poff = (size_t)(seq & 1) * (size_t)a.parity_stride;
  named_bar_sync(1, MG_CW * 32);  // every consumer warp of this CTA has stored its partial pairs
  if (tid < a.tp_size && tid != a.tp_rank) {
    __threadfence_system();
    st_release_sys(a.peer_cta_flags[tid] + (size_t)a.tp_rank * MG_CTA_FLAG_STRIDE + blockIdx.x, epoch);
    const uint32_t* f = a.peer_cta_flags[a.tp_rank] + (size_t)tid * MG_CTA_FLAG_STRIDE + blockIdx.x;
    SpinGuard sg;
    while ((int32_t)(ld_acquire_sys(f) - epoch) < 0) sg.poll();
  }
  named_bar_sync(1, MG_CW * 32);
  const int P = a.hidden >> 1;
  const int p0 = (int)(((long long)blockIdx.x * P) / gridDim.x);
  const int p1 = (int)(((long long)(blockIdx.x + 1) * P) / gridDim.x);
  const int np = p1 - p0;
  for (int i = tid; i < a.M * np; i += MG_CW * 32) {
    const int m = i / np, p = p0 + (i - m * np);
    const size_t o = (size_t)m * a.hidden + 2 * (size_t)p;
    float2 s = make_float2(0.f, 0.f);
#pragma unroll
    for (int r = 0; r < TP_MAX; ++r) {  // rank order, own partial included: bit-identical sums on every rank
      if (r < a.tp_size) {
        const float2 v = ld_relaxed_sys_f2(a.peer_partials[r] + poff + o);
        s.x += v.x;
        s.y += v.y;
      }
    }
    const uint32_t rv = __ldcg(reinterpret_cast<const uint32_t*>(a.h + o));
    *reinterpret_cast<uint32_t*>(a.h + o) = pack_bf16(bf16r(s.x) + bf_lo(rv), bf16r(s.y) + bf_hi(rv));
  }
}

// "tp_mega": 3 — wait for the pushed partials of this CTA's pair range (all ranks, own included), sum in rank order, add the
// residual, write h.  Slot reuse: a source rewrites slot (parity, pair) two allreduces later, after it received this CTA's
// push of the allreduce in between, which this CTA issues only after the grid barrier that follows these reads.
SSB_DEVINL void tp_reduce_ll(const MegaArgs& a, int seq, uint32_t epoch, int tid) {
  const int P = a.hidden >> 1;
  int p0, p1;
  part_range(P, p0, p1);  // the pairs this CTA computed and pushed (consume<EPI_LL>); other ranks may cut differently
  const int np = p1 - p0;
  const uint4* base = a.peer_ll[a.tp_rank] + (size_t)(seq & 1) * (size_t)a.ll_parity_stride;
  SpinGuard sg;
  for (int i = tid; i < a.M * np; i += MG_CW * 32) {
    const int m = i / np, p = p0 + (i - m * np);
    float2 s = make_float2(0.f, 0.f);
#pragma unroll
    for (int r = 0; r < TP_MAX; ++r) {
      if (r < a.tp_size) {
        const uint4* slot = base + (size_t)r * (size_t)a.ll_src_stride + (size_t)m * P + p;
        uint4 v = ld_relaxed_sys_v4(slot);
        while (v.y != epoch || v.w != epoch) {
          sg.poll();
          v = ld_relaxed_sys_v4(slot);
        }
        s.x += __uint_as_float(v.x);
        s.y += __uint_as_float(v.z);
      }
    }
    const size_t o = (size_t)m * a.hidden + 2 * (size_t)p;
    const uint32_t rv = __ldcg(reinterpret_cast<const uint32_t*>(a.h + o));
    *reinterpret_cast<uint32_t*>(a.h + o) = pack_bf16(bf16r(s.x) + bf_lo(rv), bf16r(s.y) + bf_hi(rv));
  }
}

template <int BT, int D, int G, bool TP = false>
__global__ void __launch_bounds__(MG_THREADS, 1) decode_mega_kernel(const MegaArgs a) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  bf16* tiles = reinterpret_cast<bf16*>(smem_raw);
  bf16* xs = tiles + (size_t)a.n_stages * MG_STAGE_ELEMS;
  uint64_t* full = reinterpret_cast<uint64_t*>(xs + (size_t)BT * a.k_max);
  uint64_t* empty = full + a.n_stages;
  float* red = reinterpret_cast<float*>(empty + a.n_stages);
  float* red_s = red + 32;  // [2][MG_CW][16][4] k-slice partial sums
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int h = a.hidden;

  for (size_t i = threadIdx.x; i < (size_t)a.n_stages * MG_STAGE_ELEMS / 8; i += MG_THREADS)
    reinterpret_cast<uint4*>(tiles)[i] = make_uint4(0, 0, 0, 0);  // k tails multiply stale ring contents by zero: keep them finite
  constexpr bool DYN = !TP;  // claimed passes on one GPU, fixed ranges under tensor parallelism (see part_range)
  if (tid == 0) {
    for (int s = 0; s < a.n_stages; ++s) {
      mbar_init(&full[s], MG_PW);
      mbar_init(&empty[s], MG_CW);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  Ring r = {0, 0};

  if (warp >= MG_CW) {
    // ================================================================ producers: every weight byte of the step, in order
    const uint64_t pol = policy_evict_first();
    const int pw = warp - MG_CW;
    // Claims run ahead of pdl_wait() and into the next matrix while the consumers are still in the current phase.  A claim
    // moves only weights (the consumers pass the grid barrier before they read the next activations), but the counters
    // must be zero when this launch starts: see the reset at the end of the kernel.
    unsigned* claim = a.grid_bar + MEGA_CLAIM_OFF;
    unsigned n_claims = 0;
    for (int l = 0; l < a.n_layers; ++l) {
      const MegaLayer& w = a.layers[l];
      produce<DYN>(w.wqkv, a.q_rows + 2 * a.kv_rows, h, tiles, full, empty, a.n_stages, r, pol, lane, pw, claim + 4 * l, n_claims);
      produce<DYN>(w.wo, h, a.q_rows, tiles, full, empty, a.n_stages, r, pol, lane, pw, claim + 4 * l + 1, n_claims);
      produce<DYN>(w.wgu, 2 * a.inter, h, tiles, full, empty, a.n_stages, r, pol, lane, pw, claim + 4 * l + 2, n_claims);
      produce<DYN>(w.wdown, h, a.inter, tiles, full, empty, a.n_stages, r, pol, lane, pw, claim + 4 * l + 3, n_claims);
    }
    produce<DYN>(a.lm_head, a.vocab, h, tiles, full, empty, a.n_stages, r, pol, lane, pw, claim + 4 * a.n_layers, n_claims);
    return;
  }

  // ================================================================== consumers
  pdl_wait();
  int n_prof = 0;
  if (a.prof && a.prof_all && tid == 0) {
    unsigned smid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    a.prof[(size_t)blockIdx.x * 1024 + 1023] = smid;
  }
  MG_STAMP();
  unsigned n_sync = 0;
  const unsigned n_ctas = gridDim.x;
  if (blockIdx.x == 0 && tid == 0) {
    *a.step += 1;
    if (a.fwd_counter) *a.fwd_counter += 1;
  }
  // embedding gather, distributed over all consumer threads of the grid
  {
    const int per_row = h / 8;
    for (int i = blockIdx.x * (MG_CW * 32) + tid; i < a.M * per_row; i += n_ctas * MG_CW * 32) {
      const int m = i / per_row, c = i - m * per_row;
      *reinterpret_cast<uint4*>(a.h + (size_t)m * h + c * 8) = ldg128(a.embed + (size_t)a.row_tok[m] * h + c * 8);
    }
  }
  grid_sync(a.grid_bar, n_sync, n_ctas);
  // epoch of allreduce `seq` of this forward = ll_epoch0 + seq (never 0; the forward counter was bumped above and is
  // visible through the grid barrier)
  [[maybe_unused]] uint32_t ll_epoch0 = 0;
  if constexpr (TP) ll_epoch0 = (uint32_t)ld_acquire_gpu(reinterpret_cast<const unsigned*>(a.fwd_counter)) * (uint32_t)(2 * a.n_layers) + 1u;

  GemvArgs g = {};
  g.M = a.M;
  g.eps = a.eps;
  g.head_dim = D;
  g.q_rows = a.q_rows;
  g.kv_rows = a.kv_rows;
  g.block_table = a.block_table;
  g.bt_stride = a.bt_stride;
  g.row_slot = a.row_slot;
  g.row_pos = a.row_pos;
  g.rope_cs = a.rope_cs;
  g.block_size = a.block_size;
  g.kvh = a.kvh;
  g.q_out = a.q;

  for (int l = 0; l < a.n_layers; ++l) {
    const MegaLayer& w = a.layers[l];
    // ---- RMSNorm + QKV + RoPE + KV append
    stage_x<BT, NORM_RMS>(a.h, h, a.M, h, w.ln1, a.eps, xs, red, tid, warp, lane);
    g.N = a.q_rows + 2 * a.kv_rows;
    g.K = h;
    g.kcache = w.kcache;
    g.vcache = w.vcache;
    MG_STAMP();  // 1: x staged
    consume<BT, EPI_QKV_ROPE, DYN>(g, tiles, xs, full, empty, a.n_stages, r, warp, lane, red_s);
    MG_STAMP();  // 2: qkv consumed
    grid_sync(a.grid_bar, n_sync, n_ctas);
    MG_STAMP();  // 3
    // ---- attention
    if constexpr (G == 8) {
      if (a.attn_cta_tile)
        attention_phase_cta<D>(a, w.kcache, w.vcache, xs, reinterpret_cast<int*>(red + 16), tid, warp, lane);
      else
        attention_phase<D, G>(a, w.kcache, w.vcache, warp, lane);
    } else {
      if (a.attn_coop)
        attention_phase_coop<D, G>(a, w.kcache, w.vcache, reinterpret_cast<float*>(xs), reinterpret_cast<int*>(red + 16), tid, warp, lane);
      else
        attention_phase<D, G>(a, w.kcache, w.vcache, warp, lane);
    }
    MG_STAMP();  // 4: attention done
    grid_sync(a.grid_bar, n_sync, n_ctas);
    MG_STAMP();  // 5
    // ---- O projection + residual
    stage_x<BT, NORM_NONE>(a.attn, a.q_rows, a.M, a.q_rows, nullptr, 0.f, xs, red, tid, warp, lane);
    g.N = h;
    g.K = a.q_rows;
    g.out_bf16 = a.h;
    g.resid = a.h;
    g.ld_out = h;
    MG_STAMP();  // 6: x staged
    if constexpr (TP) {
      g.out_f32 = a.peer_partials[a.tp_rank] + (size_t)((2 * l) & 1) * (size_t)a.parity_stride;
      if (a.tp_mode == 3) {
        const LlCtx lx = {&a, ll_epoch0 + (uint32_t)(2 * l), (size_t)((2 * l) & 1) * (size_t)a.ll_parity_stride + (size_t)a.tp_rank * (size_t)a.ll_src_stride};
        consume<BT, EPI_LL, DYN>(g, tiles, xs, full, empty, a.n_stages, r, warp, lane, red_s, &lx);
        tp_reduce_ll(a, 2 * l, lx.epoch, tid);
      } else {
      consume<BT, EPI_F32, DYN>(g, tiles, xs, full, empty, a.n_stages, r, warp, lane, red_s);
      }
      if (a.tp_mode == 3) {
      } else if (a.tp_mode == 2) {
        tp_reduce_cta(a, 2 * l, tid);
      } else {
        grid_sync(a.grid_bar, n_sync, n_ctas);
        tp_reduce_phase(a, 2 * l, tid);
      }
    } else {
      consume<BT, EPI_RESID, DYN>(g, tiles, xs, full, empty, a.n_stages, r, warp, lane, red_s);
    }
    MG_STAMP();  // 7: o consumed
    grid_sync(a.grid_bar, n_sync, n_ctas);
    MG_STAMP();  // 8
    // ---- RMSNorm + gate/up + SwiGLU
    stage_x<BT, NORM_RMS>(a.h, h, a.M, h, w.ln2, a.eps, xs, red, tid, warp, lane);
    g.N = 2 * a.inter;
    g.K = h;
    g.out_bf16 = a.act;
    g.ld_out = a.inter;
    MG_STAMP();  // 9: x staged
    consume<BT, EPI_SWIGLU, DYN>(g, tiles, xs, full, empty, a.n_stages, r, warp, lane, red_s);
    MG_STAMP();  // 10: gate/up consumed
    grid_sync(a.grid_bar, n_sync, n_ctas);
    MG_STAMP();  // 11
    // ---- down projection + residual
    stage_x<BT, NORM_NONE>(a.act, a.inter, a.M, a.inter, nullptr, 0.f, xs, red, tid, warp, lane);
    g.N = h;
    g.K = a.inter;
    g.out_bf16 = a.h;
    g.resid = a.h;
    g.ld_out = h;
    MG_STAMP();  // 12: x staged
    if constexpr (TP) {
      g.out_f32 = a.peer_partials[a.tp_rank] + (size_t)((2 * l + 1) & 1) * (size_t)a.parity_stride;
      if (a.tp_mode == 3) {
        const LlCtx lx = {&a, ll_epoch0 + (uint32_t)(2 * l + 1), (size_t)((2 * l + 1) & 1) * (size_t)a.ll_parity_stride + (size_t)a.tp_rank * (size_t)a.ll_src_stride};
        consume<BT, EPI_LL, DYN>(g, tiles, xs, full, empty, a.n_stages, r, warp, lane, red_s, &lx);
        tp_reduce_ll(a, 2 * l + 1, lx.epoch, tid);
      } else {
      consume<BT, EPI_F32, DYN>(g, tiles, xs, full, empty, a.n_stages, r, warp, lane, red_s);
      }
      if (a.tp_mode == 3) {
      } else if (a.tp_mode == 2) {
        tp_reduce_cta(a, 2 * l + 1, tid);
      } else {
        grid_sync(a.grid_bar, n_sync, n_ctas);
        tp_reduce_phase(a, 2 * l + 1, tid);
      }
    } else {
      consume<BT, EPI_RESID, DYN>(g, tiles, xs, full, empty, a.n_stages, r, warp, lane, red_s);
    }
    MG_STAMP();  // 13: down consumed
    grid_sync(a.grid_bar, n_sync, n_ctas);
    MG_STAMP();  // 14 (= 0 of the next layer)
  }
  // ---- final norm + lm_head
  stage_x<BT, NORM_RMS>(a.h, h, a.M, h, a.final_norm, a.eps, xs, red, tid, warp, lane);
  g.N = a.vocab;
  g.K = h;
  g.out_f32 = a.logits;
  g.ld_out = a.vocab;
  consume<BT, EPI_F32_BF16R, DYN>(g, tiles, xs, full, empty, a.n_stages, r, warp, lane, red_s);
  grid_sync(a.grid_bar, n_sync, n_ctas);
  // ---- greedy pick: CTA m handles row m (lowest index wins ties)
  if ((int)blockIdx.x < a.M) {
    const int m = blockIdx.x;
    const float* lg = a.logits + (size_t)m * a.vocab;
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = tid; i < a.vocab; i += MG_CW * 32) {
      const float v = __ldcg(lg + i);
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
    float* sv = red;                                     // [8] floats
    int* si = reinterpret_cast<int*>(red + MG_CW);       // [8] ints
    if (lane == 0) {
      sv[warp] = best;
      si[warp] = bi;
    }
    named_bar_sync(1, MG_CW * 32);
    if (tid == 0) {
      for (int w2 = 1; w2 < MG_CW; ++w2)
        if (sv[w2] > best || (sv[w2] == best && si[w2] < bi)) {
          best = sv[w2];
          bi = si[w2];
        }
      a.row_tok[m] = bi;
      a.hist[(size_t)(__ldcg(a.step)) * a.M + m] = bi;
      a.row_pos[m] += 1;
    }
  }
  // leave the barrier and claim counters at zero for the next launch: the last CTA through resets them.  Every producer's
  // last claim precedes the end marker its consumers waited for, so no claim of this launch can follow the reset.  The
  // kernel is launched without programmatic dependent launch (Engine::forward_mega), so the next step starts only after
  // this one has exited; with PDL its producers, which claim before pdl_wait(), could claim before these stores.
  if (tid == 0) {
    __threadfence();
    if (atomicAdd(a.grid_bar + 1, 1u) == n_ctas - 1) {
      a.grid_bar[0] = 0;
      a.grid_bar[1] = 0;
      if constexpr (DYN)
        for (int i = 0; i <= 4 * a.n_layers; ++i) a.grid_bar[MEGA_CLAIM_OFF + i] = 0;
      __threadfence();
    }
  }
}

size_t mega_smem_bytes(int bt, int k_max, int n_stages) {
  return (size_t)n_stages * MG_STAGE_ELEMS * 2 + (size_t)bt * k_max * 2 + 2 * (size_t)n_stages * 8 + 128 +
         (size_t)MG_RED_FLOATS * 4;  // dynamic part
}

int mega_pick_stages(int bt, int k_max) {
  // 227 KiB per CTA in all; 225 KiB for the dynamic part
  int s = 6;
  while (s > 2 && mega_smem_bytes(bt, k_max, s) > 225 * 1024) --s;
  return mega_smem_bytes(bt, k_max, s) <= 225 * 1024 ? s : 0;
}

template <int BT, int D, int G, bool TP = false>
static cudaError_t launch_mega_t(const MegaArgs& a, const LaunchCfg& lc) {
  const size_t smem = mega_smem_bytes(BT, a.k_max, a.n_stages);
  static std::atomic<unsigned long long> attr_mask{0};  // per instantiation, per device
  if (first_launch_on_device(attr_mask)) {
    cudaError_t e = cudaFuncSetAttribute(decode_mega_kernel<BT, D, G, TP>, cudaFuncAttributeMaxDynamicSharedMemorySize, 225 * 1024);
    if (e != cudaSuccess) return e;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(lc.n_sm);
  cfg.blockDim = dim3(MG_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = lc.stream;
  cudaLaunchAttribute attr[2];
  int na = 0;
  attr[na].id = cudaLaunchAttributeCooperative;  // all CTAs must be co-resident (grid-wide barriers)
  attr[na].val.cooperative = 1;
  ++na;
  if (lc.pdl) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  return cudaLaunchKernelEx(&cfg, decode_mega_kernel<BT, D, G, TP>, a);
}

template <int BT>
static cudaError_t launch_mega_b(const MegaArgs& a, const LaunchCfg& lc) {
  const int g = a.attn_g;
  if (a.tp_size > 1) {  // tensor-parallel variant: Llama head size only
    if (a.head_dim != 128 || a.tp_size > TP_MAX || (a.hidden & 3) || !a.peer_partials || !a.peer_flags) return cudaErrorInvalidValue;
    if (a.tp_mode == 2 && (!a.peer_cta_flags || lc.n_sm > MG_CTA_FLAG_STRIDE)) return cudaErrorInvalidValue;
    if (a.tp_mode == 3 && !a.peer_ll) return cudaErrorInvalidValue;
    switch (g) {
      case 1: return launch_mega_t<BT, 128, 1, true>(a, lc);
      case 2: return launch_mega_t<BT, 128, 2, true>(a, lc);
      case 4: return launch_mega_t<BT, 128, 4, true>(a, lc);
      case 8: return launch_mega_t<BT, 128, 8, true>(a, lc);
    }
    return cudaErrorInvalidValue;
  }
  if (a.head_dim == 128) {
    switch (g) {
      case 1: return launch_mega_t<BT, 128, 1>(a, lc);
      case 2: return launch_mega_t<BT, 128, 2>(a, lc);
      case 4: return launch_mega_t<BT, 128, 4>(a, lc);
      case 8: return launch_mega_t<BT, 128, 8>(a, lc);
    }
  } else if (a.head_dim == 64) {
    switch (g) {
      case 1: return launch_mega_t<BT, 64, 1>(a, lc);
      case 2: return launch_mega_t<BT, 64, 2>(a, lc);
      case 4: return launch_mega_t<BT, 64, 4>(a, lc);
      case 8: return launch_mega_t<BT, 64, 8>(a, lc);
    }
  }
  return cudaErrorInvalidValue;
}

cudaError_t launch_decode_mega(const MegaArgs& a, const LaunchCfg& lc) {
  if (a.M < 1 || a.M > 4 || a.n_stages < 2 || a.n_stages > MG_MAX_STAGES) return cudaErrorInvalidValue;
  if (lc.n_sm < a.M) return cudaErrorInvalidValue;  // the greedy pick runs row m on CTA m
  if (a.M == 1) return launch_mega_b<1>(a, lc);
  if (a.M == 2) return launch_mega_b<2>(a, lc);
  return launch_mega_b<4>(a, lc);
}

int mega_attn_group(int group) { return (group % 8 == 0) ? 8 : (group % 4 == 0) ? 4 : (group % 2 == 0) ? 2 : 1; }
int mega_attn_chunk(int head_dim, int g) { return (32 / (head_dim / 8)) * (g <= 2 ? 8 : 2); }
size_t mega_attn_tile_bytes(int head_dim) { return (size_t)2 * MG_ATT_TILE * head_dim * 2; }
size_t mega_attn_coop_bytes(int head_dim, int g) { return (size_t)MG_CW * g * (head_dim + 2) * sizeof(float); }

MegaGeom mega_geometry(int hidden, int n_heads, int kv_heads, int head_dim, int inter, int n_layers, int max_seq, int rows,
                       bool attn_tile) {
  MegaGeom g = {};
  g.attn_g = mega_attn_group(n_heads / kv_heads);
  const int ch = mega_attn_chunk(head_dim, g.attn_g);
  g.max_chunks = (max_seq + ch - 1) / ch;
  g.k_max = std::max(hidden, std::max(n_heads * head_dim, inter));
  g.bt = rows <= 1 ? 1 : (rows == 2 ? 2 : 4);
  g.n_stages = mega_pick_stages(g.bt, g.k_max);
  const size_t xs_bytes = (size_t)g.bt * g.k_max * sizeof(bf16);  // the attention forms borrow the activation area
  g.attn_coop = (g.attn_g < 8 && attn_tile && xs_bytes >= mega_attn_coop_bytes(head_dim, g.attn_g)) ? 1 : 0;
  g.attn_cta_tile = (g.attn_g == 8 && attn_tile && xs_bytes >= mega_attn_tile_bytes(head_dim)) ? 1 : 0;
  const size_t units = (size_t)4 * (n_heads / g.attn_g) * g.max_chunks;  // [4 rows][head units][chunks]
  g.part_o_floats = units * g.attn_g * head_dim;
  g.part_ml_floats = units * g.attn_g * 2;
  g.counter_ints = (size_t)4 * n_heads;
  g.bar_words = mega_bar_words(n_layers);
  return g;
}
