// tp_twoshot.cu — two-shot tensor-parallel allreduce(sum) + residual for PREFILL-sized activations (opt-in:
// params.json "tp_two_shot": 1).  Verified on one GPU as a single rank with its peers staged in memory
// (tests/test_tp_exchange_gpu.py: slices, gather, flags, epochs, `done`); ranks running concurrently on several GPUs are
// exercised only by the two_shot case of tests/test_tp_gpu.py, which needs two or more GPUs.
//
// The one-shot kernel (kernels.cu, tp_allreduce_resid_kernel) lets every rank pull every peer's full fp32 partial:
// (TP-1) * M * hidden * 4 bytes per rank and allreduce, which is what makes TTFT grow with TP (512 x 8192 rows at TP8:
// 117 MB per rank, 160 times per prompt).  Here each rank
//   A. publishes "my partials are complete" and waits for the same flag from its peers            (as in the one-shot),
//   B. reduces only ITS 1/TP slice of [M, hidden] (pulls (TP-1) fp32 slices), adds the residual, rounds to bf16 exactly
//      like the one-shot does, writes the slice to its own h and to its `gather` buffer in the exchange pool,
//   C. after the last of its CTAs has finished B, publishes "slice ready"; waits for the peers' slice flags and pulls
//      their bf16 slices into its own h.
// Bytes pulled per rank: (TP-1)/TP * M*hidden * (4 + 2) instead of (TP-1) * M*hidden * 4 — 5.3x less at TP8 — and all
// ranks end up with bit-identical h (every element is reduced once, by its owner).
// Buffer reuse: partials are double-buffered by allreduce parity (they are rewritten by the NEXT projection, before
// that allreduce's flag wait); `gather` is written only after phase A of the same allreduce, which a rank passes only
// once every peer has finished the previous allreduce kernel (stream order), so one buffer is enough.
#include "common.cuh"
#include "kernels.h"

namespace {
constexpr int T2_MAX = 8;
constexpr int T2_THREADS = 256;

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
SSB_DEVINL uint2 ld_relaxed_sys_u2(const uint2* p) {
  uint2 v;
  asm volatile("ld.relaxed.sys.global.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
  return v;
}

__global__ void __launch_bounds__(T2_THREADS) tp_allreduce2_kernel(const TpArgs2 a) {
  pdl_wait();  // this rank's partials (previous kernel) are complete and visible
  pdl_launch_dependents();
  const uint32_t epoch = (uint32_t)(*a.tp_step) * (uint32_t)a.n_per_step + (uint32_t)a.seq_in_step + 1u;
  const size_t poff = (size_t)(a.seq_in_step & 1) * (size_t)a.parity_stride;
  const long long total4 = (long long)a.M * a.hidden / 4;
  const int tid = threadIdx.x;
  // ---- A: partials ready
  if (blockIdx.x == 0 && tid < a.size && tid != a.rank) {
    __threadfence_system();
    st_release_sys(a.peer_flags[tid] + a.rank, epoch);
  }
  if (tid < a.size && tid != a.rank) {
    const uint32_t* f = a.peer_flags[a.rank] + tid;
    SpinGuard sg;
    while ((int32_t)(ld_acquire_sys(f) - epoch) < 0) sg.poll();
  }
  __syncthreads();
  // ---- B: reduce my slice (flattened [M*hidden/4) float4 index space, contiguous per rank)
  const long long lo = total4 * a.rank / a.size, hi = total4 * (a.rank + 1) / a.size;
  uint2* out2 = reinterpret_cast<uint2*>(a.out);
  uint2* gat2 = reinterpret_cast<uint2*>(a.peer_gather[a.rank]);
  for (long long i = lo + (long long)blockIdx.x * T2_THREADS + tid; i < hi; i += (long long)gridDim.x * T2_THREADS) {
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int r = 0; r < T2_MAX; ++r) {  // rank order, as in the one-shot kernel
      if (r < a.size) {
        const float4 v = ld_relaxed_sys_f4(a.peer_partials[r] + poff + (size_t)i * 4);
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
    out2[i] = o;
    gat2[i] = o;
  }
  // ---- slice ready: the LAST CTA to finish B tells the peers (fence + counter, then a system-scope release)
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    if (atomicAdd(a.done, 1u) == gridDim.x - 1) {
      __threadfence_system();
      *a.done = 0;  // clean for the next launch (stream order)
      for (int p = 0; p < a.size; ++p)
        if (p != a.rank) st_release_sys(a.peer_flags[p] + T2_MAX + a.rank, epoch);
    }
  }
  // ---- C: gather the peers' slices
  if (tid < a.size && tid != a.rank) {
    const uint32_t* f = a.peer_flags[a.rank] + T2_MAX + tid;
    SpinGuard sg;
    while ((int32_t)(ld_acquire_sys(f) - epoch) < 0) sg.poll();
  }
  __syncthreads();
  for (int p = 0; p < a.size; ++p) {
    if (p == a.rank) continue;
    const long long plo = total4 * p / a.size, phi = total4 * (p + 1) / a.size;
    const uint2* src = reinterpret_cast<const uint2*>(a.peer_gather[p]);
#pragma unroll 4
    for (long long i = plo + (long long)blockIdx.x * T2_THREADS + tid; i < phi; i += (long long)gridDim.x * T2_THREADS)
      out2[i] = ld_relaxed_sys_u2(src + i);
  }
}
}  // namespace

cudaError_t launch_tp_allreduce2(const TpArgs2& a, const LaunchCfg& lc) {
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  if (a.size > T2_MAX || (a.hidden & 3) || !a.peer_gather || !a.done) return cudaErrorInvalidValue;
  const long long slice4 = (long long)a.M * a.hidden / 4 / a.size;
  long long grid = (slice4 + T2_THREADS * 4 - 1) / (T2_THREADS * 4);  // ~4 float4 per thread in phase B
  grid = grid < 1 ? 1 : (grid > lc.n_sm ? lc.n_sm : grid);             // every CTA spins on flags: stay co-resident
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3(T2_THREADS);
  cfg.stream = lc.stream;
  cfg.attrs = attr;
  cfg.numAttrs = lc.pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, tp_allreduce2_kernel, a);
}
