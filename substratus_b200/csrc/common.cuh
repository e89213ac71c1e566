// common.cuh — PTX wrappers and small device helpers shared by the sm_90a kernels.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define SSB_DEVINL __device__ __forceinline__

typedef __nv_bfloat16 bf16;

// ---------------------------------------------------------------- bf16 helpers
SSB_DEVINL float bf16r(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }  // round-trip through bf16 (RNE)
SSB_DEVINL float bf_lo(uint32_t u) { return __uint_as_float(u << 16); }
SSB_DEVINL float bf_hi(uint32_t u) { return __uint_as_float(u & 0xffff0000u); }
SSB_DEVINL uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

// ---------------------------------------------------------------- shared-memory / mbarrier / bulk copy (TMA engine)
SSB_DEVINL uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

SSB_DEVINL void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
SSB_DEVINL void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
SSB_DEVINL void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
SSB_DEVINL void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
SSB_DEVINL void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
SSB_DEVINL bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
SSB_DEVINL void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// 1-D bulk async copy global -> shared (TMA engine, no tensor map); bytes % 16 == 0, both addresses 16 B aligned.
SSB_DEVINL void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// same with an L2 evict-first policy: weights are streamed exactly once per step
SSB_DEVINL uint64_t policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
SSB_DEVINL void bulk_g2s_hint(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar, uint64_t pol) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
          smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(pol)
      : "memory");
}

// ---------------------------------------------------------------- programmatic dependent launch (PDL)
// wait: block until every prerequisite grid has completed and its memory is visible.
SSB_DEVINL void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// launch_dependents: allow the next kernel in the stream to start being scheduled.
SSB_DEVINL void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

SSB_DEVINL void named_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

// ---------------------------------------------------------------- bounded cross-GPU waits
// Every spin on a flag another GPU has to write goes through SpinGuard::poll(): after SSB_SPIN_TIMEOUT_NS (20 s) of
// polling the kernel traps instead of hanging.  A peer rank that died (or a protocol bug) then surfaces on the host as a
// sticky CUDA error -> SSB_ECUDA -> the serve host exits non-zero and the Deployment restarts the pod
// (internal/controller/server_controller.go:280-296 turns that into Serving=False), instead of every later request
// blocking behind a kernel that never returns.  The clock is read once per 1024 polls, so the poll loop stays tight.
#ifndef SSB_SPIN_TIMEOUT_NS
#define SSB_SPIN_TIMEOUT_NS 20000000000ull
#endif
struct SpinGuard {
  unsigned long long t0 = 0;
  unsigned n = 0;
  SSB_DEVINL void poll() {
    if ((++n & 1023u) == 0) {
      unsigned long long now;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
      if (t0 == 0)
        t0 = now;
      else if (now - t0 > SSB_SPIN_TIMEOUT_NS)
        __trap();
    }
  }
};

// ---------------------------------------------------------------- warp reductions
SSB_DEVINL float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
SSB_DEVINL float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// 128-bit read-only global load
SSB_DEVINL uint4 ldg128(const void* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }
