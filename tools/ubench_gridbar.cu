// ubench_gridbar.cu — latency of grid-wide barrier flavours on one co-resident CTA per SM (the persistent decode kernel pays 5
// per layer, 160 per Llama-2-7B token).  Standalone:
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/bin/ubench_gridbar tools/ubench_gridbar.cu && tools/bin/ubench_gridbar
// Every flavour also carries a message (each CTA writes a word before the barrier, reads its neighbour's after it) so a
// flavour that is fast because it is wrong shows up as "BAD".
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#define DEVINL __device__ __forceinline__
constexpr int CW_THREADS = 256;  // threads taking part per CTA (the consumer warps of decode_mega_kernel)

DEVINL unsigned ld_acquire_gpu(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
DEVINL unsigned ld_relaxed_gpu(const unsigned* p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
DEVINL void st_release_gpu(unsigned* p, unsigned v) { asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
DEVINL void red_release_gpu(unsigned* p) { asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(p) : "memory"); }
DEVINL void fence_acq_rel_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
DEVINL void bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// mode 0: fence + atomicAdd + acquire poll + fence (round-1 default)      1: red.release + acquire poll
// mode 2: two-level tree (16 groups)                                      3: per-CTA flag words, one warp polls them all
// mode 4: as 3 with one flag per 128-byte line                            5: red.release + relaxed poll + one acquire fence
template <int MODE>
DEVINL void grid_sync(unsigned* bar, unsigned& n_done, unsigned n_ctas) {
  bar_sync(1, CW_THREADS);
  ++n_done;
  if (MODE == 3 || MODE == 4) {
    constexpr int STRIDE = MODE == 4 ? 32 : 1;
    if (threadIdx.x < 32) {
      if (threadIdx.x == 0) st_release_gpu(bar + 64 + blockIdx.x * STRIDE, n_done);
      for (unsigned c = threadIdx.x; c < n_ctas; c += 32) {
        while ((int)(ld_relaxed_gpu(bar + 64 + c * STRIDE) - n_done) < 0) {
        }
      }
      fence_acq_rel_gpu();
    }
  } else if (threadIdx.x == 0) {
    if (MODE == 0) {
      __threadfence();
      atomicAdd(bar, 1u);
      const unsigned target = n_done * n_ctas;
      while (ld_acquire_gpu(bar) < target) {
      }
      __threadfence();
    } else if (MODE == 1) {
      red_release_gpu(bar);
      const unsigned target = n_done * n_ctas;
      while (ld_acquire_gpu(bar) < target) {
      }
    } else if (MODE == 5) {
      red_release_gpu(bar);
      const unsigned target = n_done * n_ctas;
      while (ld_relaxed_gpu(bar) < target) {
      }
      fence_acq_rel_gpu();
    } else if (MODE == 2) {
      constexpr unsigned G = 16;
      const unsigned g = blockIdx.x % G;
      const unsigned gsize = n_ctas / G + (g < n_ctas % G ? 1u : 0u);
      __threadfence();
      const unsigned old = atomicAdd(bar + 32 + 32 * g, 1u);
      if (old + 1 == n_done * gsize) {
        __threadfence();
        atomicAdd(bar, 1u);
      }
      const unsigned target = n_done * G;
      while (ld_acquire_gpu(bar) < target) {
      }
      __threadfence();
    }
  }
  bar_sync(1, CW_THREADS);
}

template <int MODE>
__global__ void __launch_bounds__(384, 1) k(unsigned* bar, unsigned* msg, int iters, int work, unsigned* bad, unsigned long long* t_ns) {
  if (threadIdx.x >= CW_THREADS) return;  // producer warps do not take part
  unsigned n_done = 0;
  const unsigned n = gridDim.x;
  unsigned long long t0 = 0;
  unsigned errs = 0;
  float sink = 0.f;
  for (int it = 0; it < iters; ++it) {
    if (it == 8 && threadIdx.x == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    for (int w = 0; w < work; ++w) sink = sink * 1.0001f + 1.f;  // optional per-iteration work (same on every CTA)
    if (threadIdx.x == 7) msg[blockIdx.x * 32] = (unsigned)it * 1000u + blockIdx.x;  // plain store by a non-leader thread
    grid_sync<MODE>(bar, n_done, n);
    if (threadIdx.x == 9) {
      const unsigned nb = (blockIdx.x + 61) % n;
      const unsigned v = __ldcg(msg + nb * 32);
      if (v != (unsigned)it * 1000u + nb) ++errs;
    }
    grid_sync<MODE>(bar, n_done, n);  // second barrier: nobody overwrites msg before everyone has read it
  }
  if (threadIdx.x == 0) {
    unsigned long long t1;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
    if (blockIdx.x == 0) *t_ns = t1 - t0;
  }
  if (errs) atomicAdd(bad, errs);
  if (sink == 12345.f) msg[0] = 1;
}

template <int MODE>
static void run(const char* name, int n_sm, int iters, int work) {
  unsigned *bar, *msg, *bad;
  unsigned long long* t;
  cudaMalloc(&bar, 64 * 1024);
  cudaMalloc(&msg, n_sm * 128);
  cudaMalloc(&bad, 4);
  cudaMalloc(&t, 8);
  cudaMemset(bar, 0, 64 * 1024);
  cudaMemset(msg, 0, n_sm * 128);
  cudaMemset(bad, 0, 4);
  void* args[] = {&bar, &msg, &iters, &work, &bad, &t};
  cudaError_t e = cudaLaunchCooperativeKernel((void*)k<MODE>, dim3(n_sm), dim3(384), args, 0, 0);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    printf("%-46s launch failed: %s\n", name, cudaGetErrorString(e));
    return;
  }
  unsigned hb = 0;
  unsigned long long ns = 0;
  cudaMemcpy(&hb, bad, 4, cudaMemcpyDeviceToHost);
  cudaMemcpy(&ns, t, 8, cudaMemcpyDeviceToHost);
  printf("%-46s work %4d : %7.3f us per barrier  (%d barriers)  %s\n", name, work, (double)ns / 1e3 / (2.0 * (iters - 8)), 2 * (iters - 8),
         hb ? "BAD (stale reads)" : "ok");
  cudaFree(bar);
  cudaFree(msg);
  cudaFree(bad);
  cudaFree(t);
}

int main() {
  cudaDeviceProp p;
  cudaGetDeviceProperties(&p, 0);
  const int n = p.multiProcessorCount;
  printf("%s, %d SMs\n", p.name, n);
  for (int work : {0, 2000}) {
    run<0>("0 fence+atomicAdd+acquire poll+fence (default)", n, 2008, work);
    run<1>("1 red.release + acquire poll", n, 2008, work);
    run<5>("5 red.release + relaxed poll + fence", n, 2008, work);
    run<2>("2 tree (16 groups)", n, 2008, work);
    run<3>("3 flag words, warp polls all (packed)", n, 2008, work);
    run<4>("4 flag words, warp polls all (128 B apart)", n, 2008, work);
  }
  return 0;
}
