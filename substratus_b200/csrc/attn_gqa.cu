// attn_gqa.cu — paged-KV decode attention for grouped-query models (G = 4 or 8 query heads per KV head,
// e.g. Llama-2-70B 64/8, Falcon-40B 128/8).  One CTA = one (row, KV head [, head sub-group], context split);
// the K/V rows of the split are staged ONCE in shared memory (cp.async 16 B per thread, all loads in flight at once),
// then warp g computes query head g against the staged tile: dot via 16-lane shuffle reduction, fp32 online softmax,
// fp32 P.V — so the K/V stream is read once per group instead of once per head and no thread carries G accumulators.
// Splits are merged by the last-arriving CTA (same scheme and buffers as attn_decode_kernel).
// Math/rounding: HF:models/llama/modeling_llama.py:187-221 (repeat_kv + eager_attention_forward), see kernels.cu.
#include "common.cuh"
#include "kernels.h"

constexpr int GQ_TOK = 64;  // tokens staged per pass

SSB_DEVINL void cp_async16(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem)), "l"(gmem) : "memory");
}
SSB_DEVINL void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

template <int D, int G>
__global__ void __launch_bounds__(G * 32) attn_gqa_kernel(const AttnArgs a) {
  constexpr int LPR = D / 8, RPW = 32 / LPR;
  constexpr int NT = G * 32;
  __shared__ __align__(16) bf16 sK[GQ_TOK][D];
  __shared__ __align__(16) bf16 sV[GQ_TOK][D];
  __shared__ int sm_last;

  pdl_wait();
  pdl_launch_dependents();
  const int split = blockIdx.x, row = blockIdx.z;
  const int kvh = blockIdx.y / (a.group / G);
  const int head0 = blockIdx.y * G;
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
  const int HD = a.n_heads * D;
  const int* bt = a.block_table + (size_t)slot * a.bt_stride;

  float q[8];
  {
    const uint4 v = *reinterpret_cast<const uint4*>(a.q + (size_t)row * HD + (head0 + warp) * D + li * 8);
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      q[2 * i] = bf_lo(u[i]);
      q[2 * i + 1] = bf_hi(u[i]);
    }
  }
  float m = -1e30f, l = 0.f, acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;

  for (int p0 = t_begin; p0 < t_end; p0 += GQ_TOK) {
    const int np = min(GQ_TOK, t_end - p0);
    if (p0 != t_begin) __syncthreads();  // previous tile fully consumed
    for (int i = tid; i < np * LPR; i += NT) {
      const int tt = i / LPR, c = i % LPR;
      const int t = p0 + tt;
      const size_t off = (((size_t)bt[t / BS] * a.kvh + kvh) * BS + (t % BS)) * D + c * 8;
      cp_async16(&sK[tt][c * 8], a.kcache + off);
      cp_async16(&sV[tt][c * 8], a.vcache + off);
    }
    cp_async_wait_all();
    __syncthreads();
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
      const float s = bf16r(bf16r(d) * a.scale);
      const float mn = fmaxf(m, s);
      const float corr = __expf(m - mn), p = __expf(s - mn);
      m = mn;
      l = l * corr + p;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        acc[2 * i] = fmaf(p, bf_lo(vu[i]), acc[2 * i] * corr);
        acc[2 * i + 1] = fmaf(p, bf_hi(vu[i]), acc[2 * i + 1] * corr);
      }
    }
  }
  // merge the RPW token sub-groups of the warp
#pragma unroll
  for (int o = LPR; o < 32; o <<= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, o);
    const float ol = __shfl_xor_sync(0xffffffffu, l, o);
    const float mn = fmaxf(m, om);
    const float wa = __expf(m - mn), wb = __expf(om - mn);
    l = l * wa + ol * wb;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float oa = __shfl_xor_sync(0xffffffffu, acc[i], o);
      acc[i] = acc[i] * wa + oa * wb;
    }
    m = mn;
  }
  const size_t pbase = ((size_t)row * gridDim.y + blockIdx.y) * a.n_splits;
  if (n_active == 1) {
    if (sub == 0) {
      const float inv = 1.0f / l;
      uint32_t o[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) o[i] = pack_bf16(acc[2 * i] * inv, acc[2 * i + 1] * inv);
      *reinterpret_cast<uint4*>(a.out + (size_t)row * HD + (head0 + warp) * D + li * 8) = make_uint4(o[0], o[1], o[2], o[3]);
    }
    return;
  }
  if (sub == 0) {
    float* po = a.part_o + (pbase + split) * (G * D) + warp * D + li * 8;
    *reinterpret_cast<float4*>(po) = make_float4(acc[0], acc[1], acc[2], acc[3]);
    *reinterpret_cast<float4*>(po + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
    if (li == 0) {
      a.part_ml[(pbase + split) * (2 * G) + warp] = m;
      a.part_ml[(pbase + split) * (2 * G) + G + warp] = l;
    }
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) sm_last = (atomicAdd(&a.counters[row * gridDim.y + blockIdx.y], 1) == n_active - 1);
  __syncthreads();
  if (!sm_last) return;
  __threadfence();
  // warp g merges head g over the splits; lane handles 4 dims (D = 128) or lanes 0..15 (D = 64)
  for (int dd = lane * 4; dd < D; dd += 128) {
    float M2 = -1e30f;
    for (int s = 0; s < n_active; ++s) M2 = fmaxf(M2, __ldcg(&a.part_ml[(pbase + s) * (2 * G) + warp]));
    float L2 = 0.f;
    float4 O = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int s = 0; s < n_active; ++s) {
      const float w = __expf(__ldcg(&a.part_ml[(pbase + s) * (2 * G) + warp]) - M2);
      L2 += __ldcg(&a.part_ml[(pbase + s) * (2 * G) + G + warp]) * w;
      const float4 o = __ldcg(reinterpret_cast<const float4*>(a.part_o + (pbase + s) * (G * D) + warp * D + dd));
      O.x += o.x * w;
      O.y += o.y * w;
      O.z += o.z * w;
      O.w += o.w * w;
    }
    const float inv = 1.0f / L2;
    uint2 o;
    o.x = pack_bf16(O.x * inv, O.y * inv);
    o.y = pack_bf16(O.z * inv, O.w * inv);
    *reinterpret_cast<uint2*>(a.out + (size_t)row * HD + (head0 + warp) * D + dd) = o;
  }
  if (tid == 0) a.counters[row * gridDim.y + blockIdx.y] = 0;
}

template <int D, int G>
static cudaError_t launch_gqa_t(const AttnArgs& a, const LaunchCfg& lc) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(a.n_splits, a.kvh * (a.group / G), a.M);
  cfg.blockDim = dim3(G * 32);
  cfg.stream = lc.stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = lc.pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, attn_gqa_kernel<D, G>, a);
}

// gc = query heads per CTA (4 or 8)
cudaError_t launch_attn_gqa(const AttnArgs& a, int gc, const LaunchCfg& lc) {
  if (a.head_dim == 128) {
    if (gc == 8) return launch_gqa_t<128, 8>(a, lc);
    if (gc == 4) return launch_gqa_t<128, 4>(a, lc);
  } else if (a.head_dim == 64) {
    if (gc == 8) return launch_gqa_t<64, 8>(a, lc);
    if (gc == 4) return launch_gqa_t<64, 4>(a, lc);
  }
  return cudaErrorInvalidValue;
}

// =====================================================================================================================
// prefill attention on the tensor pipe (mma.sync m16n8k16 bf16, fp32 accumulate), flash-style:
// a CTA owns up to 64 consecutive query rows of one sequence and one query head (16 rows per warp); the causal key
// range is streamed through shared memory in 64-key chunks (cp.async, XOR-swizzled 16-byte chunks so ldmatrix is
// conflict-free); S = Q.K^T and O += P.V run on HMMA, the online softmax (fp32) lives in the accumulator fragments.
// Rounding points as HF eager attention (HF:models/llama/modeling_llama.py:199-221): scores rounded to bf16 and scaled
// in bf16, softmax in fp32, P cast to bf16 for P.V.  (This is the legacy-MMA tensor path on purpose: the tile is
// 16x64 per warp and lives in registers; the projections, where the FLOPs are, use wgmma.)
// =====================================================================================================================
constexpr int PF_Q = 64, PF_K = 64;

SSB_DEVINL void ldsm_x4(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
SSB_DEVINL void ldsm_x4_t(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
SSB_DEVINL void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <int D>
__global__ void __launch_bounds__(128) attn_prefill_kernel(const AttnArgs a) {
  constexpr int CH = D / 8;        // 16-byte chunks per row
  constexpr int PITCH = D * 2;     // bytes per row
  extern __shared__ __align__(128) uint8_t pf_smem[];
  uint8_t* sQ = pf_smem;
  uint8_t* sK = sQ + PF_Q * PITCH;
  uint8_t* sV = sK + PF_K * PITCH;
  auto sw = [](int row, int chunk) { return row * PITCH + ((chunk ^ (row & 7)) << 4); };

  pdl_wait();
  pdl_launch_dependents();
  const int tile = blockIdx.x, head = blockIdx.y;
  const int kvh = head / a.group;
  const int row0 = a.tile_row0[tile], nrows = a.tile_nrows[tile];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int slot = a.row_slot[row0];
  const int pos0 = a.row_pos[row0];           // rows of a tile have consecutive positions pos0, pos0+1, ...
  const int ctx = pos0 + nrows;               // keys needed by the last row
  const int BS = a.block_size;
  const int HD = a.n_heads * D;
  const int* bt = a.block_table + (size_t)slot * a.bt_stride;

  // ---- stage Q (zero rows past the tile end)
  for (int i = tid; i < PF_Q * CH; i += 128) {
    const int r = i / CH, c = i % CH;
    if (r < nrows)
      cp_async16(sQ + sw(r, c), a.q + (size_t)(row0 + r) * HD + head * D + c * 8);
    else
      *reinterpret_cast<uint4*>(sQ + sw(r, c)) = make_uint4(0, 0, 0, 0);
  }
  cp_async_wait_all();
  __syncthreads();
  uint32_t qf[D / 16][4];
#pragma unroll
  for (int ks = 0; ks < D / 16; ++ks) {
    const int r = warp * 16 + (lane & 7) + 8 * ((lane >> 3) & 1);
    ldsm_x4(qf[ks], sQ + sw(r, 2 * ks + (lane >> 4)));
  }
  float o[D / 8][4];
#pragma unroll
  for (int j = 0; j < D / 8; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
  float mrow[2] = {-1e30f, -1e30f}, lrow[2] = {0.f, 0.f};
  const int qpos0 = pos0 + warp * 16 + g;  // position of this thread's first row (second row: +8)
  const int warp_max_pos = pos0 + warp * 16 + 15;

  for (int p0 = 0; p0 < ctx; p0 += PF_K) {
    const int np = min(PF_K, ctx - p0);
    if (p0) __syncthreads();
    for (int i = tid; i < PF_K * CH; i += 128) {
      const int r = i / CH, c = i % CH;
      if (r < np) {
        const int tk = p0 + r;
        const size_t off = (((size_t)bt[tk / BS] * a.kvh + kvh) * BS + (tk % BS)) * D + c * 8;
        cp_async16(sK + sw(r, c), a.kcache + off);
        cp_async16(sV + sw(r, c), a.vcache + off);
      } else {
        *reinterpret_cast<uint4*>(sK + sw(r, c)) = make_uint4(0, 0, 0, 0);
        *reinterpret_cast<uint4*>(sV + sw(r, c)) = make_uint4(0, 0, 0, 0);
      }
    }
    cp_async_wait_all();
    __syncthreads();
    if (p0 > warp_max_pos) continue;  // chunk entirely in this warp's future (warp-uniform)

    // ---- S = Q K^T  (16 x 64 per warp)
    float sc[PF_K / 8][4];
#pragma unroll
    for (int j = 0; j < PF_K / 8; ++j) {
      sc[j][0] = sc[j][1] = sc[j][2] = sc[j][3] = 0.f;
#pragma unroll
      for (int ks = 0; ks < D / 16; ks += 2) {
        uint32_t kb[4];  // (keys j*8.., d chunks 2ks, 2ks+1, 2ks+2, 2ks+3)
        ldsm_x4(kb, sK + sw(j * 8 + (lane & 7), 2 * ks + (lane >> 3)));
        mma16816(sc[j], qf[ks], kb[0], kb[1]);
        mma16816(sc[j], qf[ks + 1], kb[2], kb[3]);
      }
    }
    // ---- rounding pins, causal mask, online softmax (rows g and g+8 of this warp's 16)
    float cmax[2] = {-1e30f, -1e30f};
#pragma unroll
    for (int j = 0; j < PF_K / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = p0 + j * 8 + 2 * t + (e & 1);
        const int qp = qpos0 + 8 * (e >> 1);
        float v = bf16r(bf16r(sc[j][e]) * a.scale);
        if (key > qp) v = -1e30f;
        sc[j][e] = v;
        cmax[e >> 1] = fmaxf(cmax[e >> 1], v);
      }
    }
    float corr[2], psum[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      cmax[r] = fmaxf(cmax[r], __shfl_xor_sync(0xffffffffu, cmax[r], 1));
      cmax[r] = fmaxf(cmax[r], __shfl_xor_sync(0xffffffffu, cmax[r], 2));
      const float mn = fmaxf(mrow[r], cmax[r]);
      corr[r] = __expf(mrow[r] - mn);
      mrow[r] = mn;
    }
    uint32_t pa[PF_K / 16][4];
#pragma unroll
    for (int j = 0; j < PF_K / 8; ++j) {
      float p[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        p[e] = sc[j][e] <= -1e29f ? 0.f : __expf(sc[j][e] - mrow[e >> 1]);
        p[e] = bf16r(p[e]);  // P is cast to bf16 before P.V
        psum[e >> 1] += p[e];
      }
      pa[j >> 1][(j & 1) * 2 + 0] = pack_bf16(p[0], p[1]);
      pa[j >> 1][(j & 1) * 2 + 1] = pack_bf16(p[2], p[3]);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      psum[r] += __shfl_xor_sync(0xffffffffu, psum[r], 1);
      psum[r] += __shfl_xor_sync(0xffffffffu, psum[r], 2);
      lrow[r] = lrow[r] * corr[r] + psum[r];
    }
    // ---- O = O * corr + P V
#pragma unroll
    for (int dj = 0; dj < D / 8; dj += 2) {
      o[dj][0] *= corr[0];
      o[dj][1] *= corr[0];
      o[dj][2] *= corr[1];
      o[dj][3] *= corr[1];
      o[dj + 1][0] *= corr[0];
      o[dj + 1][1] *= corr[0];
      o[dj + 1][2] *= corr[1];
      o[dj + 1][3] *= corr[1];
#pragma unroll
      for (int kk = 0; kk < PF_K / 16; ++kk) {
        uint32_t vb[4];  // (keys kk*16 + 0..7 | 8..15) x (d chunks dj, dj+1), transposed on load
        ldsm_x4_t(vb, sV + sw(kk * 16 + (lane & 7) + 8 * ((lane >> 3) & 1), dj + (lane >> 4)));
        mma16816(o[dj], pa[kk], vb[0], vb[1]);
        mma16816(o[dj + 1], pa[kk], vb[2], vb[3]);
      }
    }
  }
  // ---- normalise and store
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int rr = warp * 16 + g + 8 * r;
    if (rr < nrows) {
      const float inv = 1.0f / lrow[r];
      bf16* dst = a.out + (size_t)(row0 + rr) * HD + head * D + 2 * t;
#pragma unroll
      for (int dj = 0; dj < D / 8; ++dj)
        *reinterpret_cast<uint32_t*>(dst + dj * 8) = pack_bf16(o[dj][2 * r] * inv, o[dj][2 * r + 1] * inv);
    }
  }
}

int attn_prefill_tile_rows() { return PF_Q; }

cudaError_t launch_attn_prefill(const AttnArgs& a, const LaunchCfg& lc) {
  if (a.n_tiles <= 0) return cudaSuccess;
  const size_t smem = (size_t)(PF_Q + 2 * PF_K) * a.head_dim * 2;
  static std::atomic<unsigned long long> attr_mask{0};  // per instantiation, per device
  if (first_launch_on_device(attr_mask)) {
    cudaFuncSetAttribute(attn_prefill_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (PF_Q + 2 * PF_K) * 128 * 2);
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(a.n_tiles, a.n_heads);
  cfg.blockDim = dim3(128);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = lc.stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = lc.pdl ? 1 : 0;
  if (a.head_dim == 128) return cudaLaunchKernelEx(&cfg, attn_prefill_kernel<128>, a);
  if (a.head_dim == 64) return cudaLaunchKernelEx(&cfg, attn_prefill_kernel<64>, a);
  return cudaErrorInvalidValue;
}
