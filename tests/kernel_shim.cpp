// kernel_shim.cpp — test-only C entry points over the launchers of kernels.h / tc_gemm.h, so that
// tests/test_kernels_gpu.py can run one projection, attention, norm or argmax kernel at a time on torch-owned device
// buffers.  Built by the test with g++ and linked against the in-tree libsubstratus_b200.so; launches go to stream 0
// without programmatic dependent launch.  Each function returns the launcher's cudaError_t (or a negative code when a
// tensor map cannot be built).
#include "tc_gemm.h"

// Mirrored field for field by the ctypes structures in test_kernels_gpu.py: pointers first, then ints, then floats.
struct ShimProj {
  const void *W, *x, *row_map, *norm_w, *norm_b, *f32_add, *resid, *resid2, *rope_cs, *block_table, *row_slot, *row_pos;
  void *out_f32, *out_bf16, *q_out, *kcache, *vcache;
  int N, K, ldx, M, ld_out, q_rows, kv_rows, head_dim, bt_stride, block_size, kvh;
  float eps;
};

struct ShimAttn {
  const void *q, *kcache, *vcache, *block_table, *row_slot, *row_pos, *tile_row0, *tile_nrows;
  void *out, *part_o, *part_ml, *counters;
  int bt_stride, M, n_heads, kvh, group, head_dim, block_size, n_splits, n_tiles;
  float scale;
};

static GemvArgs gemv_args(const ShimProj& p) {
  GemvArgs a = {};
  a.W = (const bf16*)p.W;
  a.N = p.N;
  a.K = p.K;
  a.x = (const bf16*)p.x;
  a.ldx = p.ldx;
  a.M = p.M;
  a.row_map = (const int*)p.row_map;
  a.norm_w = (const bf16*)p.norm_w;
  a.norm_b = (const bf16*)p.norm_b;
  a.eps = p.eps;
  a.out_f32 = (float*)p.out_f32;
  a.out_bf16 = (bf16*)p.out_bf16;
  a.resid = (const bf16*)p.resid;
  a.resid2 = (const bf16*)p.resid2;
  a.f32_add = (const float*)p.f32_add;
  a.ld_out = p.ld_out;
  a.q_out = (bf16*)p.q_out;
  a.q_rows = p.q_rows;
  a.kv_rows = p.kv_rows;
  a.head_dim = p.head_dim;
  a.kcache = (bf16*)p.kcache;
  a.vcache = (bf16*)p.vcache;
  a.block_table = (const int*)p.block_table;
  a.bt_stride = p.bt_stride;
  a.row_slot = (const int*)p.row_slot;
  a.row_pos = (const int*)p.row_pos;
  a.rope_cs = (const uint32_t*)p.rope_cs;
  a.block_size = p.block_size;
  a.kvh = p.kvh;
  return a;
}

static AttnArgs attn_args(const ShimAttn& p) {
  AttnArgs a = {};
  a.q = (const bf16*)p.q;
  a.kcache = (const bf16*)p.kcache;
  a.vcache = (const bf16*)p.vcache;
  a.block_table = (const int*)p.block_table;
  a.bt_stride = p.bt_stride;
  a.row_slot = (const int*)p.row_slot;
  a.row_pos = (const int*)p.row_pos;
  a.out = (bf16*)p.out;
  a.part_o = (float*)p.part_o;
  a.part_ml = (float*)p.part_ml;
  a.counters = (int*)p.counters;
  a.M = p.M;
  a.n_heads = p.n_heads;
  a.kvh = p.kvh;
  a.group = p.group;
  a.head_dim = p.head_dim;
  a.block_size = p.block_size;
  a.n_splits = p.n_splits;
  a.scale = p.scale;
  a.tile_row0 = (const int*)p.tile_row0;
  a.tile_nrows = (const int*)p.tile_nrows;
  a.n_tiles = p.n_tiles;
  return a;
}

static LaunchCfg launch_cfg(int n_sm) {
  LaunchCfg lc;
  lc.stream = 0;
  lc.pdl = false;
  lc.n_sm = n_sm;
  return lc;
}

extern "C" {

int shim_gemv(const ShimProj* p, int epi, int norm, int n_sm) { return (int)launch_gemv(gemv_args(*p), epi, norm, launch_cfg(n_sm)); }

int shim_gemv_pick_bt(int M, int K) { return gemv_pick_bt(M, K); }

// sk_part == null: the tiled kernel (one CTA per 128-row weight tile and token tile); otherwise the stream-K kernel
// whenever M <= tn <= 64, as in the engine's batched decode
int shim_tc_gemm(const ShimProj* p, int epi, int tn, int n_sm, void* sk_part, void* sk_flags, int sk_slots) {
  TcTensorMap ta, tb;
  if (tc_make_tmap(&ta, (const bf16*)p->W, p->N, p->K, p->K, tc_weight_box_rows()) != cudaSuccess) return -1;
  if (tc_make_tmap(&tb, (const bf16*)p->x, p->M, p->K, p->ldx, tn) != cudaSuccess) return -2;
  LaunchCfg lc = launch_cfg(n_sm);
  lc.sk_part = (float*)sk_part;
  lc.sk_flags = (unsigned*)sk_flags;
  lc.sk_slots = sk_slots;
  return (int)launch_tc_gemm(ta, tb, tn, gemv_args(*p), epi, lc);
}

int shim_attn_decode(const ShimAttn* p) { return (int)launch_attn_decode(attn_args(*p), launch_cfg(1)); }

int shim_attn_prefill(const ShimAttn* p) { return (int)launch_attn_prefill(attn_args(*p), launch_cfg(1)); }

int shim_rmsnorm(const void* x, const void* w, void* out, int M, int K, float eps) {
  return (int)launch_rmsnorm((const bf16*)x, (const bf16*)w, (bf16*)out, M, K, eps, launch_cfg(1));
}

int shim_layernorm(const void* x, const void* w, const void* b, void* out, int M, int K, float eps) {
  return (int)launch_layernorm((const bf16*)x, (const bf16*)w, (const bf16*)b, (bf16*)out, M, K, eps, launch_cfg(1));
}

int shim_argmax(const void* logits, int V, int n_rows, void* tok_out, void* hist, const void* step, void* pos_inc) {
  return (int)launch_argmax((const float*)logits, V, n_rows, (int*)tok_out, (int*)hist, (const int*)step, (int*)pos_inc,
                            launch_cfg(1));
}

}  // extern "C"
