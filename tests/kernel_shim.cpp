// kernel_shim.cpp — test-only C entry points over the launchers of kernels.h / tc_gemm.h / mega.h, so that
// tests/test_kernels_gpu.py, tests/test_mega_kernel_gpu.py and tests/test_tp_exchange_gpu.py can run one projection,
// attention, norm, argmax or tensor-parallel exchange kernel, or one persistent decode step, at a time on torch-owned
// device buffers.  Built by the tests with g++ and linked against the
// in-tree libsubstratus_b200.so; launches go to stream 0 without programmatic dependent launch.  Each function returns the
// launcher's cudaError_t (or a negative code when a tensor map cannot be built).
#include <cmath>
#include <cstddef>

#include "mega.h"
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

// The persistent decode kernel (mega.cu) on one GPU.  layers = device array of MegaLayer, which the test builds as int64
// [n_layers][8] in field order.  Everything the launch geometry decides (k_max, n_stages, max_chunks, the attention form) comes
// from mega_geometry, never from the caller: a wrong value would overrun shared memory in a kernel full of spin-waits.
struct ShimMega {
  const void *layers, *embed, *lm_head, *final_norm, *row_slot, *block_table, *rope_cs;
  void *h, *q, *attn, *act, *logits, *row_tok, *row_pos, *part_o, *part_ml, *counters, *hist, *step, *fwd_counter, *grid_bar;
  int n_layers, hidden, n_heads, kvh, head_dim, inter, vocab, M, bt_stride, block_size, max_seq, attn_tile;
  float eps;
};
static_assert(sizeof(MegaLayer) == 8 * sizeof(void*) && offsetof(MegaLayer, ln2) == 5 * sizeof(void*) &&
                  offsetof(MegaLayer, vcache) == 7 * sizeof(void*),
              "tests/test_mega_kernel_gpu.py lays MegaLayer out as 8 pointers: wqkv wo wgu wdown ln1 ln2 kcache vcache");

static MegaGeom shim_geom(const ShimMega& p) {
  return mega_geometry(p.hidden, p.n_heads, p.kvh, p.head_dim, p.inter, p.n_layers, p.max_seq, p.M, p.attn_tile != 0);
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

// out[11] = attn_g, k_max, max_chunks, bt, n_stages, attn_coop, attn_cta_tile, then the buffer sizes part_o, part_ml,
// counters, grid_bar (elements), so that the test sizes every buffer from the geometry the launch uses
void shim_mega_geometry(const ShimMega* p, long long* out) {
  const MegaGeom g = shim_geom(*p);
  const long long v[11] = {g.attn_g, g.k_max, g.max_chunks, g.bt, g.n_stages, g.attn_coop, g.attn_cta_tile,
                           (long long)g.part_o_floats, (long long)g.part_ml_floats, (long long)g.counter_ints, (long long)g.bar_words};
  for (int i = 0; i < 11; ++i) out[i] = v[i];
}

}  // extern "C"

static MegaArgs mega_args(const ShimMega* p, const MegaGeom& g) {
  MegaArgs a = {};
  a.layers = (const MegaLayer*)p->layers;
  a.n_layers = p->n_layers;
  a.hidden = p->hidden;
  a.q_rows = p->n_heads * p->head_dim;
  a.kv_rows = p->kvh * p->head_dim;
  a.head_dim = p->head_dim;
  a.inter = p->inter;
  a.vocab = p->vocab;
  a.n_heads = p->n_heads;
  a.kvh = p->kvh;
  a.group = p->n_heads / p->kvh;
  a.attn_g = g.attn_g;
  a.eps = p->eps;
  a.scale = 1.0f / sqrtf((float)p->head_dim);  // as Engine::forward_mega
  a.M = p->M;
  a.embed = (const bf16*)p->embed;
  a.lm_head = (const bf16*)p->lm_head;
  a.final_norm = (const bf16*)p->final_norm;
  a.h = (bf16*)p->h;
  a.q = (bf16*)p->q;
  a.attn = (bf16*)p->attn;
  a.act = (bf16*)p->act;
  a.logits = (float*)p->logits;
  a.row_tok = (int*)p->row_tok;
  a.row_slot = (const int*)p->row_slot;
  a.row_pos = (int*)p->row_pos;
  a.block_table = (const int*)p->block_table;
  a.bt_stride = p->bt_stride;
  a.block_size = p->block_size;
  a.rope_cs = (const uint32_t*)p->rope_cs;
  a.part_o = (float*)p->part_o;
  a.part_ml = (float*)p->part_ml;
  a.counters = (int*)p->counters;
  a.max_chunks = g.max_chunks;
  a.hist = (int*)p->hist;
  a.step = (int*)p->step;
  a.fwd_counter = (int*)p->fwd_counter;
  a.grid_bar = (unsigned*)p->grid_bar;
  a.n_stages = g.n_stages;
  a.k_max = g.k_max;
  a.attn_coop = g.attn_coop;
  a.attn_cta_tile = g.attn_cta_tile;
  return a;
}

// ---- tensor-parallel exchange, one rank at a time (tests/test_tp_exchange_gpu.py).  Every pointer array (peer_*,
// push_dst, push_flags) is a DEVICE array of device pointers, as the kernels dereference it on the device.
struct ShimTpArgs {  // TpArgs
  const void *peer_partials, *peer_flags, *tp_step, *resid;
  void* out;
  int rank, size, seq_in_step, n_per_step, parity_stride, M, hidden, variant;
};

struct ShimTp2 {  // TpArgs2
  const void *peer_partials, *peer_flags, *peer_gather, *tp_step, *resid;
  void *out, *done;
  int rank, size, seq_in_step, n_per_step, M, hidden;
  long long parity_stride;
};

struct ShimTpPush {  // TpPushArgs
  const void *recv, *flags, *tp_step, *resid;
  void* out;
  int size, seq_in_step, n_per_step, M, hidden;
  long long arrivals_per_epoch, parity_stride, src_stride;
};

struct ShimTp {  // the tensor-parallel fields of MegaArgs
  const void *peer_partials, *peer_flags, *peer_cta_flags, *peer_ll;
  int tp_size, tp_rank, tp_mode;
  long long parity_stride;
};

static TpArgs tp_args(const ShimTpArgs& p) {
  TpArgs a = {};
  a.rank = p.rank;
  a.size = p.size;
  a.peer_partials = (float* const*)p.peer_partials;
  a.peer_flags = (uint32_t* const*)p.peer_flags;
  a.tp_step = (const int*)p.tp_step;
  a.seq_in_step = p.seq_in_step;
  a.n_per_step = p.n_per_step;
  a.parity_stride = p.parity_stride;
  a.M = p.M;
  a.hidden = p.hidden;
  a.resid = (const bf16*)p.resid;
  a.out = (bf16*)p.out;
  a.variant = p.variant;
  return a;
}

extern "C" {

// tp_size = 0 (single GPU), no profile stamps; cudaErrorInvalidValue without launching when the step does not
// fit the kernel's shared memory
int shim_decode_mega(const ShimMega* p, int n_sm) {
  const MegaGeom g = shim_geom(*p);
  if (g.n_stages == 0) return (int)cudaErrorInvalidValue;
  return (int)launch_decode_mega(mega_args(p, g), launch_cfg(n_sm));
}

// The tensor-parallel instantiation (decode_mega_kernel<.., TP=true>) as rank t->tp_rank of t->tp_size, with the LL strides
// of Engine::forward_mega: 4 rows of hidden/2 pairs per source, 8 sources per parity.
int shim_decode_mega_tp(const ShimMega* p, const ShimTp* t, int n_sm) {
  const MegaGeom g = shim_geom(*p);
  if (g.n_stages == 0) return (int)cudaErrorInvalidValue;
  MegaArgs a = mega_args(p, g);
  a.tp_size = t->tp_size;
  a.tp_rank = t->tp_rank;
  a.tp_mode = t->tp_mode;
  a.peer_partials = (float* const*)t->peer_partials;
  a.peer_flags = (uint32_t* const*)t->peer_flags;
  a.parity_stride = t->parity_stride;
  a.peer_cta_flags = (uint32_t* const*)t->peer_cta_flags;
  a.peer_ll = (uint4* const*)t->peer_ll;
  a.ll_src_stride = 4LL * (p->hidden / 2);
  a.ll_parity_stride = 8 * a.ll_src_stride;
  return (int)launch_decode_mega(a, launch_cfg(n_sm));
}

int shim_tp_allreduce_resid(const ShimTpArgs* p) { return (int)launch_tp_allreduce_resid(tp_args(*p), launch_cfg(1)); }

int shim_tp_allreduce_ll(const ShimTpArgs* p, const void* peer_ll, long long parity_stride, long long src_stride) {
  TpLlArgs l = {};
  l.peer_ll = (uint4* const*)peer_ll;
  l.parity_stride = parity_stride;
  l.src_stride = src_stride;
  return (int)launch_tp_allreduce_ll(tp_args(*p), l, launch_cfg(1));
}

// n_sm caps the two-shot grid
int shim_tp_allreduce2(const ShimTp2* p, int n_sm) {
  TpArgs2 a = {};
  a.rank = p->rank;
  a.size = p->size;
  a.peer_partials = (float* const*)p->peer_partials;
  a.peer_flags = (uint32_t* const*)p->peer_flags;
  a.peer_gather = (bf16* const*)p->peer_gather;
  a.tp_step = (const int*)p->tp_step;
  a.seq_in_step = p->seq_in_step;
  a.n_per_step = p->n_per_step;
  a.parity_stride = p->parity_stride;
  a.M = p->M;
  a.hidden = p->hidden;
  a.resid = (const bf16*)p->resid;
  a.out = (bf16*)p->out;
  a.done = (unsigned*)p->done;
  return (int)launch_tp_allreduce2(a, launch_cfg(n_sm));
}

int shim_tp_reduce_push(const ShimTpPush* p) {
  TpPushArgs a = {};
  a.size = p->size;
  a.recv = (const float*)p->recv;
  a.flags = (const unsigned long long*)p->flags;
  a.tp_step = (const int*)p->tp_step;
  a.seq_in_step = p->seq_in_step;
  a.n_per_step = p->n_per_step;
  a.arrivals_per_epoch = (unsigned long long)p->arrivals_per_epoch;
  a.parity_stride = p->parity_stride;
  a.src_stride = p->src_stride;
  a.M = p->M;
  a.hidden = p->hidden;
  a.resid = (const bf16*)p->resid;
  a.out = (bf16*)p->out;
  return (int)launch_tp_reduce_push(a, launch_cfg(1));
}

// the GEMV with EPI_F32_PUSH: the fp32 partial goes to slot push_off of every push_dst[r], then each CTA adds 1 to
// push_flags[r][push_rank]
int shim_gemv_push(const ShimProj* p, const void* push_dst, const void* push_flags, long long push_off, int push_n, int push_rank,
                   int n_sm) {
  GemvArgs a = gemv_args(*p);
  a.push_dst = (float* const*)push_dst;
  a.push_flags = (unsigned long long* const*)push_flags;
  a.push_off = push_off;
  a.push_n = push_n;
  a.push_rank = push_rank;
  return (int)launch_gemv(a, EPI_F32_PUSH, NORM_NONE, launch_cfg(n_sm));
}

int shim_gemv_grid_ctas(int M, int N, int K, int n_sm) { return gemv_grid_ctas(M, N, K, n_sm); }

}  // extern "C"
