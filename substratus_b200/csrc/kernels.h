// kernels.h — host-visible launch API of the sm_90a decode kernels (plain structs, no torch).
#pragma once
#include <atomic>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

typedef __nv_bfloat16 bf16;

enum GemvEpi : int {
  EPI_F32 = 0,       // out_f32[m][n] = acc                      (TP partial sums, raw fp32)
  EPI_F32_BF16R = 1, // out_f32[m][n] = float(bf16(acc))          (lm_head logits: HF Linear output is bf16, then .float())
  EPI_RESID = 2,     // out_bf16[m][n] = bf16(float(bf16(acc)) + resid[m][n])   (o_proj / down_proj + residual)
  EPI_SWIGLU = 3,    // rows (2i,2i+1) = (gate_i, up_i): out_bf16[m][i] = bf16(bf16(silu(bf16 g)) * bf16 u)
  EPI_QKV_ROPE = 4,  // pair-interleaved q|k|v rows: RoPE on q,k; q -> q_out, k/v -> paged KV cache at (slot,pos)
  EPI_BF16 = 5,      // out_bf16[m][n] = bf16(acc + bias)
  EPI_F32_PUSH = 6,  // tensor parallel, decode: raw fp32 partial PUSHED into every rank's receive slot over NVLink
  EPI_GELU = 7,      // out_bf16[m][n] = bf16(gelu_erf(bf16(acc)))                       (Falcon dense_h_to_4h + act)
  EPI_RESID2 = 8,    // out_bf16[m][n] = bf16(bf16(bf16(acc) + resid2[m][n]) + resid[m][n]) (Falcon parallel block:
                     //                  mlp_out += attn_out; out = mlp_out + residual)
};

enum NormKind : int { NORM_NONE = 0, NORM_RMS = 1, NORM_LN = 2 };  // LN = LayerNorm with weight and bias (Falcon)

struct GemvArgs {
  // y[M, N] = x[M, K] * W[N, K]^T ; W bf16 row-major (physical row order, see DESIGN.md "weight layout")
  const bf16* W;
  int N, K;
  const bf16* x;  // [*, ldx]
  int ldx, M;
  const int* row_map;  // optional: tile row m reads x row row_map[m]
  const bf16* norm_w;  // NORM_RMS / NORM_LN: weight[K]
  const bf16* norm_b;  // NORM_LN: bias[K]
  float eps;
  // outputs
  float* out_f32;
  bf16* out_bf16;
  const bf16* resid;
  const bf16* resid2;    // EPI_RESID2
  const float* f32_add;  // EPI_F32: optional fp32 addend with the layout of out_f32 (Falcon TP: attn partial + mlp partial)
  int ld_out;
  // EPI_QKV_ROPE
  bf16* q_out;       // [M, q_rows]
  int q_rows;        // H_local * head_dim
  int kv_rows;       // KVH_local * head_dim
  int head_dim;
  bf16* kcache;      // this layer: [blocks][KVH_local][block_size][head_dim]
  bf16* vcache;
  const int* block_table;  // [slots][bt_stride]
  int bt_stride;
  const int* row_slot;     // [M]
  const int* row_pos;      // [M]
  const uint32_t* rope_cs; // [max_pos][head_dim/2] packed (cos bf16 | sin bf16 << 16)
  int block_size;
  int kvh;                 // KVH_local
  // EPI_F32_PUSH (row-parallel projection under tensor parallelism)
  float* const* push_dst;                 // [push_n] peer-mapped base of each rank's receive buffer
  unsigned long long* const* push_flags;  // [push_n] peer-mapped arrival counters, [push_n] entries each (one per source)
  long long push_off;                     // element offset of (parity, this rank)'s slot inside a receive buffer
  int push_n, push_rank;
  int n_stages;  // set by launch_gemv: ring stages that fit beside the staged activations (2..6)
};

struct AttnArgs {
  const bf16* q;  // [M, H_local*D]
  const bf16* kcache;
  const bf16* vcache;
  const int* block_table;
  int bt_stride;
  const int* row_slot;
  const int* row_pos;
  bf16* out;  // [M, H_local*D]
  float* part_o;  // [M][H_local/GC][n_splits][GC*D]   (GC = heads per CTA)
  float* part_ml; // [M][H_local/GC][n_splits][2*GC]
  int* counters;  // [M][H_local/GC], zero on entry, zero on exit
  int M, n_heads, kvh, group, head_dim, block_size, n_splits;
  float scale;
  // prefill (attn_prefill_kernel): query tiles of <= 64 consecutive rows of ONE sequence, consecutive positions
  const int* tile_row0;
  const int* tile_nrows;
  int n_tiles;
};

struct LaunchCfg {
  cudaStream_t stream;
  bool pdl;
  int n_sm;
  // per-engine fp32 partial-tile workspace of the stream-K decode GEMM (tc_gemm.cu); null => one CTA per 128-row tile
  float* sk_part = nullptr;
  unsigned* sk_flags = nullptr;  // [sk_slots], zero on entry and on exit
  int sk_slots = 0;
  unsigned long long* sk_prof = nullptr;  // [n_sm][8] phase stamps of the last stream-K launch (libraries built with -DTC_SK_PROF=1)
};

// cudaFuncSetAttribute is per device: returns true the first time it is called for `mask` on the current device.  TP rank
// threads (one per device) reach the same static mask concurrently, hence the atomic read-modify-write.
inline bool first_launch_on_device(std::atomic<unsigned long long>& mask) {
  int d = 0;
  cudaGetDevice(&d);
  const unsigned long long bit = 1ull << d;
  if (mask.load(std::memory_order_acquire) & bit) return false;
  return (mask.fetch_or(bit, std::memory_order_acq_rel) & bit) == 0;
}

cudaError_t launch_gemv(const GemvArgs& a, int epi, int norm, const LaunchCfg& lc);
int gemv_pick_bt(int M, int K);
int gemv_grid_ctas(int M, int N, int K, int n_sm);  // CTAs launch_gemv will use (arrival count of the push allreduce)
cudaError_t launch_attn_decode(const AttnArgs& a, const LaunchCfg& lc);
cudaError_t launch_attn_prefill(const AttnArgs& a, const LaunchCfg& lc);
int attn_prefill_tile_rows();  // query rows per prefill-attention tile (64)
// h[m][:] = embed[row_tok[m]][:]; thread 0 of block 0 also does (*step_counter)++ when non-null
cudaError_t launch_embed(const bf16* embed, const int* row_tok, bf16* h, int M, int hidden, int* step_counter,
                         int* fwd_counter, int* push_counter, const LaunchCfg& lc);
// greedy pick per row (lowest index wins ties, as torch.argmax on CPU): tok_out[r] = argmax logits[r][:]
// hist != null: hist[(*step) * n_rows + r] = tok ; pos_inc != null: pos_inc[r] += 1
cudaError_t launch_argmax(const float* logits, int V, int n_rows, int* tok_out, int* hist, const int* step,
                          int* pos_inc, const LaunchCfg& lc);

// ---- load-time kernels
// dst[r*dst_ld + c] = bf16(src[row_idx[r]][col0 + c]), src element type: 0 bf16, 1 f16, 2 f32
cudaError_t launch_gather_rows(bf16* dst, int64_t dst_ld, const void* src, int src_dtype, int64_t src_ld,
                               const int* row_idx, int rows, int col0, int cols, cudaStream_t s);
// dst[r*dst_ld + c] = synth(seed, tid, row_idx[r]*full_cols + col0 + c)  (row_idx null => identity)
cudaError_t launch_synth_fill(bf16* dst, int64_t dst_ld, const int* row_idx, int rows, int col0, int cols, int64_t full_cols,
                              uint64_t seed, uint32_t tid, float amp, float base, cudaStream_t s);
void synth_fill_host(uint64_t seed, uint32_t tid, int64_t start, int64_t n, float amp, float base, uint16_t* dst);
cudaError_t launch_bf16_to_f32(const bf16* src, float* dst, int64_t n, cudaStream_t s);

// ---- tensor-parallel exchange (one-shot allreduce over NVLink peer memory, fused with the residual add)
struct TpArgs {
  int rank, size;
  float* const* peer_partials;   // [size] device pointers (peer-mapped) to each rank's partial buffer [2][rows_max][hidden]
  uint32_t* const* peer_flags;   // [size] device pointers to each rank's flag array [size] (flags live at the RECEIVER)
  const int* tp_step;            // device counter, +1 per forward (same on every rank)
  int seq_in_step, n_per_step;   // index of this allreduce inside the forward, allreduces per forward
  int parity_stride;             // elements between the two parity buffers (rows_max * hidden)
  int M, hidden;
  const bf16* resid;             // [M][hidden] local residual stream
  bf16* out;                     // [M][hidden] (may alias resid)
  int variant;                   // latency experiments (tools/tp_bench.py): bit0 no fence.sys before the flag store,
                                 // bit1 poll with relaxed loads + one acquire fence, bit2 push model (write partials
                                 // into the peers' slots, read locally)
};
cudaError_t launch_tp_allreduce_resid(const TpArgs& a, const LaunchCfg& lc);
// decode-sized (M <= 4) allreduce + residual with the LL wire format (16-byte {v0, epoch, v1, epoch} pushed into every
// rank's receive slots [parity][src][row][pair], receiver polls its own slots): same TpArgs (partials, epoch, residual)
struct TpLlArgs {
  uint4* const* peer_ll;                 // [size] peer-mapped receive buffers
  long long parity_stride, src_stride;   // in uint4 units
};
cudaError_t launch_tp_allreduce_ll(const TpArgs& a, const TpLlArgs& l, const LaunchCfg& lc);

// two-shot allreduce for prefill-sized activations (tp_twoshot.cu; params "tp_two_shot", experimental): each rank
// reduces its 1/size slice and the bf16 slices are gathered through `peer_gather` (one [rows_max][hidden] bf16 buffer per
// rank in the exchange pool).  "slice ready" flags are entries [8 + src] of the receiver's flag array.
struct TpArgs2 {
  int rank, size;
  float* const* peer_partials;
  uint32_t* const* peer_flags;
  bf16* const* peer_gather;
  const int* tp_step;
  int seq_in_step, n_per_step;
  long long parity_stride;
  int M, hidden;
  const bf16* resid;
  bf16* out;
  unsigned* done;  // CTA-completion counter (this rank's memory), zero on entry and on exit
};
cudaError_t launch_tp_allreduce2(const TpArgs2& a, const LaunchCfg& lc);

// push-model reduce (decode): partials were pushed into recv[parity][src][M][hidden] by the GEMV epilogues of all
// ranks; wait until every source's arrival counter reached `target`, sum the slots in rank order, add the residual.
struct TpPushArgs {
  int size;
  const float* recv;                   // this rank's receive buffer
  const unsigned long long* flags;     // this rank's arrival counters [size]
  const int* tp_step;
  int seq_in_step, n_per_step;
  unsigned long long arrivals_per_epoch;  // CTAs of the producing GEMV grid (each adds 1 per allreduce)
  long long parity_stride, src_stride;    // elements
  int M, hidden;
  const bf16* resid;
  bf16* out;
};
cudaError_t launch_tp_reduce_push(const TpPushArgs& a, const LaunchCfg& lc);

// GGUF block dequantisation (dequant.cu): src = raw tensor bytes on the device, dtype = ssb::DType, n elements
cudaError_t launch_dequant(const void* src, int dtype, int64_t n, bf16* dst, cudaStream_t s);
