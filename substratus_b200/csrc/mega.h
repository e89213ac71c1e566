// mega.h — launch API of the persistent single-kernel decode step (mega.cu).
#pragma once
#include "kernels.h"

struct MegaLayer {
  const bf16 *wqkv, *wo, *wgu, *wdown, *ln1, *ln2;
  bf16 *kcache, *vcache;
};

struct MegaArgs {
  const MegaLayer* layers;  // device array [n_layers]
  int n_layers;
  int hidden, q_rows, kv_rows, head_dim, inter, vocab;
  int n_heads, kvh, group, attn_g;  // attn_g = query heads per attention unit (all share one KV head)
  float eps, scale;
  int M;  // batch rows (1..4)
  const bf16 *embed, *lm_head, *final_norm;
  bf16 *h, *q, *attn, *act;
  float* logits;
  int* row_tok;
  const int* row_slot;
  int* row_pos;
  const int* block_table;
  int bt_stride, block_size;
  const uint32_t* rope_cs;
  float *part_o, *part_ml;  // [M][n_heads/attn_g][max_chunks][attn_g*D], [..][attn_g*2]
  int* counters;            // [M][n_heads/attn_g], zero on entry and on exit
  int max_chunks;
  int *hist, *step, *fwd_counter;
  unsigned* grid_bar;  // [mega_bar_words(n_layers)], zero on entry and on exit: [0] barrier, [1] exit counter,
                       // [MEGA_CLAIM_OFF + 4 * layer + matrix] pass claims (mega.cu: part_range)
  int n_stages, k_max;
  unsigned long long* prof;  // optional globaltimer stamps (params.mega_prof): [1024] of CTA 0, or with prof_all [n_ctas][1024]
                             // (entry 1023 of a CTA's row = its %smid) — per-phase arrival skew across the SMs
  // ---- tensor parallel (params.json "tp_mega": 1; new fields stay at the END so the single-GPU instantiations keep
  // their parameter layout).  tp_size > 1 selects decode_mega_kernel<.., TP=true>: the row-parallel projections (o,
  // down) leave fp32 partials in this rank's exchange buffer and every allreduce is
  //   grid barrier -> flag to the peers -> wait for the peers' flags -> each CTA pulls ITS slice of [M, hidden] from all
  //   ranks over NVLink, adds the residual, writes h -> grid barrier
  // i.e. one extra grid barrier and one NVLink round trip per allreduce, no kernel boundary (same epochs, flags and
  // parity double-buffering as tp_allreduce_resid_kernel, so prefill through the multi-kernel path interleaves freely).
  int tp_size, tp_rank;
  float* const* peer_partials;  // [tp_size] peer-mapped partial buffers [2][rows_max][hidden]
  uint32_t* const* peer_flags;  // [tp_size] flag arrays [tp_size], living at the receiver
  long long parity_stride;      // elements between the two parity buffers
  // "tp_mega": 2 — per-CTA exchange instead of a grid-wide one: CTA c of every rank produces the SAME output range of the
  // row-parallel projection (same grid, same dims), so it only needs the partials of the peers' CTA c.  It flags them
  // (flag [src rank][cta] at the receiver), waits for theirs, pulls their range, adds its own partial and the residual and
  // writes its range of h; the phase then ends with the ordinary grid barrier.  One grid barrier less per allreduce than
  // mode 1 and no GPU-wide skew wait.
  int tp_mode;                       // 1 | 2 | 3
  uint32_t* const* peer_cta_flags;   // [tp_size] -> u32 [8][256] at each receiver
  // "tp_mega": 3 — low-latency PUSH exchange (the wire format of NCCL's LL protocol): the row-parallel epilogue stores
  // every fp32 partial pair straight into all ranks' receive slots as ONE 16-byte word {v0, epoch, v1, epoch}; the
  // receiver polls the slot itself until both epoch halves match, so there is no separate flag, no fence and no remote
  // read on the critical path (one NVLink one-way latency per allreduce instead of flag + pull round trip).  Slots:
  // ll[parity][src rank][row][pair] (uint4), CTA c of every rank owns the same pair range, so only same-index CTAs talk.
  uint4* const* peer_ll;             // [tp_size] peer-mapped receive buffers
  long long ll_parity_stride, ll_src_stride;  // in uint4 units
  int prof_all;                      // params.mega_prof = 2: every CTA stamps
  int attn_cta_tile;                 // GQA groups of 8: one (row, KV head, split) per CTA with K/V staged in shared memory
  int attn_coop;                     // groups of 1 / 2 / 4: one (row, head unit, split) per CTA, warps combined through shared memory
  // QKV -> attention without a grid barrier ("mega_head_flags", default on with the CTA-level attention forms): head_done[slot]
  // counts the row pairs of q head / k head / v head `slot` whose epilogue has run in this launch (slots: n_heads q, kvh k, kvh v;
  // head_dim/2 pairs each per layer); an attention unit waits only for the heads it reads.  Zeroed by the kernel at entry.
  unsigned* head_done;
};

constexpr int MEGA_CLAIM_OFF = 1024;  // below: the barrier counters, including the tree-barrier experiment's 16 groups
inline size_t mega_bar_words(int n_layers) { return MEGA_CLAIM_OFF + 4 * (size_t)n_layers + 1; }
size_t mega_smem_bytes(int bt, int k_max, int n_stages);
int mega_pick_stages(int bt, int k_max);  // 0 if the step does not fit
int mega_attn_group(int group);
int mega_attn_chunk(int head_dim, int g);  // tokens per attention unit
size_t mega_attn_coop_bytes(int head_dim, int g);  // shared memory of the CTA-cooperative attention (groups of 1 / 2 / 4)
size_t mega_attn_tile_bytes(int head_dim);  // shared memory the CTA-tile attention stages K/V in (must fit the activation area)
cudaError_t launch_decode_mega(const MegaArgs& a, const LaunchCfg& lc);
