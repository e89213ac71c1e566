// engine.h — the decode engine behind include/ssb.h (one engine = one GPU rank).
#pragma once
#include <cuda_runtime.h>

#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/ssb.h"
#include "json.h"
#include "kernels.h"
#include "loader.h"
#include "mega.h"
#include "tc_gemm.h"

namespace ssb {

struct ModelCfg {
  std::string model_type = "llama";
  int hidden = 0, inter = 0, layers = 0, heads = 0, kv_heads = 0, head_dim = 0, vocab = 0, max_pos = 0;
  float eps = 1e-5f, theta = 10000.f;
  bool tie_embeddings = false;
  bool falcon = false;  // Falcon new_decoder_architecture: LayerNorm(+bias) x2 on the same input, fused grouped QKV,
                        // GELU MLP, parallel block (HF:models/falcon/modeling_falcon.py:572-636)
};

struct LayerW {
  bf16 *wqkv = nullptr, *wo = nullptr, *wgu = nullptr, *wdown = nullptr, *ln1 = nullptr, *ln2 = nullptr;
  bf16 *ln1_b = nullptr, *ln2_b = nullptr;  // Falcon LayerNorm biases (wgu = dense_h_to_4h, wdown = dense_4h_to_h)
  TcTensorMap tm_qkv, tm_o, tm_gu, tm_down;  // TMA descriptors of the four projection matrices (tensor-core path)
};

struct SeqSlot {
  bool used = false;
  int len = 0;
  std::vector<int> blocks;
};

class Engine {
 public:
  Engine() = default;
  ~Engine();
  int init(const std::string& model_dir, const std::string& params_json);
  int info(ssb_info* out) const;
  int seq_create(int* id);
  int seq_free(int id);
  int seq_len(int id, int* len) const;
  void kv_blocks(int* total, int* free_now) const {
    *total = n_blocks_;
    *free_now = (int)free_blocks_.size();
  }
  int prefill(const int* seq_ids, const int32_t* tokens, const int* lens, int nseq, int32_t* next_tok, float* logits);
  int decode(const int* seq_ids, const int32_t* last_tok, int nseq, int nsteps, int32_t* out_tok, float* logits);
  int last_timing(ssb_timing* t) const;
  void timing_reset();
  int debug_read(const char* name, float* dst, int64_t n, int* rows, int* cols);
  int bench_kernel(const char* which, int rows, int ctx, int iters, double* ms_out, int64_t* bytes_out);
  int tp_export(void* handle_out);
  int tp_connect(const void* all_handles, int n_ranks);

 private:
  // setup
  int load_config(const std::string& dir, const Json& params);
  int alloc_weights();
  int fill_weights(const std::string& dir, bool synthetic, uint64_t seed, bool validate_only);
  int alloc_runtime(const Json& params);
  template <typename T>
  int dmalloc(T** p, size_t n);
  // run
  int ensure_blocks(int slot, int new_len);
  int ensure_blocks_all(const int* slot_ids, const int* new_lens, int n);
  int upload_block_rows(const std::vector<int>& slots);
  int forward(int M, int n_logit_rows, bool decode_mode);  // enqueue one forward over the staged rows
  int build_graph(int B);
  int forward_mega(int B);
  int forward_falcon(int M, int n_logit_rows, bool decode_mode);  // one persistent kernel for the whole decode step (B <= 4, single rank)
  LaunchCfg lc(bool pdl) const {
    LaunchCfg c{stream_, pdl && use_pdl_, n_sm_};
    c.sk_part = sk_part_;
    c.sk_flags = sk_flags_;
    c.sk_slots = sk_slots_;
    return c;
  }
  float* sk_part_ = nullptr;  // stream-K workspace of the tensor-core decode projections
  unsigned* sk_flags_ = nullptr;
  int sk_slots_ = 0;
  bool tp_presharded_ = false;  // weights come from <model_dir>/ssb_tp<N>/rank<r>.safetensors (this rank's slices only)

  ModelCfg cfg_;
  int tp_size_ = 1, tp_rank_ = 0, device_ = 0, n_sm_ = 132;
  int Hl_ = 0, KVHl_ = 0, Il_ = 0;  // per-rank heads / kv heads / intermediate
  int max_batch_ = 32, max_seq_ = 4096, block_size_ = 16, n_blocks_ = 0, max_blocks_per_seq_ = 0, m_max_ = 0;
  bool use_pdl_ = true, use_graph_ = true, taps_ = false;
  bool use_mega_ = true;
  MegaLayer* d_mega_layers_ = nullptr;
  float *mega_part_o_ = nullptr, *mega_part_ml_ = nullptr;
  int* mega_counters_ = nullptr;
  unsigned* mega_bar_ = nullptr;
  unsigned long long* mega_prof_ = nullptr;
  bool mega_prof_all_ = false;
  bool mega_attn_tile_ = true;
  int mega_max_batch_ = 1;  // params "mega_max_batch": largest batch the persistent kernel serves (above: graph of per-projection kernels)
  MegaGeom mega_geom(int rows) const {  // launch geometry of the persistent kernel for a batch of `rows` (mega.h)
    return mega_geometry(cfg_.hidden, Hl_, KVHl_, cfg_.head_dim, Il_, cfg_.layers, max_seq_, rows, mega_attn_tile_);
  }
  int tc_tn_prefill_ = 0;  // params "tc_tn_prefill": force the prefill token-tile width (0 = heuristic)
  int tc_min_rows_ = 5;  // forwards with >= this many token rows run the projections on the tensor cores (wgmma)
  cudaStream_t stream_ = nullptr;
  cudaEvent_t ev0_ = nullptr, ev1_ = nullptr;

  // weights
  std::vector<LayerW> lw_;
  bf16 *embed_ = nullptr, *lm_head_ = nullptr, *final_norm_ = nullptr, *final_norm_b_ = nullptr;
  TcTensorMap tm_lm_head_;
  bf16* ao_ = nullptr;  // Falcon: attention-branch output of the parallel block
  float* falcon_scratch_ = nullptr;  // Falcon TP: local fp32 partial of the attention branch
  uint32_t* rope_cs_ = nullptr;
  // KV pool: per layer [n_blocks][KVHl][block][D]
  bf16 *kpool_ = nullptr, *vpool_ = nullptr;
  size_t kv_layer_elems_ = 0;
  // activations
  bf16 *h_ = nullptr, *q_ = nullptr, *attn_ = nullptr, *act_ = nullptr, *xn_ = nullptr;
  float *logits_ = nullptr, *part_o_ = nullptr, *part_ml_ = nullptr;
  int *counters_ = nullptr, *row_tok_ = nullptr, *row_slot_ = nullptr, *row_pos_ = nullptr, *logit_rows_ = nullptr;
  int *next_tok_ = nullptr, *hist_ = nullptr, *step_ = nullptr, *block_table_ = nullptr;
  int max_steps_ = 0;
  int *tile_row0_ = nullptr, *tile_nrows_ = nullptr;  // prefill attention query tiles of the current forward
  int n_pf_tiles_ = 0;                                 // 0 => decode-style attention
  // tensor parallel exchange (peer-mapped over NVLink; see tp_allreduce_resid_kernel)
  // one exported pool per rank: [partials 2*m_max*h f32 | recv 2*8*max_batch*h f32 | flags 8 u32 (64 B) | pflags 8 u64]
  uint8_t* tp_pool_ = nullptr;
  size_t tp_pool_bytes_ = 0, tp_off_recv_ = 0, tp_off_flags_ = 0, tp_off_pflags_ = 0;
  float* tp_partials_ = nullptr;       // pull model (prefill / tensor-core path): fp32 partial sums of this rank
  float* tp_recv_ = nullptr;           // push model (decode): [2 parity][8 src][max_batch][hidden]
  uint32_t* tp_flags_ = nullptr;       // [8] epoch flags written by the peers (pull model)
  unsigned long long* tp_pflags_ = nullptr;  // [8] arrival counters, one per source rank (push model)
  int* tp_step_ = nullptr;             // forwards executed (device counter)
  int* tp_push_step_ = nullptr;        // push-model forwards executed (device counter)
  float** d_peer_partials_ = nullptr;  // [tp_size] device array of peer-mapped pointers
  uint32_t** d_peer_flags_ = nullptr;
  float** d_peer_recv_ = nullptr;
  unsigned long long** d_peer_pflags_ = nullptr;
  std::vector<void*> ipc_opened_;
  bool tp_connected_ = false, tp_push_ = false;
  // experimental two-shot prefill allreduce (tp_twoshot.cu): gather region appended to the exchange pool when enabled
  bool tp_two_shot_ = false;
  int tp_two_shot_min_rows_ = 64;
  size_t tp_off_gather_ = 0;
  bf16** d_peer_gather_ = nullptr;
  unsigned* tp2_done_ = nullptr;
  // "tp_mega": 2 — per-CTA exchange flags [8][256] u32, appended to the exchange pool when enabled
  int tp_mega_mode_ = 0;
  size_t tp_off_ctaflags_ = 0;
  uint32_t** d_peer_cta_flags_ = nullptr;
  // "tp_mega": 3 — LL push receive buffers [2 parity][8 src][4 rows][hidden/2] uint4, appended to the exchange pool
  size_t tp_off_ll_ = 0;
  bool tp_ll_ = true;  // params "tp_ll": LL push allreduce kernel for decode-sized forwards of the multi-kernel path
  uint4** d_peer_ll_ = nullptr;
  // taps
  bf16 *tap_q0_ = nullptr, *tap_attn0_ = nullptr, *tap_h0_ = nullptr;
  int tap_rows_ = 0;
  // host state
  ModelFiles files_;
  std::vector<SeqSlot> slots_;
  std::vector<int> free_blocks_;
  std::vector<int> host_bt_;
  std::map<int, cudaGraphExec_t> graphs_;
  std::map<int, int> graph_launches_;  // kernels in graphs_[B]: launches_per_forward_ is whatever forward ran last
  std::vector<void*> allocs_;
  size_t hbm_bytes_ = 0;
  int64_t weight_bytes_step_ = 0;
  int launches_per_forward_ = 0;
  // per-kernel-class event timing of one forward (params.profile_forward=1; tools/fwd_prof.py)
  bool prof_fwd_ = false;
  std::vector<std::pair<std::string, cudaEvent_t>> prof_marks_;
  std::map<std::string, double> prof_ms_;
  void prof_mark(const char* label);
  void prof_collect();
 public:
  std::string prof_report();
 private:
  // stats
  mutable ssb_timing timing_ = {};
  int decode_splits_(int M) const;
  int attn_splits_ = 0;
};

void set_error(const std::string& s);
const char* get_error();

}  // namespace ssb
