// engine.cu — host side of the H100 decode engine: model load, paged-KV bookkeeping, CUDA-graph'd decode loop.
//
// Stands in for the model-load + generate path of the external serving image the reference's ServerReconciler
// launches (internal/controller/server_controller.go:114-205; container contract docs/container-contract.md:25-55).
// Forward structure = HF LlamaModel.forward / LlamaDecoderLayer.forward (HF:models/llama/modeling_llama.py:292-332,
// 355-500); greedy loop = HF:generation/utils.py:2658-2800.  No CPU fallback anywhere: init() fails with
// SSB_ENODEV when there is no sm_90 device.
#include <sys/stat.h>
#include "engine.h"
#include "tokenizer.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <unistd.h>

namespace ssb {

static thread_local std::string g_err;
void set_error(const std::string& s) { g_err = s; }
const char* get_error() { return g_err.c_str(); }

#define CK(expr)                                                                                         \
  do {                                                                                                   \
    cudaError_t _e = (expr);                                                                             \
    if (_e != cudaSuccess) {                                                                             \
      set_error(std::string(#expr) + ": " + cudaGetErrorString(_e) + " (" + __FILE__ + ":" + std::to_string(__LINE__) + ")"); \
      return SSB_ECUDA;                                                                                  \
    }                                                                                                    \
  } while (0)
#define RET(code, msg)   \
  do {                   \
    set_error(msg);      \
    return (code);       \
  } while (0)
#define TRY(expr)            \
  do {                       \
    int _r = (expr);         \
    if (_r != SSB_OK) return _r; \
  } while (0)

// synthetic-weight conventions; twins of oracle/synth.py (W_AMP, LMHEAD_GAIN, NORM_AMP, tensor ids)
static const float kWAmp = 0.02f * 1.7320508075688772f;
static const float kLmHeadGain = 4.0f;
static const float kNormAmp = 0.1f;
enum { K_Q = 0, K_K, K_V, K_O, K_GATE, K_UP, K_DOWN, K_LN1, K_LN2 };
static const uint32_t kGlobal = 1u << 20;

Engine::~Engine() {
  if (device_ >= 0) cudaSetDevice(device_);
  for (auto& g : graphs_) cudaGraphExecDestroy(g.second);
  for (void* p : ipc_opened_) cudaIpcCloseMemHandle(p);
  for (void* p : allocs_) cudaFree(p);
  if (ev0_) cudaEventDestroy(ev0_);
  if (ev1_) cudaEventDestroy(ev1_);
  if (stream_) cudaStreamDestroy(stream_);
}

template <typename T>
int Engine::dmalloc(T** p, size_t n) {
  void* v = nullptr;
  size_t bytes = std::max<size_t>(n * sizeof(T), 256);
  cudaError_t e = cudaMalloc(&v, bytes);
  if (e != cudaSuccess) {
    set_error(std::string("cudaMalloc(") + std::to_string(bytes) + "): " + cudaGetErrorString(e));
    return SSB_ENOMEM;
  }
  allocs_.push_back(v);
  hbm_bytes_ += bytes;
  *p = (T*)v;
  return SSB_OK;
}

int Engine::load_config(const std::string& dir, const Json& params) {
  if (files_.is_gguf()) {
    // GGUF carries its own hyper-parameters (llama.cpp convention `<arch>.<key>`); there is no config.json
    // (examples/llama2-13b-chat-gguf/base-model.yaml:8-9 stores a single `model.bin`).
    const Json& m = files_.gguf_meta();
    const std::string arch = m.get_str("general.architecture", "llama");
    if (arch != "llama") RET(SSB_EINVAL, "GGUF architecture '" + arch + "' is not supported (llama only)");
    cfg_.model_type = "llama";
    cfg_.hidden = (int)m.get_int(arch + ".embedding_length", 0);
    cfg_.inter = (int)m.get_int(arch + ".feed_forward_length", 0);
    cfg_.layers = (int)m.get_int(arch + ".block_count", 0);
    cfg_.heads = (int)m.get_int(arch + ".attention.head_count", 0);
    cfg_.kv_heads = (int)m.get_int(arch + ".attention.head_count_kv", cfg_.heads);
    cfg_.head_dim = (int)m.get_int(arch + ".attention.key_length", cfg_.heads ? cfg_.hidden / cfg_.heads : 0);
    cfg_.max_pos = (int)m.get_int(arch + ".context_length", 2048);
    cfg_.eps = (float)m.get_num(arch + ".attention.layer_norm_rms_epsilon", 1e-5);
    cfg_.theta = (float)m.get_num(arch + ".rope.freq_base", 10000.0);
    const TensorView* te = files_.find("token_embd.weight");
    if (!te) RET(SSB_EIO, "GGUF file has no token_embd.weight");
    cfg_.vocab = (int)te->rows();
    cfg_.tie_embeddings = files_.find("output.weight") == nullptr;
  } else {
  std::string txt;
  if (!read_text_file(dir + "/config.json", &txt)) RET(SSB_EIO, "cannot read " + dir + "/config.json");
  Json c;
  try {
    c = json_parse(txt);
  } catch (std::exception& e) {
    RET(SSB_EINVAL, std::string("config.json: ") + e.what());
  }
  cfg_.model_type = c.get_str("model_type", "llama");
  if (cfg_.model_type != "llama" && cfg_.model_type != "falcon")
    RET(SSB_EINVAL, "unsupported model_type '" + cfg_.model_type + "' (llama and falcon families)");
  cfg_.falcon = cfg_.model_type == "falcon";
  cfg_.hidden = (int)c.get_int("hidden_size", 0);
  cfg_.inter = (int)c.get_int("intermediate_size", 0);
  cfg_.layers = (int)c.get_int("num_hidden_layers", 0);
  cfg_.heads = (int)c.get_int("num_attention_heads", 0);
  cfg_.kv_heads = (int)c.get_int("num_key_value_heads", cfg_.heads);
  if (cfg_.falcon) {
    // examples/falcon-40b: new_decoder_architecture (two LayerNorms, grouped fused QKV, parallel block), no biases, RoPE
    if (c.get_num("new_decoder_architecture", 0) == 0) RET(SSB_EINVAL, "falcon: only new_decoder_architecture=true (falcon-40b class) is supported");
    if (c.get_num("alibi", 0) != 0 || c.get_num("bias", 0) != 0) RET(SSB_EINVAL, "falcon: alibi / linear biases are not supported");
    if (c.has("num_ln_in_parallel_attn") && c.get_int("num_ln_in_parallel_attn", 2) != 2) RET(SSB_EINVAL, "falcon: num_ln_in_parallel_attn must be 2");
    cfg_.kv_heads = (int)c.get_int("num_kv_heads", cfg_.heads);
    cfg_.inter = (int)c.get_int("ffn_hidden_size", 4 * cfg_.hidden);
  }
  cfg_.head_dim = (int)c.get_int("head_dim", cfg_.heads ? cfg_.hidden / cfg_.heads : 0);
  cfg_.vocab = (int)c.get_int("vocab_size", 0);
  cfg_.max_pos = (int)c.get_int("max_position_embeddings", 2048);
  cfg_.eps = (float)c.get_num(cfg_.falcon ? "layer_norm_epsilon" : "rms_norm_eps", cfg_.falcon ? 1e-5 : 1e-6);
  cfg_.theta = (float)c.get_num("rope_theta", 10000.0);
  if (const Json* rp = c.find("rope_parameters"))
    if (rp->kind == Json::Obj) cfg_.theta = (float)rp->get_num("rope_theta", cfg_.theta);
  if (const Json* rs = c.find("rope_scaling"))
    if (rs->kind == Json::Obj && rs->get_str("rope_type", rs->get_str("type", "default")) != "default")
      RET(SSB_EINVAL, "rope_scaling other than 'default' is not supported");
  cfg_.tie_embeddings = c.get_num("tie_word_embeddings", 0) != 0;
  }
  if (cfg_.hidden <= 0 || cfg_.inter <= 0 || cfg_.layers <= 0 || cfg_.heads <= 0 || cfg_.vocab <= 0)
    RET(SSB_EINVAL, "config.json: missing model dimensions");
  if (cfg_.head_dim != 64 && cfg_.head_dim != 128) RET(SSB_EINVAL, "head_dim must be 64 or 128");
  if (cfg_.hidden % 8 || cfg_.inter % 8 || cfg_.vocab % 2) RET(SSB_EINVAL, "hidden/intermediate must be multiples of 8, vocab even");
  if (cfg_.heads % cfg_.kv_heads) RET(SSB_EINVAL, "num_attention_heads must be a multiple of num_key_value_heads");
  const int group = cfg_.heads / cfg_.kv_heads;
  if (group > 8 && group % 8) RET(SSB_EINVAL, "GQA group must be <= 8 or a multiple of 8");
  tp_size_ = (int)params.get_int("tp_size", 1);
  tp_rank_ = (int)params.get_int("tp_rank", 0);
  if (tp_size_ < 1 || tp_rank_ < 0 || tp_rank_ >= tp_size_) RET(SSB_EINVAL, "bad tp_size/tp_rank");
  if (cfg_.kv_heads % tp_size_ || cfg_.inter % (8 * tp_size_)) RET(SSB_EINVAL, "tp_size must divide kv heads and intermediate_size/8");
  Hl_ = cfg_.heads / tp_size_;
  KVHl_ = cfg_.kv_heads / tp_size_;
  Il_ = cfg_.inter / tp_size_;
  return SSB_OK;
}

int Engine::alloc_weights() {
  const size_t h = cfg_.hidden, D = cfg_.head_dim;
  const size_t qkv_rows = (size_t)(Hl_ + 2 * KVHl_) * D;
  lw_.resize(cfg_.layers);
  for (auto& w : lw_) {
    TRY(dmalloc(&w.wqkv, qkv_rows * h));
    TRY(dmalloc(&w.wo, h * (size_t)Hl_ * D));
    TRY(dmalloc(&w.wgu, (cfg_.falcon ? 1 : 2) * (size_t)Il_ * h));
    TRY(dmalloc(&w.wdown, h * (size_t)Il_));
    TRY(dmalloc(&w.ln1, h));
    TRY(dmalloc(&w.ln2, h));
    if (cfg_.falcon) {
      TRY(dmalloc(&w.ln1_b, h));
      TRY(dmalloc(&w.ln2_b, h));
    }
  }
  if (cfg_.falcon) TRY(dmalloc(&final_norm_b_, h));
  TRY(dmalloc(&embed_, (size_t)cfg_.vocab * h));
  if (cfg_.tie_embeddings)
    lm_head_ = embed_;
  else
    TRY(dmalloc(&lm_head_, (size_t)cfg_.vocab * h));
  TRY(dmalloc(&final_norm_, h));
  weight_bytes_step_ = 2 * ((int64_t)cfg_.layers * (int64_t)(qkv_rows * h + h * Hl_ * D + (cfg_.falcon ? 2 : 3) * (size_t)Il_ * h) +
                            (int64_t)cfg_.vocab * h);
  return SSB_OK;
}

// One destination matrix region filled either from a checkpoint tensor or from the synthetic generator.
struct FillJob {
  bf16* dst;            // destination (row r at dst + r*dst_ld)
  int64_t dst_ld;
  std::vector<int> rows;  // logical source rows (empty => identity 0..n_rows-1)
  int n_rows;
  int col0, cols;
  int64_t full_cols;    // logical columns of the HF tensor
  std::string name;     // HF tensor name
  uint32_t tid;
  float amp, base;
};

int Engine::fill_weights(const std::string& dir, bool synthetic, uint64_t seed, bool validate_only) {
  const int h = cfg_.hidden, D = cfg_.head_dim, half = D / 2;
  // a pre-sharded artifact holds this rank's slices only: the same jobs with every offset zero and the row-parallel
  // matrices as wide as the slice (the device-side gather / interleave is unchanged)
  const bool pre = tp_presharded_ && !synthetic;
  const int h0 = pre ? 0 : tp_rank_ * Hl_, kv0 = pre ? 0 : tp_rank_ * KVHl_, i0 = pre ? 0 : tp_rank_ * Il_;
  const int64_t o_cols = pre ? (int64_t)Hl_ * cfg_.head_dim : (int64_t)cfg_.heads * cfg_.head_dim, down_cols = pre ? Il_ : cfg_.inter;
  std::vector<FillJob> jobs;
  auto ident = [](int start, int n) {
    std::vector<int> v(n);
    for (int i = 0; i < n; ++i) v[i] = start + i;
    return v;
  };
  // pair-interleave so that physical rows (2p, 2p+1) = logical (head*D + j, head*D + j + D/2): RoPE partners adjacent
  auto rope_rows = [&](int head0, int nheads) {
    std::vector<int> v((size_t)nheads * D);
    for (int r = 0; r < nheads * D; ++r) {
      int p = r >> 1, hd = p / half, j = p % half;
      v[r] = (head0 + hd) * D + j + (r & 1) * half;
    }
    return v;
  };
  if (cfg_.falcon) {
    // fused query_key_value rows are grouped per KV head: [G query heads | k | v] x KVH  (modeling_falcon.py:259-270)
    const int G = cfg_.heads / cfg_.kv_heads, gs = (G + 2) * D;
    auto q_rows = [&]() {
      std::vector<int> v((size_t)Hl_ * D);
      for (int r = 0; r < Hl_ * D; ++r) {
        const int pp = r >> 1, hd = pp / half, j = pp % half, head = h0 + hd;
        v[r] = (head / G) * gs + (head % G) * D + j + (r & 1) * half;
      }
      return v;
    };
    auto k_rows = [&]() {
      std::vector<int> v((size_t)KVHl_ * D);
      for (int r = 0; r < KVHl_ * D; ++r) {
        const int pp = r >> 1, hd = pp / half, j = pp % half;
        v[r] = (kv0 + hd) * gs + G * D + j + (r & 1) * half;
      }
      return v;
    };
    auto v_rows = [&]() {
      std::vector<int> v((size_t)KVHl_ * D);
      for (int r = 0; r < KVHl_ * D; ++r) v[r] = (kv0 + r / D) * gs + (G + 1) * D + r % D;
      return v;
    };
    for (int l = 0; l < cfg_.layers; ++l) {
      const std::string p = "transformer.h." + std::to_string(l) + ".";
      const uint32_t t = (uint32_t)l * 16;
      LayerW& w = lw_[l];
      const std::string qkv = p + "self_attention.query_key_value.weight";
      jobs.push_back({w.wqkv, h, q_rows(), Hl_ * D, 0, h, h, qkv, t + 11, kWAmp, 0.f});
      jobs.push_back({w.wqkv + (size_t)Hl_ * D * h, h, k_rows(), KVHl_ * D, 0, h, h, qkv, t + 11, kWAmp, 0.f});
      jobs.push_back({w.wqkv + (size_t)(Hl_ + KVHl_) * D * h, h, v_rows(), KVHl_ * D, 0, h, h, qkv, t + 11, kWAmp, 0.f});
      jobs.push_back({w.wo, (int64_t)Hl_ * D, {}, h, h0 * D, Hl_ * D, o_cols, p + "self_attention.dense.weight", t + K_O, kWAmp, 0.f});
      jobs.push_back({w.wgu, h, ident(i0, Il_), Il_, 0, h, h, p + "mlp.dense_h_to_4h.weight", t + 9, kWAmp, 0.f});
      jobs.push_back({w.wdown, Il_, {}, h, i0, Il_, down_cols, p + "mlp.dense_4h_to_h.weight", t + 10, kWAmp, 0.f});
      jobs.push_back({w.ln1, h, {}, 1, 0, h, h, p + "ln_attn.weight", t + K_LN1, kNormAmp, 1.f});
      jobs.push_back({w.ln1_b, h, {}, 1, 0, h, h, p + "ln_attn.bias", t + 12, kNormAmp, 0.f});
      jobs.push_back({w.ln2, h, {}, 1, 0, h, h, p + "ln_mlp.weight", t + K_LN2, kNormAmp, 1.f});
      jobs.push_back({w.ln2_b, h, {}, 1, 0, h, h, p + "ln_mlp.bias", t + 13, kNormAmp, 0.f});
    }
    jobs.push_back({embed_, h, {}, cfg_.vocab, 0, h, h, "transformer.word_embeddings.weight", kGlobal + 0, kWAmp, 0.f});
    if (!cfg_.tie_embeddings) jobs.push_back({lm_head_, h, {}, cfg_.vocab, 0, h, h, "lm_head.weight", kGlobal + 2, kWAmp * kLmHeadGain, 0.f});
    jobs.push_back({final_norm_, h, {}, 1, 0, h, h, "transformer.ln_f.weight", kGlobal + 1, kNormAmp, 1.f});
    jobs.push_back({final_norm_b_, h, {}, 1, 0, h, h, "transformer.ln_f.bias", kGlobal + 3, kNormAmp, 0.f});
  }
  for (int l = 0; l < (cfg_.falcon ? 0 : cfg_.layers); ++l) {
    const std::string p = "model.layers." + std::to_string(l) + ".";
    const uint32_t t = (uint32_t)l * 16;
    LayerW& w = lw_[l];
    jobs.push_back({w.wqkv, h, rope_rows(h0, Hl_), Hl_ * D, 0, h, h, p + "self_attn.q_proj.weight", t + K_Q, kWAmp, 0.f});
    jobs.push_back({w.wqkv + (size_t)Hl_ * D * h, h, rope_rows(kv0, KVHl_), KVHl_ * D, 0, h, h, p + "self_attn.k_proj.weight", t + K_K, kWAmp, 0.f});
    jobs.push_back({w.wqkv + (size_t)(Hl_ + KVHl_) * D * h, h, ident(kv0 * D, KVHl_ * D), KVHl_ * D, 0, h, h, p + "self_attn.v_proj.weight", t + K_V, kWAmp, 0.f});
    jobs.push_back({w.wo, (int64_t)Hl_ * D, {}, h, h0 * D, Hl_ * D, o_cols, p + "self_attn.o_proj.weight", t + K_O, kWAmp, 0.f});
    // gate/up interleaved row-wise: physical row 2i = gate_i, 2i+1 = up_i (SwiGLU partners adjacent)
    jobs.push_back({w.wgu, 2 * (int64_t)h, ident(i0, Il_), Il_, 0, h, h, p + "mlp.gate_proj.weight", t + K_GATE, kWAmp, 0.f});
    jobs.push_back({w.wgu + h, 2 * (int64_t)h, ident(i0, Il_), Il_, 0, h, h, p + "mlp.up_proj.weight", t + K_UP, kWAmp, 0.f});
    jobs.push_back({w.wdown, Il_, {}, h, i0, Il_, down_cols, p + "mlp.down_proj.weight", t + K_DOWN, kWAmp, 0.f});
    jobs.push_back({w.ln1, h, {}, 1, 0, h, h, p + "input_layernorm.weight", t + K_LN1, kNormAmp, 1.f});
    jobs.push_back({w.ln2, h, {}, 1, 0, h, h, p + "post_attention_layernorm.weight", t + K_LN2, kNormAmp, 1.f});
  }
  if (!cfg_.falcon) {
    jobs.push_back({embed_, h, {}, cfg_.vocab, 0, h, h, "model.embed_tokens.weight", kGlobal + 0, kWAmp, 0.f});
    if (!cfg_.tie_embeddings) jobs.push_back({lm_head_, h, {}, cfg_.vocab, 0, h, h, "lm_head.weight", kGlobal + 2, kWAmp * kLmHeadGain, 0.f});
    jobs.push_back({final_norm_, h, {}, 1, 0, h, h, "model.norm.weight", kGlobal + 1, kNormAmp, 1.f});
  }

  ModelFiles& files = files_;
  size_t max_src = 0, max_deq = 0;
  const bool gguf = !synthetic && files.is_gguf();
  if (gguf) {
    // HF name -> GGUF name (llama.cpp convert_hf_to_gguf tensor map).  GGUF stores q/k rows already permuted per head
    // to (j, j + d/2) -> (2j, 2j+1) for llama.cpp's interleaved RoPE; that IS this engine's pair-interleaved layout,
    // so q/k rows are taken in file order.
    auto rename = [](std::string n) {
      auto rep = [&](const std::string& a, const std::string& b) {
        size_t p = n.find(a);
        if (p != std::string::npos) n.replace(p, a.size(), b);
      };
      rep("model.layers.", "blk.");
      rep("self_attn.q_proj", "attn_q");
      rep("self_attn.k_proj", "attn_k");
      rep("self_attn.v_proj", "attn_v");
      rep("self_attn.o_proj", "attn_output");
      rep("mlp.gate_proj", "ffn_gate");
      rep("mlp.up_proj", "ffn_up");
      rep("mlp.down_proj", "ffn_down");
      rep("input_layernorm", "attn_norm");
      rep("post_attention_layernorm", "ffn_norm");
      if (n == "model.embed_tokens.weight") n = "token_embd.weight";
      if (n == "model.norm.weight") n = "output_norm.weight";
      if (n == "lm_head.weight") n = "output.weight";
      return n;
    };
    for (auto& j : jobs) {
      const bool qk = j.name.find("q_proj") != std::string::npos || j.name.find("k_proj") != std::string::npos;
      if (qk) {
        const bool isq = j.name.find("q_proj") != std::string::npos;
        j.rows = ident((isq ? h0 : kv0) * D, (isq ? Hl_ : KVHl_) * D);
      }
      j.name = rename(j.name);
    }
  }
  if (!synthetic) {
    for (auto& j : jobs) {
      const TensorView* tv = files.find(j.name);
      if (!tv) RET(SSB_EIO, "checkpoint is missing tensor " + j.name);
      if (tv->dtype == DT_OTHER || (!gguf && tv->dtype > DT_F32)) RET(SSB_EINVAL, "unsupported dtype for " + j.name);
      if (tv->cols() != j.full_cols) RET(SSB_EINVAL, "unexpected shape for " + j.name);
      int64_t max_row = j.rows.empty() ? j.n_rows - 1 : 0;
      for (int r : j.rows) max_row = std::max<int64_t>(max_row, r);
      if (max_row >= tv->rows()) RET(SSB_EINVAL, "tensor " + j.name + " has too few rows for this config");
      if (pre && files.is_gguf()) RET(SSB_EINVAL, "a pre-sharded artifact cannot be GGUF");
      max_src = std::max(max_src, tv->nbytes);
      if (tv->dtype >= DT_Q4_0) {
        int64_t n = 1;
        for (auto d : tv->shape) n *= d;
        max_deq = std::max(max_deq, (size_t)n * 2);
      }
    }
  }
  if (validate_only) return SSB_OK;  // host-side inventory check only (runs before any device is touched)
  int* d_rows = nullptr;
  size_t max_rows = 0;
  for (auto& j : jobs) max_rows = std::max(max_rows, j.rows.size());
  CK(cudaMalloc(&d_rows, std::max<size_t>(max_rows, 1) * sizeof(int)));
  void* d_src = nullptr;
  bf16* d_deq = nullptr;
  if (max_src) CK(cudaMalloc(&d_src, max_src));
  if (max_deq) CK(cudaMalloc(&d_deq, max_deq));
  int rc = SSB_OK;
  for (auto& j : jobs) {
    const int* rows = nullptr;
    if (!j.rows.empty()) {
      cudaMemcpyAsync(d_rows, j.rows.data(), j.rows.size() * sizeof(int), cudaMemcpyHostToDevice, stream_);
      rows = d_rows;
    }
    cudaError_t e;
    if (synthetic) {
      e = launch_synth_fill(j.dst, j.dst_ld, rows, j.n_rows, j.col0, j.cols, j.full_cols, seed, j.tid, j.amp, j.base, stream_);
    } else {
      const TensorView* tv = files.find(j.name);
      cudaMemcpyAsync(d_src, tv->data, tv->nbytes, cudaMemcpyHostToDevice, stream_);
      timing_.h2d_bytes += (int64_t)tv->nbytes;
      if (tv->dtype >= DT_Q4_0) {  // GGUF block formats: dequantise the whole tensor to bf16, then permute/shard
        int64_t n = 1;
        for (auto d : tv->shape) n *= d;
        e = launch_dequant(d_src, tv->dtype, n, d_deq, stream_);
        if (e == cudaSuccess)
          e = launch_gather_rows(j.dst, j.dst_ld, d_deq, DT_BF16, tv->cols(), rows, j.n_rows, j.col0, j.cols, stream_);
      } else {
        e = launch_gather_rows(j.dst, j.dst_ld, d_src, tv->dtype, tv->cols(), rows, j.n_rows, j.col0, j.cols, stream_);
      }
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream_);  // d_rows / d_src are reused by the next job
    if (e != cudaSuccess) {
      set_error(std::string("weight fill ") + j.name + ": " + cudaGetErrorString(e));
      rc = SSB_ECUDA;
      break;
    }
  }
  cudaFree(d_rows);
  if (d_src) cudaFree(d_src);
  if (d_deq) cudaFree(d_deq);
  return rc;
}

void Engine::prof_mark(const char* label) {
  if (!prof_fwd_) return;
  cudaEvent_t e;
  cudaEventCreate(&e);
  cudaEventRecord(e, stream_);
  prof_marks_.emplace_back(label, e);
}
void Engine::prof_collect() {
  if (!prof_fwd_ || prof_marks_.empty()) return;
  cudaStreamSynchronize(stream_);
  for (size_t i = 1; i < prof_marks_.size(); ++i) {
    float ms = 0;
    cudaEventElapsedTime(&ms, prof_marks_[i - 1].second, prof_marks_[i].second);
    prof_ms_[prof_marks_[i].first] += ms;  // time since the previous mark is attributed to the kernel that just ran
  }
  for (auto& m : prof_marks_) cudaEventDestroy(m.second);
  prof_marks_.clear();
}
std::string Engine::prof_report() {
  prof_collect();
  std::string s = "{";
  for (auto& kv : prof_ms_) s += (s.size() > 1 ? "," : "") + std::string("\"") + kv.first + "\":" + std::to_string(kv.second);
  prof_ms_.clear();
  return s + "}";
}

int Engine::decode_splits_(int M) const {
  const int group = cfg_.heads / cfg_.kv_heads;
  const int gc = (group % 8 == 0) ? 8 : (group % 4 == 0) ? 4 : (group % 2 == 0) ? 2 : 1;
  if (attn_splits_ > 0) return std::min(attn_splits_, gc >= 4 ? 16 : 32);  // params "attn_splits": sweep knob, 0 = heuristic
  const int ctas = M * (Hl_ / gc);
  int s = ((gc >= 4 ? 2 : 4) * n_sm_ + ctas - 1) / ctas;
  return std::max(1, std::min(s, gc >= 4 ? 16 : 32));
}

int Engine::alloc_runtime(const Json& params) {
  const int h = cfg_.hidden, D = cfg_.head_dim;
  max_batch_ = (int)params.get_int("max_batch", 32);
  max_seq_ = (int)params.get_int("max_seq_len", cfg_.max_pos);
  block_size_ = (int)params.get_int("kv_block_size", 16);
  if (max_batch_ < 1 || max_seq_ < 1 || (block_size_ != 8 && block_size_ != 16 && block_size_ != 32 && block_size_ != 64))
    RET(SSB_EINVAL, "bad max_batch / max_seq_len / kv_block_size (8|16|32|64)");
  max_blocks_per_seq_ = (max_seq_ + block_size_ - 1) / block_size_;
  attn_splits_ = (int)params.get_int("attn_splits", 0);
  m_max_ = std::max(max_batch_, (int)params.get_int("prefill_chunk", 1024));
  max_steps_ = max_seq_;
  // rope table
  {
    const int half = D / 2;
    std::vector<uint32_t> cs((size_t)max_seq_ * half);
    std::vector<float> inv(half);
    // HF: inv_freq = 1 / theta^(2j/d) in fp32; freqs = pos * inv_freq (fp32); cos/sin fp32 -> bf16
    for (int j = 0; j < half; ++j) inv[j] = 1.0f / powf(cfg_.theta, (float)(2 * j) / (float)D);
    for (int p = 0; p < max_seq_; ++p)
      for (int j = 0; j < half; ++j) {
        const float f = (float)p * inv[j];
        __nv_bfloat16 c = __float2bfloat16_rn(cosf(f)), s = __float2bfloat16_rn(sinf(f));
        uint16_t cb, sb;
        memcpy(&cb, &c, 2);
        memcpy(&sb, &s, 2);
        cs[(size_t)p * half + j] = (uint32_t)cb | ((uint32_t)sb << 16);
      }
    TRY(dmalloc(&rope_cs_, cs.size()));
    CK(cudaMemcpy(rope_cs_, cs.data(), cs.size() * 4, cudaMemcpyHostToDevice));
  }
  TRY(dmalloc(&h_, (size_t)m_max_ * h));
  TRY(dmalloc(&q_, (size_t)m_max_ * Hl_ * D));
  TRY(dmalloc(&attn_, (size_t)m_max_ * Hl_ * D));
  TRY(dmalloc(&act_, (size_t)m_max_ * Il_));
  TRY(dmalloc(&xn_, (size_t)m_max_ * h));
  if (cfg_.falcon) TRY(dmalloc(&ao_, (size_t)m_max_ * h));
  if (cfg_.falcon && tp_size_ > 1) TRY(dmalloc(&falcon_scratch_, (size_t)m_max_ * h));
  TRY(dmalloc(&tp_step_, 1));
  CK(cudaMemset(tp_step_, 0, sizeof(int)));
  TRY(dmalloc(&tp_push_step_, 1));
  CK(cudaMemset(tp_push_step_, 0, sizeof(int)));
  if (tp_size_ > 1) {
    // one plain cudaMalloc (not a pool) so the whole exchange area is exported with a single cudaIpcGetMemHandle
    const size_t b_part = 2 * (size_t)m_max_ * h * sizeof(float);
    const size_t b_recv = 2 * 8 * (size_t)max_batch_ * h * sizeof(float);
    tp_off_recv_ = b_part;
    tp_off_flags_ = b_part + b_recv;
    tp_off_pflags_ = tp_off_flags_ + 64;
    tp_pool_bytes_ = tp_off_pflags_ + 64;
    // prefill-sized forwards (>= tp_two_shot_min_rows rows): reduce-scatter + bf16 gather instead of every rank pulling every
    // peer's full fp32 partial.  Default ON (parity: tests/test_tp_gpu.py two_shot)
    tp_two_shot_ = params.get_int("tp_two_shot", 1) != 0 && !cfg_.falcon;
    tp_two_shot_min_rows_ = std::max(1, (int)params.get_int("tp_two_shot_min_rows", 64));
    if (tp_two_shot_) {  // opt-in: the default pool layout (and its size check in tp_connect) is unchanged
      tp_off_gather_ = tp_pool_bytes_;
      tp_pool_bytes_ += (size_t)m_max_ * h * sizeof(bf16);
      TRY(dmalloc(&d_peer_gather_, 8));
      TRY(dmalloc(&tp2_done_, 1));
      CK(cudaMemset(tp2_done_, 0, sizeof(unsigned)));
    }
    // decode under tensor parallelism: 3 (default) = the persistent kernel with the 16-byte {value, epoch} push exchange;
    // 0 = the multi-kernel path, 1 / 2 = flag + pull variants.  Llama-family head size only
    tp_mega_mode_ = D == 128 && !cfg_.falcon ? (int)params.get_int("tp_mega", 3) : 0;
    if (tp_mega_mode_ == 2) {
      tp_off_ctaflags_ = tp_pool_bytes_;
      tp_pool_bytes_ += 8 * 256 * sizeof(uint32_t);
      TRY(dmalloc(&d_peer_cta_flags_, 8));
    }
    tp_ll_ = params.get_int("tp_ll", 1) != 0;  // decode-sized allreduce of the multi-kernel path: LL push kernel (0 = one-shot pull)
    if (tp_mega_mode_ == 3 || tp_ll_) {
      tp_off_ll_ = (tp_pool_bytes_ + 255) & ~(size_t)255;
      tp_pool_bytes_ = tp_off_ll_ + 2 * 8 * 4 * (size_t)(h / 2) * sizeof(uint4);
      TRY(dmalloc(&d_peer_ll_, 8));
    }
    TRY(dmalloc(&tp_pool_, tp_pool_bytes_));
    if (tp_mega_mode_ == 2) CK(cudaMemset(tp_pool_ + tp_off_ctaflags_, 0, 8 * 256 * sizeof(uint32_t)));
    if (tp_off_ll_) CK(cudaMemset(tp_pool_ + tp_off_ll_, 0, tp_pool_bytes_ - tp_off_ll_));  // epoch 0 = never written
    CK(cudaMemset(tp_pool_ + tp_off_flags_, 0, 128));
    tp_partials_ = (float*)tp_pool_;
    tp_recv_ = (float*)(tp_pool_ + tp_off_recv_);
    tp_flags_ = (uint32_t*)(tp_pool_ + tp_off_flags_);
    tp_pflags_ = (unsigned long long*)(tp_pool_ + tp_off_pflags_);
    TRY(dmalloc(&d_peer_partials_, 8));
    TRY(dmalloc(&d_peer_flags_, 8));
    TRY(dmalloc(&d_peer_recv_, 8));
    TRY(dmalloc(&d_peer_pflags_, 8));
  }
  TRY(dmalloc(&logits_, (size_t)max_batch_ * cfg_.vocab));
  const int max_splits = 32;
  TRY(dmalloc(&part_o_, (size_t)max_batch_ * Hl_ * max_splits * D));
  TRY(dmalloc(&part_ml_, (size_t)max_batch_ * Hl_ * max_splits * 2));
  TRY(dmalloc(&counters_, (size_t)m_max_ * Hl_));
  CK(cudaMemset(counters_, 0, (size_t)m_max_ * Hl_ * sizeof(int)));
  TRY(dmalloc(&row_tok_, (size_t)m_max_));
  TRY(dmalloc(&row_slot_, (size_t)m_max_));
  TRY(dmalloc(&row_pos_, (size_t)m_max_));
  TRY(dmalloc(&logit_rows_, (size_t)max_batch_));
  TRY(dmalloc(&tile_row0_, (size_t)m_max_));
  TRY(dmalloc(&tile_nrows_, (size_t)m_max_));
  TRY(dmalloc(&next_tok_, (size_t)max_batch_));
  TRY(dmalloc(&hist_, (size_t)max_steps_ * max_batch_));
  TRY(dmalloc(&step_, 1));
  TRY(dmalloc(&block_table_, (size_t)max_batch_ * max_blocks_per_seq_));
  CK(cudaMemset(block_table_, 0, (size_t)max_batch_ * max_blocks_per_seq_ * sizeof(int)));
  host_bt_.assign((size_t)max_batch_ * max_blocks_per_seq_, 0);
  taps_ = params.get_int("debug_taps", 0) != 0;
  if (taps_) {
    TRY(dmalloc(&tap_q0_, (size_t)m_max_ * Hl_ * D));
    TRY(dmalloc(&tap_attn0_, (size_t)m_max_ * Hl_ * D));
    TRY(dmalloc(&tap_h0_, (size_t)m_max_ * h));
  }
  // KV pool
  const size_t block_elems = (size_t)KVHl_ * block_size_ * D;
  const size_t block_bytes_all_layers = block_elems * 2 /*bf16*/ * 2 /*K,V*/ * cfg_.layers;
  int64_t want = params.get_int("kv_blocks", (int64_t)max_batch_ * max_blocks_per_seq_);
  size_t free_b = 0, total_b = 0;
  CK(cudaMemGetInfo(&free_b, &total_b));
  const int64_t fit = (int64_t)((double)free_b * 0.92 / (double)block_bytes_all_layers);
  n_blocks_ = (int)std::min<int64_t>(want, fit);
  if (n_blocks_ < max_blocks_per_seq_ && n_blocks_ < want) RET(SSB_ENOMEM, "not enough HBM for the KV block pool");
  kv_layer_elems_ = (size_t)n_blocks_ * block_elems;
  TRY(dmalloc(&kpool_, kv_layer_elems_ * cfg_.layers));
  TRY(dmalloc(&vpool_, kv_layer_elems_ * cfg_.layers));
  free_blocks_.resize(n_blocks_);
  for (int i = 0; i < n_blocks_; ++i) free_blocks_[i] = n_blocks_ - 1 - i;
  slots_.assign(max_batch_, SeqSlot());
  {  // stream-K workspace of the tensor-core decode projections
    if (params.get_int("tc_streamk", 1) != 0) {
      sk_slots_ = 2 * n_sm_;
      TRY(dmalloc(&sk_part_, (size_t)sk_slots_ * 64 * 128));
      TRY(dmalloc(&sk_flags_, (size_t)sk_slots_));
      CK(cudaMemset(sk_flags_, 0, sk_slots_ * sizeof(unsigned)));
      if (params.get_int("sk_prof", 0)) {
        TRY(dmalloc(&sk_prof_, (size_t)n_sm_ * 8));
        CK(cudaMemset(sk_prof_, 0, (size_t)n_sm_ * 8 * sizeof(unsigned long long)));
      }
    }
  }
  // persistent decode kernel (mega.cu): per-layer pointer table, attention chunk partials, grid barrier
  // under tensor parallelism the persistent kernel carries the allreduce itself ("tp_mega", see above; 0 = multi-kernel path)
  const bool tp_mega = tp_size_ > 1 && tp_mega_mode_ != 0;
  use_mega_ = params.get_int("use_mega", 1) != 0 && (tp_size_ == 1 || tp_mega) && !cfg_.falcon && !prof_fwd_;
  if (use_mega_) {
    const int group = cfg_.heads / cfg_.kv_heads, ag = mega_attn_group(group);
    const int ch = mega_attn_chunk(D, ag);
    mega_max_chunks_ = (max_seq_ + ch - 1) / ch;
    mega_k_max_ = std::max(h, std::max(Hl_ * D, Il_));
    if (mega_pick_stages(1, mega_k_max_) == 0) {
      use_mega_ = false;
    } else {
      std::vector<MegaLayer> ml(cfg_.layers);
      for (int l = 0; l < cfg_.layers; ++l)
        ml[l] = MegaLayer{lw_[l].wqkv, lw_[l].wo, lw_[l].wgu, lw_[l].wdown, lw_[l].ln1, lw_[l].ln2,
                          kpool_ + (size_t)l * kv_layer_elems_, vpool_ + (size_t)l * kv_layer_elems_};
      TRY(dmalloc(&d_mega_layers_, ml.size()));
      CK(cudaMemcpy(d_mega_layers_, ml.data(), ml.size() * sizeof(MegaLayer), cudaMemcpyHostToDevice));
      const size_t units = (size_t)4 * (Hl_ / ag) * mega_max_chunks_;
      TRY(dmalloc(&mega_part_o_, units * ag * D));
      TRY(dmalloc(&mega_part_ml_, units * ag * 2));
      TRY(dmalloc(&mega_counters_, (size_t)4 * Hl_));
      CK(cudaMemset(mega_counters_, 0, (size_t)4 * Hl_ * sizeof(int)));
      if (params.get_int("mega_prof", 0)) {  // 1: CTA 0 stamps its phases; 2: every CTA does (arrival skew across the SMs)
        mega_prof_all_ = params.get_int("mega_prof", 0) >= 2;
        const size_t n = mega_prof_all_ ? (size_t)n_sm_ * 1024 : 1024;
        TRY(dmalloc(&mega_prof_, n));
        CK(cudaMemset(mega_prof_, 0, n * sizeof(unsigned long long)));
      }
      if (params.get_int("mega_head_flags", 0) != 0) {  // needs a library built with -DMG_HEAD_FLAGS=1; measured slower (mega.cu)
        TRY(dmalloc(&mega_head_done_, (size_t)Hl_ + 2 * KVHl_ + 32));
        CK(cudaMemset(mega_head_done_, 0, ((size_t)Hl_ + 2 * KVHl_ + 32) * sizeof(unsigned)));
      }
      // [0] barrier counter, [1] exit counter, [32 + 32 g] group counters of the tree-barrier experiment, then the pass claims
      TRY(dmalloc(&mega_bar_, mega_bar_words(cfg_.layers)));
      CK(cudaMemset(mega_bar_, 0, mega_bar_words(cfg_.layers) * sizeof(unsigned)));
    }
  }
  return SSB_OK;
}

int Engine::init(const std::string& model_dir, const std::string& params_json) {
  Json params;
  try {
    params = json_parse(params_json.empty() ? "{}" : params_json);
  } catch (std::exception& e) {
    RET(SSB_EINVAL, std::string("params.json: ") + e.what());
  }
  if (params.kind != Json::Obj) RET(SSB_EINVAL, "params.json must be a JSON object");
  device_ = -1;
  // 1. everything that needs no GPU: params, checkpoint containers, config, tensor inventory (names / dtypes / shapes)
  const std::string wmode = params.get_str("weights", "file");
  if (wmode != "file" && wmode != "synthetic") RET(SSB_EINVAL, "params.weights must be 'file' or 'synthetic'");
  if (wmode == "file") {
    std::string err;
    // A tensor-parallel rank prefers its pre-sharded artifact (SURVEY 8f #2; written by tools/tp_shard.py): ONE safetensors
    // file with exactly this rank's slices of the projections plus the replicated tensors, so a rank reads ~1/N of the
    // checkpoint at pod start instead of mapping all of it.  "tp_presharded": 0 ignores it.
    const long long tps = params.get_int("tp_size", 1), tpr = params.get_int("tp_rank", 0);
    const std::string shard = std::string(model_dir) + "/ssb_tp" + std::to_string(tps) + "/rank" + std::to_string(tpr) + ".safetensors";
    struct stat st;
    if (tps > 1 && params.get_int("tp_presharded", 1) != 0 && stat(shard.c_str(), &st) == 0) {
      if (!files_.open_file(shard, &err)) RET(SSB_EIO, err);
      const auto& md = files_.metadata();
      auto get = [&](const char* k) {
        auto it = md.find(k);
        return it == md.end() ? std::string() : it->second;
      };
      if (get("format") != "ssb-tp" || get("tp_size") != std::to_string(tps) || get("tp_rank") != std::to_string(tpr))
        RET(SSB_EINVAL, shard + " is not the pre-sharded artifact of rank " + std::to_string(tpr) + " of " + std::to_string(tps) +
                            " (metadata format / tp_size / tp_rank)");
      tp_presharded_ = true;
    } else if (!files_.open(model_dir, &err)) {
      RET(SSB_EIO, err);
    }
  }
  TRY(load_config(model_dir, params));
  if (tp_size_ > 8) RET(SSB_EINVAL, "tp_size > 8 is not supported (one NVSwitch domain)");
  if (wmode == "file") {
    lw_.assign(cfg_.layers, LayerW());
    TRY(fill_weights(model_dir, false, 0, /*validate_only=*/true));
  }
  // 2. the device: no CPU fallback
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    RET(SSB_ENODEV, "no CUDA device: libsubstratus_b200 has no CPU fallback");
  device_ = (int)params.get_int("device", tp_rank_ % ndev);
  if (device_ < 0 || device_ >= ndev) RET(SSB_EINVAL, "bad device index");
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, device_));
  if (prop.major != 9 || prop.minor != 0) {
    RET(SSB_ENODEV, std::string("device ") + prop.name + " is sm_" + std::to_string(prop.major * 10 + prop.minor) +
                        "; this library contains sm_90a code only");
  }
  CK(cudaSetDevice(device_));
  n_sm_ = prop.multiProcessorCount;
  CK(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
  CK(cudaEventCreate(&ev0_));
  CK(cudaEventCreate(&ev1_));
  prof_fwd_ = params.get_int("profile_forward", 0) != 0;
  use_pdl_ = params.get_int("use_pdl", 1) != 0;
  tp_push_ = params.get_int("tp_push", 0) != 0;  // push-model allreduce (default: pull, DESIGN.md §6)
  use_graph_ = params.get_int("use_graph", 1) != 0;
  if (prof_fwd_) use_pdl_ = use_graph_ = false;  // event marks between launches need plain stream order
  TRY(alloc_weights());
  TRY(fill_weights(model_dir, wmode == "synthetic", (uint64_t)params.get_int("seed", 0), false));
  TRY(alloc_runtime(params));
  {
    const std::string gp = params.get_str("gemm_path", "auto");  // "auto" | "gemv" (CUDA cores only) | "tc" (tensor cores always)
    if (gp == "gemv")
      tc_min_rows_ = 1 << 30;
    else if (gp == "tc")
      tc_min_rows_ = 1;
    else if (gp == "auto")
      // tensor-core stream-K from 5 rows up: 5-7 rows would take TWO passes of the 4-row kernel (weights streamed twice)
      tc_min_rows_ = (int)params.get_int("tc_min_rows", 5);
    else
      RET(SSB_EINVAL, "params.gemm_path must be auto|gemv|tc");
    mega_attn_tile_ = params.get_int("mega_attn_tile", 1) != 0;
    mega_max_batch_ = (int)params.get_int("mega_max_batch", 1);
    tc_tn_prefill_ = (int)params.get_int("tc_tn_prefill", 0);  // 0 = per-projection heuristic; 128 | 256 force (tests, A/B)
    if (tc_tn_prefill_ != 0 && tc_tn_prefill_ != 128 && tc_tn_prefill_ != 256) RET(SSB_EINVAL, "params.tc_tn_prefill must be 0, 128 or 256");
    const int h = cfg_.hidden, D = cfg_.head_dim, br = tc_weight_box_rows();
    for (auto& w : lw_) {
      CK(tc_make_tmap(&w.tm_qkv, w.wqkv, (int64_t)(Hl_ + 2 * KVHl_) * D, h, h, br));
      CK(tc_make_tmap(&w.tm_o, w.wo, h, (int64_t)Hl_ * D, (int64_t)Hl_ * D, br));
      CK(tc_make_tmap(&w.tm_gu, w.wgu, (cfg_.falcon ? 1 : 2) * (int64_t)Il_, h, h, br));
      CK(tc_make_tmap(&w.tm_down, w.wdown, h, Il_, Il_, br));
    }
    CK(tc_make_tmap(&tm_lm_head_, lm_head_, cfg_.vocab, h, h, br));
  }
  CK(cudaStreamSynchronize(stream_));
  timing_reset();
  return SSB_OK;
}

int Engine::info(ssb_info* o) const {
  memset(o, 0, sizeof(*o));
  o->vocab_size = cfg_.vocab;
  o->hidden_size = cfg_.hidden;
  o->n_layers = cfg_.layers;
  o->n_heads = cfg_.heads;
  o->n_kv_heads = cfg_.kv_heads;
  o->head_dim = cfg_.head_dim;
  o->intermediate_size = cfg_.inter;
  o->max_seq_len = max_seq_;
  o->max_batch = max_batch_;
  o->kv_block_size = block_size_;
  o->tp_size = tp_size_;
  o->tp_rank = tp_rank_;
  o->n_sm = n_sm_;
  o->device = device_;
  o->weight_bytes_per_step = weight_bytes_step_;
  o->kv_bytes_per_token = (int64_t)2 * cfg_.layers * KVHl_ * cfg_.head_dim * 2;
  o->hbm_bytes_allocated = (int64_t)hbm_bytes_;
  snprintf(o->model_type, sizeof o->model_type, "%s", cfg_.model_type.c_str());
  snprintf(o->dtype, sizeof o->dtype, "bf16");
  return SSB_OK;
}

int Engine::seq_create(int* id) {
  for (int i = 0; i < max_batch_; ++i)
    if (!slots_[i].used) {
      slots_[i].used = true;
      slots_[i].len = 0;
      slots_[i].blocks.clear();
      *id = i;
      return SSB_OK;
    }
  RET(SSB_ENOMEM, "all sequence slots are in use (max_batch)");
}

int Engine::seq_free(int id) {
  if (id < 0 || id >= max_batch_ || !slots_[id].used) RET(SSB_EINVAL, "bad seq_id");
  for (int b : slots_[id].blocks) free_blocks_.push_back(b);
  slots_[id] = SeqSlot();
  return SSB_OK;
}

int Engine::seq_len(int id, int* len) const {
  if (id < 0 || id >= max_batch_ || !slots_[id].used) RET(SSB_EINVAL, "bad seq_id");
  *len = slots_[id].len;
  return SSB_OK;
}

int Engine::ensure_blocks(int slot, int new_len) {
  if (new_len > max_seq_) RET(SSB_EINVAL, "sequence would exceed max_seq_len");
  SeqSlot& s = slots_[slot];
  const int need = (new_len + block_size_ - 1) / block_size_;
  // all or nothing per sequence: a refused call leaves the pool as it found it (the host retires ONE request and retries)
  if (need - (int)s.blocks.size() > (int)free_blocks_.size()) RET(SSB_ENOMEM, "KV block pool exhausted");
  while ((int)s.blocks.size() < need) {
    const int b = free_blocks_.back();
    free_blocks_.pop_back();
    host_bt_[(size_t)slot * max_blocks_per_seq_ + s.blocks.size()] = b;
    s.blocks.push_back(b);
  }
  return SSB_OK;
}

// the blocks of several sequences in one step: checks every length and the pool first, then grants — nothing changes on error
int Engine::ensure_blocks_all(const int* slot_ids, const int* new_lens, int n) {
  long long need = 0;
  for (int i = 0; i < n; ++i) {
    if (new_lens[i] > max_seq_) RET(SSB_EINVAL, "sequence would exceed max_seq_len");
    const int want = (new_lens[i] + block_size_ - 1) / block_size_ - (int)slots_[slot_ids[i]].blocks.size();
    if (want > 0) need += want;
  }
  if (need > (long long)free_blocks_.size()) RET(SSB_ENOMEM, "KV block pool exhausted");
  for (int i = 0; i < n; ++i) TRY(ensure_blocks(slot_ids[i], new_lens[i]));
  return SSB_OK;
}

int Engine::upload_block_rows(const std::vector<int>& slots) {
  for (int s : slots) {
    const size_t n = slots_[s].blocks.size();
    if (!n) continue;
    CK(cudaMemcpyAsync(block_table_ + (size_t)s * max_blocks_per_seq_, host_bt_.data() + (size_t)s * max_blocks_per_seq_,
                       n * sizeof(int), cudaMemcpyHostToDevice, stream_));
    timing_.h2d_bytes += (int64_t)(n * sizeof(int));
  }
  return SSB_OK;
}

// Enqueue one forward pass over the M staged rows (row_tok_/row_slot_/row_pos_).  The last-position logits of the
// n_logit_rows rows listed in logit_rows_ go to logits_; greedy picks to next_tok_.  decode_mode: rows == batch,
// argmax feeds row_tok_ back, appends to hist_ and advances row_pos_ (device-resident loop, graph-capturable).
int Engine::forward(int M, int n_logit_rows, bool decode_mode) {
  if (cfg_.falcon) return forward_falcon(M, n_logit_rows, decode_mode);
  const int h = cfg_.hidden, D = cfg_.head_dim;
  const int group = cfg_.heads / cfg_.kv_heads;
  int launches = 0;
  const bool tp = tp_size_ > 1;
  // push-model allreduce (decode-sized forwards on the GEMV path): partials are written straight into every rank's
  // receive slots by the projection epilogue; pull model otherwise (prefill / tensor-core path)
  const bool tp_push = tp && tp_push_ && M <= 4 && M < tc_min_rows_ && M <= max_batch_;
  prof_mark("start");
  CK(launch_embed(embed_, row_tok_, h_, M, h, decode_mode ? step_ : nullptr, tp_step_, tp_push ? tp_push_step_ : nullptr, lc(true)));
  prof_mark("embed");
  TpArgs ta = {};
  if (tp) {
    ta.rank = tp_rank_;
    ta.size = tp_size_;
    ta.peer_partials = d_peer_partials_;
    ta.peer_flags = d_peer_flags_;
    ta.tp_step = tp_step_;
    ta.n_per_step = 2 * cfg_.layers;
    ta.parity_stride = m_max_ * h;
    ta.M = M;
    ta.hidden = h;
    ta.resid = h_;
    ta.out = h_;
    ta.variant = 1;  // st.release.sys alone orders the partials before the flag (no separate fence before the store)
  }
  // decode-sized forwards (<= 4 rows): the allreduce kernel pushes 16-byte {value, epoch} words and polls its own slots
  // (one NVLink one-way latency) instead of flag + pull (kernels.cu: tp_allreduce_ll_kernel)
  const bool tp_ll = tp && tp_ll_ && tp_off_ll_ && M <= 4 && !tp_push;
  TpLlArgs tl = {};
  tl.peer_ll = d_peer_ll_;
  tl.src_stride = 4LL * (h / 2);
  tl.parity_stride = 8 * tl.src_stride;
  // experimental: prefill-sized forwards reduce-scatter + gather bf16 slices instead of pulling every peer's full partial
  const bool tp_two = tp && tp_two_shot_ && M >= tp_two_shot_min_rows_;
  TpArgs2 t2 = {};
  if (tp_two) {
    t2.rank = tp_rank_;
    t2.size = tp_size_;
    t2.peer_partials = d_peer_partials_;
    t2.peer_flags = d_peer_flags_;
    t2.peer_gather = d_peer_gather_;
    t2.tp_step = tp_step_;
    t2.n_per_step = 2 * cfg_.layers;
    t2.parity_stride = (long long)m_max_ * h;
    t2.M = M;
    t2.hidden = h;
    t2.resid = h_;
    t2.out = h_;
    t2.done = tp2_done_;
  }
  TpPushArgs tpa = {};
  if (tp_push) {
    tpa.size = tp_size_;
    tpa.recv = tp_recv_;
    tpa.flags = tp_pflags_;
    tpa.tp_step = tp_push_step_;
    tpa.n_per_step = 2 * cfg_.layers;
    tpa.parity_stride = 8LL * max_batch_ * h;
    tpa.src_stride = (long long)max_batch_ * h;
    tpa.M = M;
    tpa.hidden = h;
    tpa.resid = h_;
    tpa.out = h_;
  }
  auto set_push = [&](GemvArgs& g, int seq) {
    g.push_dst = d_peer_recv_;
    g.push_flags = d_peer_pflags_;
    g.push_n = tp_size_;
    g.push_rank = tp_rank_;
    g.push_off = (long long)(seq & 1) * 8LL * max_batch_ * h + (long long)tp_rank_ * max_batch_ * h;
    tpa.seq_in_step = seq;
    tpa.arrivals_per_epoch = (unsigned long long)gemv_grid_ctas(g.M, g.N, g.K, n_sm_);
  };
  ++launches;
  const int n_splits = (M <= max_batch_) ? decode_splits_(M) : 1;
  // projections: CUDA-core GEMV (weights streamed once, M <= 4 rows per pass) or wgmma GEMM (tokens = wgmma N)
  const bool tc = M >= tc_min_rows_;
  const int tn = tc_pick_tn(M);
  // token-tile width per projection (prefill-sized forwards only differ): the activation tensor map's box follows it
  auto pick = [&](int N) { return (tc_tn_prefill_ && M > 128) ? tc_tn_prefill_ : tc_pick_tn_prefill(M, N, n_sm_); };
  const int tn_qkv = pick((Hl_ + 2 * KVHl_) * D), tn_o = pick(h), tn_gu = pick(2 * Il_), tn_down = tn_o;
  TcTensorMap tm_xn, tm_xn_gu, tm_attn, tm_act;
  if (tc) {
    CK(tc_make_tmap(&tm_xn, xn_, M, h, h, tn_qkv));
    CK(tc_make_tmap(&tm_xn_gu, xn_, M, h, h, tn_gu));
    CK(tc_make_tmap(&tm_attn, attn_, M, (int64_t)Hl_ * D, (int64_t)Hl_ * D, tn_o));
    CK(tc_make_tmap(&tm_act, act_, M, Il_, Il_, tn_down));
  }
  for (int l = 0; l < cfg_.layers; ++l) {
    const LayerW& w = lw_[l];
    GemvArgs g = {};
    g.W = w.wqkv;
    g.N = (Hl_ + 2 * KVHl_) * D;
    g.K = h;
    g.x = h_;
    g.ldx = h;
    g.M = M;
    g.norm_w = w.ln1;
    g.eps = cfg_.eps;
    g.q_out = q_;
    g.q_rows = Hl_ * D;
    g.kv_rows = KVHl_ * D;
    g.head_dim = D;
    g.kcache = kpool_ + (size_t)l * kv_layer_elems_;
    g.vcache = vpool_ + (size_t)l * kv_layer_elems_;
    g.block_table = block_table_;
    g.bt_stride = max_blocks_per_seq_;
    g.row_slot = row_slot_;
    g.row_pos = row_pos_;
    g.rope_cs = rope_cs_;
    g.block_size = block_size_;
    g.kvh = KVHl_;
    if (tc) {
      CK(launch_rmsnorm(h_, w.ln1, xn_, M, h, cfg_.eps, lc(true)));
      prof_mark("norm");
      CK(launch_tc_gemm(w.tm_qkv, tm_xn, tn_qkv, g, EPI_QKV_ROPE, lc(true)));
      ++launches;
    } else {
      CK(launch_gemv(g, EPI_QKV_ROPE, NORM_RMS, lc(true)));
    }
    prof_mark("qkv");

    AttnArgs a = {};
    a.q = q_;
    a.kcache = g.kcache;
    a.vcache = g.vcache;
    a.block_table = block_table_;
    a.bt_stride = max_blocks_per_seq_;
    a.row_slot = row_slot_;
    a.row_pos = row_pos_;
    a.out = attn_;
    a.part_o = part_o_;
    a.part_ml = part_ml_;
    a.counters = counters_;
    a.M = M;
    a.n_heads = Hl_;
    a.kvh = KVHl_;
    a.group = group;
    a.head_dim = D;
    a.block_size = block_size_;
    a.n_splits = n_splits;
    a.scale = 1.0f / sqrtf((float)D);
    a.tile_row0 = tile_row0_;
    a.tile_nrows = tile_nrows_;
    a.n_tiles = n_pf_tiles_;
    if (n_pf_tiles_ > 0)
      CK(launch_attn_prefill(a, lc(true)));
    else
      CK(launch_attn_decode(a, lc(true)));
    prof_mark("attn");
    if (taps_ && l == 0) {
      CK(cudaMemcpyAsync(tap_q0_, q_, (size_t)M * Hl_ * D * 2, cudaMemcpyDeviceToDevice, stream_));
      CK(cudaMemcpyAsync(tap_attn0_, attn_, (size_t)M * Hl_ * D * 2, cudaMemcpyDeviceToDevice, stream_));
    }

    GemvArgs o = {};
    o.W = w.wo;
    o.N = h;
    o.K = Hl_ * D;
    o.x = attn_;
    o.ldx = Hl_ * D;
    o.M = M;
    o.out_bf16 = h_;
    o.resid = h_;
    o.ld_out = h;
    const int epi_rowpar = tp_push ? EPI_F32_PUSH : tp ? EPI_F32 : EPI_RESID;  // row-parallel under TP: fp32 partial -> allreduce + residual
    if (tp) o.out_f32 = tp_partials_ + (size_t)((2 * l) & 1) * m_max_ * h;
    if (tp_push) set_push(o, 2 * l);
    if (tc)
      CK(launch_tc_gemm(w.tm_o, tm_attn, tn_o, o, epi_rowpar, lc(true)));
    else
      CK(launch_gemv(o, epi_rowpar, NORM_NONE, lc(true)));
    prof_mark("o");
    if (tp_push) {
      CK(launch_tp_reduce_push(tpa, lc(true)));
      ++launches;
    } else if (tp_two) {
      t2.seq_in_step = 2 * l;
      CK(launch_tp_allreduce2(t2, lc(true)));
      ++launches;
    } else if (tp) {
      ta.seq_in_step = 2 * l;
      if (tp_ll)
        CK(launch_tp_allreduce_ll(ta, tl, lc(true)));
      else
        CK(launch_tp_allreduce_resid(ta, lc(true)));
      ++launches;
    }

    GemvArgs u = {};
    u.W = w.wgu;
    u.N = 2 * Il_;
    u.K = h;
    u.x = h_;
    u.ldx = h;
    u.M = M;
    u.norm_w = w.ln2;
    u.eps = cfg_.eps;
    u.out_bf16 = act_;
    u.ld_out = Il_;
    prof_mark("allreduce");
    if (tc) {
      CK(launch_rmsnorm(h_, w.ln2, xn_, M, h, cfg_.eps, lc(true)));
      prof_mark("norm");
      CK(launch_tc_gemm(w.tm_gu, tm_xn_gu, tn_gu, u, EPI_SWIGLU, lc(true)));
      ++launches;
    } else {
      CK(launch_gemv(u, EPI_SWIGLU, NORM_RMS, lc(true)));
    }
    prof_mark("gate_up");

    GemvArgs d = {};
    d.W = w.wdown;
    d.N = h;
    d.K = Il_;
    d.x = act_;
    d.ldx = Il_;
    d.M = M;
    d.out_bf16 = h_;
    d.resid = h_;
    d.ld_out = h;
    if (tp) d.out_f32 = tp_partials_ + (size_t)((2 * l + 1) & 1) * m_max_ * h;
    if (tp_push) set_push(d, 2 * l + 1);
    if (tc)
      CK(launch_tc_gemm(w.tm_down, tm_act, tn_down, d, epi_rowpar, lc(true)));
    else
      CK(launch_gemv(d, epi_rowpar, NORM_NONE, lc(true)));
    prof_mark("down");
    if (tp_push) {
      CK(launch_tp_reduce_push(tpa, lc(true)));
      ++launches;
    } else if (tp_two) {
      t2.seq_in_step = 2 * l + 1;
      CK(launch_tp_allreduce2(t2, lc(true)));
      ++launches;
    } else if (tp) {
      ta.seq_in_step = 2 * l + 1;
      if (tp_ll)
        CK(launch_tp_allreduce_ll(ta, tl, lc(true)));
      else
        CK(launch_tp_allreduce_resid(ta, lc(true)));
      ++launches;
    }
    launches += 5;
    prof_mark("allreduce");
    if (taps_ && l == 0) {
      CK(cudaMemcpyAsync(tap_h0_, h_, (size_t)M * h * 2, cudaMemcpyDeviceToDevice, stream_));
      tap_rows_ = M;
    }
  }
  if (n_logit_rows > 0) {
    GemvArgs g = {};
    g.W = lm_head_;
    g.N = cfg_.vocab;
    g.K = h;
    g.x = h_;
    g.ldx = h;
    g.M = n_logit_rows;
    g.row_map = decode_mode ? nullptr : logit_rows_;
    g.norm_w = final_norm_;
    g.eps = cfg_.eps;
    g.out_f32 = logits_;
    g.ld_out = cfg_.vocab;
    if (tc && decode_mode && n_logit_rows == M) {  // batched decode: lm_head on the tensor cores too (stream-K)
      CK(launch_rmsnorm(h_, final_norm_, xn_, M, h, cfg_.eps, lc(true)));
      CK(launch_tc_gemm(tm_lm_head_, tm_xn, tn, g, EPI_F32_BF16R, lc(true)));
      ++launches;
    } else {
      CK(launch_gemv(g, EPI_F32_BF16R, NORM_RMS, lc(true)));
    }
    CK(launch_argmax(logits_, cfg_.vocab, n_logit_rows, decode_mode ? row_tok_ : next_tok_, decode_mode ? hist_ : nullptr,
                     step_, decode_mode ? row_pos_ : nullptr, lc(true)));
    launches += 2;
    prof_mark("lm_head+argmax");
  }
  launches_per_forward_ = launches;
  timing_.kernel_launches += launches;
  prof_collect();
  return SSB_OK;
}

int Engine::prefill(const int* seq_ids, const int32_t* tokens, const int* lens, int nseq, int32_t* next_tok, float* logits) {
  if (nseq < 1 || nseq > max_batch_) RET(SSB_EINVAL, "nseq out of range");
  if (tp_size_ > 1 && !tp_connected_) RET(SSB_ESTATE, "tensor-parallel engine: call ssb_tp_connect first");
  CK(cudaSetDevice(device_));
  int total = 0;
  std::vector<int> slots(seq_ids, seq_ids + nseq);
  for (int i = 0; i < nseq; ++i) {
    const int s = seq_ids[i];
    if (s < 0 || s >= max_batch_ || !slots_[s].used) RET(SSB_EINVAL, "bad seq_id");
    if (lens[i] < 1) RET(SSB_EINVAL, "empty prompt");
    for (int j = 0; j < i; ++j)
      if (seq_ids[j] == s) RET(SSB_EINVAL, "duplicate seq_id");
    total += lens[i];
  }
  for (int i = 0, o = 0; i < nseq; o += lens[i], ++i)
    for (int t = 0; t < lens[i]; ++t)
      if (tokens[o + t] < 0 || tokens[o + t] >= cfg_.vocab) RET(SSB_EINVAL, "token id out of range");
  // blocks last, and for the whole call or not at all: a refused call leaves the pool as it found it
  {
    std::vector<int> new_len(nseq);
    for (int i = 0; i < nseq; ++i) new_len[i] = slots_[seq_ids[i]].len + lens[i];
    TRY(ensure_blocks_all(seq_ids, new_len.data(), nseq));
  }
  TRY(upload_block_rows(slots));
  // flatten rows
  std::vector<int> r_tok(total), r_slot(total), r_pos(total), r_last(total, -1);
  for (int i = 0, o = 0; i < nseq; o += lens[i], ++i)
    for (int t = 0; t < lens[i]; ++t) {
      r_tok[o + t] = tokens[o + t];
      r_slot[o + t] = seq_ids[i];
      r_pos[o + t] = slots_[seq_ids[i]].len + t;
      if (t == lens[i] - 1) r_last[o + t] = i;
    }
  CK(cudaEventRecord(ev0_, stream_));
  std::vector<int> h_next(nseq, 0);
  for (int base = 0; base < total; base += m_max_) {
    const int M = std::min(m_max_, total - base);
    std::vector<int> lrows, lseq;
    for (int r = 0; r < M; ++r)
      if (r_last[base + r] >= 0) {
        lrows.push_back(r);
        lseq.push_back(r_last[base + r]);
      }
    CK(cudaMemcpyAsync(row_tok_, r_tok.data() + base, M * sizeof(int), cudaMemcpyHostToDevice, stream_));
    CK(cudaMemcpyAsync(row_slot_, r_slot.data() + base, M * sizeof(int), cudaMemcpyHostToDevice, stream_));
    CK(cudaMemcpyAsync(row_pos_, r_pos.data() + base, M * sizeof(int), cudaMemcpyHostToDevice, stream_));
    timing_.h2d_bytes += 3LL * M * sizeof(int);
    if (!lrows.empty()) {
      CK(cudaMemcpyAsync(logit_rows_, lrows.data(), lrows.size() * sizeof(int), cudaMemcpyHostToDevice, stream_));
      timing_.h2d_bytes += (int64_t)(lrows.size() * sizeof(int));
    }
    // query tiles of the tensor-pipe prefill attention: <= 64 consecutive rows of one sequence (rows are (slot, pos)-ordered)
    std::vector<int> t0, tn_;
    if (M > max_batch_ || M >= 16) {
      const int tq = attn_prefill_tile_rows();
      for (int r = 0; r < M;) {
        int n = 1;
        while (n < tq && r + n < M && r_slot[base + r + n] == r_slot[base + r]) ++n;
        t0.push_back(r);
        tn_.push_back(n);
        r += n;
      }
      CK(cudaMemcpyAsync(tile_row0_, t0.data(), t0.size() * sizeof(int), cudaMemcpyHostToDevice, stream_));
      CK(cudaMemcpyAsync(tile_nrows_, tn_.data(), tn_.size() * sizeof(int), cudaMemcpyHostToDevice, stream_));
      timing_.h2d_bytes += (int64_t)(2 * t0.size() * sizeof(int));
    }
    n_pf_tiles_ = (int)t0.size();
    int frc = forward(M, (int)lrows.size(), false);
    n_pf_tiles_ = 0;
    TRY(frc);
    if (!lrows.empty()) {
      std::vector<int> tmp(lrows.size());
      CK(cudaMemcpyAsync(tmp.data(), next_tok_, lrows.size() * sizeof(int), cudaMemcpyDeviceToHost, stream_));
      timing_.d2h_bytes += (int64_t)(lrows.size() * sizeof(int));
      if (logits) {
        // rows of logits_ are in lrows order; scatter to the caller's [nseq, V]
        std::vector<float> lt(lrows.size() * (size_t)cfg_.vocab);
        CK(cudaMemcpyAsync(lt.data(), logits_, lt.size() * sizeof(float), cudaMemcpyDeviceToHost, stream_));
        CK(cudaStreamSynchronize(stream_));
        timing_.d2h_bytes += (int64_t)(lt.size() * sizeof(float));
        for (size_t k = 0; k < lrows.size(); ++k)
          memcpy(logits + (size_t)lseq[k] * cfg_.vocab, lt.data() + k * cfg_.vocab, (size_t)cfg_.vocab * sizeof(float));
      } else {
        CK(cudaStreamSynchronize(stream_));
      }
      for (size_t k = 0; k < lrows.size(); ++k) h_next[lseq[k]] = tmp[k];
    }
  }
  CK(cudaEventRecord(ev1_, stream_));
  CK(cudaStreamSynchronize(stream_));
  float ms = 0;
  CK(cudaEventElapsedTime(&ms, ev0_, ev1_));
  timing_.prefill_ms = ms;
  for (int i = 0; i < nseq; ++i) {
    slots_[seq_ids[i]].len += lens[i];
    next_tok[i] = h_next[i];
  }
  return SSB_OK;
}

// Falcon (new decoder architecture) forward: per layer
//   a = LN_attn(x), m = LN_mlp(x);  attn = dense(attention(rope(qkv(a))));  out = x + (dense_4h_to_h(gelu(dense_h_to_4h(m))) + attn)
// (HF:models/falcon/modeling_falcon.py:594-636).  Same kernels as Llama with the LayerNorm prologue and the GELU /
// two-addend residual epilogues; under tensor parallelism the two row-parallel partials are summed locally first, so
// there is ONE allreduce per layer.
int Engine::forward_falcon(int M, int n_logit_rows, bool decode_mode) {
  const int h = cfg_.hidden, D = cfg_.head_dim, group = cfg_.heads / cfg_.kv_heads;
  int launches = 0;
  const bool tp = tp_size_ > 1;
  CK(launch_embed(embed_, row_tok_, h_, M, h, decode_mode ? step_ : nullptr, tp_step_, nullptr, lc(true)));
  ++launches;
  const int n_splits = (M <= max_batch_) ? decode_splits_(M) : 1;
  const bool tc = M >= tc_min_rows_;
  auto pick = [&](int N) { return (tc_tn_prefill_ && M > 128) ? tc_tn_prefill_ : tc_pick_tn_prefill(M, N, n_sm_); };
  const int tn_qkv = pick((Hl_ + 2 * KVHl_) * D), tn_o = pick(h), tn_gu = pick(Il_), tn_down = tn_o;
  TcTensorMap tm_xn, tm_xn_gu, tm_attn, tm_act;
  if (tc) {
    CK(tc_make_tmap(&tm_xn, xn_, M, h, h, tn_qkv));
    CK(tc_make_tmap(&tm_xn_gu, xn_, M, h, h, tn_gu));
    CK(tc_make_tmap(&tm_attn, attn_, M, (int64_t)Hl_ * D, (int64_t)Hl_ * D, tn_o));
    CK(tc_make_tmap(&tm_act, act_, M, Il_, Il_, tn_down));
  }
  TpArgs ta = {};
  if (tp) {
    ta.rank = tp_rank_;
    ta.size = tp_size_;
    ta.peer_partials = d_peer_partials_;
    ta.peer_flags = d_peer_flags_;
    ta.tp_step = tp_step_;
    ta.n_per_step = cfg_.layers;
    ta.parity_stride = m_max_ * h;
    ta.M = M;
    ta.hidden = h;
    ta.resid = h_;
    ta.out = h_;
    ta.variant = 1;
  }
  for (int l = 0; l < cfg_.layers; ++l) {
    const LayerW& w = lw_[l];
    GemvArgs g = {};
    g.W = w.wqkv;
    g.N = (Hl_ + 2 * KVHl_) * D;
    g.K = h;
    g.x = h_;
    g.ldx = h;
    g.M = M;
    g.norm_w = w.ln1;
    g.norm_b = w.ln1_b;
    g.eps = cfg_.eps;
    g.q_out = q_;
    g.q_rows = Hl_ * D;
    g.kv_rows = KVHl_ * D;
    g.head_dim = D;
    g.kcache = kpool_ + (size_t)l * kv_layer_elems_;
    g.vcache = vpool_ + (size_t)l * kv_layer_elems_;
    g.block_table = block_table_;
    g.bt_stride = max_blocks_per_seq_;
    g.row_slot = row_slot_;
    g.row_pos = row_pos_;
    g.rope_cs = rope_cs_;
    g.block_size = block_size_;
    g.kvh = KVHl_;
    if (tc) {
      CK(launch_layernorm(h_, w.ln1, w.ln1_b, xn_, M, h, cfg_.eps, lc(true)));
      CK(launch_tc_gemm(w.tm_qkv, tm_xn, tn_qkv, g, EPI_QKV_ROPE, lc(true)));
      ++launches;
    } else {
      CK(launch_gemv(g, EPI_QKV_ROPE, NORM_LN, lc(true)));
    }
    AttnArgs a = {};
    a.q = q_;
    a.kcache = g.kcache;
    a.vcache = g.vcache;
    a.block_table = block_table_;
    a.bt_stride = max_blocks_per_seq_;
    a.row_slot = row_slot_;
    a.row_pos = row_pos_;
    a.out = attn_;
    a.part_o = part_o_;
    a.part_ml = part_ml_;
    a.counters = counters_;
    a.M = M;
    a.n_heads = Hl_;
    a.kvh = KVHl_;
    a.group = group;
    a.head_dim = D;
    a.block_size = block_size_;
    a.n_splits = n_splits;
    a.scale = 1.0f / sqrtf((float)D);
    a.tile_row0 = tile_row0_;
    a.tile_nrows = tile_nrows_;
    a.n_tiles = n_pf_tiles_;
    if (n_pf_tiles_ > 0)
      CK(launch_attn_prefill(a, lc(true)));
    else
      CK(launch_attn_decode(a, lc(true)));
    if (taps_ && l == 0) {
      CK(cudaMemcpyAsync(tap_q0_, q_, (size_t)M * Hl_ * D * 2, cudaMemcpyDeviceToDevice, stream_));
      CK(cudaMemcpyAsync(tap_attn0_, attn_, (size_t)M * Hl_ * D * 2, cudaMemcpyDeviceToDevice, stream_));
    }
    // attention branch output (row-parallel): bf16 ao_ (TP1) or fp32 partial (TP)
    GemvArgs o = {};
    o.W = w.wo;
    o.N = h;
    o.K = Hl_ * D;
    o.x = attn_;
    o.ldx = Hl_ * D;
    o.M = M;
    o.out_bf16 = ao_;
    o.ld_out = h;
    float* part_attn = tp ? falcon_scratch_ : nullptr;  // local fp32 scratch (the exchange buffers may still be read by peers)
    if (tp) o.out_f32 = part_attn;
    const int epi_o = tp ? EPI_F32 : EPI_BF16;
    if (tc)
      CK(launch_tc_gemm(w.tm_o, tm_attn, tn_o, o, epi_o, lc(true)));
    else
      CK(launch_gemv(o, epi_o, NORM_NONE, lc(true)));
    // MLP branch on LN_mlp(x)
    GemvArgs u = {};
    u.W = w.wgu;
    u.N = Il_;
    u.K = h;
    u.x = h_;
    u.ldx = h;
    u.M = M;
    u.norm_w = w.ln2;
    u.norm_b = w.ln2_b;
    u.eps = cfg_.eps;
    u.out_bf16 = act_;
    u.ld_out = Il_;
    if (tc) {
      CK(launch_layernorm(h_, w.ln2, w.ln2_b, xn_, M, h, cfg_.eps, lc(true)));
      CK(launch_tc_gemm(w.tm_gu, tm_xn_gu, tn_gu, u, EPI_GELU, lc(true)));
      ++launches;
    } else {
      CK(launch_gemv(u, EPI_GELU, NORM_LN, lc(true)));
    }
    GemvArgs d = {};
    d.W = w.wdown;
    d.N = h;
    d.K = Il_;
    d.x = act_;
    d.ldx = Il_;
    d.M = M;
    d.out_bf16 = h_;
    d.resid = h_;
    d.resid2 = ao_;
    d.ld_out = h;
    if (tp) {
      d.out_f32 = tp_partials_ + (size_t)(l & 1) * m_max_ * h;
      d.f32_add = part_attn;
    }
    const int epi_d = tp ? EPI_F32 : EPI_RESID2;
    if (tc)
      CK(launch_tc_gemm(w.tm_down, tm_act, tn_down, d, epi_d, lc(true)));
    else
      CK(launch_gemv(d, epi_d, NORM_NONE, lc(true)));
    launches += 5;
    if (tp) {
      ta.seq_in_step = l;
      if (tp_ll_ && tp_off_ll_ && M <= 4) {
        TpLlArgs tl = {};
        tl.peer_ll = d_peer_ll_;
        tl.src_stride = 4LL * (h / 2);
        tl.parity_stride = 8 * tl.src_stride;
        CK(launch_tp_allreduce_ll(ta, tl, lc(true)));
      } else {
        CK(launch_tp_allreduce_resid(ta, lc(true)));
      }
      ++launches;
    }
    if (taps_ && l == 0) {
      CK(cudaMemcpyAsync(tap_h0_, h_, (size_t)M * h * 2, cudaMemcpyDeviceToDevice, stream_));
      tap_rows_ = M;
    }
  }
  if (n_logit_rows > 0) {
    GemvArgs g = {};
    g.W = lm_head_;
    g.N = cfg_.vocab;
    g.K = h;
    g.x = h_;
    g.ldx = h;
    g.M = n_logit_rows;
    g.row_map = decode_mode ? nullptr : logit_rows_;
    g.norm_w = final_norm_;
    g.norm_b = final_norm_b_;
    g.eps = cfg_.eps;
    g.out_f32 = logits_;
    g.ld_out = cfg_.vocab;
    CK(launch_gemv(g, EPI_F32_BF16R, NORM_LN, lc(true)));
    CK(launch_argmax(logits_, cfg_.vocab, n_logit_rows, decode_mode ? row_tok_ : next_tok_, decode_mode ? hist_ : nullptr,
                     step_, decode_mode ? row_pos_ : nullptr, lc(true)));
    launches += 2;
  }
  launches_per_forward_ = launches;
  timing_.kernel_launches += launches;
  return SSB_OK;
}

int Engine::forward_mega(int B) {
  const int D = cfg_.head_dim, group = cfg_.heads / cfg_.kv_heads;
  MegaArgs a = {};
  a.layers = d_mega_layers_;
  a.n_layers = cfg_.layers;
  a.hidden = cfg_.hidden;
  a.q_rows = Hl_ * D;
  a.kv_rows = KVHl_ * D;
  a.head_dim = D;
  a.inter = Il_;
  a.vocab = cfg_.vocab;
  a.n_heads = Hl_;
  a.kvh = KVHl_;
  a.group = group;
  a.attn_g = mega_attn_group(group);
  a.eps = cfg_.eps;
  a.scale = 1.0f / sqrtf((float)D);
  a.M = B;
  a.embed = embed_;
  a.lm_head = lm_head_;
  a.final_norm = final_norm_;
  a.h = h_;
  a.q = q_;
  a.attn = attn_;
  a.act = act_;
  a.logits = logits_;
  a.row_tok = row_tok_;
  a.row_slot = row_slot_;
  a.row_pos = row_pos_;
  a.block_table = block_table_;
  a.bt_stride = max_blocks_per_seq_;
  a.block_size = block_size_;
  a.rope_cs = rope_cs_;
  a.part_o = mega_part_o_;
  a.part_ml = mega_part_ml_;
  a.counters = mega_counters_;
  a.max_chunks = mega_max_chunks_;
  a.hist = hist_;
  a.step = step_;
  a.fwd_counter = tp_step_;
  a.grid_bar = mega_bar_;
  a.k_max = mega_k_max_;
  a.prof = mega_prof_;
  a.prof_all = mega_prof_all_ ? 1 : 0;
  if (mega_prof_all_) CK(cudaMemsetAsync(mega_prof_, 0, (size_t)n_sm_ * 1024 * sizeof(unsigned long long), stream_));
  a.n_stages = mega_pick_stages(B == 1 ? 1 : (B == 2 ? 2 : 4), mega_k_max_);
  // GQA groups of 8: CTA-tile attention when the K/V tile fits the activation staging area (params "mega_attn_tile": 0 = off)
  a.head_done = mega_head_done_;
  a.attn_coop = (a.attn_g < 8 && mega_attn_tile_ &&
                 (size_t)(B == 1 ? 1 : (B == 2 ? 2 : 4)) * mega_k_max_ * sizeof(bf16) >= mega_attn_coop_bytes(D, a.attn_g)) ? 1 : 0;
  a.attn_cta_tile = (a.attn_g == 8 && mega_attn_tile_ &&
                     (size_t)(B == 1 ? 1 : (B == 2 ? 2 : 4)) * mega_k_max_ * sizeof(bf16) >= mega_attn_tile_bytes(D)) ? 1 : 0;
  if (a.n_stages == 0) RET(SSB_EINVAL, "decode step does not fit the persistent kernel's shared memory");
  if (tp_size_ > 1) {  // "tp_mega": allreduce inside the kernel, same exchange pool / epochs as launch_tp_allreduce_resid
    a.tp_size = tp_size_;
    a.tp_rank = tp_rank_;
    a.peer_partials = d_peer_partials_;
    a.peer_flags = d_peer_flags_;
    a.parity_stride = (long long)m_max_ * cfg_.hidden;
    a.tp_mode = tp_mega_mode_ >= 2 ? tp_mega_mode_ : 1;
    a.peer_cta_flags = d_peer_cta_flags_;
    a.peer_ll = d_peer_ll_;
    a.ll_src_stride = 4LL * (cfg_.hidden / 2);
    a.ll_parity_stride = 8 * a.ll_src_stride;
  }
  // no PDL: the kernel resets its pass-claim counters at exit, and the next step must not claim before that (mega.cu)
  CK(launch_decode_mega(a, LaunchCfg{stream_, false, n_sm_}));
  launches_per_forward_ = 1;
  timing_.kernel_launches += 1;
  return SSB_OK;
}

int Engine::build_graph(int B) {
  cudaGraph_t graph = nullptr;
  CK(cudaStreamBeginCapture(stream_, cudaStreamCaptureModeThreadLocal));
  int rc = forward(B, B, true);
  cudaError_t e = cudaStreamEndCapture(stream_, &graph);
  if (rc != SSB_OK) {
    if (graph) cudaGraphDestroy(graph);
    return rc;
  }
  if (e != cudaSuccess) RET(SSB_ECUDA, std::string("cudaStreamEndCapture: ") + cudaGetErrorString(e));
  cudaGraphExec_t exec = nullptr;
  e = cudaGraphInstantiate(&exec, graph, 0);
  cudaGraphDestroy(graph);
  if (e != cudaSuccess) RET(SSB_ECUDA, std::string("cudaGraphInstantiate: ") + cudaGetErrorString(e));
  graphs_[B] = exec;
  graph_launches_[B] = launches_per_forward_;
  timing_.kernel_launches -= launches_per_forward_;  // capture enqueued nothing
  return SSB_OK;
}

int Engine::decode(const int* seq_ids, const int32_t* last_tok, int nseq, int nsteps, int32_t* out_tok, float* logits) {
  if (nseq < 1 || nseq > max_batch_) RET(SSB_EINVAL, "nseq out of range");
  if (nsteps < 1 || nsteps > max_steps_) RET(SSB_EINVAL, "nsteps out of range");
  if (tp_size_ > 1 && !tp_connected_) RET(SSB_ESTATE, "tensor-parallel engine: call ssb_tp_connect first");
  CK(cudaSetDevice(device_));
  std::vector<int> slots(seq_ids, seq_ids + nseq), pos(nseq);
  for (int i = 0; i < nseq; ++i) {
    const int s = seq_ids[i];
    if (s < 0 || s >= max_batch_ || !slots_[s].used) RET(SSB_EINVAL, "bad seq_id");
    for (int j = 0; j < i; ++j)
      if (seq_ids[j] == s) RET(SSB_EINVAL, "duplicate seq_id");
    if (last_tok[i] < 0 || last_tok[i] >= cfg_.vocab) RET(SSB_EINVAL, "token id out of range");
    pos[i] = slots_[s].len;
  }
  {
    std::vector<int> new_len(nseq);
    for (int i = 0; i < nseq; ++i) new_len[i] = pos[i] + nsteps;
    TRY(ensure_blocks_all(seq_ids, new_len.data(), nseq));
  }
  TRY(upload_block_rows(slots));
  CK(cudaMemcpyAsync(row_tok_, last_tok, nseq * sizeof(int), cudaMemcpyHostToDevice, stream_));
  CK(cudaMemcpyAsync(row_slot_, slots.data(), nseq * sizeof(int), cudaMemcpyHostToDevice, stream_));
  CK(cudaMemcpyAsync(row_pos_, pos.data(), nseq * sizeof(int), cudaMemcpyHostToDevice, stream_));
  CK(cudaMemsetAsync(step_, 0xFF, sizeof(int), stream_));  // -1: the embed kernel pre-increments
  timing_.h2d_bytes += 3LL * nseq * sizeof(int);
  // persistent kernel for batch <= mega_max_batch_ (default 1); from 2 rows the graph + PDL multi-kernel step, whose
  // proj_rows_kernel runs on the tensor pipe with a 6-deep ring (DESIGN.md §4 gives the H100 comparison)
  const bool mega = use_mega_ && !taps_ && nseq <= mega_max_batch_ && nseq <= 4 && nseq < tc_min_rows_ && mega_pick_stages(nseq == 1 ? 1 : (nseq == 2 ? 2 : 4), mega_k_max_) > 0;
  const bool graph = use_graph_ && !taps_ && !mega;
  if (graph && !graphs_.count(nseq)) {
    CK(cudaStreamSynchronize(stream_));
    TRY(build_graph(nseq));
  }
  CK(cudaEventRecord(ev0_, stream_));
  for (int s = 0; s < nsteps; ++s) {
    if (mega) {
      TRY(forward_mega(nseq));
    } else if (graph) {
      CK(cudaGraphLaunch(graphs_[nseq], stream_));
      timing_.kernel_launches += graph_launches_[nseq];
    } else {
      TRY(forward(nseq, nseq, true));
    }
    if (logits) {
      CK(cudaMemcpyAsync(logits + (size_t)s * nseq * cfg_.vocab, logits_, (size_t)nseq * cfg_.vocab * sizeof(float),
                         cudaMemcpyDeviceToHost, stream_));
      timing_.d2h_bytes += (int64_t)nseq * cfg_.vocab * sizeof(float);
    }
  }
  CK(cudaEventRecord(ev1_, stream_));
  std::vector<int> hist((size_t)nsteps * nseq);
  CK(cudaMemcpyAsync(hist.data(), hist_, hist.size() * sizeof(int), cudaMemcpyDeviceToHost, stream_));
  CK(cudaStreamSynchronize(stream_));
  timing_.d2h_bytes += (int64_t)(hist.size() * sizeof(int));
  float ms = 0;
  CK(cudaEventElapsedTime(&ms, ev0_, ev1_));
  timing_.decode_ms = ms;
  for (int i = 0; i < nseq; ++i) {
    for (int s = 0; s < nsteps; ++s) out_tok[(size_t)i * nsteps + s] = hist[(size_t)s * nseq + i];
    slots_[seq_ids[i]].len += nsteps;
  }
  return SSB_OK;
}

// Times `iters` back-to-back launches of one kernel class, cycling over the layers' weights (so nothing is served
// from L2), between CUDA events on the engine stream.  rows = batch rows; ctx = cached length for "attn".
int Engine::bench_kernel(const char* which, int rows, int ctx, int iters, double* ms_out, int64_t* bytes_out) {
  if (rows < 1 || rows > max_batch_ || iters < 1) RET(SSB_EINVAL, "bad rows/iters");
  CK(cudaSetDevice(device_));
  std::string w = which ? which : "";
  // "<name>@l2": reuse layer 0's weights every launch (L2-resident when the matrix fits the 50 MB L2) — separates the
  // kernel's own consumption rate from the HBM rate
  bool same_layer = false;
  if (w.size() > 3 && w.compare(w.size() - 3, 3, "@l2") == 0) {
    same_layer = true;
    w.resize(w.size() - 3);
  }
  int variant = 0;       // "allreduce@v<bits>[n]": latency experiments, trailing 'n' = no PDL
  bool bench_pdl = true;
  bool bench_ll = false;
  if (w == "allreduce_ll" || w == "allreduce_lln") {
    bench_ll = true;
    bench_pdl = w.back() != 'n';
    w = "allreduce";
  }
  if (w.rfind("allreduce@v", 0) == 0) {
    variant = atoi(w.c_str() + 11);
    if (w.back() == 'n') bench_pdl = false;
    w = "allreduce";
  }
  const int h = cfg_.hidden, D = cfg_.head_dim;
  // stage a decode-like batch: rows sequences of length ctx (slots 0..rows-1 must be free)
  std::vector<int> sl(rows), tok(rows, 1), pos(rows, ctx - 1);
  for (int i = 0; i < rows; ++i) {
    if (slots_[i].used) RET(SSB_ESTATE, "bench_kernel needs free sequence slots");
    sl[i] = i;
  }
  for (int i = 0; i < rows; ++i) {
    slots_[i].used = true;
    int rc = ensure_blocks(i, ctx);
    if (rc != SSB_OK) {
      for (int j = 0; j <= i; ++j) seq_free(j);
      return rc;
    }
  }
  int rc = upload_block_rows(sl);
  if (rc == SSB_OK) {
    cudaMemcpyAsync(row_tok_, tok.data(), rows * sizeof(int), cudaMemcpyHostToDevice, stream_);
    cudaMemcpyAsync(row_slot_, sl.data(), rows * sizeof(int), cudaMemcpyHostToDevice, stream_);
    cudaMemcpyAsync(row_pos_, pos.data(), rows * sizeof(int), cudaMemcpyHostToDevice, stream_);
    cudaMemsetAsync(h_, 0, (size_t)rows * h * 2, stream_);
    cudaMemsetAsync(attn_, 0, (size_t)rows * Hl_ * D * 2, stream_);
    cudaMemsetAsync(act_, 0, (size_t)rows * Il_ * 2, stream_);
    cudaMemsetAsync(q_, 0, (size_t)rows * Hl_ * D * 2, stream_);
  }
  int64_t bytes = 0;
  const bool btc = rows >= tc_min_rows_ && !cfg_.falcon;  // mirror forward(): tensor-core projections from tc_min_rows up
  const int btn = tc_pick_tn(rows);
  TcTensorMap btm_xn, btm_attn, btm_act;
  if (btc) {
    CK(tc_make_tmap(&btm_xn, xn_, rows, h, h, btn));
    CK(tc_make_tmap(&btm_attn, attn_, rows, (int64_t)Hl_ * D, (int64_t)Hl_ * D, btn));
    CK(tc_make_tmap(&btm_act, act_, rows, Il_, Il_, btn));
    cudaMemsetAsync(xn_, 0, (size_t)rows * h * 2, stream_);
  }
  auto one = [&](int l) -> int {
    if (same_layer) l = 0;
    const LayerW& lwv = lw_[l % cfg_.layers];
    GemvArgs g = {};
    g.x = h_;
    g.ldx = h;
    g.K = h;
    g.M = rows;
    g.eps = cfg_.eps;
    if (w == "qkv") {
      g.W = lwv.wqkv;
      g.N = (Hl_ + 2 * KVHl_) * D;
      g.norm_w = lwv.ln1;
      g.q_out = q_;
      g.q_rows = Hl_ * D;
      g.kv_rows = KVHl_ * D;
      g.head_dim = D;
      g.kcache = kpool_ + (size_t)(l % cfg_.layers) * kv_layer_elems_;
      g.vcache = vpool_ + (size_t)(l % cfg_.layers) * kv_layer_elems_;
      g.block_table = block_table_;
      g.bt_stride = max_blocks_per_seq_;
      g.row_slot = row_slot_;
      g.row_pos = row_pos_;
      g.rope_cs = rope_cs_;
      g.block_size = block_size_;
      g.kvh = KVHl_;
      g.norm_b = lwv.ln1_b;
      bytes = 2LL * g.N * g.K;
      if (btc)
        CK(launch_tc_gemm(lwv.tm_qkv, btm_xn, btn, g, EPI_QKV_ROPE, lc(true)));
      else
        CK(launch_gemv(g, EPI_QKV_ROPE, cfg_.falcon ? NORM_LN : NORM_RMS, lc(true)));
    } else if (w == "gate_up") {
      g.W = lwv.wgu;
      g.N = (cfg_.falcon ? 1 : 2) * Il_;
      g.norm_w = lwv.ln2;
      g.norm_b = lwv.ln2_b;
      g.out_bf16 = act_;
      g.ld_out = Il_;
      bytes = 2LL * g.N * g.K;
      if (btc)
        CK(launch_tc_gemm(lwv.tm_gu, btm_xn, btn, g, EPI_SWIGLU, lc(true)));
      else
        CK(launch_gemv(g, cfg_.falcon ? EPI_GELU : EPI_SWIGLU, cfg_.falcon ? NORM_LN : NORM_RMS, lc(true)));
    } else if (w == "o") {
      g.W = lwv.wo;
      g.N = h;
      g.K = Hl_ * D;
      g.x = attn_;
      g.ldx = Hl_ * D;
      g.out_bf16 = h_;
      g.resid = h_;
      g.ld_out = h;
      bytes = 2LL * g.N * g.K;
      if (btc)
        CK(launch_tc_gemm(lwv.tm_o, btm_attn, btn, g, EPI_RESID, lc(true)));
      else
        CK(launch_gemv(g, EPI_RESID, NORM_NONE, lc(true)));
    } else if (w == "down") {
      g.W = lwv.wdown;
      g.N = h;
      g.K = Il_;
      g.x = act_;
      g.ldx = Il_;
      g.out_bf16 = h_;
      g.resid = h_;
      g.ld_out = h;
      bytes = 2LL * g.N * g.K;
      if (btc)
        CK(launch_tc_gemm(lwv.tm_down, btm_act, btn, g, EPI_RESID, lc(true)));
      else
        CK(launch_gemv(g, EPI_RESID, NORM_NONE, lc(true)));
    } else if (w == "lm_head") {
      g.W = lm_head_;
      g.N = cfg_.vocab;
      g.norm_w = final_norm_;
      g.norm_b = final_norm_b_;
      g.out_f32 = logits_;
      g.ld_out = cfg_.vocab;
      bytes = 2LL * g.N * g.K;
      if (btc) {  // mirror forward(): batched decode runs lm_head on the tensor cores (norm kernel + stream-K GEMM)
        CK(launch_rmsnorm(h_, final_norm_, xn_, rows, h, cfg_.eps, lc(true)));
        CK(launch_tc_gemm(tm_lm_head_, btm_xn, btn, g, EPI_F32_BF16R, lc(true)));
      } else {
        CK(launch_gemv(g, EPI_F32_BF16R, cfg_.falcon ? NORM_LN : NORM_RMS, lc(true)));
      }
    } else if (w == "attn") {
      AttnArgs a = {};
      a.q = q_;
      a.kcache = kpool_ + (size_t)(l % cfg_.layers) * kv_layer_elems_;
      a.vcache = vpool_ + (size_t)(l % cfg_.layers) * kv_layer_elems_;
      a.block_table = block_table_;
      a.bt_stride = max_blocks_per_seq_;
      a.row_slot = row_slot_;
      a.row_pos = row_pos_;
      a.out = attn_;
      a.part_o = part_o_;
      a.part_ml = part_ml_;
      a.counters = counters_;
      a.M = rows;
      a.n_heads = Hl_;
      a.kvh = KVHl_;
      a.group = cfg_.heads / cfg_.kv_heads;
      a.head_dim = D;
      a.block_size = block_size_;
      a.n_splits = decode_splits_(rows);
      a.scale = 1.0f / sqrtf((float)D);
      bytes = 2LL * rows * ctx * KVHl_ * D * 2;
      CK(launch_attn_decode(a, lc(true)));
    } else if (w == "allreduce") {
      // collective: every rank must run the same bench_kernel("allreduce", ...) call at the same time
      if (tp_size_ < 2 || !tp_connected_) RET(SSB_ESTATE, "allreduce bench needs a connected tensor-parallel engine");
      TpArgs ta = {};
      ta.rank = tp_rank_;
      ta.size = tp_size_;
      ta.peer_partials = d_peer_partials_;
      ta.peer_flags = d_peer_flags_;
      ta.tp_step = tp_step_;
      ta.n_per_step = iters + 3;
      ta.seq_in_step = l;
      ta.parity_stride = m_max_ * h;
      ta.M = rows;
      ta.hidden = h;
      ta.resid = h_;
      ta.out = h_;
      ta.variant = variant;
      bytes = (int64_t)(tp_size_ - 1) * rows * h * 4;
      if (bench_ll) {  // "allreduce_ll": the LL push kernel (decode-sized forwards of the multi-kernel path)
        if (!tp_off_ll_ || rows > 4) RET(SSB_ESTATE, "allreduce_ll needs params.tp_ll / tp_mega 3 and rows <= 4");
        TpLlArgs tl = {};
        tl.peer_ll = d_peer_ll_;
        tl.src_stride = 4LL * (h / 2);
        tl.parity_stride = 8 * tl.src_stride;
        CK(launch_tp_allreduce_ll(ta, tl, lc(bench_pdl)));
      } else {
        CK(launch_tp_allreduce_resid(ta, lc(bench_pdl)));
      }
    } else {
      RET(SSB_EINVAL, "unknown kernel '" + w + "' (qkv|o|gate_up|down|lm_head|attn|allreduce)");
    }
    return SSB_OK;
  };
  if (w == "allreduce") {  // a fresh epoch range for this run: one forward-counter tick, sequence numbers 0..iters+2
    CK(launch_embed(embed_, row_tok_, h_, rows, h, nullptr, tp_step_, nullptr, lc(false)));
    cudaMemsetAsync(tp_partials_, 0, 2 * (size_t)m_max_ * h * sizeof(float), stream_);
  }
  for (int i = 0; i < 3 && rc == SSB_OK; ++i) rc = one(i);
  if (rc == SSB_OK) {
    cudaEventRecord(ev0_, stream_);
    for (int i = 0; i < iters && rc == SSB_OK; ++i) rc = one(i + 3);
    cudaEventRecord(ev1_, stream_);
    cudaError_t e = cudaStreamSynchronize(stream_);
    if (rc == SSB_OK && e != cudaSuccess) {
      set_error(std::string("bench_kernel: ") + cudaGetErrorString(e));
      rc = SSB_ECUDA;
    }
    float ms = 0;
    if (rc == SSB_OK) {
      cudaEventElapsedTime(&ms, ev0_, ev1_);
      *ms_out = (double)ms / iters;
      *bytes_out = bytes;
      timing_.kernel_launches += iters + 3;
    }
  }
  for (int i = 0; i < rows; ++i) seq_free(i);
  return rc;
}

// ---- tensor-parallel bootstrap: exchange buffers are exported as CUDA IPC handles (or raw pointers inside one process)
struct TpHandle {
  uint32_t magic;
  int32_t rank, size, device;
  int64_t pid;
  cudaIpcMemHandle_t pool;
  uint64_t raw_pool, pool_bytes;
};
static_assert(sizeof(TpHandle) <= 256, "ssb_tp_handle_size");

int Engine::tp_export(void* out) {
  if (tp_size_ < 2) RET(SSB_ESTATE, "engine is not tensor parallel");
  CK(cudaSetDevice(device_));
  TpHandle hd;
  memset(&hd, 0, sizeof hd);
  hd.magic = 0x53534254u;
  hd.rank = tp_rank_;
  hd.size = tp_size_;
  hd.device = device_;
  hd.pid = (int64_t)getpid();
  CK(cudaIpcGetMemHandle(&hd.pool, tp_pool_));
  hd.raw_pool = (uint64_t)(uintptr_t)tp_pool_;
  hd.pool_bytes = (uint64_t)tp_pool_bytes_;
  memset(out, 0, 256);
  memcpy(out, &hd, sizeof hd);
  return SSB_OK;
}

int Engine::tp_connect(const void* all, int n) {
  if (tp_size_ < 2) RET(SSB_ESTATE, "engine is not tensor parallel");
  if (n != tp_size_) RET(SSB_EINVAL, "n_ranks != tp_size");
  CK(cudaSetDevice(device_));
  std::vector<uint8_t*> pool(8, nullptr);
  for (int r = 0; r < n; ++r) {
    TpHandle hd;
    memcpy(&hd, (const char*)all + (size_t)r * 256, sizeof hd);
    if (hd.magic != 0x53534254u || hd.rank != r || hd.size != tp_size_ || hd.pool_bytes != (uint64_t)tp_pool_bytes_)
      RET(SSB_EINVAL, "bad TP handle for rank " + std::to_string(r) + " (ranks must be created with identical params)");
    if (r == tp_rank_) {
      pool[r] = tp_pool_;
    } else if (hd.pid == (int64_t)getpid()) {  // several ranks in one process (serve host): plain peer access
      if (hd.device != device_) {
        cudaError_t e = cudaDeviceEnablePeerAccess(hd.device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) CK(e);
        cudaGetLastError();
      }
      pool[r] = (uint8_t*)(uintptr_t)hd.raw_pool;
    } else {
      void* a = nullptr;
      CK(cudaIpcOpenMemHandle(&a, hd.pool, cudaIpcMemLazyEnablePeerAccess));
      ipc_opened_.push_back(a);
      pool[r] = (uint8_t*)a;
    }
  }
  std::vector<float*> pp(8, nullptr), pr(8, nullptr);
  std::vector<uint32_t*> pf(8, nullptr);
  std::vector<unsigned long long*> pq(8, nullptr);
  for (int r = 0; r < n; ++r) {
    pp[r] = (float*)pool[r];
    pr[r] = (float*)(pool[r] + tp_off_recv_);
    pf[r] = (uint32_t*)(pool[r] + tp_off_flags_);
    pq[r] = (unsigned long long*)(pool[r] + tp_off_pflags_);
  }
  CK(cudaMemcpy(d_peer_partials_, pp.data(), 8 * sizeof(float*), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_peer_flags_, pf.data(), 8 * sizeof(uint32_t*), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_peer_recv_, pr.data(), 8 * sizeof(float*), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_peer_pflags_, pq.data(), 8 * sizeof(unsigned long long*), cudaMemcpyHostToDevice));
  if (tp_mega_mode_ == 2) {
    std::vector<uint32_t*> pc(8, nullptr);
    for (int r = 0; r < n; ++r) pc[r] = (uint32_t*)(pool[r] + tp_off_ctaflags_);
    CK(cudaMemcpy(d_peer_cta_flags_, pc.data(), 8 * sizeof(uint32_t*), cudaMemcpyHostToDevice));
  }
  if (tp_off_ll_) {
    std::vector<uint4*> pl(8, nullptr);
    for (int r = 0; r < n; ++r) pl[r] = (uint4*)(pool[r] + tp_off_ll_);
    CK(cudaMemcpy(d_peer_ll_, pl.data(), 8 * sizeof(uint4*), cudaMemcpyHostToDevice));
  }
  if (tp_two_shot_) {
    std::vector<bf16*> pg(8, nullptr);
    for (int r = 0; r < n; ++r) pg[r] = (bf16*)(pool[r] + tp_off_gather_);
    CK(cudaMemcpy(d_peer_gather_, pg.data(), 8 * sizeof(bf16*), cudaMemcpyHostToDevice));
  }
  tp_connected_ = true;
  return SSB_OK;
}

int Engine::last_timing(ssb_timing* t) const {
  *t = timing_;
  return SSB_OK;
}

void Engine::timing_reset() { timing_ = ssb_timing{}; }

int Engine::debug_read(const char* name, float* dst, int64_t n, int* rows, int* cols) {
  const std::string nm = name ? name : "";
  if (nm == "sk_prof") {  // [n_sm][8] stamps of the last stream-K projection launch, us from the earliest (0 = not stamped)
    if (!sk_prof_) RET(SSB_ESTATE, "engine was not created with params.sk_prof=1");
    if (n < (int64_t)n_sm_ * 8) RET(SSB_EINVAL, "destination too small");
    CK(cudaSetDevice(device_));
    CK(cudaStreamSynchronize(stream_));
    std::vector<unsigned long long> t((size_t)n_sm_ * 8);
    CK(cudaMemcpy(t.data(), sk_prof_, t.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    unsigned long long t0 = ~0ull;
    for (size_t i = 0; i < t.size(); ++i)
      if (i % 8 != 7 && t[i] && t[i] < t0) t0 = t[i];
    for (size_t i = 0; i < t.size(); ++i)  // column 7 is a count (segments of the CTA's range), not a time
      dst[i] = i % 8 == 7 ? (float)t[i] : (t[i] ? (float)((double)(t[i] - t0) * 1e-3) : -1.0f);
    *rows = n_sm_;
    *cols = 8;
    return SSB_OK;
  }
  if (nm == "mega_prof_all") {  // [n_ctas][1024]: per-CTA phase stamps of the LAST step in us from the earliest one; column 1023 = %smid
    if (!mega_prof_ || !mega_prof_all_) RET(SSB_ESTATE, "engine was not created with params.mega_prof=2");
    if (n < (int64_t)n_sm_ * 1024) RET(SSB_EINVAL, "destination too small");
    CK(cudaSetDevice(device_));
    std::vector<unsigned long long> t((size_t)n_sm_ * 1024);
    CK(cudaMemcpy(t.data(), mega_prof_, t.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    unsigned long long t0 = ~0ull;
    for (int c = 0; c < n_sm_; ++c)
      if (t[(size_t)c * 1024] && t[(size_t)c * 1024] < t0) t0 = t[(size_t)c * 1024];
    for (int c = 0; c < n_sm_; ++c)
      for (int i = 0; i < 1024; ++i) {
        const unsigned long long v = t[(size_t)c * 1024 + i];
        dst[(size_t)c * 1024 + i] = i == 1023 ? (float)v : (v ? (float)((double)(v - t0) * 1e-3) : -1.0f);
      }
    *rows = n_sm_;
    *cols = 1024;
    return SSB_OK;
  }
  if (nm == "mega_prof") {  // phase timestamps of CTA 0 of the LAST persistent decode step, in microseconds from its start
    if (!mega_prof_) RET(SSB_ESTATE, "engine was not created with params.mega_prof=1");
    if (n < 1024) RET(SSB_EINVAL, "destination too small");
    std::vector<unsigned long long> t(1024);
    CK(cudaMemcpy(t.data(), mega_prof_, 1024 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    int cnt = 0;
    while (cnt < 1024 && t[cnt] != 0) ++cnt;
    for (int i = 0; i < cnt; ++i) dst[i] = (float)((double)(t[i] - t[0]) * 1e-3);
    *rows = 1;
    *cols = cnt;
    return SSB_OK;
  }
  if (!taps_) RET(SSB_ESTATE, "engine was not created with params.debug_taps=1");
  CK(cudaSetDevice(device_));
  const bf16* src = nullptr;
  int c = 0;
  if (nm == "q0") {
    src = tap_q0_;
    c = Hl_ * cfg_.head_dim;
  } else if (nm == "attn0") {
    src = tap_attn0_;
    c = Hl_ * cfg_.head_dim;
  } else if (nm == "h0") {
    src = tap_h0_;
    c = cfg_.hidden;
  } else if (nm == "h") {
    src = h_;
    c = cfg_.hidden;
  } else {
    RET(SSB_EINVAL, "unknown tap '" + nm + "'");
  }
  const int64_t need = (int64_t)tap_rows_ * c;
  *rows = tap_rows_;
  *cols = c;
  if (n < need) RET(SSB_EINVAL, "destination too small");
  float* tmp = nullptr;
  CK(cudaMalloc(&tmp, (size_t)need * sizeof(float)));
  cudaError_t e = launch_bf16_to_f32(src, tmp, need, stream_);
  if (e == cudaSuccess) e = cudaMemcpyAsync(dst, tmp, (size_t)need * sizeof(float), cudaMemcpyDeviceToHost, stream_);
  if (e == cudaSuccess) e = cudaStreamSynchronize(stream_);
  cudaFree(tmp);
  if (e != cudaSuccess) RET(SSB_ECUDA, cudaGetErrorString(e));
  return SSB_OK;
}

}  // namespace ssb

// ===================================================================================================================
// C ABI (include/ssb.h)
// ===================================================================================================================
using ssb::Engine;
struct ssb_engine {
  Engine impl;
};

extern "C" {

int ssb_engine_create(const char* model_dir, const char* params_json, ssb_engine** out) {
  if (!model_dir || !out) {
    ssb::set_error("null argument");
    return SSB_EINVAL;
  }
  *out = nullptr;
  ssb_engine* e = new (std::nothrow) ssb_engine();
  if (!e) return SSB_ENOMEM;
  int rc;
  try {
    rc = e->impl.init(model_dir, params_json ? params_json : "{}");
  } catch (std::exception& ex) {
    ssb::set_error(std::string("exception: ") + ex.what());
    rc = SSB_EINVAL;
  }
  if (rc != SSB_OK) {
    std::string keep = ssb::get_error();
    delete e;
    ssb::set_error(keep);
    return rc;
  }
  *out = e;
  return SSB_OK;
}

void ssb_engine_destroy(ssb_engine* e) { delete e; }

#define GUARD(e)                        \
  if (!(e)) {                           \
    ssb::set_error("null engine");      \
    return SSB_EINVAL;                  \
  }

int ssb_engine_info(ssb_engine* e, ssb_info* out) {
  GUARD(e);
  return out ? e->impl.info(out) : SSB_EINVAL;
}
int ssb_seq_create(ssb_engine* e, int* seq_id) {
  GUARD(e);
  return seq_id ? e->impl.seq_create(seq_id) : SSB_EINVAL;
}
int ssb_seq_free(ssb_engine* e, int seq_id) {
  GUARD(e);
  return e->impl.seq_free(seq_id);
}
int ssb_seq_len(ssb_engine* e, int seq_id, int* len) {
  GUARD(e);
  return len ? e->impl.seq_len(seq_id, len) : SSB_EINVAL;
}
int ssb_kv_blocks(ssb_engine* e, int* total, int* free_now) {
  GUARD(e);
  if (!total || !free_now) return SSB_EINVAL;
  e->impl.kv_blocks(total, free_now);
  return SSB_OK;
}
int ssb_prefill(ssb_engine* e, const int* seq_ids, const int32_t* tokens, const int* lens, int nseq, int32_t* next_tok,
                float* logits_opt) {
  GUARD(e);
  if (!seq_ids || !tokens || !lens || !next_tok) {
    ssb::set_error("null argument");
    return SSB_EINVAL;
  }
  try {
    return e->impl.prefill(seq_ids, tokens, lens, nseq, next_tok, logits_opt);
  } catch (std::exception& ex) {
    ssb::set_error(std::string("exception: ") + ex.what());
    return SSB_ENOMEM;
  }
}
int ssb_decode(ssb_engine* e, const int* seq_ids, const int32_t* last_tok, int nseq, int nsteps, int32_t* out_tok,
               float* logits_opt) {
  GUARD(e);
  if (!seq_ids || !last_tok || !out_tok) {
    ssb::set_error("null argument");
    return SSB_EINVAL;
  }
  try {
    return e->impl.decode(seq_ids, last_tok, nseq, nsteps, out_tok, logits_opt);
  } catch (std::exception& ex) {
    ssb::set_error(std::string("exception: ") + ex.what());
    return SSB_ENOMEM;
  }
}
int ssb_last_timing(ssb_engine* e, ssb_timing* out) {
  GUARD(e);
  return out ? e->impl.last_timing(out) : SSB_EINVAL;
}
int ssb_timing_reset(ssb_engine* e) {
  GUARD(e);
  e->impl.timing_reset();
  return SSB_OK;
}
int ssb_tp_handle_size(void) { return 256; }
int ssb_tp_export(ssb_engine* e, void* handle_out) {
  GUARD(e);
  return handle_out ? e->impl.tp_export(handle_out) : SSB_EINVAL;
}
int ssb_tp_connect(ssb_engine* e, const void* all_handles, int n_ranks) {
  GUARD(e);
  return all_handles ? e->impl.tp_connect(all_handles, n_ranks) : SSB_EINVAL;
}
const char* ssb_debug_profile(ssb_engine* e) {
  static thread_local std::string rep;
  if (!e) return "{}";
  rep = e->impl.prof_report();
  return rep.c_str();
}
int ssb_bench_kernel(ssb_engine* e, const char* which, int rows, int ctx, int iters, double* ms_per_launch,
                     int64_t* algorithmic_bytes) {
  GUARD(e);
  if (!ms_per_launch || !algorithmic_bytes) return SSB_EINVAL;
  return e->impl.bench_kernel(which, rows, ctx, iters, ms_per_launch, algorithmic_bytes);
}
int ssb_debug_read(ssb_engine* e, const char* name, float* dst, int64_t dst_elems, int* rows, int* cols) {
  GUARD(e);
  if (!dst || !rows || !cols) return SSB_EINVAL;
  return e->impl.debug_read(name, dst, dst_elems, rows, cols);
}
int ssb_debug_dequant(int ggml_type, const void* blocks, int64_t nbytes, int64_t n_elems, uint16_t* dst_bf16) {
  if (!blocks || !dst_bf16 || n_elems <= 0) return SSB_EINVAL;
  int dt;
  switch (ggml_type) {
    case 0: dt = ssb::DT_F32; break;
    case 1: dt = ssb::DT_F16; break;
    case 2: dt = ssb::DT_Q4_0; break;
    case 8: dt = ssb::DT_Q8_0; break;
    case 12: dt = ssb::DT_Q4_K; break;
    case 14: dt = ssb::DT_Q6_K; break;
    case 30: dt = ssb::DT_BF16; break;
    default: ssb::set_error("unsupported ggml type"); return SSB_EINVAL;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    ssb::set_error("no CUDA device: libsubstratus_b200 has no CPU fallback");
    return SSB_ENODEV;
  }
  void* d_src = nullptr;
  bf16* d_dst = nullptr;
  cudaError_t e = cudaMalloc(&d_src, (size_t)nbytes);
  if (e == cudaSuccess) e = cudaMalloc(&d_dst, (size_t)n_elems * 2);
  if (e == cudaSuccess) e = cudaMemcpy(d_src, blocks, (size_t)nbytes, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = launch_dequant(d_src, dt, n_elems, d_dst, 0);
  if (e == cudaSuccess) e = cudaMemcpy(dst_bf16, d_dst, (size_t)n_elems * 2, cudaMemcpyDeviceToHost);
  cudaFree(d_src);
  cudaFree(d_dst);
  if (e != cudaSuccess) {
    ssb::set_error(cudaGetErrorString(e));
    return SSB_ECUDA;
  }
  return SSB_OK;
}
int ssb_synth_fill_host(uint64_t seed, uint32_t tid, int64_t start, int64_t n, float amp, float base, uint16_t* dst) {
  if (!dst || n < 0) return SSB_EINVAL;
  synth_fill_host(seed, tid, start, n, amp, base, dst);
  return SSB_OK;
}
struct ssb_tokenizer {
  ssb::Tokenizer impl;
};
int ssb_tok_load(const char* path, ssb_tokenizer** out) {
  if (!path || !out) return SSB_EINVAL;
  *out = nullptr;
  ssb_tokenizer* t = new (std::nothrow) ssb_tokenizer();
  if (!t) return SSB_ENOMEM;
  std::string err;
  bool ok = false;
  try {
    ok = t->impl.load(path, &err);
  } catch (std::exception& ex) {
    err = ex.what();
  }
  if (!ok) {
    delete t;
    ssb::set_error(err);
    return err.rfind("cannot read", 0) == 0 ? SSB_EIO : SSB_EINVAL;
  }
  *out = t;
  return SSB_OK;
}
void ssb_tok_free(ssb_tokenizer* t) { delete t; }
int ssb_tok_encode(ssb_tokenizer* t, const char* text, int add_special, int32_t* ids, int cap, int* n_out) {
  if (!t || !text || !n_out || (cap > 0 && !ids)) return SSB_EINVAL;
  const std::vector<int32_t> v = t->impl.encode(text, add_special != 0);
  *n_out = (int)v.size();
  if ((int)v.size() > cap) {
    ssb::set_error("id buffer too small");
    return SSB_ENOMEM;
  }
  if (!v.empty()) memcpy(ids, v.data(), v.size() * sizeof(int32_t));
  return SSB_OK;
}
int ssb_tok_decode(ssb_tokenizer* t, const int32_t* ids, int n, int skip_special, char* buf, int cap, int* len_out) {
  if (!t || (n > 0 && !ids) || !len_out || (cap > 0 && !buf)) return SSB_EINVAL;
  const std::string s = t->impl.decode(std::vector<int32_t>(ids, ids + n), skip_special != 0);
  *len_out = (int)s.size();
  if ((int)s.size() > cap) {
    ssb::set_error("text buffer too small");
    return SSB_ENOMEM;
  }
  if (!s.empty()) memcpy(buf, s.data(), s.size());
  return SSB_OK;
}
const char* ssb_last_error(void) { return ssb::get_error(); }
#ifdef SSB_VARIANT
const char* ssb_version(void) { return "substratus_b200 0.1 (sm_90a) variant=" SSB_VARIANT; }
#else
const char* ssb_version(void) { return "substratus_b200 0.1 (sm_90a)"; }
#endif

}  // extern "C"
