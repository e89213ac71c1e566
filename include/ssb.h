/* ssb.h — C ABI of libsubstratus_b200.so, the H100-native engine behind the
 * Substratus `Server` CRD's serving container.
 *
 * What this replaces.  The reference (substratusai/substratus @ 7352fb0) defines
 * NO in-process interface for inference: its ServerReconciler only emits a Pod
 * (internal/controller/server_controller.go:114-205: container "serve", port
 * 8080 "http-serve", readiness GET /, model mounted RO at /content/model,
 * /content/params.json from .spec.params via internal/controller/
 * params_reconciler.go:28-104) and the container contract
 * (docs/container-contract.md:50-55) is "listen on :8080, 200 on /".  The
 * model-load + generate path runs inside external images
 * (examples/llama2-7b/server.yaml:6 `substratusai/model-server-basaran`).  This
 * header is the seam north_star asks for between a thin (Go/cgo or C++) serve
 * host and the CUDA engine: each entry point cites the step of that external
 * path it stands in for.  Pure C: opaque handle, caller-owned host buffers,
 * int return codes (0 = ok, <0 = error; text via ssb_last_error()), no
 * callbacks, no torch types.  Calls on one engine are not re-entrant; the host
 * serialises them (also satisfies cgo's pointer rules: only ints/bytes cross).
 *
 * There is NO CPU fallback: every compute entry point fails with SSB_ENODEV if
 * no sm_90 device is present.
 */
#ifndef SSB_H
#define SSB_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SSB_OK 0
#define SSB_EINVAL (-1)  /* bad argument / bad config / bad params.json          */
#define SSB_EIO (-2)     /* model directory / safetensors / .bin / gguf could not be read */
#define SSB_ENODEV (-3)  /* no CUDA device of compute capability 10.x            */
#define SSB_ENOMEM (-4)  /* HBM or KV-block pool exhausted                       */
#define SSB_ECUDA (-5)   /* CUDA runtime error (message in ssb_last_error)       */
#define SSB_ESTATE (-6)  /* call not valid in this state (e.g. TP not connected) */

typedef struct ssb_engine ssb_engine;

typedef struct ssb_info {
  int32_t vocab_size, hidden_size, n_layers, n_heads, n_kv_heads, head_dim;
  int32_t intermediate_size, max_seq_len, max_batch, kv_block_size;
  int32_t tp_size, tp_rank, n_sm, device;
  int64_t weight_bytes_per_step;  /* algorithmic Linear-weight bytes one decode step streams on THIS rank (SURVEY §8d: 2*P_dec/TP) */
  int64_t kv_bytes_per_token;     /* K+V bytes per cached token on THIS rank, all layers                                      */
  int64_t hbm_bytes_allocated;
  char model_type[32];            /* "llama" | "falcon" | "opt"                                                                */
  char dtype[8];                  /* arithmetic type: "bf16"                                                                   */
} ssb_info;

typedef struct ssb_timing {
  double prefill_ms;      /* device time of the last ssb_prefill, CUDA events on the engine stream (excludes host copies) */
  double decode_ms;       /* device time of the last ssb_decode (all nsteps), same clock                                    */
  int64_t kernel_launches;/* engine kernels launched (graph nodes count as launches) since the last ssb_timing_reset        */
  int64_t h2d_bytes, d2h_bytes; /* bytes copied across PCIe since the last reset                                            */
} ssb_timing;

/* Model load: stands in for the external image's `from_pretrained(/content/model)`
 * at pod start (SURVEY §3.2; docs/container-contract.md:25-36).  model_dir is an
 * HF snapshot dir (config.json + *.safetensors, else pytorch_model*.bin [+ index]) or holds a single GGUF
 * file; params_json is the text of /content/params.json (internal/controller/
 * params_reconciler.go:36-53), may be NULL or "{}".  Recognised params:
 *   "max_batch" (32), "max_seq_len" (config's), "kv_block_size" (16), "kv_blocks" (auto),
 *   "weights": "file" | "synthetic" (seeded hash weights at config.json's shapes; "seed"),
 *   "tp_size", "tp_rank" (1, 0), "device" (tp_rank),
 *   "tp_presharded" (1: with tp_size N > 1, if <model_dir>/ssb_tp<N>/rank<tp_rank>.safetensors exists — written by
 *   tools/tp_shard.py: this rank's slices of the projections + the replicated tensors — the rank loads that file alone),
 *   "use_pdl" (1), "use_graph" (1), "use_mega" (1: persistent single-kernel decode step for batches up to
 *   "mega_max_batch"; Llama layouts only), "mega_max_batch" (1; at most 4, larger values act as 4): larger batches
 *   take the graph + PDL multi-kernel step, and so do batches of "tc_min_rows" or more rows and batches whose step does
 *   not fit the persistent kernel's shared memory (e.g. 4 rows at Llama-2-70B widths); ssb_timing.kernel_launches tells
 *   the paths apart: the persistent kernel is one launch per decode step,
 *   "gemm_path": "auto" | "gemv" | "tc", "tc_min_rows" (5), "tc_streamk" (1), "prefill_chunk" (1024),
 *   "tc_tn_prefill" (0 = per-projection heuristic | 128 | 256: token-tile width of the prefill GEMMs),
 *   "attn_splits" (0 = heuristic; context splits of the decode attention kernels, a sweep knob),
 *   "mega_attn_tile" (1: CTA-tile attention for GQA groups of 8 inside the persistent kernel),
 *   tensor-parallel decode exchange, "tp_mega": 3 (default: the persistent kernel pushes 16-byte {value, epoch} words into
 *   every rank's receive slots over NVLink peer memory and polls its own) | 1, 2 (flag + pull inside the persistent kernel,
 *   grid-wide / per CTA) | 0 (multi-kernel step with the one-shot pull allreduce kernel); prefill-sized forwards always
 *   use the allreduce kernels: "tp_two_shot": 1 (default) reduce-scatter + bf16 gather from "tp_two_shot_min_rows" (64)
 *   rows up, one-shot pull below (and with "tp_two_shot": 0); "tp_push" (push-model allreduce kernel, measured slower).  All cross-GPU waits are bounded (20 s, then the
 *   kernel traps and the call returns SSB_ECUDA).  There is no NCCL call on the data path; the NCCL baseline the engine's
 *   exchange is measured against is tools/nccl_ar_bench.py.
 *   diagnostics (read back with ssb_debug_read): "mega_prof" 1 | 2 (phase stamps of the persistent kernel: CTA 0 | every CTA),
 *   "sk_prof" 1 (phase stamps of the stream-K projections; needs the library variant built with -DTC_SK_PROF=1).
 * Keys the engine does not know are ignored (the serve host keeps its own keys in the same file: "batching",
 * "batch_tick", "stream_chunk", "stop_at_eos", "eos_token_id", "eos_check_every").
 * With tp_size > 1 the engine is usable only after ssb_tp_connect(). */
int ssb_engine_create(const char* model_dir, const char* params_json, ssb_engine** out);
void ssb_engine_destroy(ssb_engine* e);
int ssb_engine_info(ssb_engine* e, ssb_info* out);

/* Sequence slots (one per in-flight request; a slot owns a paged-KV block list). */
int ssb_seq_create(ssb_engine* e, int* seq_id);
int ssb_seq_free(ssb_engine* e, int seq_id);

/* Prompt processing: stands in for the first `forward(T=prompt_len)` of HF greedy
 * generation (HF generation/utils.py:2658-2800 as wrapped by Basaran).  tokens is
 * the concatenation of the nseq prompts (lens[i] ids each, host memory).  Appends to
 * each sequence's KV cache, returns the greedy next token per sequence and, if
 * logits_opt != NULL, the fp32 last-position logits [nseq, vocab]. */
int ssb_prefill(ssb_engine* e, const int* seq_ids, const int32_t* tokens, const int* lens, int nseq,
                int32_t* next_tok, float* logits_opt);

/* Decode loop: nsteps greedy steps for nseq sequences, fed on-device (one H2D of
 * last_tok, one D2H of out_tok [nseq, nsteps] row-major).  logits_opt, if not NULL,
 * receives the fp32 logits of every step [nsteps, nseq, vocab]. */
int ssb_decode(ssb_engine* e, const int* seq_ids, const int32_t* last_tok, int nseq, int nsteps,
               int32_t* out_tok, float* logits_opt);

/* Current cached length of a sequence (tokens in its KV cache). */
int ssb_seq_len(ssb_engine* e, int seq_id, int* len);

/* KV block pool of this engine: *total blocks of ssb_info.kv_block_size tokens, *free_now of them unassigned.  A sequence
 * of n cached tokens holds ceil(n / kv_block_size) blocks until ssb_seq_free; ssb_prefill / ssb_decode return SSB_ENOMEM
 * (state untouched) when the pool cannot cover the tokens they would add.  The host scheduler admits a request only when
 * prompt + max_new_tokens blocks are available (host/scheduler.h) — the reference has no such limit to mirror: its
 * container serves one request at a time (internal/controller/server_controller.go:115). */
int ssb_kv_blocks(ssb_engine* e, int* total, int* free_now);

int ssb_last_timing(ssb_engine* e, ssb_timing* out);
int ssb_timing_reset(ssb_engine* e);

/* Tensor-parallel bootstrap for the one-process-per-GPU launch (torchrun / one
 * container per GPU).  Each rank exports an opaque handle (CUDA IPC handles of its
 * exchange buffers + an NCCL unique id slot), the host all-gathers them by any
 * means (torch.distributed, a file, the Pod's localhost) and hands every rank the
 * concatenation, rank-major.  ssb_tp_handle_size() bytes per rank. */
int ssb_tp_handle_size(void);
int ssb_tp_export(ssb_engine* e, void* handle_out);
int ssb_tp_connect(ssb_engine* e, const void* all_handles, int n_ranks);

/* Measurement hook (bench.py's `roofline` object): times `iters` back-to-back launches of ONE kernel class of the
 * decode step ("qkv" | "o" | "gate_up" | "down" | "lm_head" | "attn"), cycling over the layers' weights so nothing is
 * served from L2, between CUDA events on the engine's own stream.  rows = batch rows, ctx = cached length (attn).
 * Returns the average device ms per launch and the ALGORITHMIC bytes one launch must move (2*N*K for a projection,
 * 2*rows*ctx*KVH*D*2 for attention). */
int ssb_bench_kernel(ssb_engine* e, const char* which, int rows, int ctx, int iters, double* ms_per_launch,
                     int64_t* algorithmic_bytes);

/* Per-kernel-class device time (ms, JSON object) accumulated over the forwards since the last call, for engines
 * created with params.profile_forward=1 (CUDA events between plain stream-ordered launches; no graph, no PDL). */
const char* ssb_debug_profile(ssb_engine* e);

/* Debug/parity taps (tests only): copy an internal activation of the LAST forward
 * to host as fp32.  name: "h" (residual stream after the last layer), "q0", "attn0",
 * "h0" (layer-0 taps).  rows/cols returned through the out params. */
int ssb_debug_read(ssb_engine* e, const char* name, float* dst, int64_t dst_elems, int* rows, int* cols);

/* GGUF block dequantisation kernel exposed for the bit-exact check against llama.cpp's gguf-py (tests only):
 * ggml_type = GGML type id (0 F32, 1 F16, 2 Q4_0, 8 Q8_0, 12 Q4_K, 14 Q6_K, 30 BF16); blocks = raw bytes (host);
 * dst = n_elems bf16 bit patterns (host).  Runs the load-time CUDA kernel. */
int ssb_debug_dequant(int ggml_type, const void* blocks, int64_t nbytes, int64_t n_elems, uint16_t* dst_bf16);

/* Model-artifact inspection without a device: opens model_dir with the engine's own container readers (safetensors,
 * pytorch_model*.bin torch.save zips, GGUF — SURVEY §8f #2) and returns one tensor's raw stored bytes.  dtype: 0 bf16,
 * 1 f16, 2 f32, 10 Q4_0, 11 Q4_K, 12 Q6_K, 13 Q8_0, 99 other; shape (outermost first) into shape[0..*ndim), at most 4
 * dims.  name == NULL: *nbytes_out = number of tensors in the artifact.  dst may be NULL (cap 0) to query sizes.
 * SSB_EIO if the artifact or tensor is missing, SSB_ENOMEM if cap is too small.  Used by tests/ and by operators
 * checking an artifact before scheduling a GPU pod; never on the request path. */
int ssb_model_read_tensor(const char* model_dir, const char* name, void* dst, int64_t cap, int64_t* nbytes_out, int* dtype,
                          int64_t* shape, int* ndim);

/* Deterministic synthetic-weight generator exposed for the oracle cross-check
 * (tests/: bit-exact against oracle/synth.py).  Fills dst (host, uint16 bf16 bits). */
int ssb_synth_fill_host(uint64_t seed, uint32_t tid, int64_t start, int64_t n, float amp, float base, uint16_t* dst);

/* Text path (SURVEY §8f #1; the reference's one request carries text: test/system.sh:73-78).  Native reader of HF
 * `tokenizer.json` (Llama-2 SentencePiece-style BPE with byte fallback, GPT-2/OPT byte-level BPE); CPU only, no GPU
 * needed.  Unsupported tokenizer components fail at load (SSB_EINVAL) instead of tokenising approximately.
 * encode: returns the id count through n_out (even when > cap, so the caller can retry); decode: bytes through len_out. */
typedef struct ssb_tokenizer ssb_tokenizer;
int ssb_tok_load(const char* tokenizer_json_path, ssb_tokenizer** out);
void ssb_tok_free(ssb_tokenizer* t);
int ssb_tok_encode(ssb_tokenizer* t, const char* text_utf8, int add_special, int32_t* ids, int cap, int* n_out);
int ssb_tok_decode(ssb_tokenizer* t, const int32_t* ids, int n, int skip_special, char* buf, int cap, int* len_out);

const char* ssb_last_error(void);
const char* ssb_version(void);

#ifdef __cplusplus
}
#endif
#endif /* SSB_H */
