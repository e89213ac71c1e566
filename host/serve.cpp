// serve.cpp — the serve host of the H100 container: the process the reference's ServerReconciler launches as
// container "serve" (internal/controller/server_controller.go:149-173).  Contract it honours
// (docs/container-contract.md:5-11,25-55):
//   * WORKDIR /content; model mounted read-only at /content/model; params at /content/params.json
//   * listen on TCP 8080 (port name http-serve); GET / -> 200 only when ready to serve (kubelet readiness probe)
//   * exit != 0 on fatal errors so the Deployment restarts the pod (server_controller.go:280-296)
// Inference API: the reference specifies none; the only request it ever sends is
// POST /v1/completions {"prompt", "max_tokens"} (test/system.sh:73-78).  We serve that (prompt = array of token ids;
// text prompts need the tokenizer of SURVEY §8f #1) and POST /generate (north_star).  All compute goes through the
// C ABI of include/ssb.h; this file contains no arithmetic and there is no CPU fallback.
//
// Stand-in for the Go host north_star names (`containertools/cmd/serve`): no Go toolchain exists in this image, so
// the host is C++ over the same C ABI; the cgo twin is in INTEGRATION.md.
#include <arpa/inet.h>
#include <netinet/in.h>
#include <netinet/tcp.h>
#include <signal.h>
#include <sys/socket.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../include/ssb.h"
#include "../substratus_b200/csrc/json.h"
#include "sampler.h"
#include "scheduler.h"

using ssb::Json;
using ssbhost::Sampling;

static std::atomic<int> g_ready{0};  // 0 loading, 1 ready, -1 failed
// SIGTERM (pod deletion / rollout): stop accepting, answer the readiness probe with 503 so the Service drops the pod,
// let the requests in flight finish, exit 0 — inside the default 30 s terminationGracePeriodSeconds of the Deployment
// the reconciler creates (server_controller.go:122-178 sets none, so the Kubernetes default applies).
static std::atomic<bool> g_draining{false};
static std::atomic<int> g_inflight{0};
static int g_listen_fd = -1;
static void on_sigterm(int) {
  g_draining = true;
  if (g_listen_fd >= 0) shutdown(g_listen_fd, SHUT_RD);  // wakes accept(); async-signal-safe
}
static ssb_engine* g_engine = nullptr;
static ssb_info g_info;
static std::mutex g_engine_mu;  // ssb_* calls on one engine are not re-entrant
static std::atomic<long long> g_requests{0}, g_tokens{0}, g_errors{0};
static std::atomic<long long> g_ttft_us_sum{0}, g_decode_us_sum{0};  // integer microseconds: fetch_add is atomic
static std::atomic<int> g_conns{0};
static const int kMaxConns = 256;  // concurrent connections (each holds a thread); above it: 503
// A device-side failure is not recoverable inside the process (CUDA errors are sticky; under tensor parallelism the other
// ranks would wait for a peer that is gone): fail readiness and exit non-zero so the Deployment restarts the pod
// (the container contract's error path: server_controller.go:280-296).
[[noreturn]] static void fatal_exit(const std::string& why) {
  g_ready = -1;
  fprintf(stderr, "serve: fatal engine error, exiting for a pod restart: %s\n", why.c_str());
  fflush(stderr);
  _exit(1);
}
static std::string g_load_error;
static ssb_tokenizer* g_tok = nullptr;  // <model_dir>/tokenizer.json, if present and supported (text prompts)
// Tensor parallel inside the ONE container the reconciler grants N GPUs to (resources.gpu.count -> nvidia.com/gpu: N,
// internal/resources/resources.go:39-47): rank 0 is g_engine, ranks 1..N-1 live here; every rank runs in its own
// host thread per request (the ranks' kernels wait for each other over NVLink, so the calls must be concurrent).
static std::vector<ssb_engine*> g_peers;

// opt-in continuous batching (params.json {"batching": 1, "batch_tick": 8}); policy and its CPU test: scheduler.h
struct AbiEngine {
  ssb_engine* e;
  std::string err;
  int seq_create(int* sid) { return note(ssb_seq_create(e, sid)); }
  int seq_free(int sid) { return ssb_seq_free(e, sid); }
  int prefill(const int* sids, const int32_t* toks, const int* lens, int nseq, int32_t* next) {
    return note(ssb_prefill(e, sids, toks, lens, nseq, next, nullptr));
  }
  int decode(const int* sids, const int32_t* last, int nseq, int nsteps, int32_t* out) {
    return note(ssb_decode(e, sids, last, nseq, nsteps, out, nullptr));
  }
  int note(int rc) {
    if (rc != SSB_OK) err = ssb_last_error();
    return rc;
  }
  std::string last_error() { return err; }
};
static AbiEngine g_abi;
static ssbhost::BatchScheduler<AbiEngine>* g_sched = nullptr;

static std::string getenv_or(const char* k, const char* d) {
  const char* v = getenv(k);
  return v && *v ? v : d;
}

static bool read_file(const std::string& p, std::string* out) {
  FILE* f = fopen(p.c_str(), "rb");
  if (!f) return false;
  char buf[65536];
  size_t n;
  out->clear();
  while ((n = fread(buf, 1, sizeof buf, f)) > 0) out->append(buf, n);
  fclose(f);
  return true;
}

// The container contract documents params both as /content/params.json and as PARAM_{UPPER(key)} environment variables
// (docs/container-contract.md:36-48); the reconciler at this commit only mounts the file
// (internal/controller/params_reconciler.go:78-104).  Tolerate both: env entries fill in keys the file does not set.
extern char** environ;
static std::string merge_param_env(const std::string& params) {
  std::vector<std::pair<std::string, std::string>> extra;
  Json have;
  try {
    have = ssb::json_parse(params.empty() ? "{}" : params);
  } catch (std::exception&) {
    return params;  // the engine reports the JSON error
  }
  if (have.kind != Json::Obj) return params;
  for (char** e = environ; e && *e; ++e) {
    if (strncmp(*e, "PARAM_", 6) != 0) continue;
    const char* eq = strchr(*e, '=');
    if (!eq || eq == *e + 6) continue;
    std::string key((const char*)*e + 6, eq);
    for (auto& c : key) c = (char)tolower((unsigned char)c);
    if (have.find(key)) continue;
    extra.emplace_back(key, eq + 1);
  }
  if (extra.empty()) return params;
  std::string out = "{";
  for (auto& kv : extra) {
    std::string v = kv.second;
    bool raw = false;  // numbers / true / false / null pass through, everything else becomes a JSON string
    try {
      const Json j = ssb::json_parse(v);
      raw = j.kind == Json::Num || j.kind == Json::Bool || j.kind == Json::Null;
    } catch (std::exception&) {
    }
    out += "\"" + ssb::json_escape(kv.first) + "\":" + (raw ? v : "\"" + ssb::json_escape(v) + "\"") + ",";
  }
  const size_t brace = params.find('{');
  const std::string rest = brace == std::string::npos ? "}" : params.substr(brace + 1);
  if (rest.find_first_not_of(" \t\r\n") == rest.find('}')) out.pop_back();  // file object is empty: drop the trailing comma
  return out + rest;
}

static bool send_all(int fd, const std::string& s) {
  size_t off = 0;
  while (off < s.size()) {
    ssize_t n = send(fd, s.data() + off, s.size() - off, MSG_NOSIGNAL);
    if (n <= 0) return false;  // peer went away (or SO_SNDTIMEO expired)
    off += (size_t)n;
  }
  return true;
}

static void respond(int fd, int code, const char* status, const std::string& body, const char* ctype = "application/json") {
  char hdr[256];
  snprintf(hdr, sizeof hdr, "HTTP/1.1 %d %s\r\nContent-Type: %s\r\nContent-Length: %zu\r\nConnection: close\r\n\r\n", code, status,
           ctype, body.size());
  send_all(fd, std::string(hdr) + body);
}

static std::string err_json(const std::string& m) { return "{\"error\":\"" + ssb::json_escape(m) + "\"}"; }

struct GenResult {
  std::vector<int32_t> tokens;
  double ttft_ms = 0, decode_ms = 0;
  bool hit_eos = false;  // stopped at an end-of-sequence id (which is NOT included in tokens)
  std::string error;
  bool fatal = false;  // the engine is unusable (SSB_ECUDA, or tensor-parallel ranks failed / disagreed)
};

// Called with the ids produced since the previous call (first call: the prefill's token).  Returning false stops the
// generation early (client went away); only honoured where one engine serves the request (the ranks of a TP group must
// stay in lock-step, so there the request runs on regardless of the client).
using TokenSink = std::function<bool(const int32_t*, int)>;

// index of the first end-of-sequence id in ids[0..n), or n
static int find_eos(const std::vector<int32_t>& eos, const int32_t* ids, int n) {
  for (int i = 0; i < n; ++i)
    for (int32_t e : eos)
      if (ids[i] == e) return i;
  return n;
}

// one rank's share of a request: identical inputs on every rank, identical greedy ids out.  `chunk` = decode steps per
// ssb_decode call: max_new-1 for a plain request (ONE call, as the bench measures it), params.json "stream_chunk" (1)
// for "stream": true, "eos_check_every" (16) when the request stops at EOS.  `eos` (may be empty) is checked after every
// call on EVERY rank — the ids are identical across ranks, so all ranks stop at the same call.
// With samp.on() the engine is driven one step per call and the token is drawn on the host from the step's logits
// (sampler.h); every rank of a TP group draws from bit-identical logits with the same seed.
static const Sampling kGreedy;
static int run_rank(ssb_engine* e, const std::vector<int32_t>& prompt, int max_new, int chunk, const std::vector<int32_t>& eos,
                    const TokenSink& sink, bool may_stop, std::vector<int32_t>* toks, bool* hit_eos, double* ttft_ms, double* decode_ms,
                    std::string* error, const Sampling& samp = kGreedy) {
  int sid = -1;
  int rc = ssb_seq_create(e, &sid);
  if (rc != SSB_OK) {
    *error = ssb_last_error();
    return rc;
  }
  auto t0 = std::chrono::steady_clock::now();
  int n = (int)prompt.size();
  int32_t first = 0;
  toks->assign(max_new, 0);
  *hit_eos = false;
  std::vector<float> logits(samp.on() ? (size_t)g_info.vocab_size : 0);
  std::vector<std::pair<float, int>> cand;
  ssbhost::Rng rng{samp.seed};
  rc = ssb_prefill(e, &sid, prompt.data(), &n, 1, &first, samp.on() ? logits.data() : nullptr);
  auto t1 = std::chrono::steady_clock::now();
  int done = 0;
  if (rc == SSB_OK) {
    if (samp.on()) first = ssbhost::sample_token(logits.data(), g_info.vocab_size, samp, rng, cand);
    (*toks)[0] = first;
    // deliver the ids of one engine call: cut at the first EOS, feed the sink, decide whether to go on
    auto deliver = [&](int from, int count) {
      const int keep = find_eos(eos, toks->data() + from, count);
      done = from + keep;
      *hit_eos = keep < count;
      const bool client_ok = !sink || keep == 0 || sink(toks->data() + from, keep);
      return !*hit_eos && (client_ok || !may_stop);
    };
    bool go = deliver(0, 1);
    while (rc == SSB_OK && go && done < max_new) {
      const int steps = samp.on() ? 1 : std::min(std::max(1, chunk), max_new - done);
      const int32_t last = (*toks)[done - 1];
      rc = ssb_decode(e, &sid, &last, 1, steps, toks->data() + done, samp.on() ? logits.data() : nullptr);
      if (rc != SSB_OK) break;
      if (samp.on()) (*toks)[done] = ssbhost::sample_token(logits.data(), g_info.vocab_size, samp, rng, cand);
      go = deliver(done, steps);
    }
  }
  auto t2 = std::chrono::steady_clock::now();
  if (rc != SSB_OK) *error = ssb_last_error();  // thread-local in the library: read it on the calling thread
  toks->resize(done);
  ssb_seq_free(e, sid);
  *ttft_ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
  *decode_ms = std::chrono::duration<double, std::milli>(t2 - t1).count();
  return rc;
}

static GenResult generate_tp(const std::vector<int32_t>& prompt, int max_new, int chunk, const std::vector<int32_t>& eos,
                             const TokenSink& sink, const Sampling& samp) {
  GenResult r;
  std::lock_guard<std::mutex> lk(g_engine_mu);
  const size_t n = g_peers.size() + 1;
  std::vector<std::vector<int32_t>> toks(n);
  std::vector<double> ttft(n, 0), dec(n, 0);
  std::vector<std::string> errs(n);
  std::vector<char> hit(n, 0);
  std::vector<std::thread> th;
  for (size_t i = 1; i < n; ++i)
    th.emplace_back([&, i] {
      bool h = false;
      const int rc = run_rank(g_peers[i - 1], prompt, max_new, chunk, eos, nullptr, false, &toks[i], &h, &ttft[i], &dec[i], &errs[i], samp);
      // the other ranks may be spinning on this rank's flags (bounded, SpinGuard): do not wait for them
      if (rc == SSB_ECUDA) fatal_exit("rank " + std::to_string(i) + ": " + errs[i]);
      hit[i] = h;
    });
  const int rc0 = run_rank(g_engine, prompt, max_new, chunk, eos, sink, false, &toks[0], &r.hit_eos, &ttft[0], &dec[0], &errs[0], samp);
  if (rc0 == SSB_ECUDA) fatal_exit("rank 0: " + errs[0]);
  for (auto& t : th) t.join();
  for (size_t i = 0; i < n; ++i) {
    if (!errs[i].empty()) r.error = "rank " + std::to_string(i) + ": " + errs[i];
    if (i && r.error.empty() && toks[i] != toks[0]) r.error = "tensor-parallel ranks disagree on the generated ids";
  }
  r.fatal = !r.error.empty();  // ranks out of lock-step (one failed, or ids differ): the group cannot serve the next request
  r.tokens = toks[0];
  r.ttft_ms = *std::max_element(ttft.begin(), ttft.end());
  r.decode_ms = *std::max_element(dec.begin(), dec.end());
  return r;
}

static const std::vector<int32_t> kNoEos;
static GenResult generate(const std::vector<int32_t>& prompt, int max_new, int chunk = 1 << 30, const TokenSink& sink = nullptr,
                          const std::vector<int32_t>& eos = kNoEos, const Sampling& samp = kGreedy) {
  if (!g_peers.empty()) return generate_tp(prompt, max_new, chunk, eos, sink, samp);
  GenResult r;
  if (g_sched && samp.on()) {
    r.error = "sampling (temperature > 0) is not available while continuous batching is on: the shared decode loop is greedy";
    return r;
  }
  if (g_sched) {  // concurrent clients share prefill / decode calls; the sink is fed once per scheduler tick
    ssbhost::Request rq;
    rq.prompt = prompt;
    rq.max_new = max_new;
    size_t kept = 0;  // ids accepted so far (everything before the first EOS)
    if (sink || !eos.empty())
      rq.on_tokens = [&](const int32_t* ids, int n) {
        const int keep = find_eos(eos, ids, n);
        kept += (size_t)keep;
        r.hit_eos = keep < n;
        const bool client_ok = !sink || keep == 0 || sink(ids, keep);
        return !r.hit_eos && client_ok;
      };
    g_sched->submit(&rq);
    r.tokens = rq.tokens;
    if (r.hit_eos) r.tokens.resize(kept);
    r.error = rq.error;
    r.fatal = rq.error_code == SSB_ECUDA;  // the device is gone for every later request too: the caller exits for a restart
    r.ttft_ms = rq.ttft_ms;
    r.decode_ms = rq.total_ms - rq.ttft_ms;
    return r;
  }
  std::lock_guard<std::mutex> lk(g_engine_mu);
  const int rc = run_rank(g_engine, prompt, max_new, chunk, eos, sink, true, &r.tokens, &r.hit_eos, &r.ttft_ms, &r.decode_ms, &r.error, samp);
  r.fatal = rc == SSB_ECUDA;
  return r;
}

static bool parse_ids(const Json* j, int vocab, std::vector<int32_t>* out, std::string* err) {
  if (!j || j->kind != Json::Arr || j->arr.empty()) {
    *err = "expected a non-empty array of token ids";
    return false;
  }
  for (auto& v : j->arr) {
    if (v.kind != Json::Num || v.num < 0 || v.num >= vocab || v.num != (double)(long long)v.num) {
      *err = "token ids must be integers in [0, vocab_size)";
      return false;
    }
    out->push_back((int32_t)v.num);
  }
  return true;
}

static std::string ids_json(const std::vector<int32_t>& v) {
  std::string s = "[";
  for (size_t i = 0; i < v.size(); ++i) s += (i ? "," : "") + std::to_string(v[i]);
  return s + "]";
}

// Longest prefix of s[from..] that ends on a UTF-8 character boundary and not in a U+FFFD the decoder substituted for
// a byte-fallback run that later ids may still complete.
static size_t utf8_safe_len(const std::string& s) {
  size_t n = s.size();
  size_t i = n;
  int back = 0;
  while (i > 0 && back < 4 && ((unsigned char)s[i - 1] & 0xC0) == 0x80) {
    --i;
    ++back;
  }
  if (i > 0) {
    const unsigned char lead = (unsigned char)s[i - 1];
    const int need = lead >= 0xF0 ? 4 : lead >= 0xE0 ? 3 : lead >= 0xC0 ? 2 : 1;
    if (need > 1 && back + 1 < need) n = i - 1;  // incomplete multi-byte tail: hold it back
  }
  while (n >= 3 && (unsigned char)s[n - 3] == 0xEF && (unsigned char)s[n - 2] == 0xBF && (unsigned char)s[n - 1] == 0xBD) n -= 3;
  return n;
}

// "stream": true — server-sent events, one per decode chunk (params.json "stream_chunk", default 1 token), in the
// OpenAI completions-stream shape the reference's browser UI consumes (internal/tui/serve.go:282-289 points users at
// Basaran's streaming playground); terminated by `data: [DONE]`.  Text is detokenised incrementally: every event carries
// the new suffix of decode(all ids so far), cut at a UTF-8 boundary, so the concatenation equals the non-streamed text.
static int g_stream_chunk = 1;
// End-of-sequence handling.  The synthetic benchmark request never stops early (SURVEY.md §8d: "no EOS stop"), so a
// request stops at EOS only when it says "stop_at_eos": true (or params.json sets "stop_at_eos": 1 as the default).
// Ids come from params.json "eos_token_id", else <model_dir>/generation_config.json, else config.json (int or list).
// The EOS id itself is not returned; finish_reason becomes "stop".  Without streaming the ids are checked every
// "eos_check_every" (16) decode steps, so at most that many steps are computed past the end.
static std::vector<int32_t> g_eos;
static bool g_stop_default = false;
static int g_eos_every = 16;
static void stream_response(int fd, bool oai, const std::vector<int32_t>& prompt, int max_new, bool text_mode,
                            const std::vector<int32_t>& eos, const Sampling& samp) {
  send_all(fd, "HTTP/1.1 200 OK\r\nContent-Type: text/event-stream\r\nCache-Control: no-cache\r\nConnection: close\r\n\r\n");
  std::vector<int32_t> all;
  size_t emitted = 0;
  const std::string model = g_info.model_type;
  auto event = [&](const int32_t* ids, int n, const std::string& piece, const char* finish, const std::string& extra) {
    const std::string idj = ids_json(std::vector<int32_t>(ids, ids + n));
    std::string e = "data: ";
    if (oai)
      e += "{\"object\":\"text_completion\",\"model\":\"" + model + "\",\"choices\":[{\"index\":0,\"text\":\"" + ssb::json_escape(piece) +
           "\",\"tokens\":" + idj + ",\"finish_reason\":" + (finish ? "\"" + std::string(finish) + "\"" : std::string("null")) + "}]" + extra + "}";
    else
      e += "{\"tokens\":" + idj + ",\"text\":\"" + ssb::json_escape(piece) + "\",\"done\":" + (finish ? "true" : "false") + extra + "}";
    return send_all(fd, e + "\n\n");
  };
  auto next_piece = [&](bool flush) {
    std::string piece;
    if (text_mode && g_tok && !all.empty()) {
      std::vector<char> buf(16 * all.size() + 64);
      int len = 0;
      if (ssb_tok_decode(g_tok, all.data(), (int)all.size(), 1, buf.data(), (int)buf.size(), &len) == SSB_OK) {
        const std::string full(buf.data(), (size_t)len);
        const size_t upto = flush ? full.size() : utf8_safe_len(full);
        if (upto > emitted) {
          piece = full.substr(emitted, upto - emitted);
          emitted = upto;
        }
      }
    }
    return piece;
  };
  TokenSink sink = [&](const int32_t* ids, int n) {
    all.insert(all.end(), ids, ids + n);
    return event(ids, n, next_piece(false), nullptr, "");
  };
  GenResult r = generate(prompt, max_new, g_stream_chunk, sink, eos, samp);
  if (!r.error.empty()) {
    g_errors++;
    send_all(fd, "data: " + err_json(r.error) + "\n\n");
    if (r.fatal) {
      send_all(fd, "data: [DONE]\n\n");
      fatal_exit(r.error);
    }
  } else {
    g_tokens += (long long)r.tokens.size();
    g_ttft_us_sum.fetch_add((long long)(r.ttft_ms * 1e3));
    g_decode_us_sum.fetch_add((long long)(r.decode_ms * 1e3));
    char tail[320];
    const double tps = r.decode_ms > 0 && r.tokens.size() > 1 ? (r.tokens.size() - 1) * 1e3 / r.decode_ms : 0.0;
    snprintf(tail, sizeof tail,
             ",\"usage\":{\"prompt_tokens\":%zu,\"completion_tokens\":%zu},\"ttft_ms\":%.3f,\"decode_ms\":%.3f,\"decode_tokens_per_sec\":%.2f",
             prompt.size(), r.tokens.size(), r.ttft_ms, r.decode_ms, tps);
    event(nullptr, 0, next_piece(true), r.hit_eos ? "stop" : (int)r.tokens.size() >= max_new ? "length" : "cancelled", tail);
  }
  send_all(fd, "data: [DONE]\n\n");
}

struct InflightGuard {
  InflightGuard() { ++g_inflight; }
  ~InflightGuard() { --g_inflight; }
};

struct ConnGuard {
  ConnGuard() { ++g_conns; }
  ~ConnGuard() { --g_conns; }
};

// Largest request body accepted: a prompt can never exceed max_seq_len ids (<= 11 characters each in JSON) or, as text,
// a few bytes per token; 1 MiB floor for the fixed fields.  The JSON tree costs ~100 B per number, so an uncapped id
// array is a cheap way to run the pod out of memory.
static size_t max_body_bytes() {
  const size_t per_seq = g_ready.load() == 1 ? (size_t)g_info.max_seq_len * 32 : 0;
  return std::max<size_t>(1u << 20, per_seq);
}

static void handle(int fd) {
  ConnGuard conn;
  if (g_conns.load() > kMaxConns) {
    respond(fd, 503, "Service Unavailable", err_json("too many connections"));
    close(fd);
    return;
  }
  {  // an idle or slow client must not pin a thread (and the SIGTERM drain) for ever
    timeval tv{10, 0};
    setsockopt(fd, SOL_SOCKET, SO_RCVTIMEO, &tv, sizeof tv);
  }
  InflightGuard guard;
  std::string req;
  char buf[8192];
  size_t hdr_end = std::string::npos;
  while (hdr_end == std::string::npos && req.size() < (1u << 20)) {
    ssize_t n = recv(fd, buf, sizeof buf, 0);
    if (n <= 0) break;
    req.append(buf, (size_t)n);
    hdr_end = req.find("\r\n\r\n");
  }
  if (hdr_end == std::string::npos) {
    close(fd);
    return;
  }
  size_t clen = 0;
  {
    std::string low = req.substr(0, hdr_end);
    for (auto& c : low) c = (char)tolower(c);
    size_t p = low.find("\r\ncontent-length:");  // a header NAME starts a line (not e.g. "x-content-length:")
    if (p != std::string::npos) clen = (size_t)strtoull(low.c_str() + p + 17, nullptr, 10);
  }
  if (clen > max_body_bytes()) {
    respond(fd, 413, "Payload Too Large", err_json("body too large"));
    close(fd);
    return;
  }
  while (req.size() < hdr_end + 4 + clen) {
    ssize_t n = recv(fd, buf, sizeof buf, 0);
    if (n <= 0) break;
    req.append(buf, (size_t)n);
  }
  if (req.size() < hdr_end + 4 + clen) {  // client stalled (SO_RCVTIMEO) or went away mid-body
    respond(fd, 408, "Request Timeout", err_json("request body incomplete"));
    close(fd);
    return;
  }
  const std::string line = req.substr(0, req.find("\r\n"));
  const size_t sp1 = line.find(' '), sp2 = line.find(' ', sp1 + 1);
  const std::string method = line.substr(0, sp1);
  std::string path = sp2 == std::string::npos ? "" : line.substr(sp1 + 1, sp2 - sp1 - 1);
  if (size_t q = path.find('?'); q != std::string::npos) path.resize(q);
  const std::string body = req.size() >= hdr_end + 4 ? req.substr(hdr_end + 4, clen) : "";

  if (method == "GET" && (path == "/" || path == "/healthz" || path == "/readyz")) {
    // readiness: 200 only when weights are on the device and the engine answered ssb_engine_info
    const int st = g_draining.load() ? 2 : g_ready.load();
    if (st == 2)
      respond(fd, 503, "Service Unavailable", "{\"status\":\"draining\"}");
    else if (st == 1)
      respond(fd, 200, "OK", "{\"status\":\"ready\",\"engine\":\"" + std::string(ssb_version()) + "\",\"model_type\":\"" +
                                 std::string(g_info.model_type) + "\"}");
    else
      respond(fd, 503, "Service Unavailable", st == 0 ? "{\"status\":\"loading\"}" : err_json(g_load_error));
  } else if (method == "GET" && path == "/metrics") {
    char m[1024];
    snprintf(m, sizeof m,
             "# TYPE ssb_requests_total counter\nssb_requests_total %lld\n# TYPE ssb_generated_tokens_total counter\n"
             "ssb_generated_tokens_total %lld\n# TYPE ssb_errors_total counter\nssb_errors_total %lld\n"
             "# TYPE ssb_ttft_ms_sum counter\nssb_ttft_ms_sum %.3f\n# TYPE ssb_decode_ms_sum counter\nssb_decode_ms_sum %.3f\n",
             g_requests.load(), g_tokens.load(), g_errors.load(), g_ttft_us_sum.load() / 1e3, g_decode_us_sum.load() / 1e3);
    std::string ms = m;
    if (g_sched) {  // continuous batching: how full the shared steps are and how often admission waited for KV blocks
      snprintf(m, sizeof m,
               "# TYPE ssb_sched_decode_calls_total counter\nssb_sched_decode_calls_total %lld\n"
               "# TYPE ssb_sched_step_rows_total counter\nssb_sched_step_rows_total %lld\n"
               "# TYPE ssb_sched_max_rows gauge\nssb_sched_max_rows %d\n"
               "# TYPE ssb_sched_kv_deferred_total counter\nssb_sched_kv_deferred_total %lld\n",
               g_sched->steps(), g_sched->step_rows(), g_sched->max_rows_seen(), g_sched->deferred());
      ms += m;
    }
    respond(fd, 200, "OK", ms, "text/plain; version=0.0.4");
  } else if (method == "POST" && (path == "/generate" || path == "/v1/completions")) {
    if (g_ready.load() != 1) {
      respond(fd, 503, "Service Unavailable", err_json("model is not loaded yet"));
    } else {
      g_requests++;
      std::string err;
      std::vector<int32_t> prompt;
      int max_new = 16;
      bool ok = true, text_mode = false, stream = false, stop_eos = g_stop_default;
      Sampling samp;
      try {
        Json j = ssb::json_parse(body);
        const bool oai = path == "/v1/completions";
        const Json* p = j.find(oai ? "prompt" : "tokens");
        const Json* ptxt = oai ? p : j.find("prompt");  // /generate also takes {"prompt": "text"}
        if (ptxt && ptxt->kind == Json::Str && (oai || !p)) {
          if (!g_tok) {
            ok = false;
            err = "text prompts need <model_dir>/tokenizer.json (Llama-2 or GPT-2 style BPE); pass the prompt as an array of token ids";
          } else {
            std::vector<int32_t> ids(4 * ptxt->str.size() + 16);
            int n = 0;
            if (ssb_tok_encode(g_tok, ptxt->str.c_str(), 1, ids.data(), (int)ids.size(), &n) != SSB_OK || n < 1) {
              ok = false;
              err = std::string("tokenizer: ") + ssb_last_error();
            } else {
              prompt.assign(ids.begin(), ids.begin() + n);
              for (int32_t t : prompt)
                if (t < 0 || t >= g_info.vocab_size) {
                  ok = false;
                  err = "tokenizer produced an id outside the model's vocabulary";
                }
              text_mode = true;
            }
          }
        } else {
          ok = parse_ids(p, g_info.vocab_size, &prompt, &err);
        }
        max_new = (int)j.get_int(oai ? "max_tokens" : "max_new_tokens", 16);
        if (const Json* st = j.find("stream")) stream = (st->kind == Json::Bool && st->b) || (st->kind == Json::Num && st->num != 0);
        if (const Json* st = j.find("stop_at_eos")) stop_eos = (st->kind == Json::Bool && st->b) || (st->kind == Json::Num && st->num != 0);
        samp.temperature = (float)j.get_num("temperature", 0.0);  // 0 (default) = greedy, the engine's device-resident loop
        samp.top_p = (float)j.get_num("top_p", 1.0);
        samp.top_k = (int)j.get_int("top_k", 0);
        if (const Json* sd = j.find("seed"); sd && sd->kind == Json::Num)
          samp.seed = (uint64_t)sd->num;
        else
          samp.seed = (uint64_t)std::chrono::steady_clock::now().time_since_epoch().count() ^ ((uint64_t)g_requests.load() << 32);
        if (ok && (samp.temperature < 0 || !(samp.top_p > 0 && samp.top_p <= 1) || samp.top_k < 0)) {
          ok = false;
          err = "temperature must be >= 0, top_p in (0, 1], top_k >= 0";
        }
        if (ok && samp.on() && g_sched) {
          ok = false;
          err = "sampling (temperature > 0) is not available while continuous batching is on: the shared decode loop is greedy";
        }
        if (ok && stop_eos && g_eos.empty()) {
          ok = false;
          err = "stop_at_eos: no eos_token_id in params.json, generation_config.json or config.json";
        }
        if (ok && (max_new < 1 || (int)prompt.size() + max_new > g_info.max_seq_len)) {
          ok = false;
          err = "prompt length + max tokens exceeds max_seq_len";
        }
      } catch (std::exception& e) {
        ok = false;
        err = e.what();
      }
      if (!ok) {
        g_errors++;
        respond(fd, 400, "Bad Request", err_json(err));
      } else if (stream) {
        stream_response(fd, path == "/v1/completions", prompt, max_new, text_mode, stop_eos ? g_eos : kNoEos, samp);
      } else {
        GenResult r = (stop_eos || samp.on()) ? generate(prompt, max_new, stop_eos ? g_eos_every : 1 << 30, nullptr, stop_eos ? g_eos : kNoEos, samp)
                                              : generate(prompt, max_new);
        if (!r.error.empty()) {
          g_errors++;
          respond(fd, 500, "Internal Server Error", err_json(r.error));
          if (r.fatal) fatal_exit(r.error);
        } else {
          g_tokens += (long long)r.tokens.size();
          g_ttft_us_sum.fetch_add((long long)(r.ttft_ms * 1e3));
          g_decode_us_sum.fetch_add((long long)(r.decode_ms * 1e3));
          char tail[256];
          const double tps = r.decode_ms > 0 && r.tokens.size() > 1 ? (r.tokens.size() - 1) * 1e3 / r.decode_ms : 0.0;
          snprintf(tail, sizeof tail, "\"ttft_ms\":%.3f,\"decode_ms\":%.3f,\"decode_tokens_per_sec\":%.2f", r.ttft_ms, r.decode_ms, tps);
          std::string text;
          if (text_mode && g_tok) {
            std::vector<char> buf(16 * r.tokens.size() + 64);
            int len = 0;
            if (ssb_tok_decode(g_tok, r.tokens.data(), (int)r.tokens.size(), 1, buf.data(), (int)buf.size(), &len) == SSB_OK)
              text.assign(buf.data(), (size_t)len);
          }
          if (path == "/generate")
            respond(fd, 200, "OK", "{\"tokens\":" + ids_json(r.tokens) + ",\"text\":\"" + ssb::json_escape(text) + "\",\"finish_reason\":\"" +
                                       (r.hit_eos ? "stop" : "length") + "\"," + tail + "}");
          else
            respond(fd, 200, "OK",
                    "{\"object\":\"text_completion\",\"model\":\"" + std::string(g_info.model_type) +
                        "\",\"choices\":[{\"index\":0,\"text\":\"" + ssb::json_escape(text) + "\",\"tokens\":" + ids_json(r.tokens) +
                        ",\"finish_reason\":\"" + (r.hit_eos ? "stop" : "length") + "\"}],\"usage\":{\"prompt_tokens\":" + std::to_string(prompt.size()) +
                        ",\"completion_tokens\":" + std::to_string(r.tokens.size()) + "}," + tail + "}");
        }
      }
    }
  } else {
    respond(fd, 404, "Not Found", err_json("no such endpoint"));
  }
  shutdown(fd, SHUT_RDWR);
  close(fd);
}

int main(int argc, char** argv) {
  signal(SIGPIPE, SIG_IGN);
  signal(SIGTERM, on_sigterm);
  const std::string model_dir = (argc > 1 && argv[1][0] != '-') ? argv[1] : getenv_or("MODEL_DIR", "/content/model");
  const std::string params_file = getenv_or("PARAMS_FILE", "/content/params.json");
  const int port = atoi(getenv_or("PORT", "8080").c_str());
  std::string params = "{}";
  read_file(params_file, &params);  // {} if absent (params_reconciler.go mounts it only when .spec.params is set)
  params = merge_param_env(params);
  if (argc > 1 && strcmp(argv[1], "--print-params") == 0) {  // what the engine will be created with (no GPU needed)
    printf("%s\n", params.c_str());
    return 0;
  }

  int ls = socket(AF_INET, SOCK_STREAM, 0);
  int one = 1;
  setsockopt(ls, SOL_SOCKET, SO_REUSEADDR, &one, sizeof one);
  sockaddr_in addr{};
  addr.sin_family = AF_INET;
  addr.sin_addr.s_addr = htonl(INADDR_ANY);
  addr.sin_port = htons((uint16_t)port);
  if (bind(ls, (sockaddr*)&addr, sizeof addr) != 0 || listen(ls, 128) != 0) {
    perror("serve: bind/listen");
    return 2;
  }
  fprintf(stderr, "serve: listening on :%d, loading %s\n", port, model_dir.c_str());

  // model load runs beside the accept loop so the readiness probe sees 503 (not a refused connection) while loading
  // tp_size from params.json: one engine rank per GPU of this container, all in this process
  int tp = 1;
  try {
    tp = (int)ssb::json_parse(params).get_int("tp_size", 1);
  } catch (std::exception&) {
  }
  std::thread loader([&, tp] {
    int rc = SSB_OK;
    if (tp <= 1) {
      rc = ssb_engine_create(model_dir.c_str(), params.c_str(), &g_engine);
    } else {
      // per-rank params: {"tp_rank": r, "device": r, <the CRD's params>}  (first key wins in the engine's parser)
      const size_t brace = params.find('{');
      const std::string rest = brace == std::string::npos ? "}" : params.substr(brace + 1);
      const bool empty_obj = rest.find_first_not_of(" \t\r\n") == rest.find('}');
      std::vector<ssb_engine*> eng(tp, nullptr);
      std::vector<int> rcs(tp, SSB_OK);
      std::vector<std::string> errs(tp);
      std::vector<std::thread> th;
      for (int r = 0; r < tp; ++r)
        th.emplace_back([&, r] {
          const std::string pj = "{\"tp_rank\":" + std::to_string(r) + ",\"device\":" + std::to_string(r) + (empty_obj ? "" : ",") + rest;
          rcs[r] = ssb_engine_create(model_dir.c_str(), pj.c_str(), &eng[r]);
          if (rcs[r] != SSB_OK) errs[r] = ssb_last_error();
        });
      for (auto& t : th) t.join();
      for (int r = 0; r < tp && rc == SSB_OK; ++r)
        if (rcs[r] != SSB_OK) {
          rc = rcs[r];
          g_load_error = "rank " + std::to_string(r) + ": " + errs[r];
        }
      if (rc == SSB_OK) {
        const int hs = ssb_tp_handle_size();
        std::vector<char> handles((size_t)hs * tp);
        for (int r = 0; r < tp && rc == SSB_OK; ++r) rc = ssb_tp_export(eng[r], handles.data() + (size_t)r * hs);
        for (int r = 0; r < tp && rc == SSB_OK; ++r) rc = ssb_tp_connect(eng[r], handles.data(), tp);
        if (rc != SSB_OK) g_load_error = ssb_last_error();
      }
      if (rc == SSB_OK) {
        g_engine = eng[0];
        g_peers.assign(eng.begin() + 1, eng.end());
      }
    }
    if (rc != SSB_OK) {
      if (g_load_error.empty()) g_load_error = ssb_last_error();
      fprintf(stderr, "serve: engine create failed (%d): %s\n", rc, g_load_error.c_str());
      g_ready = -1;
      // fatal: exit non-zero so the Deployment restarts the pod; no CPU fallback
      std::this_thread::sleep_for(std::chrono::milliseconds(200));
      _exit(rc == SSB_ENODEV ? 3 : 1);
    }
    ssb_engine_info(g_engine, &g_info);
    try {
      const Json pj = ssb::json_parse(params);
      g_stream_chunk = std::max(1, (int)pj.get_int("stream_chunk", 1));
      g_stop_default = pj.get_int("stop_at_eos", 0) != 0;
      g_eos_every = std::max(1, (int)pj.get_int("eos_check_every", 16));
      // .spec.params is map[string]IntOrString (api/v1/server_types.go:30): params.json may say "eos_token_id": "2"
      auto one_eos = [](const Json& x) {
        if (x.kind == Json::Num) g_eos.push_back((int32_t)x.num);
        if (x.kind == Json::Str && !x.str.empty()) {
          char* end = nullptr;
          const long v = strtol(x.str.c_str(), &end, 10);
          if (end && *end == 0 && v >= 0) g_eos.push_back((int32_t)v);
        }
      };
      auto take_eos = [&](const Json* v) {
        if (!v) return;
        if (v->kind == Json::Arr)
          for (auto& x : v->arr) one_eos(x);
        else
          one_eos(*v);
      };
      take_eos(pj.find("eos_token_id"));
      for (const char* f : {"/generation_config.json", "/config.json"}) {
        std::string txt;
        if (!g_eos.empty() || !read_file(model_dir + f, &txt)) continue;
        try {
          take_eos(ssb::json_parse(txt).find("eos_token_id"));
        } catch (std::exception&) {
        }
      }
      if (pj.get_int("batching", 0) != 0 && g_peers.empty()) {
        g_abi.e = g_engine;
        int kv_total = 0, kv_free = 0;
        if (ssb_kv_blocks(g_engine, &kv_total, &kv_free) != SSB_OK) kv_total = 0;  // no accounting: ENOMEM is the limit
        g_sched = new ssbhost::BatchScheduler<AbiEngine>(&g_abi, g_info.max_batch, (int)pj.get_int("batch_tick", 8), kv_total,
                                                         g_info.kv_block_size);
        fprintf(stderr, "serve: continuous batching on (max_batch %d, %d KV blocks of %d tokens)\n", g_info.max_batch, kv_total,
                g_info.kv_block_size);
      }
    } catch (std::exception&) {
    }
    if (ssb_tok_load((model_dir + "/tokenizer.json").c_str(), &g_tok) != SSB_OK) {
      fprintf(stderr, "serve: no usable tokenizer.json (%s): text prompts disabled, token-id prompts only\n", ssb_last_error());
      g_tok = nullptr;
    }
    fprintf(stderr, "serve: ready (%s, %d layers, %.2f GB HBM)\n", g_info.model_type, g_info.n_layers,
            g_info.hbm_bytes_allocated / 1e9);
    g_ready = 1;
  });
  loader.detach();

  g_listen_fd = ls;
  for (;;) {
    int fd = accept(ls, nullptr, nullptr);
    if (g_draining.load()) {
      if (fd >= 0) close(fd);
      break;
    }
    if (fd < 0) continue;
    setsockopt(fd, IPPROTO_TCP, TCP_NODELAY, &one, sizeof one);
    timeval snd{10, 0};  // a stalled streaming client must not hold the engine (or the batch scheduler) for ever
    setsockopt(fd, SOL_SOCKET, SO_SNDTIMEO, &snd, sizeof snd);
    std::thread(handle, fd).detach();
  }
  close(ls);
  fprintf(stderr, "serve: SIGTERM, draining %d request(s)\n", g_inflight.load());
  for (int i = 0; i < 250 && g_inflight.load() > 0; ++i) std::this_thread::sleep_for(std::chrono::milliseconds(100));
  fprintf(stderr, "serve: exit\n");
  _exit(0);  // engine teardown is the process exit: the device context goes with it
}
