// scheduler.h — continuous batching for the serve host (SURVEY.md §8f #4; opt-in with params.json {"batching": 1}).
//
// The reference serves one request at a time per replica (Deployment `replicas := 1`, one Basaran process,
// internal/controller/server_controller.go:115,134); the engine streams its weights once per decode step no
// matter how many sequences ride along (batch 32 costs 2.3x a batch-1 step, not 32x), so concurrent clients should
// share steps.  This is the policy, written against the five calls of include/ssb.h so it can be unit-tested with a
// fake engine on a CPU box (tests/test_scheduler_cpu.py) and used unchanged over the real one:
//
//   loop:  admit waiting requests while slots are free        -> ONE ssb_prefill over all newcomers
//          run min(tick, min remaining) decode steps          -> ONE ssb_decode over all active sequences
//          retire sequences that produced max_new tokens      -> fulfil their promise, free their slot
//
// Failure isolation: SSB_ENOMEM (a resource limit, engine state untouched) costs ONE request — newcomers are re-prefilled
// one by one, a decode retires its most recently admitted sequence and retries the rest; any other engine error fails the
// batch only if it is SSB_ECUDA (the host then exits for a pod restart); an argument the engine rejects (validated before
// any state changes) makes that tick run sequence by sequence so only the offender is retired.  With the pool size known
// (ssb_kv_blocks) requests are admitted only while their prompt + max_new blocks are unreserved, so ENOMEM stays a backstop.
//
// Decode never overshoots a request (the step count is the minimum remaining), newcomers wait at most one tick, and
// greedy decoding makes every request's ids independent of who shared its batch (checked by the test).  A request may
// carry an on_tokens callback (streaming): it sees its ids once per tick and can retire the request early.
#pragma once
#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdint>
#include <deque>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

namespace ssbhost {

struct Request {
  std::vector<int32_t> prompt;
  int max_new = 0;
  // optional: fed the ids produced since the previous call (first the prefill's token, then once per tick) from the
  // scheduler thread; returning false retires the request early and frees its slot ("stream": true, client went away)
  std::function<bool(const int32_t*, int)> on_tokens;
  // result
  std::vector<int32_t> tokens;
  std::string error;
  int error_code = 0;  // the engine's return code behind `error` (0 for the scheduler's own validation errors)
  double ttft_ms = 0, total_ms = 0;
  bool done = false;
  double t0 = 0;  // submit time (scheduler-internal)
};

// EngineT must provide (all return 0 on success, error text through last_error()):
//   int seq_create(int* sid); int seq_free(int sid);
//   int prefill(const int* sids, const int32_t* toks, const int* lens, int nseq, int32_t* next);
//   int decode(const int* sids, const int32_t* last, int nseq, int nsteps, int32_t* out /*[nseq][nsteps]*/);
//   std::string last_error();
// SSB_ENOMEM of include/ssb.h: a per-call resource limit (sequence slots, KV blocks) — the engine's state is untouched
constexpr int kPerSequenceError = -4;
// SSB_ECUDA: the device (or a tensor-parallel peer) is gone — nothing can be retried, the host exits for a pod restart
constexpr int kFatalError = -5;

template <class EngineT>
class BatchScheduler {
 public:
  // kv_total_blocks / kv_block_size (ssb_kv_blocks, ssb_info.kv_block_size): when given, a request is admitted only while
  // the blocks its prompt + max_new tokens will need are unreserved, and waits in the queue otherwise — so one long
  // request cannot run the pool dry under the others mid-decode.  0 = no accounting (the engine's SSB_ENOMEM is the limit).
  BatchScheduler(EngineT* eng, int max_batch, int tick, int kv_total_blocks = 0, int kv_block_size = 0)
      : eng_(eng), max_batch_(max_batch), tick_(std::max(1, tick)), kv_total_(kv_total_blocks), kv_bs_(kv_block_size) {
    worker_ = std::thread([this] { run(); });
  }
  ~BatchScheduler() {
    {
      std::lock_guard<std::mutex> lk(mu_);
      stop_ = true;
    }
    cv_.notify_all();
    worker_.join();
  }
  // blocks until the request is finished (called from the per-connection threads of the host)
  void submit(Request* r) {
    std::unique_lock<std::mutex> lk(mu_);
    r->t0 = now_ms();
    waiting_.push_back(r);
    cv_.notify_all();
    done_cv_.wait(lk, [r] { return r->done; });
  }
  // statistics (for /metrics and the test)
  long long steps() const { return steps_; }
  long long step_rows() const { return step_rows_; }  // sum over decode calls of nseq * nsteps
  int max_rows_seen() const { return max_rows_; }
  long long deferred() const { return deferred_; }  // admission passes that left a request queued for want of KV blocks

 private:
  struct Active {
    Request* r;
    int sid;
    int32_t last;
    int blocks;  // KV blocks reserved at admission (0 without accounting)
  };
  int blocks_for(const Request* r) const {
    if (kv_total_ <= 0 || kv_bs_ <= 0) return 0;
    return (int)(((long long)r->prompt.size() + std::max(0, r->max_new) + kv_bs_ - 1) / kv_bs_);
  }
  static double now_ms() {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
  }
  void finish(Request* r, const std::string& err, int code = 0) {
    std::lock_guard<std::mutex> lk(mu_);
    r->error = err;
    r->error_code = code;
    r->total_ms = now_ms() - r->t0;
    r->done = true;
    done_cv_.notify_all();
  }
  void run() {
    std::vector<Active> active;
    for (;;) {
      std::vector<Request*> fresh, too_big;
      {
        std::unique_lock<std::mutex> lk(mu_);
        cv_.wait(lk, [&] { return stop_ || !waiting_.empty() || !active.empty(); });
        if (stop_ && active.empty() && waiting_.empty()) return;
        int reserved = 0;
        for (const Active& a : active) reserved += a.blocks;
        while (!waiting_.empty() && (int)(active.size() + fresh.size()) < max_batch_) {
          Request* r = waiting_.front();
          const int need = blocks_for(r);
          if (need > kv_total_ && kv_total_ > 0) {  // can never fit: fail it alone, now
            too_big.push_back(r);
            waiting_.pop_front();
            continue;
          }
          if (reserved + need > kv_total_ && need > 0) {
            ++deferred_;  // FIFO: wait for running requests to retire rather than overtake
            break;
          }
          reserved += need;
          fresh.push_back(r);
          waiting_.pop_front();
        }
      }
      for (Request* r : too_big)
        finish(r, "KV block pool exhausted: the request needs " + std::to_string(blocks_for(r)) + " blocks of " +
                      std::to_string(kv_bs_) + " tokens, the pool holds " + std::to_string(kv_total_),
               kPerSequenceError);
      // ---- admit: one prefill over all newcomers
      if (!fresh.empty()) {
        std::vector<int> sids, lens;
        std::vector<int32_t> toks;
        std::vector<Request*> ok;
        for (Request* r : fresh) {
          int sid = -1;
          if (r->prompt.empty() || r->max_new < 1) {
            finish(r, "empty prompt or max_new < 1");
          } else if (int crc = eng_->seq_create(&sid)) {
            finish(r, eng_->last_error(), crc);
          } else {
            sids.push_back(sid);
            lens.push_back((int)r->prompt.size());
            toks.insert(toks.end(), r->prompt.begin(), r->prompt.end());
            ok.push_back(r);
          }
        }
        if (!ok.empty()) {
          std::vector<int32_t> next(ok.size());
          int prc = eng_->prefill(sids.data(), toks.data(), lens.data(), (int)ok.size(), next.data());
          if (prc != 0 && prc != kFatalError && ok.size() > 1) {
            // a resource limit (e.g. the KV block pool) or a rejected argument of ONE prompt must not fail every newcomer:
            // the engine rejects before it touches any state, so prefill them one by one and fail only the offenders
            prc = 0;
            std::vector<Request*> ok2;
            std::vector<int> sids2;
            std::vector<int32_t> next2;
            for (size_t i = 0, o = 0; i < ok.size(); o += (size_t)lens[i], ++i) {
              int32_t nx = 0;
              if (int rc1 = eng_->prefill(&sids[i], toks.data() + o, &lens[i], 1, &nx)) {
                const std::string e = eng_->last_error();
                eng_->seq_free(sids[i]);
                finish(ok[i], e, rc1);
              } else {
                ok2.push_back(ok[i]);
                sids2.push_back(sids[i]);
                next2.push_back(nx);
              }
            }
            ok.swap(ok2);
            sids.swap(sids2);
            next.swap(next2);
          }
          if (prc != 0) {
            const std::string e = eng_->last_error();
            for (size_t i = 0; i < ok.size(); ++i) {
              eng_->seq_free(sids[i]);
              finish(ok[i], e, prc);
            }
          } else {
            for (size_t i = 0; i < ok.size(); ++i) {
              Request* r = ok[i];
              r->ttft_ms = now_ms() - r->t0;
              r->tokens.assign(1, next[i]);
              const bool go = !r->on_tokens || r->on_tokens(&next[i], 1);
              if (r->max_new == 1 || !go) {
                eng_->seq_free(sids[i]);
                finish(r, "");
              } else {
                active.push_back({r, sids[i], next[i], blocks_for(r)});
              }
            }
          }
        }
      }
      if (active.empty()) continue;
      // ---- one decode tick over all active sequences, never past the shortest remaining request
      int nsteps = tick_;
      for (auto& a : active) nsteps = std::min(nsteps, a.r->max_new - (int)a.r->tokens.size());
      std::vector<int> sids(active.size());
      std::vector<int32_t> last(active.size()), out(active.size() * (size_t)nsteps);
      for (size_t i = 0; i < active.size(); ++i) {
        sids[i] = active[i].sid;
        last[i] = active[i].last;
      }
      int n = (int)active.size();
      int drc = eng_->decode(sids.data(), last.data(), n, nsteps, out.data());
      if (drc != 0 && drc != kPerSequenceError && drc != kFatalError && n > 1) {
        // a rejected argument of ONE sequence (the engine validates everything before it touches any) must not fail its
        // batch mates: run this tick sequence by sequence, retire the ones the engine refuses, carry on with the others
        std::vector<Active> keep;
        std::vector<int32_t> out2, one((size_t)nsteps);
        drc = 0;
        for (int i = 0; i < n && drc != kFatalError; ++i) {
          const int rc1 = eng_->decode(&sids[i], &last[i], 1, nsteps, one.data());
          if (rc1 == 0) {
            keep.push_back(active[i]);
            out2.insert(out2.end(), one.begin(), one.end());
          } else if (rc1 == kFatalError) {
            drc = rc1;  // the device is gone: everybody fails below
          } else {
            const std::string e = eng_->last_error();
            eng_->seq_free(active[i].sid);
            finish(active[i].r, e, rc1);
            active[i].r = nullptr;
          }
        }
        if (drc == kFatalError) {
          std::vector<Active> left;
          for (auto& a : active)
            if (a.r) left.push_back(a);
          active.swap(left);
        } else {
          active.swap(keep);
          out.swap(out2);
          n = (int)active.size();
          if (n == 0) continue;
        }
      }
      if (drc == kPerSequenceError && n > 1) {
        // resource limit (KV blocks for the next steps): the engine refused before changing any sequence.  Retire the most
        // recently admitted request with the error and retry the others on the next pass instead of failing the whole batch.
        const std::string e = eng_->last_error();
        eng_->seq_free(active.back().sid);
        finish(active.back().r, e, drc);
        active.pop_back();
        continue;
      }
      if (drc != 0) {
        const std::string e = eng_->last_error();
        for (auto& a : active) {
          eng_->seq_free(a.sid);
          finish(a.r, e, drc);
        }
        active.clear();
        continue;
      }
      ++steps_;
      step_rows_ += (long long)n * nsteps;
      if (n > max_rows_.load()) max_rows_ = n;
      std::vector<Active> still;
      for (int i = 0; i < n; ++i) {
        Active& a = active[i];
        a.r->tokens.insert(a.r->tokens.end(), out.begin() + (size_t)i * nsteps, out.begin() + (size_t)(i + 1) * nsteps);
        a.last = a.r->tokens.back();
        const bool go = !a.r->on_tokens || a.r->on_tokens(a.r->tokens.data() + a.r->tokens.size() - nsteps, nsteps);
        if ((int)a.r->tokens.size() >= a.r->max_new || !go) {
          eng_->seq_free(a.sid);
          finish(a.r, "");
        } else {
          still.push_back(a);
        }
      }
      active.swap(still);
    }
  }

  EngineT* eng_;
  int max_batch_, tick_, kv_total_ = 0, kv_bs_ = 0;
  std::atomic<long long> deferred_{0};  // counters are read by the /metrics thread while the worker runs
  std::mutex mu_;
  std::condition_variable cv_, done_cv_;
  std::deque<Request*> waiting_;
  bool stop_ = false;
  std::thread worker_;
  std::atomic<long long> steps_{0}, step_rows_{0};
  std::atomic<int> max_rows_{0};
};

}  // namespace ssbhost
