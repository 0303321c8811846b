// hx_callers.cpp — the reference's calling pattern as a load generator: N concurrent callers, ONE query per call
// (ValidatedVectorReadIndex::search is invoked once per request from its own tokio task:
//  crates/db/src/search/vector/read_index.rs:81-101 <- execution/interpreter/access/search/storage.rs:142-192).
//
// A C++ host linked against libhelix_b200.so through host/vector_index.hpp (the C++ mirror of the reference interface);
// built as libhx_callers.so so that bench.py and the tests can drive it (ctypes) and check every result bit for bit.
//   mode 0  blocking : n_callers OS threads, each `svc.search(q)` in a loop (thread-per-request hosts, spawn_blocking)
//   mode 1  tasks    : n_threads OS threads, each multiplexing n_callers / n_threads logical callers with
//                      submit() / poll()  (what a tokio worker does with the tasks it owns)
//   mode 2  direct   : n_callers OS threads, each one blocking B = 1 hx_search call per query (no service: the
//                      round-1 path, kept as the comparison)
// hx_callers_run_restricted plays search_restricted the same way (one query + its candidate set per call); its direct
// mode is one blocking B = 1 hx_search_restricted per call.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstring>
#include <functional>
#include <thread>
#include <vector>

#include "vector_index.hpp"

using clk = std::chrono::steady_clock;

extern "C" {
typedef struct {
  double seconds, qps, mean_us, p50_us, p90_us, p99_us, max_us;
  uint64_t completed, errors;
} hx_callers_report;

}

// one blocking call for query qi (service search, or the direct library call), and the async submit for query qi
using BlockingCall = std::function<void(size_t qi, uint64_t* ids, float* scores, uint32_t* count)>;
using SubmitCall = std::function<uint64_t(size_t qi)>;

// Caller c walks queries c, c + n_callers, ... (wrapping) until `seconds` have passed and every query has been answered
// at least once.  out_*: the answer recorded for each query index (n_queries x k).
static int run_callers(hx_service* svc, size_t n_queries, uint32_t k, uint32_t n_callers, uint32_t n_threads, int mode,
                       double seconds, const BlockingCall& call, const SubmitCall& submit, uint64_t* out_ids,
                       float* out_scores, uint32_t* out_counts, hx_callers_report* rep) {
  if (mode != 1) n_threads = n_callers;
  if (n_threads == 0) n_threads = 1;
  n_threads = std::min(n_threads, n_callers);
  std::atomic<uint64_t> completed{0}, errors{0};
  std::atomic<bool> go{false};
  std::vector<std::vector<float>> lat(n_threads);
  const auto deadline_after = std::chrono::duration<double>(seconds);
  clk::time_point t_start;

  auto record = [&](size_t qi, const uint64_t* ids, const float* sc, uint32_t cnt) {
    if (out_ids) memcpy(out_ids + qi * k, ids, k * sizeof(uint64_t));
    if (out_scores) memcpy(out_scores + qi * k, sc, k * sizeof(float));
    if (out_counts) out_counts[qi] = cnt;
  };

  auto worker = [&](uint32_t t) {
    try {
      std::vector<float>& L = lat[t];
      L.reserve(1 << 16);
      while (!go.load(std::memory_order_acquire)) std::this_thread::yield();
      const auto t_end = t_start + std::chrono::duration_cast<clk::duration>(deadline_after);
      if (mode == 0 || mode == 2) {
        std::vector<uint64_t> ids(k);
        std::vector<float> sc(k);
        size_t qi = t % n_queries, done_here = 0;
        const size_t mine = (n_queries + n_callers - 1 - t) / n_callers;   // queries this caller must cover once
        while (clk::now() < t_end || done_here < mine) {
          uint32_t cnt = 0;
          const auto a = clk::now();
          call(qi, ids.data(), sc.data(), &cnt);
          const auto b = clk::now();
          L.push_back(std::chrono::duration<float, std::micro>(b - a).count());
          record(qi, ids.data(), sc.data(), cnt);
          completed.fetch_add(1, std::memory_order_relaxed);
          done_here++;
          qi += n_callers;
          if (qi >= n_queries) qi = t % n_queries;
        }
      } else {
        // logical callers owned by this thread: c = t, t + n_threads, ...
        struct Task { uint32_t c; size_t qi; uint64_t ticket; bool busy; clk::time_point t0; size_t done; };
        std::vector<Task> tasks;
        for (uint32_t c = t; c < n_callers; c += n_threads) tasks.push_back(Task{c, c % n_queries, 0, false, {}, 0});
        std::vector<uint64_t> ids(k);
        std::vector<float> sc(k);
        size_t active = tasks.size();
        std::vector<bool> finished(tasks.size(), false);
        while (active) {
          const bool past = clk::now() >= t_end;
          for (size_t i = 0; i < tasks.size(); ++i) {
            Task& T = tasks[i];
            if (finished[i]) continue;
            if (!T.busy) {
              const size_t mine = (n_queries + n_callers - 1 - T.c) / n_callers;
              if (past && T.done >= mine) { finished[i] = true; active--; continue; }
              T.t0 = clk::now();
              T.ticket = submit(T.qi);
              T.busy = true;
            } else {
              uint32_t cnt = 0;
              int32_t done = 0;
              helix::check(hx_service_poll(svc, T.ticket, &done, ids.data(), sc.data(), &cnt));
              if (done) {
                L.push_back(std::chrono::duration<float, std::micro>(clk::now() - T.t0).count());
                record(T.qi, ids.data(), sc.data(), cnt);
                completed.fetch_add(1, std::memory_order_relaxed);
                T.busy = false;
                T.done++;
                T.qi += n_callers;
                if (T.qi >= n_queries) T.qi = T.c % n_queries;
              }
            }
          }
        }
      }
    } catch (const std::exception&) {
      errors.fetch_add(1);
    }
  };

  std::vector<std::thread> th;
  for (uint32_t t = 0; t < n_threads; ++t) th.emplace_back(worker, t);
  t_start = clk::now();
  go.store(true, std::memory_order_release);
  for (auto& x : th) x.join();
  const double secs = std::chrono::duration<double>(clk::now() - t_start).count();
  std::vector<float> all;
  for (auto& l : lat) all.insert(all.end(), l.begin(), l.end());
  std::sort(all.begin(), all.end());
  memset(rep, 0, sizeof(*rep));
  rep->seconds = secs;
  rep->completed = completed.load();
  rep->errors = errors.load();
  rep->qps = secs > 0 ? rep->completed / secs : 0.0;
  if (!all.empty()) {
    double sum = 0;
    for (float v : all) sum += v;
    rep->mean_us = sum / all.size();
    rep->p50_us = all[all.size() / 2];
    rep->p90_us = all[(size_t)(all.size() * 0.90)];
    rep->p99_us = all[std::min(all.size() - 1, (size_t)(all.size() * 0.99))];
    rep->max_us = all.back();
  }
  return rep->errors ? 2 : 0;
}

extern "C" {
// queries: n_queries x dim
int hx_callers_run(hx_service* svc, hx_index* index, uint32_t ef, const float* queries, size_t n_queries, uint32_t dim,
                   uint32_t k, uint32_t n_callers, uint32_t n_threads, int mode, double seconds, uint64_t* out_ids,
                   float* out_scores, uint32_t* out_counts, hx_callers_report* rep) {
  if (!queries || !rep || n_callers == 0 || n_queries == 0 || (mode != 2 && !svc) || (mode == 2 && !index)) return 1;
  hx_search_params p{};
  p.k = k;
  p.ef = ef;
  p.simhash_mode = HX_SIMHASH_OFF;
  p.pre_sampling_ratio = 1.0f;
  const helix::SearchService S(svc, k, false);
  const BlockingCall call = [&](size_t qi, uint64_t* ids, float* sc, uint32_t* cnt) {
    if (mode == 0) S.search(queries + qi * dim, ids, sc, cnt);
    else helix::check(hx_search(index, queries + qi * dim, 1, &p, ids, sc, cnt, nullptr));
  };
  const SubmitCall submit = [&](size_t qi) { return S.submit(queries + qi * dim); };
  return run_callers(svc, n_queries, k, n_callers, n_threads, mode, seconds, call, submit, out_ids, out_scores, out_counts,
                     rep);
}

// search_restricted callers: query qi scans cand_ids[cand_offsets[qi] .. cand_offsets[qi + 1]), or the device set
// sets[qi] when `sets` is given (the direct mode then calls hx_search_restricted_sets with that one set)
int hx_callers_run_restricted(hx_service* svc, hx_index* index, const float* queries, size_t n_queries, uint32_t dim,
                              uint32_t k, const uint64_t* cand_ids, const uint64_t* cand_offsets, hx_candidates* const* sets,
                              uint32_t n_callers, uint32_t n_threads, int mode, double seconds, uint64_t* out_ids,
                              float* out_scores, uint32_t* out_counts, hx_callers_report* rep) {
  if (!queries || !rep || n_callers == 0 || n_queries == 0 || (mode != 2 && !svc) || (mode == 2 && !index) ||
      (!sets && (!cand_ids || !cand_offsets)))
    return 1;
  hx_search_params p{};
  p.k = k;
  p.simhash_mode = HX_SIMHASH_OFF;
  p.pre_sampling_ratio = 1.0f;
  const helix::RestrictedSearchService S(svc, k, false);
  const BlockingCall call = [&](size_t qi, uint64_t* ids, float* sc, uint32_t* cnt) {
    const float* q = queries + qi * dim;
    if (sets) {
      if (mode == 0) helix::check(hx_service_search_restricted_set(svc, q, sets[qi], ids, sc, cnt));
      else helix::check(hx_search_restricted_sets(index, q, 1, &p, sets + qi, 1, ids, sc, cnt, nullptr));
      return;
    }
    const uint64_t* c = cand_ids + cand_offsets[qi];
    const size_t n = cand_offsets[qi + 1] - cand_offsets[qi];
    if (mode == 0) S.search(q, c, n, ids, sc, cnt);
    else helix::check(hx_search_restricted(index, q, 1, &p, c, n, ids, sc, cnt, nullptr));
  };
  const SubmitCall submit = [&](size_t qi) {
    const float* q = queries + qi * dim;
    if (sets) return S.submit(q, sets[qi]);
    return S.submit(q, cand_ids + cand_offsets[qi], cand_offsets[qi + 1] - cand_offsets[qi]);
  };
  return run_callers(svc, n_queries, k, n_callers, n_threads, mode, seconds, call, submit, out_ids, out_scores, out_counts,
                     rep);
}
}
