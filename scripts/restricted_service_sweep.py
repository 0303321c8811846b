#!/usr/bin/env python
"""search_restricted's calling pattern (one query + one candidate set per call, many concurrent callers) on the C2 corpus
(1M x 768 cosine, `embedding` recipe, k = 10), three paths in one run:
  service : the restricted query service (hx_restricted_service_create), C++ callers (tasks on 8 threads, blocking)
  direct  : one blocking B = 1 hx_search_restricted per call (hx_search_restricted_sets for device sets)
  batched : every query in ONE hx_search_restricted_multi call (the rate the scan reaches without per-call overhead)
Candidate sets of 100 / 1 000 / 10 000 ids, contiguous and random, plus one device-set run.  Every answer is compared with
hx_search_restricted_multi's.  Writes JSON lines to stdout; the first line names the card and its power limit."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import helix_db_b200 as hx  # noqa: E402
from helix_db_b200 import callers  # noqa: E402

SEED = 0x0DB9ED1A


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired) as e:
        out = f"unavailable: {e}"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--queries", type=int, default=2048)
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--sizes", default="100,1000,10000")
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    ix = hx.VectorIndex(hx.Metric.Cosine, hx.VectorIndexConfig("c2", "embedding", a.dim))
    ix.generate_vectors(0, a.n, SEED, 1024, 1.0, 32)
    ix.load_graph(0, np.array([0], np.uint64), [0, 0], [])   # the exact scan needs no graph: entry point only
    ix.set_entry(0, 0)
    q = ix.generate_queries(SEED, a.queries, first_query=10_000_000, n_centroids=1024, sigma=1.0, kind=32)
    nq, k = a.queries, 10
    rng = np.random.default_rng(SEED)
    svc = ix.restricted_service(k, capacity=2048)
    p = hx.SearchParams.strict(k)

    def one(path, shape, rep, ids, sc, cnt, ref, launches=None):
        # row by row up to each count (entries past a count are whatever the caller's buffer held)
        same = bool(cnt.tolist() == ref[2].tolist() and all(
            ids[i, :c].tolist() == ref[0][i, :c].tolist() and sc[i, :c].tobytes() == ref[1][i, :c].tobytes()
            for i, c in enumerate(cnt.tolist())))
        row = {"path": path, **shape, "qps": rep["qps"], "p50_us": rep["p50_us"], "p99_us": rep["p99_us"],
               "completed": rep["completed"], "errors": rep["errors"], "answers_match": same}
        if launches is not None:
            row["launches_per_query"] = round(launches / max(1, rep["completed"]), 4)
        print(json.dumps(row), flush=True)

    for size in [int(x) for x in a.sizes.split(",")]:
        for kind in ("contiguous", "random"):
            if kind == "contiguous":
                starts = rng.integers(0, a.n - size, size=nq)
                cands = [np.arange(s, s + size, dtype=np.uint64) for s in starts]
            else:
                cands = [np.sort(rng.choice(a.n, size=size, replace=False)).astype(np.uint64) for _ in range(nq)]
            flat = np.concatenate(cands)
            offs = np.concatenate([[0], np.cumsum([size] * nq)]).astype(np.uint64)
            ref = ix.search_restricted_multi(q, p, flat, offs)   # warm-up + the answers every path must reproduce
            shape = {"candidates": size, "ids": kind, "k": k}
            reps = 3
            t0 = time.perf_counter()
            for _ in range(reps):
                bi, bs, bc = ix.search_restricted_multi(q, p, flat, offs)
            dt = (time.perf_counter() - t0) / reps
            print(json.dumps({"path": "batched hx_search_restricted_multi", **shape, "queries_per_call": nq,
                              "qps": round(nq / dt, 1), "call_ms": round(dt * 1e3, 3),
                              "answers_match": bool(bi.tolist() == ref[0].tolist() and bs.tobytes() == ref[1].tobytes())}),
                  flush=True)
            for mode, ncall, nthr in (("tasks", 1, 1), ("tasks", 16, 8), ("tasks", 256, 8), ("blocking", 256, 0)):
                l0 = svc.stats()["launches"]
                rep, ids, sc, cnt = callers.run_restricted(svc, ix, q, k, ncall, cand_ids=flat, cand_offsets=offs, mode=mode,
                                                           n_threads=nthr, seconds=a.seconds)
                one(f"service {mode}", {**shape, "callers": ncall, "threads": rep["threads"]}, rep, ids, sc, cnt, ref,
                    svc.stats()["launches"] - l0)
            for ncall in (1, 16, 256):
                rep, ids, sc, cnt = callers.run_restricted(None, ix, q, k, ncall, cand_ids=flat, cand_offsets=offs,
                                                           mode="direct", seconds=a.seconds)
                one("direct hx_search_restricted B=1", {**shape, "callers": ncall}, rep, ids, sc, cnt, ref)
    # device-resident sets (hx_candidates): 1 000 random ids per query, no ids cross PCIe per call
    size = 1000
    cands = [np.sort(rng.choice(a.n, size=size, replace=False)).astype(np.uint64) for _ in range(nq)]
    sets = [ix.cache_candidates(hx.RestrictedVectorCandidates(c)) for c in cands]
    ref = ix.search_restricted_sets(q, p, sets)
    shape = {"candidates": size, "ids": "device set", "k": k}
    for mode, ncall, nthr in (("tasks", 256, 8), ("blocking", 256, 0)):
        l0 = svc.stats()["launches"]
        rep, ids, sc, cnt = callers.run_restricted(svc, ix, q, k, ncall, sets=sets, mode=mode, n_threads=nthr,
                                                   seconds=a.seconds)
        one(f"service {mode}", {**shape, "callers": ncall, "threads": rep["threads"]}, rep, ids, sc, cnt, ref,
            svc.stats()["launches"] - l0)
    rep, ids, sc, cnt = callers.run_restricted(None, ix, q, k, 256, sets=sets, mode="direct", seconds=a.seconds)
    one("direct hx_search_restricted_sets B=1", {**shape, "callers": 256}, rep, ids, sc, cnt, ref)
    print(json.dumps({"service_stats": svc.stats()}), flush=True)
    svc.close()
    for s in sets:
        s.close()
    ix.close()


if __name__ == "__main__":
    main()
