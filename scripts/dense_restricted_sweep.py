#!/usr/bin/env python
"""Prefiltered search with one candidate set shared by the B queries of a call: the tensor-core path
(hx_search_dense_restricted / _set) against the exact scan (hx_search_restricted / _sets), on the bench's corpus
(1M x 768 cosine, `embedding` recipe, generated on the device), k = 10.

Sets: the reference's contiguous prefilter shapes (1k / 10k / 100k ids), a random 10 % of the ids, and every id.
B in {1, 64, 256, 1024}.  Per (set, B): q/s of the four entry points (host clock around blocking calls), recall@10 of the
dense answer against the exact scan, whether every returned score is the exact scan's fp32 score bit for bit, and the
k_dense_scores time (hx_last_kernel_ms).  Per set, one profiled B = 64 call splits the device time by kernel: candidate
mapping + compaction, the gather of the set's rows into bf16 (k_to_bf16 over the set), and k_dense_scores.
The first line names the card and its power limit.  JSON lines go to stdout and to --out."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import helix_db_b200 as hx  # noqa: E402

SEED = 0x0DB9ED1A   # bench.py's embedding recipe
N_CENTROIDS, SIGMA, KIND = 1024, 1.0, 32


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired) as e:
        out = f"unavailable: {e}"
    return out


def timed(fn, min_s, max_reps):
    fn()   # warm-up: scratch buffers, tensor maps
    reps, t0 = 0, time.perf_counter()
    ms = []
    while True:
        out = fn()
        reps += 1
        ms.append(out[1])
        if time.perf_counter() - t0 >= min_s or reps >= max_reps:
            break
    return (time.perf_counter() - t0) / reps, out[0], float(np.median(ms))


def profile_kernels(torch, fn, present):
    """Device time per kernel of one call of fn (torch.profiler, CUDA activities), in microseconds."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    path = os.path.join(tempfile.mkdtemp(), "trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        ev = json.load(f)["traceEvents"]
    out = {}
    set_grid = (present + 7) // 8
    for e in ev:
        if e.get("cat") != "kernel":
            continue
        name = e["name"].split("(")[0].split("<")[0].replace("void ", "")
        if name == "k_to_bf16":
            name = "k_to_bf16 (set rows)" if e.get("args", {}).get("grid", [0])[0] == set_grid else "k_to_bf16 (queries)"
        out[name] = round(out.get(name, 0.0) + float(e["dur"]), 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--batches", default="1,64,256,1024")
    ap.add_argument("--seconds", type=float, default=0.3, help="least timed time per entry point and shape")
    ap.add_argument("--max-reps", type=int, default=50)
    ap.add_argument("--out", default=str(ROOT / "scripts_out" / "dense_restricted_sweep.json"))
    a = ap.parse_args()
    import torch
    torch.cuda.init()
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    sink = open(a.out, "w")

    def emit(row):
        line = json.dumps(row)
        print(line, flush=True)
        sink.write(line + "\n")

    emit({"card": card(), "n": a.n, "dim": a.dim, "metric": "cosine", "k": 10})
    ix = hx.VectorIndex(hx.Metric.Cosine, hx.VectorIndexConfig("sweep", "embedding", a.dim))
    ix.generate_vectors(0, a.n, SEED, N_CENTROIDS, SIGMA, KIND)
    ix.load_graph(0, np.array([0], np.uint64), [0, 0], [])
    ix.set_entry(0, 0)
    k = 10
    p = hx.SearchParams.strict(k)
    bmax = max(int(b) for b in a.batches.split(","))
    qall = ix.generate_queries(SEED, bmax, first_query=50_000_000, n_centroids=N_CENTROIDS, sigma=SIGMA, kind=KIND)
    rng = np.random.default_rng(SEED)
    sets = [("contiguous-1000", np.arange(100, 1_100, dtype=np.uint64)),
            ("contiguous-10000", np.arange(1_100, 11_100, dtype=np.uint64)),
            ("contiguous-100000", np.arange(11_100, 111_100, dtype=np.uint64)),
            ("random-10%", np.sort(rng.choice(a.n, size=a.n // 10, replace=False)).astype(np.uint64)),
            ("all", np.arange(a.n, dtype=np.uint64))]

    def call(fn):
        def run():
            r = fn()
            return r, ix.last_kernel_ms()[0]
        return run

    for name, ids in sets:
        cset = hx.RestrictedVectorCandidates(ids)
        dset = ix.cache_candidates(cset)
        for B in [int(b) for b in a.batches.split(",")]:
            q = np.ascontiguousarray(qall[:B])
            paths = {"exact hx_search_restricted": call(lambda: ix.search_restricted_batch(q, p, cset)),
                     "exact hx_search_restricted_sets": call(lambda: ix.search_restricted_sets(q, p, dset)),
                     "dense hx_search_dense_restricted": call(lambda: ix.search_dense_restricted_batch(q, p, cset)),
                     "dense hx_search_dense_restricted_set": call(lambda: ix.search_dense_restricted_sets(q, p, dset))}
            res = {}
            for path, fn in paths.items():
                dt, res[path], kms = timed(fn, a.seconds, a.max_reps)
                emit({"set": name, "candidates": int(ids.size), "B": B, "path": path, "qps": round(B / dt, 1),
                      "call_ms": round(dt * 1e3, 3), "kernel_ms": round(kms, 4)})
            ei, es, ec = res["exact hx_search_restricted"]
            for path in ("dense hx_search_dense_restricted", "dense hx_search_dense_restricted_set"):
                di, ds, dc = res[path]
                hits = sum(len(set(di[b, :dc[b]].tolist()) & set(ei[b, :ec[b]].tolist())) for b in range(B))
                # exact score bits of every returned id: the exact scan restricted to each query's own answer
                offs = np.concatenate([[0], np.cumsum(dc.astype(np.uint64))]).astype(np.uint64)
                flat = np.concatenate([np.sort(di[b, :dc[b]]) for b in range(B)]).astype(np.uint64)
                xi, xs, xc = ix.search_restricted_multi(q, p, flat, offs)
                exact_bits = bool(xc.tolist() == dc.tolist() and all(
                    xi[b, :xc[b]].tolist() == di[b, :dc[b]].tolist() and xs[b, :xc[b]].tobytes() == ds[b, :dc[b]].tobytes()
                    for b in range(B)))
                emit({"set": name, "B": B, "path": path, "recall_at_10": round(hits / max(1, int(ec.sum())), 5),
                      "scores_are_exact_bits": exact_bits, "counts_match": bool(dc.tolist() == ec.tolist())})
        q64 = np.ascontiguousarray(qall[:64])
        emit({"set": name, "B": 64, "path": "dense hx_search_dense_restricted", "device_us_by_kernel":
              profile_kernels(torch, lambda: ix.search_dense_restricted_batch(q64, p, cset), int(ids.size))})
        dset.close()
    ix.close()
    sink.close()


if __name__ == "__main__":
    main()
