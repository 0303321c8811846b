#!/usr/bin/env python
"""Resident candidate sets (hx_candidates_make_resident) against the per-call gather and the exact scan, on the bench's
corpus (1M x 768 cosine, `embedding` recipe, generated on the device), k = 10.

Sets: contiguous 10k and 100k ids, a random 10 % of the ids, and every id.  B in {1, 8, 64, 256, 1024}.  Per (set, B), q/s
of five entries:
  * the exact scan (hx_search_restricted_sets);
  * the set entry through a non-resident set (hx_search_dense_restricted_set: compaction, gather, pass);
  * the set entry through a resident set;
  * the stream-ordered entry through the resident set (hx_search_dense_restricted_set_device), timed with CUDA events on a
    torch stream, B x calls / elapsed;
  * the exact entry through the resident set (hx_search_dense_restricted_exact_set).
Host-buffer entries are timed with the host clock around blocking calls.  For each tensor-core entry: recall@10 against the
exact scan, and whether every returned score is the exact scan's fp32 score bit for bit.  Per set: the one-time
make_resident cost, one profiled B = 64 call of each set entry split by kernel, the first resident call after a one-row
upsert against a steady call, and the smallest B at which each resident entry overtakes the exact scan.
The first line names the card and its power limit.  JSON lines go to stdout and to --out."""
import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))
import helix_db_b200 as hx  # noqa: E402
from dense_restricted_sweep import N_CENTROIDS, SEED, SIGMA, KIND, card, timed  # noqa: E402


def profile_kernels(torch, fn):
    """Device time per kernel of one call of fn (torch.profiler, CUDA activities), in microseconds."""
    import os
    import tempfile
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
    for e in ev:
        if e.get("cat") != "kernel":
            continue
        name = e["name"].split("(")[0].split("<")[0].replace("void ", "")
        if name == "k_to_bf16":   # the query tile has B / 8 blocks, the gather of the set's rows present / 8
            name = "k_to_bf16 (queries)" if e.get("args", {}).get("grid", [0])[0] <= 8 else "k_to_bf16 (set rows)"
        out[name] = round(out.get(name, 0.0) + float(e["dur"]), 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--batches", default="1,8,64,256,1024")
    ap.add_argument("--seconds", type=float, default=0.3, help="least timed time per entry point and shape")
    ap.add_argument("--max-reps", type=int, default=50)
    ap.add_argument("--out", default=str(ROOT / "scripts_out" / "dense_resident_sweep.json"))
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
    batches = [int(b) for b in a.batches.split(",")]
    qall = ix.generate_queries(SEED, max(batches), first_query=50_000_000, n_centroids=N_CENTROIDS, sigma=SIGMA, kind=KIND)
    rng = np.random.default_rng(SEED)
    sets = [("contiguous-10000", np.arange(1_100, 11_100, dtype=np.uint64)),
            ("contiguous-100000", np.arange(11_100, 111_100, dtype=np.uint64)),
            ("random-10%", np.sort(rng.choice(a.n, size=a.n // 10, replace=False)).astype(np.uint64)),
            ("all", np.arange(a.n, dtype=np.uint64))]
    stream = torch.cuda.Stream()

    def call(fn):
        def run():
            r = fn()
            return r, ix.last_kernel_ms()[0]
        return run

    def device_entry(q, dset):
        """The stream-ordered entry: (qps from CUDA events over repeated calls, answer of the last call)."""
        B = len(q)
        dq = torch.from_numpy(q).cuda()
        di = torch.zeros((B, k), dtype=torch.int64, device="cuda")
        ds = torch.zeros((B, k), dtype=torch.float32, device="cuda")
        dc = torch.zeros(B, dtype=torch.int32, device="cuda")
        stream.wait_stream(torch.cuda.current_stream())

        def one():
            ix.search_dense_restricted_set_device(dq.data_ptr(), B, p, dset, di.data_ptr(), ds.data_ptr(), dc.data_ptr(),
                                                  None, stream.cuda_stream)
        with torch.cuda.stream(stream):
            one()   # warm-up
            stream.synchronize()
            reps, t0 = 0, time.perf_counter()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            while reps < a.max_reps and (time.perf_counter() - t0 < a.seconds or reps < 3):
                one()
                reps += 1
            e1.record(stream)
        stream.synchronize()
        ms = e0.elapsed_time(e1) / reps
        flags, status = ix.device_flags(stream.cuda_stream)
        assert status == hx.HX_OK, flags
        got = (di.cpu().numpy().view(np.uint64), ds.cpu().numpy(), dc.cpu().numpy().view(np.uint32))
        return B / (ms * 1e-3), ms, got

    for name, ids in sets:
        plain = ix.cache_candidates(hx.RestrictedVectorCandidates(ids))
        res = ix.cache_candidates(hx.RestrictedVectorCandidates(ids))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res.make_resident()
        emit({"set": name, "candidates": int(ids.size), "make_resident_ms": round((time.perf_counter() - t0) * 1e3, 3),
              "resident_bytes": res.resident_bytes})
        qps = {}
        for B in batches:
            q = np.ascontiguousarray(qall[:B])
            paths = {"exact hx_search_restricted_sets": call(lambda: ix.search_restricted_sets(q, p, plain)),
                     "set entry, not resident": call(lambda: ix.search_dense_restricted_sets(q, p, plain)),
                     "set entry, resident": call(lambda: ix.search_dense_restricted_sets(q, p, res)),
                     "exact set entry, resident": call(lambda: ix.search_dense_restricted_exact_sets(q, p, res)[:3])}
            out = {}
            for path, fn in paths.items():
                dt, out[path], kms = timed(fn, a.seconds, a.max_reps)
                qps[(path, B)] = B / dt
                emit({"set": name, "candidates": int(ids.size), "B": B, "path": path, "qps": round(B / dt, 1),
                      "call_ms": round(dt * 1e3, 3), "kernel_ms": round(kms, 4)})
            dq, dms, out["device entry, resident"] = device_entry(q, res)
            qps[("device entry, resident", B)] = dq
            emit({"set": name, "candidates": int(ids.size), "B": B, "path": "device entry, resident", "qps": round(dq, 1),
                  "call_ms": round(dms, 3), "timed_with": "cuda events"})
            ei, es, ec = out["exact hx_search_restricted_sets"]
            for path in ("set entry, not resident", "set entry, resident", "device entry, resident",
                         "exact set entry, resident"):
                di, ds, dc = out[path]
                hits = sum(len(set(di[b, :dc[b]].tolist()) & set(ei[b, :ec[b]].tolist())) for b in range(B))
                offs = np.concatenate([[0], np.cumsum(dc.astype(np.uint64))]).astype(np.uint64)
                flat = np.concatenate([np.sort(di[b, :dc[b]]) for b in range(B)]).astype(np.uint64)
                xi, xs, xc = ix.search_restricted_multi(q, p, flat, offs)
                exact_bits = bool(xc.tolist() == dc.tolist() and all(
                    xi[b, :xc[b]].tolist() == di[b, :dc[b]].tolist() and xs[b, :xc[b]].tobytes() == ds[b, :dc[b]].tobytes()
                    for b in range(B)))
                same = bool(dc.tolist() == out["set entry, not resident"][2].tolist() and all(
                    di[b, :dc[b]].tolist() == out["set entry, not resident"][0][b, :dc[b]].tolist() and
                    ds[b, :dc[b]].tobytes() == out["set entry, not resident"][1][b, :dc[b]].tobytes() for b in range(B)))
                emit({"set": name, "B": B, "path": path, "recall_at_10": round(hits / max(1, int(ec.sum())), 5),
                      "scores_are_exact_bits": exact_bits, "same_as_not_resident": same,
                      "same_as_exact_scan": bool(dc.tolist() == ec.tolist() and all(
                          di[b, :dc[b]].tolist() == ei[b, :ec[b]].tolist() for b in range(B)))})
        for path in ("set entry, resident", "device entry, resident", "exact set entry, resident", "set entry, not resident"):
            wins = [B for B in batches if qps[(path, B)] > qps[("exact hx_search_restricted_sets", B)]]
            emit({"set": name, "path": path, "overtakes_exact_scan_from_B": min(wins) if wins else None,
                  "faster_at_B": wins})
        q64 = np.ascontiguousarray(qall[:64])
        for label, dset in (("not resident", plain), ("resident", res)):
            emit({"set": name, "B": 64, "path": f"set entry, {label}", "device_us_by_kernel":
                  profile_kernels(torch, lambda: ix.search_dense_restricted_sets(q64, p, dset))})
        # the first resident call after a one-row upsert (a row of the set overwritten with a query) re-gathers the tile
        steady = timed(call(lambda: ix.search_dense_restricted_sets(q64, p, res)), a.seconds, a.max_reps)[0]
        ix.upsert_vectors(np.array([ids[ids.size // 2]], np.uint64), np.ascontiguousarray(qall[:1]))
        t0 = time.perf_counter()
        ix.search_dense_restricted_sets(q64, p, res)
        first = time.perf_counter() - t0
        emit({"set": name, "B": 64, "path": "set entry, resident", "first_call_after_upsert_ms": round(first * 1e3, 3),
              "steady_call_ms": round(steady * 1e3, 3)})
        plain.close()
        res.close()
    ix.close()
    sink.close()


if __name__ == "__main__":
    main()
