#!/usr/bin/env python
"""Exact tensor-core search (hx_search_dense_exact, hx_search_dense_restricted_exact) against the plain entries it extends,
on the C4 shape: 1.25M x 768 rows of the bench's `embedding` recipe, generated on the device, cosine and Euclidean, k = 10.

Points: the whole corpus at B in {128, 1024, 4096}, and restricted sets of 1e5 and 1e6 random ids at the same B.  Per point,
the plain and the exact entry are called alternately on the same queries (host clock around each blocking call, median of
--reps pairs), and the exact call's answer is compared with the plain one on every certified query.  Printed per point:
both call times, the certified / rescanned shares, and the rescan's scan-kernel time (hx_last_kernel_ms after an exact call
that rescanned; 0 when nothing was).  The first line names the card and its power limit.  JSON lines go to stdout and
to --out.

--predict-cpu: no GPU.  Predicts the certified share from the nominee cut alone (the bucket tails can only lower it) on
the CPU margin study's corpus (scripts/dense_margin_cpu.py): per query, certified iff floor(k'-th approximate score) > the
k-th exact score, with floor = hxd_exact_floor restated in tests/test_dense_exact_reference.py."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

SEED = 0x0DB9ED1A   # bench.py's embedding recipe
N_CENTROIDS, SIGMA, KIND = 1024, 1.0, 32
K = 10


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired) as e:
        out = f"unavailable: {e}"
    return out


def predict_cpu(n, nq=256):
    sys.path[:0] = [str(ROOT / "scripts"), str(ROOT / "tests")]
    import dense_margin_cpu as dm
    from oracle import hxo
    from test_dense_exact_reference import exact_floor
    kp = min(max(4 * K, 64), 800)
    draw, _ = dm.corpus(n)
    rows, queries = draw(n), draw(nq)
    qb, xb = dm.bf16_round(queries).astype(np.float64), dm.bf16_round(rows).astype(np.float64)
    dot = queries @ rows.T                                   # f32 stands in for the reference's exact score here
    adot = qb @ xb.T
    xn, qn = (xb * xb).sum(1), (qb * qb).sum(1)
    for metric in ("cosine", "euclidean"):
        cert, gaps = 0, []
        for q in range(nq):
            if metric == "cosine":                               # unit rows: (1 - dot) / 2
                ex = 0.5 - 0.5 * dot[q].astype(np.float64)
                ap = 0.5 - 0.5 * adot[q] / np.sqrt(qn[q] * xn)
                floor = lambda L: exact_floor(hxo.COSINE, 768, L)
            else:
                ex = 2.0 - 2.0 * dot[q].astype(np.float64)
                ap = qn[q] + xn - 2.0 * adot[q]
                floor = lambda L: exact_floor(hxo.EUCLIDEAN, 768, L, float(np.float32(qn[q])), float(np.float32(xn.max())))
            sk = np.partition(ex, K - 1)[K - 1]
            L = np.partition(ap, kp - 1)[kp - 1]
            cert += bool(floor(L) > sk)
            gaps.append((L - sk, L - floor(L)))
        g = np.array(gaps)
        print(json.dumps({"predict_cpu": metric, "rows": n, "queries": nq, "k": K, "k_prime": kp,
                          "certified_share_nominee_cut": cert / nq, "gap_L_minus_Sk": {"min": float(g[:, 0].min()),
                          "median": float(np.median(g[:, 0]))}, "E_at_L": {"max": float(g[:, 1].max()),
                          "median": float(np.median(g[:, 1]))}}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_250_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--batches", default="128,1024,4096")
    ap.add_argument("--sets", default="100000,1000000")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--metrics", default="cosine,euclidean")
    ap.add_argument("--predict-cpu", type=int, default=0, metavar="ROWS", help="CPU prediction only, at ROWS rows")
    ap.add_argument("--out", default=str(ROOT / "scripts_out" / "dense_exact_sweep.json"))
    a = ap.parse_args()
    if a.predict_cpu:
        predict_cpu(a.predict_cpu)
        return
    import helix_db_b200 as hx
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    sink = open(a.out, "w")

    def emit(row):
        line = json.dumps(row)
        print(line, flush=True)
        sink.write(line + "\n")

    emit({"card": card(), "n": a.n, "dim": a.dim, "k": K})
    p = hx.SearchParams.strict(K)
    batches = [int(b) for b in a.batches.split(",")]
    for metric in a.metrics.split(","):
        gm = hx.Metric.Cosine if metric == "cosine" else hx.Metric.Euclidean
        ix = hx.VectorIndex(gm, hx.VectorIndexConfig("sweep", "embedding", a.dim), storage=1)
        ix.generate_vectors(0, a.n, SEED, N_CENTROIDS, SIGMA, KIND)
        ix.load_graph(0, np.array([0], np.uint64), [0, 0], [])
        ix.set_entry(0, 0)
        qall = ix.generate_queries(SEED, max(batches), first_query=60_000_000, n_centroids=N_CENTROIDS, sigma=SIGMA,
                                   kind=KIND)
        rng = np.random.default_rng(SEED)
        views = [("all", None)] + [(f"random-{s}", hx.RestrictedVectorCandidates(
            np.sort(rng.choice(a.n, size=min(s, a.n), replace=False)).astype(np.uint64))) for s in
            (int(x) for x in a.sets.split(","))]
        for name, cset in views:
            for B in batches:
                q = np.ascontiguousarray(qall[:B])
                if cset is None:
                    plain = lambda: ix.search_dense_batch(q, p)
                    exact = lambda: ix.search_dense_exact_batch(q, p)
                else:
                    plain = lambda: ix.search_dense_restricted_batch(q, p, cset)
                    exact = lambda: ix.search_dense_restricted_exact_batch(q, p, cset)
                plain(), exact()   # warm-up: scratch buffers, tensor maps, the bf16 copy
                tp, te, rescan_ms = [], [], []
                for _ in range(a.reps):
                    t0 = time.perf_counter()
                    pr = plain()
                    t1 = time.perf_counter()
                    er = exact()
                    t2 = time.perf_counter()
                    tp.append(t1 - t0)
                    te.append(t2 - t1)
                    how = er[3]
                    rescan_ms.append(ix.last_kernel_ms()[0] if (how == 1).any() else 0.0)
                c0 = np.flatnonzero(how == 0)
                same = bool(er[2][c0].tolist() == pr[2][c0].tolist() and all(
                    er[0][b, :er[2][b]].tolist() == pr[0][b, :pr[2][b]].tolist() and
                    er[1][b, :er[2][b]].tobytes() == pr[1][b, :pr[2][b]].tobytes() for b in c0))
                emit({"metric": metric, "view": name, "B": B, "plain_ms": round(1e3 * float(np.median(tp)), 3),
                      "exact_ms": round(1e3 * float(np.median(te)), 3),
                      "certified_share": round(float((how == 0).mean()), 5),
                      "rescanned_share": round(float((how == 1).mean()), 5), "exact_scan_share": float((how == 2).mean()),
                      "rescan_kernel_ms": round(float(np.median(rescan_ms)), 4), "certified_equal_plain": same})
        ix.close()
    sink.close()


if __name__ == "__main__":
    main()
