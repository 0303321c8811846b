#!/usr/bin/env python
"""Batched device build vs the sequential-equivalent build (HX_BUILD_SEQUENTIAL: one insert_hnsw at a time, the graph the
reference would build) on the same vectors, same level sequence: build time, degree statistics and recall@10 at ef 100 / 200
against the exact scan — on the bench's embedding recipe and on SURVEY §8d's recipe.

    python scripts/build_quality.py [rows]          # default 200 000 rows x 768 (the sequential build is ~0.1 ms per insert)
"""
import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import helix_db_b200 as hx  # noqa: E402
import bench  # noqa: E402


def per_query(ids, truth):
    return np.array([len(set(a.tolist()) & set(b.tolist())) for a, b in zip(ids, truth)])


def one(n, recipe, sequential, nq=512):
    kind, sigma = bench.RECIPES[recipe]["kind"], bench.RECIPES[recipe]["sigma"]
    ix = hx.VectorIndex(hx.Metric.Cosine, hx.VectorIndexConfig("q", "embedding", 768))
    ix.generate_vectors(0, n, bench.SEED, bench.N_CENTROIDS, sigma, kind)
    t0 = time.perf_counter()
    ix.build(seed=bench.SEED, sequential=sequential)
    torch.cuda.synchronize()
    secs = time.perf_counter() - t0
    q = ix.generate_queries(bench.SEED, nq, n_centroids=bench.N_CENTROIDS, sigma=sigma, kind=kind)
    truth = bench.exact_topk_device(hx, torch, ix, q, n, 0, 10)
    res = dict(rows=n, recipe=recipe, build="sequential (insert_hnsw order)" if sequential else "batched rounds", build_s=round(secs, 2))
    for ef in (100, 200):
        st = hx.SearchStats()
        p = hx.SearchParams.strict(10, ef)
        p.collect_stats = True
        ids, sc, cnt = ix.search_batch(q, p, st)
        res[f"recall_at_10_ef{ef}"] = round(float(per_query(ids, truth).mean()) / 10, 4)
        res[f"distance_computations_ef{ef}"] = round(st.distance_computations / nq, 1)
    g = ix.download_graph()
    res["layer0_degree_mean"] = round(float(g["deg0"].mean()), 2)
    res["layer0_degree_below_8"] = round(float((g["deg0"] < 8).mean()), 4)
    res["max_layer"] = int(g["max_layer"])
    ix.close()
    print(json.dumps(res), flush=True)
    return res


if __name__ == "__main__":
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 200_000
    out = [one(n, recipe, seq) for recipe in ("embedding", "survey") for seq in (False, True)]
    (ROOT / "scripts_out").mkdir(exist_ok=True)
    (ROOT / "scripts_out" / f"build_quality_{n}.json").write_text(json.dumps(out, indent=1))
