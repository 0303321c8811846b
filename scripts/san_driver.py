#!/usr/bin/env python
"""Small end-to-end exercise of every kernel family for compute-sanitizer (memcheck / racecheck / synccheck).
  compute-sanitizer --tool memcheck  python scripts/san_driver.py
  compute-sanitizer --tool racecheck python scripts/san_driver.py
Sizes are tiny on purpose: the tools slow kernels down 10-100x."""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import helix_db_b200 as hx  # noqa: E402

which = set(sys.argv[1:]) or {"build", "ring", "cta", "policy", "scan", "dense", "service", "seq", "mirror"}
rng = np.random.default_rng(1)
n, dim = 1500, 64
rows = rng.standard_normal((n, dim)).astype(np.float32)
ids = np.arange(n, dtype=np.uint64)
ix = hx.VectorIndex(hx.Metric.Cosine, hx.VectorIndexConfig("san", "embedding", dim).with_m(8).with_m0(16).with_ef_construction(40),
                    storage=1)
ix.load_vectors(ids, rows)
if "seq" in which:
    small = hx.VectorIndex(hx.Metric.Euclidean, hx.VectorIndexConfig("s", "embedding", dim).with_m(8).with_m0(16).with_ef_construction(40))
    small.load_vectors(ids[:300], rows[:300])
    small.build(seed=3, sequential=True)
    print("sequential build ok", small.graph_info())
    small.close()
ix.build(seed=7)                                             # k_build_* (batched)
print("build ok", ix.graph_info())
q = rng.standard_normal((400, dim)).astype(np.float32)
p = hx.SearchParams.strict(10, 40)
if "ring" in which:
    a = ix.search_batch(q, p)                                # k_hnsw_search_ring (B >= #SMs), fused validation, pipelined? (B<1024: no)
    print("ring ok", int(a[2].sum()))
if "cta" in which:
    a = ix.search_batch(q[:20], p)                           # k_hnsw_search_cta_ring
    b = ix.search_batch(q[:1], p)
    print("cta ok", int(a[2].sum()), int(b[2].sum()))
if "policy" in which:
    planes = rng.standard_normal((64, dim)).astype(np.float32)
    ix.set_simhash_planes(planes)
    ix.compute_simhash()                                     # k_simhash_project
    pn = hx.SearchParams.new(10).with_ef(40)
    a = ix.search_ex(q[:200], pn)                            # k_hnsw_search_policy (warp build)
    b = ix.search_ex(q[:4], pn)                              # ... CTA build
    print("policy ok", int(a[2].sum()), int(b[2].sum()))
if "scan" in which:
    cand = hx.RestrictedVectorCandidates(ids[::3].copy())
    a = ix.search_restricted_batch(q[:50], hx.SearchParams.strict(10), cand)      # k_scan_topk (fused)
    b = ix.search_restricted_batch(q[:10], hx.SearchParams.strict(40), cand)      # k_scan + k_select
    print("scan ok", int(a[2].sum()), int(b[2].sum()))
if "dense" in which:
    a = ix.search_dense_batch(q[:130], hx.SearchParams.strict(10))               # k_dense_scores (wgmma) + re-rank
    print("dense ok", int(a[2].sum()))
if "service" in which:
    with ix.service(10, 40, capacity=64, max_batch=16) as svc:
        t = [svc.submit(q[i]) for i in range(40)]
        done = 0
        while t:
            for x in list(t):
                if svc.poll(x) is not None:
                    t.remove(x)
                    done += 1
        print("service ok", done, svc.stats()["launches"])
if "mirror" in which:
    ix.upsert_vectors(np.arange(n, n + 10, dtype=np.uint64), rng.standard_normal((10, dim)).astype(np.float32))
    ix.set_levels(np.arange(n, n + 10, dtype=np.uint64), np.zeros(10, dtype=np.uint16))
    ix.upsert_neighbor_rows(0, np.array([n], np.uint64), np.array([0, 2], np.uint32), np.array([1, 2], np.uint64))
    ix.delete_vectors([5])
    a = ix.search_batch(q[:20], p)
    print("mirror ok", int(a[2].sum()))
ix.close()
print("done")
