"""Diagnose device-build graph quality: per-query recall histogram, effect of the round size, comparison recipe."""
import json, os, sys, time
from pathlib import Path
import numpy as np
import torch
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import helix_db_b200 as hx
import bench

def per_query(ids, truth):
    return np.array([len(set(a.tolist()) & set(b.tolist())) for a, b in zip(ids, truth)])

def run(n, ncl, sigma, max_batch, nq=512, tag="", kind=0):
    if max_batch: os.environ["HX_BUILD_MAX_BATCH"] = str(max_batch)
    else: os.environ.pop("HX_BUILD_MAX_BATCH", None)
    ix = hx.VectorIndex(hx.Metric.Cosine, hx.VectorIndexConfig("p", "embedding", 768))
    ix.generate_vectors(0, n, bench.SEED, ncl, sigma, kind)
    t0 = time.perf_counter(); ix.build(seed=bench.SEED); torch.cuda.synchronize(); bs = time.perf_counter() - t0
    q = ix.generate_queries(bench.SEED, nq, n_centroids=ncl, sigma=sigma, kind=kind)
    truth = bench.exact_topk_device(hx, torch, ix, q, n, 0, 10)
    res = dict(tag=tag, n=n, ncl=ncl, sigma=sigma, kind=kind, max_batch=max_batch, build_s=round(bs, 2))
    for ef in (100, 200):
        st = hx.SearchStats(); p = hx.SearchParams.strict(10, ef); p.collect_stats = True
        ids, sc, cnt = ix.search_batch(q, p, st)
        pq = per_query(ids, truth)
        res[f"recall_ef{ef}"] = round(float(pq.mean()) / 10, 4)
        res[f"hist_ef{ef}"] = np.bincount(pq, minlength=11).tolist()
        res[f"dc_ef{ef}"] = round(st.distance_computations / nq, 1)
    g = ix.download_graph() if n <= 200000 else None
    if g is not None:
        res["deg0_mean"] = round(float(g["deg0"].mean()), 2); res["deg_lt8"] = round(float((g["deg0"] < 8).mean()), 4)
    print(json.dumps(res), flush=True)
    ix.close()
    return res

out = []
n = int(sys.argv[1]) if len(sys.argv) > 1 else 1000000
for kind, sigma in ((16, 0.5), (24, 0.5), (32, 0.5), (32, 1.0), (48, 0.7)):
    out.append(run(n, 1024, sigma, 0, tag=f"latent rank {kind} sigma {sigma}", kind=kind))
(ROOT / "scripts_out").mkdir(exist_ok=True)
(ROOT / "scripts_out" / "recall_diag_latent.json").write_text(json.dumps(out, indent=1))
