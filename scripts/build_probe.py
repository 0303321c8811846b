"""On-GPU probe of the device HNSW build: time, degree statistics, recall@10 at ef=100 vs the exact scan."""
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

out = []
for n in [int(x) for x in (sys.argv[1:] or ["20000", "100000"])]:
    class A:
        pass
    a = A()
    a.metric, a.dim = "cosine", 768
    ix = hx.VectorIndex(hx.Metric.Cosine, hx.VectorIndexConfig("p", "embedding", 768))
    ix.generate_vectors(0, n, bench.SEED, bench.N_CENTROIDS, bench.SIGMA, bench.KIND)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ix.build(seed=bench.SEED)
    torch.cuda.synchronize()
    build_s = time.perf_counter() - t0
    gi = ix.graph_info()
    q = ix.generate_queries(bench.SEED, 256, n_centroids=bench.N_CENTROIDS, sigma=bench.SIGMA, kind=bench.KIND)
    truth = bench.exact_topk_device(hx, torch, ix, q, n, 0, 10)
    res = {"n": n, "build_s": round(build_s, 2), "max_layer": gi["max_layer"]}
    for ef in (50, 100, 200):
        st = hx.SearchStats()
        p = hx.SearchParams.strict(10, ef)
        p.collect_stats = True
        ids, sc, cnt = ix.search_batch(q, p, st)
        res[f"recall_ef{ef}"] = round(bench.recall_at_k(ids, truth), 4)
        res[f"dc_ef{ef}"] = round(st.distance_computations / 256, 1)
        res[f"exp_ef{ef}"] = round(st.expansion_steps / 256, 1)
    if n <= 200000:
        g = ix.download_graph()
        res["deg0_mean"] = round(float(g["deg0"].mean()), 2)
        res["deg0_min"] = int(g["deg0"].min())
        res["deg0_zero"] = int((g["deg0"] == 0).sum())
    print(json.dumps(res), flush=True)
    out.append(res)
    ix.close()
(ROOT / "scripts_out").mkdir(exist_ok=True)
(ROOT / "scripts_out" / "build_probe.json").write_text(json.dumps(out, indent=1))
