"""On-GPU A/B of the HNSW traversal builds and their knobs on the C2 corpus (1M x 768, embedding recipe).

One index build, then for every variant (launch knobs of hx_tuning, given as their HX_* environment names and re-read with VectorIndex.tune()): warm-up, timed launches
through hx_search_device, kernel time from the library's own CUDA events, algorithmic GB/s from the SearchStats counters,
and a bit-for-bit comparison of ids/scores with the first variant.  Not the bench — writes scripts_out/hnsw_sweep.json.

  python scripts/hnsw_sweep.py [--n 1000000] [--B 8192,16384] [--variants name=K:V,K:V;name2=...]
"""
import argparse
import json
import os
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
import helix_db_b200 as hx  # noqa: E402

KNOBS = ("HX_RING_WARPS", "HX_RING_R", "HX_VT_CAP_LOG2", "HX_L2_HINT", "HX_VT_POOL", "HX_LAT_WARPS", "HX_PHASE_PROF", "HX_LAT_SPEC",
         "HX_LAT_ADMIT", "HX_POL_WARPS", "HX_POL_MINR", "HX_POL_EARLY_SIM", "HX_POL_CTA", "HX_PREFETCH_BELOW", "HX_PIPELINE")
DEFAULT_VARIANTS = [
    ("ring16", {}),
    ("ring16_nohint", {"HX_L2_HINT": "0"}),
    ("ring16_vt12", {"HX_VT_CAP_LOG2": "12"}),
    ("ring12", {"HX_RING_WARPS": "12"}),
    ("ring14", {"HX_RING_WARPS": "14"}),
    ("ring12_R4", {"HX_RING_WARPS": "12", "HX_RING_R": "4"}),
    ("ring16_R3", {"HX_RING_R": "3"}),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--B", default="8192")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--metric", default="cosine")
    ap.add_argument("--variants", default="")
    ap.add_argument("--batch1", action="store_true", help="also time one-query calls for every variant")
    ap.add_argument("--policy", action="store_true", help="time the production-default mode (hx_search_ex) instead")
    ap.add_argument("--out", default="hnsw_sweep.json")
    a = ap.parse_args()
    variants = DEFAULT_VARIANTS
    if a.variants:
        variants = []
        for item in a.variants.split(";"):
            name, _, kv = item.partition("=")
            variants.append((name, dict(p.split(":") for p in kv.split(",") if p)))
    args = argparse.Namespace(metric=a.metric, dim=a.dim)
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream().cuda_stream
    ix, setup = bench.build_index(hx, args, 0, 0, a.n)
    out = {"setup": setup, "n": a.n, "dim": a.dim, "runs": []}
    peak, _ = bench.measured_peaks()
    k = 10
    if a.policy:
        planes = np.random.default_rng(42).standard_normal((64, a.dim)).astype(np.float32)
        ix.set_simhash_planes(planes)
        ix.compute_simhash()
        B = int(a.B.split(",")[0])
        qs = [ix.generate_queries(bench.SEED, B, first_query=s * B, n_centroids=bench.N_CENTROIDS, sigma=bench.SIGMA,
                                  kind=bench.KIND) for s in range(a.reps + 1)]
        ref = None
        for name, env in variants:
            for key in KNOBS:
                os.environ.pop(key, None)
            os.environ.update(env)
            ix.tune()   # the handle reads the environment at creation: re-read it (hx_index_set_tuning(NULL))
            p = hx.SearchParams.new(k)
            ids0, sc0, cnt0 = ix.search_ex(qs[0], p)
            got = (ids0.tobytes(), sc0.tobytes())
            same = True if ref is None else got == ref
            ref = ref or got
            kms = 0.0
            for s in range(a.reps):
                ix.search_ex(qs[1 + s], p)
                kms += ix.last_kernel_ms()[0]
            kms /= a.reps
            run = {"variant": name, "env": env, "B": B, "policy_kernel_ms": round(kms, 3), "kernel_qps": round(B / kms * 1e3, 1),
                   "same_bits_as_first": same}
            print(json.dumps(run), flush=True)
            out["runs"].append(run)
        (ROOT / "scripts_out").mkdir(exist_ok=True)
        (ROOT / "scripts_out" / a.out).write_text(json.dumps(out, indent=1))
        ix.close()
        return
    for B in [int(x) for x in a.B.split(",")]:
        qs = [ix.generate_queries(bench.SEED, B, first_query=s * B, n_centroids=bench.N_CENTROIDS, sigma=bench.SIGMA,
                                  kind=bench.KIND) for s in range(a.reps + 1)]
        dq = [torch.from_numpy(q).to(dev) for q in qs]
        o_ids = torch.zeros((B, k), dtype=torch.int64, device=dev)
        o_sc = torch.zeros((B, k), dtype=torch.float32, device=dev)
        o_cnt = torch.zeros((B,), dtype=torch.int32, device=dev)
        ref = None
        for name, env in variants:
            for key in KNOBS:
                os.environ.pop(key, None)
            os.environ.update(env)
            ix.tune()   # the handle reads the environment at creation: re-read it (hx_index_set_tuning(NULL))
            p = hx.SearchParams.strict(k, bench.EF)
            p.collect_stats = True
            st = hx.SearchStats()
            ix.search_device(dq[0].data_ptr(), B, p, o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr(), stream, st)
            torch.cuda.synchronize()
            got = (o_ids.cpu().numpy().tobytes(), o_sc.cpu().numpy().tobytes(), o_cnt.cpu().numpy().tobytes())
            same = True if ref is None else got == ref
            if ref is None:
                ref = got
            p.collect_stats = False
            ix.last_kernel_ms()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for s in range(a.reps):
                ix.search_device(dq[1 + s].data_ptr(), B, p, o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr(), stream)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / a.reps
            kms, kl = ix.last_kernel_ms()
            kms /= max(kl, 1)
            gbs = st.algorithmic_bytes / (kms * 1e-3) / 1e9
            run = {"variant": name, "env": env, "B": B, "step_ms": round(ms, 3), "kernel_ms": round(kms, 3),
                   "qps": round(B / ms * 1e3, 1), "alg_GBps": round(gbs, 1), "frac": round(gbs / peak, 4),
                   "same_bits_as_first": same, "dc_per_query": round(st.distance_computations / B, 1)}
            if a.batch1:
                nb = 100
                for i in range(10):
                    ix.search_device(dq[0][i:i + 1].data_ptr(), 1, p, o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr(), stream)
                torch.cuda.synchronize()
                e0.record()
                for i in range(nb):
                    ix.search_device(dq[0][i:i + 1].data_ptr(), 1, p, o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr(), stream)
                e1.record()
                torch.cuda.synchronize()
                run["batch1_us"] = round(e0.elapsed_time(e1) / nb * 1e3, 1)
                kms1, kl1 = ix.last_kernel_ms()
                run["batch1_kernel_us"] = round(kms1 / max(kl1, 1) * 1e3, 1)
                b1 = (o_ids[0].cpu().numpy().tobytes(), o_sc[0].cpu().numpy().tobytes())
                run["batch1_last_ids"] = o_ids[0].cpu().numpy().view(np.uint64).tolist()
            print(json.dumps(run), flush=True)
            out["runs"].append(run)
    (ROOT / "scripts_out").mkdir(exist_ok=True)
    (ROOT / "scripts_out" / a.out).write_text(json.dumps(out, indent=1))
    ix.close()


if __name__ == "__main__":
    main()
