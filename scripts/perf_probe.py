"""Quick on-GPU probe (not the bench): scan GB/s and HNSW QPS at small/medium scale, written to scripts_out/ (git-ignored)."""
import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import helix_db_b200 as hx  # noqa: E402

out = {}
dev = torch.device("cuda:0")
stream = torch.cuda.current_stream().cuda_stream


def scan_probe(metric, n=1_000_000, dim=768, B=256, sel=100, reps=5):
    ix = hx.VectorIndex(metric, hx.VectorIndexConfig("p", "embedding", dim))
    t0 = time.time()
    ix.generate_vectors(0, n, 0x0DB9ED1A)
    ix.load_graph(0, np.array([0], np.uint64), np.array([0, 0], np.uint32), np.zeros(0, np.uint64))
    ix.set_entry(0, 0)
    gen_s = time.time() - t0
    q = ix.generate_queries(0x0DB9ED1A, B)
    dq = torch.from_numpy(q).to(dev)
    per = n // sel
    slots = np.concatenate([np.arange(b % sel, n, sel, dtype=np.uint32)[:per] for b in range(B)])
    offs = np.arange(0, (B + 1) * per, per, dtype=np.uint64)
    d_slots = torch.from_numpy(slots.view(np.int32)).to(dev)
    d_offs = torch.from_numpy(offs.view(np.int64)).to(dev)
    k = 10
    o_ids = torch.zeros((B, k), dtype=torch.int64, device=dev)
    o_sc = torch.zeros((B, k), dtype=torch.float32, device=dev)
    o_cnt = torch.zeros((B,), dtype=torch.int32, device=dev)
    p = hx.SearchParams.strict(k)
    for _ in range(2):
        ix.search_restricted_device(dq.data_ptr(), B, p, d_slots.data_ptr(), d_offs.data_ptr(), len(slots), per,
                                    o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr(), stream)
    torch.cuda.synchronize()
    ix.last_kernel_ms()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        ix.search_restricted_device(dq.data_ptr(), B, p, d_slots.data_ptr(), d_offs.data_ptr(), len(slots), per,
                                    o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr(), stream)
    e1.record()
    torch.cuda.synchronize()
    total_ms = e0.elapsed_time(e1) / reps
    kms, kl = ix.last_kernel_ms()
    bytes_ = len(slots) * dim * 4
    res = dict(metric=metric.name, n=n, dim=dim, B=B, cands_per_query=per, gen_s=round(gen_s, 2),
               step_ms=round(total_ms, 4), scan_kernel_ms=round(kms / max(kl, 1), 4),
               scan_GBps=round(bytes_ / (kms / max(kl, 1)) / 1e6, 1), qps=round(B / total_ms * 1e3, 1))
    # single query latency
    e0.record()
    for _ in range(20):
        ix.search_restricted_device(dq.data_ptr(), 1, p, d_slots.data_ptr(), 0, per, per,
                                    o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr(), stream)
    e1.record()
    torch.cuda.synchronize()
    res["single_query_us"] = round(e0.elapsed_time(e1) / 20 * 1e3, 1)
    ix.close()
    return res


def hnsw_probe(n=20000, dim=768, B=4096, reps=3):
    from oracle import hxo
    rng = np.random.default_rng(0)
    cent = rng.standard_normal((64, dim)).astype(np.float32)
    rows = cent[rng.integers(0, 64, n)] + 0.3 * rng.standard_normal((n, dim)).astype(np.float32)
    rows /= np.linalg.norm(rows, axis=1, keepdims=True)
    q = cent[rng.integers(0, 64, B)] + 0.3 * rng.standard_normal((B, dim)).astype(np.float32)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    q = q.astype(np.float32)
    ora = hxo.Index(hxo.COSINE, dim)
    ml = hxo.lib().hxo_default_ml_for_m(16)
    t0 = time.time()
    for i in range(n):
        ora.insert(i, rows[i], int(hxo.lib().hxo_select_layer_from_uniform(ml, float(rng.random(dtype=np.float32)))))
    build_s = time.time() - t0
    ix = hx.VectorIndex(hx.Metric.Cosine, hx.VectorIndexConfig("h", "embedding", dim))
    sys.path.insert(0, str(Path(__file__).resolve().parent.parent / 'tests'))
    from hx_testutil import mirror_from_oracle
    mirror_from_oracle(ix, ora)
    p = hx.SearchParams.strict(10)
    dq = torch.from_numpy(q).to(dev)
    o_ids = torch.zeros((B, 10), dtype=torch.int64, device=dev)
    o_sc = torch.zeros((B, 10), dtype=torch.float32, device=dev)
    o_cnt = torch.zeros((B,), dtype=torch.int32, device=dev)
    st = hx.SearchStats()
    p.collect_stats = True
    ix.search_device(dq.data_ptr(), B, p, o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr(), stream, st)
    p.collect_stats = False
    torch.cuda.synchronize()
    ix.last_kernel_ms()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        ix.search_device(dq.data_ptr(), B, p, o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr(), stream)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    kms, kl = ix.last_kernel_ms()
    res = dict(n=n, dim=dim, B=B, oracle_build_s=round(build_s, 1), step_ms=round(ms, 3), qps=round(B / ms * 1e3, 1),
               kernel_ms=round(kms / max(kl, 1), 3), stats=st.as_dict(),
               GBps=round(st.algorithmic_bytes / (kms / max(kl, 1)) / 1e6, 1))
    # batch-1 latency
    e0.record()
    for i in range(50):
        ix.search_device(dq[i:i + 1].data_ptr(), 1, p, o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr(), stream)
    e1.record()
    torch.cuda.synchronize()
    res["batch1_us"] = round(e0.elapsed_time(e1) / 50 * 1e3, 1)
    # CPU oracle for comparison
    oi, os_, oc, ost, secs = ora.search_batch(q[:512], 10, 0, threads=8)
    res["cpu_qps_8thr"] = round(512 / secs, 1)
    res["parity_first_512"] = bool(o_ids[:512].cpu().numpy().view(np.uint64).tolist() == oi.tolist())
    ix.close()
    return res


if __name__ == "__main__":
    Path(ROOT / "scripts_out").mkdir(exist_ok=True)
    which = sys.argv[1:] or ["scan", "hnsw"]
    if "scan" in which:
        for m in (hx.Metric.Euclidean, hx.Metric.Cosine):
            out[f"scan_{m.name}"] = scan_probe(m)
            print(json.dumps(out[f"scan_{m.name}"]), flush=True)
    if "hnsw" in which:
        out["hnsw"] = hnsw_probe()
        print(json.dumps(out["hnsw"]), flush=True)
    (ROOT / "scripts_out" / "perf_probe.json").write_text(json.dumps(out, indent=1))
