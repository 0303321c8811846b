#!/usr/bin/env python
"""A fixed, seeded matrix through every dense entry point and the exact-scan entries they share code with; one JSON
document of per-case digests.  Two builds of the library (HELIX_B200_LIB selects one) that compute the same thing give
the same document, so `diff` of two runs is an equivalence check of a host-code change.

Entries: hx_search_dense[_exact], hx_search_dense_restricted[_exact][_set], hx_search_dense_restricted_set_device,
hx_search_sharded[_device] with HX_SHARD_DENSE (one shard), hx_search_restricted[_multi], hx_search_restricted_sets.
Matrix: cosine and Euclidean; corpora below and above hx_dense_min_rows(k), with deleted rows; B = 1, 5, 129; k = 1, 10,
800; host ids, device sets and resident device sets.  Error cases: a NaN at B = 3 and at B = 20, a zero-norm query, k = 0
and 900, a dimension mismatch, storage 0, L1, an empty and an unpopulated index, a set of another index, and a
non-resident set passed to the stream-ordered entry.

Per case: the return code, hx_last_error_index, every hx_stats field, and (return code 0) a SHA-256 of the counts, the
first count ids and score bits of each query, and `how`.  Usage: dense_entry_digest.py --out FILE."""
import argparse
import ctypes as C
import hashlib
import json
import os
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import helix_db_b200 as hx  # noqa: E402

HX_SHARD_DENSE = 1
DIM = 96
L = hx.load_library()
u64p, u32p, fp, u8p = C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.POINTER(C.c_float), C.POINTER(C.c_uint8)


def ptr(a, t):
    return a.ctypes.data_as(t)


def params(k, qdim=0):
    return hx._Params(k, 0, 0, -1.0, 0, qdim)


def make_index(metric, n, storage=1, deleted=True, populate=True, seed=0):
    """n rows of DIM, ids 100.., entry = first id; every 7th id after the first deleted."""
    ix = hx.VectorIndex(metric, hx.VectorIndexConfig("digest", "embedding", DIM), storage=storage)
    if n == 0:
        return ix, np.zeros(0, np.uint64)
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((16, DIM)).astype(np.float32)
    rows = (centres[rng.integers(0, 16, n)] + 0.3 * rng.standard_normal((n, DIM))).astype(np.float32)
    ids = np.arange(100, 100 + n, dtype=np.uint64)
    ix.load_vectors(ids, rows)
    if populate:
        ix.load_graph(0, ids[:1], [0, 0], [])
        ix.set_entry(int(ids[0]), 0)
    if deleted:
        ix.delete_vectors(ids[7::7])
    return ix, ids


def queries(B, seed, bad=None):
    q = np.random.default_rng(1000 + seed).standard_normal((B, DIM)).astype(np.float32)
    if bad == "nan":
        q[B // 2, 5] = np.nan
    elif bad == "zero":
        q[B - 1] = 0.0
    return q


def digest(rc, B, k, ids, sc, cnt, how, st):
    rec = {"rc": int(rc), "err_index": int(L.hx_last_error_index())}
    if st is not None:
        rec["stats"] = {f: int(getattr(st, f)) for f, _ in hx.SearchStats._fields_}
    if rc == 0:
        h = hashlib.sha256()
        c = np.minimum(cnt.astype(np.int64), k)
        h.update(cnt.astype(np.uint32).tobytes())
        for b in range(B):
            h.update(ids[b, :c[b]].tobytes())
            h.update(sc[b, :c[b]].view(np.uint32).tobytes())
        if how is not None:
            h.update(how.tobytes())
        rec["digest"] = h.hexdigest()[:24]
    return rec


def outputs(B, k):
    return np.zeros((B, k), np.uint64), np.zeros((B, k), np.float32), np.zeros(B, np.uint32), np.full(B, 255, np.uint8)


def host_entry(name, ix, q, k, qdim=0, cand=None, dset=None, sets=None):
    B = len(q)
    ids, sc, cnt, how = outputs(B, k)
    st = hx.SearchStats()
    p = params(k, qdim)
    qp = ptr(q, fp)
    o = (ptr(ids, u64p), ptr(sc, fp), ptr(cnt, u32p))
    exact = "exact" in name
    if name in ("dense", "dense_exact"):
        fn = L.hx_search_dense_exact if exact else L.hx_search_dense
        rc = fn(ix.h, qp, B, C.byref(p), *o, *((ptr(how, u8p),) if exact else ()), C.byref(st))
    elif name in ("dense_restricted", "dense_restricted_exact"):
        fn = L.hx_search_dense_restricted_exact if exact else L.hx_search_dense_restricted
        rc = fn(ix.h, qp, B, C.byref(p), ptr(cand, u64p), cand.size, *o, *((ptr(how, u8p),) if exact else ()), C.byref(st))
    elif name in ("dense_restricted_set", "dense_restricted_exact_set"):
        fn = L.hx_search_dense_restricted_exact_set if exact else L.hx_search_dense_restricted_set
        rc = fn(ix.h, qp, B, C.byref(p), dset.h, *o, *((ptr(how, u8p),) if exact else ()), C.byref(st))
    elif name == "restricted":
        rc = L.hx_search_restricted(ix.h, qp, B, C.byref(p), ptr(cand, u64p), cand.size, *o, C.byref(st))
    elif name == "restricted_multi":
        allc = np.tile(cand, B)
        offs = np.arange(B + 1, dtype=np.uint64) * np.uint64(cand.size)
        rc = L.hx_search_restricted_multi(ix.h, qp, B, C.byref(p), ptr(allc, u64p), ptr(offs, u64p), *o, C.byref(st))
    elif name == "restricted_sets":
        arr = (C.c_void_p * len(sets))(*[s.h for s in sets])
        rc = L.hx_search_restricted_sets(ix.h, qp, B, C.byref(p), arr, len(sets), *o, C.byref(st))
    else:
        raise ValueError(name)
    return digest(rc, B, k, ids, sc, cnt, how if exact else None, st)


def device_entry(name, ix, q, k, torch, dset=None, group=None, qdim=0):
    B = len(q)
    dq = torch.from_numpy(np.ascontiguousarray(q)).cuda()
    di = torch.zeros((B, k), dtype=torch.int64, device="cuda")
    dsc = torch.zeros((B, k), dtype=torch.float32, device="cuda")
    dc = torch.zeros(B, dtype=torch.int32, device="cuda")
    dh = torch.full((B,), 255, dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    p = params(k, qdim)
    with torch.cuda.stream(s):
        if name == "dense_restricted_set_device":
            rc = L.hx_search_dense_restricted_set_device(ix.h, dq.data_ptr(), B, C.byref(p), dset.h, di.data_ptr(),
                                                         dsc.data_ptr(), dc.data_ptr(), dh.data_ptr(), s.cuda_stream)
        else:
            rc = L.hx_search_sharded_device(group.h, HX_SHARD_DENSE, dq.data_ptr(), B, C.byref(p), k, di.data_ptr(),
                                            dsc.data_ptr(), dc.data_ptr(), s.cuda_stream)
    s.synchronize()
    how = dh.cpu().numpy() if name == "dense_restricted_set_device" else None
    return digest(rc, B, k, di.cpu().numpy().view(np.uint64), dsc.cpu().numpy(), dc.cpu().numpy().view(np.uint32), how,
                  None)


def sharded_host(group, q, k, qdim=0):
    B = len(q)
    ids, sc, cnt, _ = outputs(B, k)
    p = params(k, qdim)
    rc = L.hx_search_sharded(group.h, HX_SHARD_DENSE, ptr(q, fp), B, C.byref(p), k, ptr(ids, u64p), ptr(sc, fp),
                             ptr(cnt, u32p))
    return digest(rc, B, k, ids, sc, cnt, None, None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    import torch
    from helix_db_b200.sharding import ShardGroup
    out = {"lib": os.environ.get("HELIX_B200_LIB", "default"), "cases": {}}
    cases = out["cases"]
    metrics = {"cos": hx.Metric.Cosine, "euc": hx.Metric.Euclidean}
    for mname, metric in metrics.items():
        for cname, n in (("small", 400), ("large", 8000)):
            ix, ids = make_index(metric, n, seed=n)
            group = ShardGroup(ix, 1, 0, None)
            half = ids[::2].copy()
            set_ids = {"all": ids, "half": half}
            dsets = {}
            for sname, cand in set_ids.items():
                dsets[sname] = ix.cache_candidates(hx.RestrictedVectorCandidates(cand))
                dsets[sname + "_res"] = ix.cache_candidates(hx.RestrictedVectorCandidates(cand)).make_resident()
            for B in (1, 5, 129):
                for k in (1, 10, 800):
                    q = queries(B, B * 1000 + k)
                    tag = f"{mname}/{cname}/B{B}/k{k}"
                    for e in ("dense", "dense_exact"):
                        cases[f"{tag}/{e}"] = host_entry(e, ix, q, k)
                    cases[f"{tag}/sharded"] = sharded_host(group, q, k)
                    cases[f"{tag}/sharded_device"] = device_entry("sharded_device", ix, q, k, torch, group=group)
                    for sname, cand in set_ids.items():
                        for e in ("dense_restricted", "dense_restricted_exact", "restricted", "restricted_multi"):
                            cases[f"{tag}/{sname}/{e}"] = host_entry(e, ix, q, k, cand=cand)
                        for suffix in ("", "_res"):
                            ds = dsets[sname + suffix]
                            for e in ("dense_restricted_set", "dense_restricted_exact_set"):
                                cases[f"{tag}/{sname}{suffix}/{e}"] = host_entry(e, ix, q, k, dset=ds)
                            cases[f"{tag}/{sname}{suffix}/restricted_sets"] = host_entry("restricted_sets", ix, q, k,
                                                                                          sets=[ds])
                        cases[f"{tag}/{sname}_res/dense_restricted_set_device"] = device_entry(
                            "dense_restricted_set_device", ix, q, k, torch, dset=dsets[sname + "_res"])
            # error cases on this corpus
            for B in (3, 20):
                bads = ("nan", "zero") if mname == "cos" else ("nan",)
                for bad in bads:
                    q = queries(B, 7, bad)
                    tag = f"{mname}/{cname}/err_{bad}_B{B}"
                    for e in ("dense", "dense_exact"):
                        cases[f"{tag}/{e}"] = host_entry(e, ix, q, 10)
                    cases[f"{tag}/sharded"] = sharded_host(group, q, 10)
                    for e in ("dense_restricted", "dense_restricted_exact", "restricted"):
                        cases[f"{tag}/{e}"] = host_entry(e, ix, q, 10, cand=ids)
                    for e in ("dense_restricted_set", "dense_restricted_exact_set"):
                        cases[f"{tag}/{e}"] = host_entry(e, ix, q, 10, dset=dsets["all"])
                        cases[f"{tag}/{e}_res"] = host_entry(e, ix, q, 10, dset=dsets["all_res"])
                    cases[f"{tag}/restricted_sets"] = host_entry("restricted_sets", ix, q, 10, sets=[dsets["all"]])
            q = queries(5, 11)
            for k in (0, 900):
                tag = f"{mname}/{cname}/err_k{k}"
                for e in ("dense", "dense_exact"):
                    cases[f"{tag}/{e}"] = host_entry(e, ix, q, k)
                for e in ("dense_restricted", "dense_restricted_exact", "restricted"):
                    cases[f"{tag}/{e}"] = host_entry(e, ix, q, k, cand=ids)
                for e in ("dense_restricted_set", "dense_restricted_exact_set"):
                    cases[f"{tag}/{e}"] = host_entry(e, ix, q, k, dset=dsets["all_res"])
                cases[f"{tag}/dense_restricted_set_device"] = device_entry("dense_restricted_set_device", ix, q, k, torch,
                                                                           dset=dsets["all_res"])
            tag = f"{mname}/{cname}/err_dim"
            for e in ("dense", "dense_exact"):
                cases[f"{tag}/{e}"] = host_entry(e, ix, q, 10, qdim=DIM + 1)
            for e in ("dense_restricted", "dense_restricted_exact"):
                cases[f"{tag}/{e}"] = host_entry(e, ix, q, 10, qdim=DIM + 1, cand=ids)
            cases[f"{tag}/dense_restricted_set"] = host_entry("dense_restricted_set", ix, q, 10, qdim=DIM + 1,
                                                              dset=dsets["all"])
            cases[f"{tag}/dense_restricted_set_device"] = device_entry("dense_restricted_set_device", ix, q, 10, torch,
                                                                       dset=dsets["all_res"], qdim=DIM + 1)
            # a set of another index, and a non-resident set on the stream-ordered entry
            other, oids = make_index(metric, 600, seed=3)
            foreign = other.cache_candidates(hx.RestrictedVectorCandidates(oids))
            tag = f"{mname}/{cname}/err_set"
            for e in ("dense_restricted_set", "dense_restricted_exact_set"):
                cases[f"{tag}/foreign/{e}"] = host_entry(e, ix, q, 10, dset=foreign)
            cases[f"{tag}/foreign/restricted_sets"] = host_entry("restricted_sets", ix, q, 10, sets=[foreign])
            cases[f"{tag}/foreign/dense_restricted_set_device"] = device_entry("dense_restricted_set_device", ix, q, 10,
                                                                               torch, dset=foreign)
            cases[f"{tag}/not_resident/dense_restricted_set_device"] = device_entry("dense_restricted_set_device", ix, q,
                                                                                    10, torch, dset=dsets["all"])
            foreign.close()
            other.close()
            for d in dsets.values():
                d.close()
            group.close()
            ix.close()
        # index-level error cases: storage 0, empty, unpopulated; L1 once below
        q = queries(5, 13)
        for iname, (n, storage, populate) in {"storage0": (8000, 0, True), "empty": (0, 1, True),
                                              "unpopulated": (8000, 1, False)}.items():
            ix, ids = make_index(metric, n, storage=storage, populate=populate, seed=5)
            tag = f"{mname}/{iname}"
            for e in ("dense", "dense_exact"):
                cases[f"{tag}/{e}"] = host_entry(e, ix, q, 10)
                cases[f"{tag}/nan/{e}"] = host_entry(e, ix, queries(3, 9, "nan"), 10)
            cand = ids if n else np.arange(100, 200, dtype=np.uint64)
            for e in ("dense_restricted", "dense_restricted_exact", "restricted"):
                cases[f"{tag}/{e}"] = host_entry(e, ix, q, 10, cand=cand)
                cases[f"{tag}/nan/{e}"] = host_entry(e, ix, queries(3, 9, "nan"), 10, cand=cand)
            if n:
                ds = ix.cache_candidates(hx.RestrictedVectorCandidates(ids)).make_resident()
                for e in ("dense_restricted_set", "dense_restricted_exact_set"):
                    cases[f"{tag}/{e}"] = host_entry(e, ix, q, 10, dset=ds)
                cases[f"{tag}/dense_restricted_set_device"] = device_entry("dense_restricted_set_device", ix, q, 10, torch,
                                                                           dset=ds)
                ds.close()
            ix.close()
    l1, ids = make_index(hx.Metric.Manhattan, 600, seed=8)
    q = queries(5, 17)
    for e in ("dense", "dense_exact"):
        cases[f"l1/{e}"] = host_entry(e, l1, q, 10)
    for e in ("dense_restricted", "dense_restricted_exact", "restricted"):
        cases[f"l1/{e}"] = host_entry(e, l1, q, 10, cand=ids)
    ds = l1.cache_candidates(hx.RestrictedVectorCandidates(ids))
    for e in ("dense_restricted_set", "dense_restricted_exact_set"):
        cases[f"l1/{e}"] = host_entry(e, l1, q, 10, dset=ds)
    cases["l1/dense_restricted_set_device"] = device_entry("dense_restricted_set_device", l1, q, 10, torch, dset=ds)
    ds.close()
    l1.close()
    Path(args.out).parent.mkdir(parents=True, exist_ok=True)
    Path(args.out).write_text(json.dumps(out, indent=1, sort_keys=True) + "\n")
    print(f"{len(cases)} cases -> {args.out}")


if __name__ == "__main__":
    main()
