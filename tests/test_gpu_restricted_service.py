"""search_restricted's calling pattern (one query and one candidate set per call, many concurrent callers:
read_index.rs:92-101) through the restricted query service.

Every answer must equal hx_search_restricted's for the same query, k and candidates, bit for bit (ids, order, score bits,
count), and the CPU oracle's search_restricted.
"""
import threading

import numpy as np
import pytest

import helix_db_b200 as hx
from oracle import hxo

pytestmark = pytest.mark.gpu

METRICS = [(hx.Metric.Euclidean, hxo.EUCLIDEAN, 64), (hx.Metric.Cosine, hxo.COSINE, 768),
           (hx.Metric.Manhattan, hxo.MANHATTAN, 40)]


def _corpus(gm, om, n, dim, gapped, seed=5):
    """n rows with ids 0..n-1 (contiguous-id mapping) or 10, 13, 16, ... (binary-search mapping); no graph but the entry."""
    rng = np.random.default_rng(seed)
    rows = rng.standard_normal((n, dim)).astype(np.float32)
    ids = (np.arange(n, dtype=np.uint64) * 3 + 10) if gapped else np.arange(n, dtype=np.uint64)
    ora = hxo.Index(om, dim)
    ora.put_vectors(ids, rows)
    ora.put_neighbors(0, int(ids[0]), [])
    ora.set_entry(int(ids[0]), 0)
    gpu = hx.VectorIndex(gm, hx.VectorIndexConfig("rs", "embedding", dim))
    gpu.load_vectors(ids, rows)
    gpu.load_graph(0, ids[:1], [0, 0], [])
    gpu.set_entry(int(ids[0]), 0)
    return gpu, ora, ids, rng


def _pairs(results):
    return [(r.entity_id(), np.float32(r.score()).tobytes()) for r in results]


def _rows(ids, sc, cnt):
    return list(zip(ids[:cnt].tolist(), [np.float32(x).tobytes() for x in sc[:cnt]]))


def _same_answers(gi, gs, gc, ei, es, ec):
    """Row by row up to each count: the entries past a count are whatever the caller's buffer held."""
    return gc.tolist() == ec.tolist() and all(_rows(gi[q], gs[q], gc[q]) == _rows(ei[q], es[q], ec[q]) for q in range(len(ec)))


def _cands(rng, ids, size):
    """`size` ascending unique ids: mostly present, some absent from the index (odd offsets / past the end)."""
    universe = int(ids[-1]) + 50
    return np.sort(rng.choice(np.arange(0, universe, dtype=np.uint64), size=size, replace=False))


@pytest.mark.parametrize("gm,om,dim", METRICS)
@pytest.mark.parametrize("gapped", [False, True])
def test_bit_exact_against_search_restricted_and_the_oracle(gm, om, dim, gapped):
    n = 70000
    gpu, ora, ids, rng = _corpus(gm, om, n, dim, gapped)
    victims = ids[rng.choice(n, size=40, replace=False)]
    gpu.delete_vectors(victims.tolist())
    vset = set(victims.tolist())
    queries = rng.standard_normal((2, dim)).astype(np.float32)
    for k in (1, 10, 32, 33, 100, 800):
        shapes = [1, k - 1, 256, 257, 5000, 60000]
        sets = []
        for size in shapes:
            c = _cands(rng, ids, size)
            c = np.unique(np.concatenate([c, victims[:3]])) if size >= 256 else c   # removed rows among the candidates
            sets.append(c)
        with gpu.restricted_service(k, capacity=64) as svc:
            pending = {}
            for si, c in enumerate(sets):
                for qi in range(len(queries)):
                    pending[svc.submit(queries[qi], hx.RestrictedVectorCandidates(c))] = (si, qi)
            got = {}
            while pending:
                for t in list(pending):
                    r = svc.poll(t)
                    if r is not None:
                        got[pending.pop(t)] = _pairs(r)
            st = svc.stats()
            assert st["submitted"] == st["completed"] == len(sets) * len(queries)
        for si, c in enumerate(sets):
            gi, gs, gc = gpu.search_restricted_batch(queries, hx.SearchParams.strict(k), hx.RestrictedVectorCandidates(c))
            for qi in range(len(queries)):
                assert got[(si, qi)] == _rows(gi[qi], gs[qi], gc[qi]), f"k={k} |C|={len(c)} q={qi}"
            live = np.array([x for x in c.tolist() if x not in vset], dtype=np.uint64)
            oi, os_ = ora.search_restricted(queries[0], k, live)
            assert got[(si, 0)] == list(zip(oi.tolist(), [np.float32(x).tobytes() for x in os_])), f"oracle k={k} |C|={len(c)}"
    gpu.close()


def test_concurrent_callers_lists_and_device_sets_mixed():
    gm, om, dim = hx.Metric.Euclidean, hxo.EUCLIDEAN, 64
    gpu, ora, ids, rng = _corpus(gm, om, 20000, dim, gapped=True)
    nq, k = 400, 10
    queries = rng.standard_normal((nq, dim)).astype(np.float32)
    sizes = rng.choice([1, 9, 100, 256, 257, 1000, 4000, 20000], size=nq)
    cands = [_cands(rng, ids, int(s)) for s in sizes]
    offs = np.concatenate([[0], np.cumsum([len(c) for c in cands])]).astype(np.uint64)
    ei, es, ec = gpu.search_restricted_multi(queries, hx.SearchParams.strict(k), np.concatenate(cands), offs)
    expect = [_rows(ei[q], es[q], ec[q]) for q in range(nq)]
    dsets = [gpu.cache_candidates(hx.RestrictedVectorCandidates(c)) for c in cands]
    allowed = [dsets[q] if q % 3 == 0 else hx.RestrictedVectorCandidates(cands[q]) for q in range(nq)]
    with gpu.restricted_service(k, capacity=256) as svc:
        got = [None] * nq
        errs = []

        def blocking(t):
            try:
                for q in range(t, nq // 2, 24):
                    got[q] = _pairs(svc.search(queries[q], allowed[q]))
            except Exception as e:   # pragma: no cover
                errs.append(e)

        def async_caller():
            try:
                pending, nxt = {}, nq // 2
                while nxt < nq or pending:
                    while nxt < nq and len(pending) < 200:
                        pending[svc.submit(queries[nxt], allowed[nxt])] = nxt
                        nxt += 1
                    for t in list(pending):
                        r = svc.poll(t)
                        if r is not None:
                            got[pending.pop(t)] = _pairs(r)
            except Exception as e:   # pragma: no cover
                errs.append(e)

        ths = [threading.Thread(target=blocking, args=(t,)) for t in range(24)] + [threading.Thread(target=async_caller)]
        [t.start() for t in ths]
        [t.join() for t in ths]
        assert not errs, errs
        for q in range(nq):
            assert got[q] == expect[q], f"query {q} (|C| = {len(cands[q])})"
        st = svc.stats()
        assert st["submitted"] == st["completed"] == nq and 1 <= st["launches"] <= nq
        # the C++ host harness (host/hx_callers.cpp): 64 concurrent callers, lists and device sets, both styles
        from helix_db_b200 import callers
        for mode, threads in (("blocking", 0), ("tasks", 4)):
            rep, ci, cs, cc = callers.run_restricted(svc, gpu, queries, k, 64, cand_ids=np.concatenate(cands),
                                                     cand_offsets=offs, mode=mode, n_threads=threads, seconds=0.2)
            assert rep["rc"] == 0 and rep["errors"] == 0 and rep["completed"] >= nq
            assert _same_answers(ci, cs, cc, ei, es, ec), mode
        rep, ci, cs, cc = callers.run_restricted(svc, gpu, queries, k, 64, sets=dsets, mode="blocking", seconds=0.2)
        assert rep["rc"] == 0 and rep["errors"] == 0
        assert _same_answers(ci, cs, cc, ei, es, ec)
        st = svc.stats()
        assert st["submitted"] == st["completed"]
    for d in dsets:
        d.close()
    gpu.close()


def test_admission_follows_search_restricted():
    gm, om, dim = hx.Metric.Cosine, hxo.COSINE, 32
    gpu, ora, ids, rng = _corpus(gm, om, 3000, dim, gapped=False)
    q = rng.standard_normal(dim).astype(np.float32)
    good = hx.RestrictedVectorCandidates(ids[:500])
    stale = gpu.cache_candidates(good)
    with gpu.restricted_service(10) as svc:
        expect = _pairs(gpu.search_restricted(q, hx.SearchParams.strict(10), good))
        assert _pairs(svc.search(q, good)) == expect
        assert svc.search(q, hx.RestrictedVectorCandidates(np.array([], np.uint64))) == []
        nan = q.copy()
        nan[0] = np.nan
        assert svc.search(nan, hx.RestrictedVectorCandidates(np.array([], np.uint64))) == []   # no validation when empty
        with pytest.raises(hx.HelixDbError) as e:
            svc.search(q, hx.RestrictedVectorCandidates(np.array([5, 3, 9], np.uint64)))
        assert e.value.variant == "VectorParameterError"
        with pytest.raises(hx.HelixDbError) as e:
            svc.search(q, hx.RestrictedVectorCandidates(np.arange(1_000_001, dtype=np.uint64)))
        assert e.value.variant == "Query"
        nan[7] = np.nan
        with pytest.raises(hx.HelixDbError) as e:   # a bad query fails alone, at submit
            svc.submit(nan, good)
        assert e.value.variant == "InvalidVectorComponent"
        assert _pairs(svc.search(q, good)) == expect
        t = svc.submit(q, good)
        assert _pairs(svc.wait(t)) == expect
        with pytest.raises(hx.HelixDbError):        # a consumed ticket is refused
            svc.poll(t)
        with pytest.raises(hx.HelixDbError) as e:   # kind mismatch: the HNSW submit on a restricted service
            lib = hx.load_library()
            tk = hx.C.c_uint64()
            hx._ck(lib.hx_service_submit(svc.h, q.ctypes.data_as(hx.C.POINTER(hx.C.c_float)), hx.C.byref(tk)))
        assert e.value.variant == "VectorParameterError"
        assert svc.stats()["submitted"] == svc.stats()["completed"]
        # a set made before the vectors were reloaded belongs to an older image
        gpu.load_vectors(ids, gpu.download_vectors(0, len(ids))[1])
        gpu.load_graph(0, ids[:1], [0, 0], [])
        gpu.set_entry(int(ids[0]), 0)
        with pytest.raises(hx.HelixDbError) as e:
            svc.search(q, stale)
        assert e.value.variant == "InvariantViolation"
    # kind mismatch the other way: a restricted submit on an HNSW service
    from test_gpu_parity import build_pair
    rows = rng.standard_normal((500, dim)).astype(np.float32)
    hg, _ = build_pair(gm, om, rows, m=8, m0=16, efc=40)
    with hg.service(10) as hs:
        ids_ = np.ascontiguousarray(good.ids)
        tk = hx.C.c_uint64()
        rc = hx.load_library().hx_service_submit_restricted(hs.h, q.ctypes.data_as(hx.C.POINTER(hx.C.c_float)),
                                                            ids_.ctypes.data_as(hx.C.POINTER(hx.C.c_uint64)), ids_.size,
                                                            hx.C.byref(tk))
        assert rc == hx.HX_ERR_INVALID_PARAMETER
        assert hs.stats()["submitted"] == 0
    stale.close()
    hg.close()
    gpu.close()


def test_arena_pressure_completes():
    """arena_ids = 1e6 and 8 threads submitting 300 000-id sets: a full arena is back-pressure, never a hang."""
    gm, om, dim = hx.Metric.Euclidean, hxo.EUCLIDEAN, 32
    gpu, ora, ids, rng = _corpus(gm, om, 400000, dim, gapped=False)
    k = 10
    queries = rng.standard_normal((8, dim)).astype(np.float32)
    sets = [np.sort(rng.choice(ids, size=300000, replace=False)) for _ in range(8)]
    expect = []
    for t in range(8):
        gi, gs, gc = gpu.search_restricted_batch(queries[t:t + 1], hx.SearchParams.strict(k), hx.RestrictedVectorCandidates(sets[t]))
        expect.append(_rows(gi[0], gs[0], gc[0]))
    errs, bad = [], []
    with gpu.restricted_service(k, arena_ids=1_000_000) as svc:
        def worker(t):
            try:
                for _ in range(4):
                    if _pairs(svc.search(queries[t], hx.RestrictedVectorCandidates(sets[t]))) != expect[t]:
                        bad.append(t)
            except Exception as e:   # pragma: no cover
                errs.append(e)

        ths = [threading.Thread(target=worker, args=(t,)) for t in range(8)]
        [t.start() for t in ths]
        [t.join(timeout=300) for t in ths]
        assert not any(t.is_alive() for t in ths), "a submitter is stuck"
        assert not errs and not bad, (errs, bad)
        st = svc.stats()
        assert st["submitted"] == st["completed"] == 32
    gpu.close()


@pytest.mark.parametrize("arena_ids,sizes", [(1_000_000, (1, 1_000_000)), (1_000_000, (500_000, 600_000)),
                                             (1_500_000, (700_000, 900_000))])
def test_a_set_that_skips_the_arena_end_is_not_stuck(arena_ids, sizes):
    """A set that does not fit before the arena end starts the next lap.  Once everything before it is released the whole
    arena is free, even when the set is larger than both the space left before the end and the space freed at the start."""
    gm, om, dim = hx.Metric.Euclidean, hxo.EUCLIDEAN, 32
    gpu, ora, ids, rng = _corpus(gm, om, 20000, dim, gapped=True)
    q = rng.standard_normal((len(sizes), dim)).astype(np.float32)
    sets = [np.arange(7, 7 + s, dtype=np.uint64) for s in sizes]   # present and absent ids mixed
    expect = []
    for i, c in enumerate(sets):
        gi, gs, gc = gpu.search_restricted_batch(q[i:i + 1], hx.SearchParams.strict(10), hx.RestrictedVectorCandidates(c))
        expect.append(_rows(gi[0], gs[0], gc[0]))
    svc = gpu.restricted_service(10, arena_ids=arena_ids)
    got, errs = [], []

    def caller():   # one blocking caller, one set after the other
        try:
            for _ in range(2):
                for i, c in enumerate(sets):
                    got.append(_pairs(svc.search(q[i], hx.RestrictedVectorCandidates(c))))
        except Exception as e:   # pragma: no cover
            errs.append(e)

    th = threading.Thread(target=caller, daemon=True)
    th.start()
    th.join(timeout=120)
    if th.is_alive():   # pragma: no cover  (the service is left open: closing it under a stuck submitter is unsafe)
        pytest.fail(f"a {sizes} sequence with arena_ids = {arena_ids} never completed")
    assert not errs, errs
    assert got == expect * 2
    assert svc.stats()["submitted"] == svc.stats()["completed"] == 2 * len(sets)
    svc.close()
    gpu.close()


def test_staged_queries_and_ids_across_arena_laps():
    """HX_SERVICE_STAGE_QUERIES: queries, cosine headers and candidate ids are copied to the device before the launch.  A
    dimension that is not a multiple of 32, and 64 concurrent callers whose ~30 000-id sets go round a 1e6-id arena many
    times, so that coalesced runs span the arena end (their ids are copied in two pieces)."""
    gm, om, dim = hx.Metric.Cosine, hxo.COSINE, 48
    gpu, ora, ids, rng = _corpus(gm, om, 100000, dim, gapped=False)
    nq, k = 256, 10
    queries = rng.standard_normal((nq, dim)).astype(np.float32)
    cands = [np.sort(rng.choice(120000, size=int(s), replace=False)).astype(np.uint64)
             for s in rng.integers(20000, 40000, size=nq)]
    offs = np.concatenate([[0], np.cumsum([len(c) for c in cands])]).astype(np.uint64)
    ei, es, ec = gpu.search_restricted_multi(queries, hx.SearchParams.strict(k), np.concatenate(cands), offs)
    from helix_db_b200 import callers
    with gpu.restricted_service(k, arena_ids=1_000_000, flags=2) as svc:   # 2 = HX_SERVICE_STAGE_QUERIES
        for q in range(0, nq, 37):
            assert _pairs(svc.search(queries[q], hx.RestrictedVectorCandidates(cands[q]))) == _rows(ei[q], es[q], ec[q])
        rep, ci, cs, cc = callers.run_restricted(svc, gpu, queries, k, 64, cand_ids=np.concatenate(cands), cand_offsets=offs,
                                                 mode="tasks", n_threads=4, seconds=0.5)
        assert rep["rc"] == 0 and rep["errors"] == 0 and rep["completed"] >= nq
        assert _same_answers(ci, cs, cc, ei, es, ec)
        st = svc.stats()
        assert st["submitted"] == st["completed"] and st["max_batch_seen"] > 1
    gpu.close()
