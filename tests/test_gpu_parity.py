"""Parity tests proper: the CUDA path (through the C ABI) against the CPU oracle on identical inputs.

Bar: neighbour ids, ordering, scores AND the reference's SearchStats counters are compared bit for bit —
the octet kernel reproduces the reference's AVX+FMA accumulation order, so no tolerance is needed for
Euclidean / Cosine / Manhattan.  The independent f64 tolerance the reference states for its own kernels,
max(d*2^-23, 1e-5) relative (tests/production_support/vector/magnitude_regressions.rs:286-328), is checked too.
"""
import math
import struct

import numpy as np
import pytest

import helix_db_b200 as hx
from oracle import hxo
from hx_testutil import mirror_from_oracle

pytestmark = pytest.mark.gpu

METRICS = [(hx.Metric.Euclidean, hxo.EUCLIDEAN), (hx.Metric.Cosine, hxo.COSINE), (hx.Metric.Manhattan, hxo.MANHATTAN)]


def bits(x):
    return struct.unpack("<I", struct.pack("<f", float(x)))[0]


def levels_for(n, m, seed):
    rng = np.random.default_rng(seed)
    ml = hxo.lib().hxo_default_ml_for_m(m)
    return [int(hxo.lib().hxo_select_layer_from_uniform(ml, float(u))) for u in rng.random(n, dtype=np.float32)]


def build_pair(gm, om, rows, ids=None, m=16, m0=32, efc=200, seed=1):
    n, dim = rows.shape
    ids = np.arange(n, dtype=np.uint64) if ids is None else np.asarray(ids, dtype=np.uint64)
    ora = hxo.Index(om, dim, m=m, m0=m0, ef_construction=efc)
    for i, lv in zip(range(n), levels_for(n, m, seed)):
        ora.insert(int(ids[i]), rows[i], lv)
    gpu = hx.VectorIndex(gm, hx.VectorIndexConfig("t", "embedding", dim).with_m(m).with_m0(m0).with_ef_construction(efc))
    mirror_from_oracle(gpu, ora)
    return gpu, ora


def assert_same(gpu_ids, gpu_sc, gpu_cnt, ora_ids, ora_sc, what=""):
    assert int(gpu_cnt) == len(ora_ids), f"{what}: count {gpu_cnt} vs {len(ora_ids)}"
    assert gpu_ids[:gpu_cnt].tolist() == ora_ids.tolist(), f"{what}: ids differ"
    assert gpu_sc[:gpu_cnt].tobytes() == ora_sc.tobytes(), f"{what}: score bits differ"


# ---- SURVEY §8c item 1: phase-0 public result baseline through the C ABI ------------------------------------
def test_phase0_public_result_and_io_baseline():
    ora = hxo.Index(hxo.COSINE, 2, m=4, m0=8, ef_construction=16)
    for node_id, vec, layer in [(1, [1.0, 0.0], 0), (2, [0.0, 1.0], 1), (3, [-1.0, 0.0], 2), (4, [0.0, -1.0], 0)]:
        ora.insert(node_id, vec, layer)
    gpu = hx.VectorIndex(hx.Metric.Cosine, hx.VectorIndexConfig("phase0", "embedding", 2).with_m(4).with_m0(8)
                         .with_ef_construction(16))
    mirror_from_oracle(gpu, ora)
    params = hx.SearchParams.new(4).with_ef(16).with_simhash_mode(hx.SimHashMode.Off).with_pre_simhash_sampling_ratio(1.0)
    results, stats = gpu.search_with_stats([1.0, 0.0], params)
    plain = gpu.search([1.0, 0.0], params)
    assert [(r.entity_id(), bits(r.score())) for r in plain] == [(r.entity_id(), bits(r.score())) for r in results]
    assert [(r.entity_id(), bits(r.score())) for r in results] == [
        (1, bits(0.0)), (2, bits(0.5)), (4, bits(0.5)), (3, bits(1.0))]
    assert stats.expansion_steps == 4
    assert stats.neighbors_examined == 12
    assert stats.vectors_loaded == 3
    assert stats.distance_computations == 4


# ---- item 7: validation order + empty index -------------------------------------------------------------------
def test_validation_order_and_empty_index():
    gpu = hx.VectorIndex(hx.Metric.Cosine, hx.VectorIndexConfig("v", "embedding", 3))
    p = hx.SearchParams.strict(1)
    assert gpu.search([1.0, 0.0, 0.0], p) == []                       # empty index -> Ok([])
    gpu.load_vectors([100, 101], [[0.0, 1.0, 0.0], [1.0, 0.0, 0.0]])
    gpu.load_graph(1, [100, 101], [0, 2, 3], [99, 101, 100])           # 99 has no vector row
    gpu.load_graph(0, [100, 101], [0, 1, 2], [101, 100])
    gpu.set_entry(100, 1)
    bad = hx.SearchParams.strict(1)
    bad.query_dimension = 2
    with pytest.raises(hx.HelixDbError) as e:
        gpu._search_raw(np.array([[1.0, 0.0]], dtype=np.float32), bad)
    assert e.value.variant == "InvalidDimension"
    with pytest.raises(hx.HelixDbError) as e:
        gpu.search([1.0, float("nan"), 0.0], p)
    assert e.value.variant == "InvalidVectorComponent" and e.value.index == 1
    with pytest.raises(hx.HelixDbError) as e:
        gpu.search([0.0, 0.0, 0.0], p)
    assert e.value.variant == "ZeroNormCosineVector"
    with pytest.raises(hx.HelixDbError) as e:                          # the default (Adaptive) mode filters on SimHash rows:
        gpu.search([1.0, 0.0, 0.0], hx.SearchParams.new(1))           # without them the search is refused, not degraded
    assert e.value.variant == "InvalidVectorConfig"
    # greedy KAT (tests/production_support/vector/search.rs:231-291): from 100 on layer 1 the walk ends at 101
    r = gpu.search([1.0, 0.0, 0.0], p)
    assert [x.entity_id() for x in r] == [101] and bits(r[0].score()) == bits(0.0)
    # the same validation runs on the device for larger batches (B > 8)
    q = np.tile(np.array([[1.0, 0.0, 0.0]], dtype=np.float32), (20, 1))
    q[13, 2] = np.inf
    with pytest.raises(hx.HelixDbError) as e:
        gpu.search_batch(q, p)
    assert e.value.variant == "InvalidVectorComponent" and e.value.index == 2
    e_gpu = hx.VectorIndex(hx.Metric.Euclidean, hx.VectorIndexConfig("m", "embedding", 2))
    e_gpu.load_vectors([1], [[1.0, 2.0]])
    e_gpu.load_graph(0, [1], [0, 0], [])
    e_gpu.set_entry(1, 0)
    lim = hxo.component_limit(hxo.EUCLIDEAN, 2)
    over = float(np.nextafter(np.float32(lim), np.float32(np.inf)))
    with pytest.raises(hx.HelixDbError) as e:
        e_gpu.search([0.0, over], hx.SearchParams.strict(1))
    assert e.value.variant == "VectorComponentMagnitudeExceeded" and e.value.index == 1
    assert len(e_gpu.search([0.0, lim], hx.SearchParams.strict(1))) == 1
    with pytest.raises(hx.HelixDbError) as e:                          # rows are validated like decode_item_borrowed
        e_gpu.load_vectors([1, 2], [[1.0, 2.0], [float("nan"), 0.0]])
    assert e.value.variant == "InvalidVectorComponent"


# ---- item 5: tie stability ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("gm,om", METRICS)
def test_tie_stability(gm, om):
    ora = hxo.Index(om, 2, m=4, m0=8, ef_construction=16)
    for node_id in (2, 1, 3):
        ora.insert(node_id, [1.0, 0.0], 0)
    gpu = hx.VectorIndex(gm, hx.VectorIndexConfig("tie", "embedding", 2).with_m(4).with_m0(8).with_ef_construction(16))
    mirror_from_oracle(gpu, ora)
    r = gpu.search_restricted([1.0, 0.0], hx.SearchParams.strict(3), hx.RestrictedVectorCandidates.from_ids([3, 1, 2]))
    assert [x.entity_id() for x in r] == [1, 2, 3] and [float(x.score()) for x in r] == [0.0, 0.0, 0.0]
    r = gpu.search([1.0, 0.0], hx.SearchParams.strict(3, 16))
    assert [x.entity_id() for x in r] == [1, 2, 3]


# ---- item 6: circle fixtures (rows seeded directly, m=32/m0=64, cosine, ef=64) -----------------------------------------
def circle_pair(n):
    ora = hxo.Index(hxo.COSINE, 2, m=32, m0=64, ef_construction=200)
    ids = np.arange(1, n + 1, dtype=np.uint64)
    rows = np.stack([hxo.circle_vector(int(e), n) for e in ids])
    ora.put_vectors(ids, rows)
    offs, nb = [0], []
    for e in ids:
        r = hxo.skip_neighbors(int(e), n)
        ora.put_neighbors(0, int(e), r)
        nb.append(r)
        offs.append(offs[-1] + len(r))
    ora.set_entry(1, 0)
    gpu = hx.VectorIndex(hx.Metric.Cosine, hx.VectorIndexConfig("circle", "embedding", 2).with_m(32).with_m0(64))
    gpu.load_vectors(ids, rows)
    gpu.load_graph(0, ids, np.array(offs, dtype=np.uint32), np.concatenate(nb))
    gpu.set_entry(1, 0)
    return gpu, ora


@pytest.mark.parametrize("n,floor", [(24, 1.0), (10_000, 0.995)])
def test_circle_fixture(n, floor):
    gpu, ora = circle_pair(n)
    params = hx.SearchParams.strict(10, 64)
    params.collect_stats = True
    matched = 0
    for qi in range(24):
        e = 1 + qi * (n // 24)
        q = hxo.circle_vector(e, n)
        st = hx.SearchStats()
        ids, sc, cnt = gpu.search_batch(q.reshape(1, -1), params, st)
        oi, os_, ost = ora.search(q, 10, ef=64, with_stats=True)
        assert_same(ids[0], sc[0], cnt[0], oi, os_, f"circle n={n} q={qi}")          # exact ties at the beam edge included
        assert st.expansion_steps == ost["expansion_steps"]
        assert st.neighbors_examined == ost["neighbors_examined"]
        assert st.distance_computations == ost["distance_computations"]
        exact, _ = ora.search_exact(q, 10)
        matched += len(set(ids[0, :cnt[0]].tolist()) & set(exact.tolist()))
    assert matched / 240.0 >= floor


# ---- C1: xorshift 128-d fixture, reference-style build, three metrics, bit-exact batch parity + stats ------------------
@pytest.mark.parametrize("gm,om", METRICS)
def test_c1_xorshift_hnsw_parity(gm, om):
    n, dim, nq = 3000, 128, 64
    rows = hxo.xorshift_vectors(0, n, dim)
    queries = hxo.xorshift_vectors(n, nq, dim)
    gpu, ora = build_pair(gm, om, rows)
    params = hx.SearchParams.strict(10)
    ids, sc, cnt = gpu.search_batch(queries, params)
    recall = 0
    for q in range(nq):
        oi, os_ = ora.search(queries[q], 10)
        assert_same(ids[q], sc[q], cnt[q], oi, os_, f"{gm.name} q={q}")
        ex, _ = ora.search_exact(queries[q], 10)
        recall += len(set(oi.tolist()) & set(ex.tolist()))
    assert recall / (10.0 * nq) >= 0.95
    # per-query counters, one query per call
    params.collect_stats = True
    for q in range(8):
        st = hx.SearchStats()
        gpu.search_batch(queries[q:q + 1], params, st)
        _, _, ost = ora.search(queries[q], 10, with_stats=True)
        for f in ("expansion_steps", "neighbors_examined", "distance_computations", "vectors_loaded"):
            assert getattr(st, f) == ost[f], (f, q)
        assert st.algorithmic_bytes == st.expansion_steps * (5 + 8 * 32) + st.distance_computations * (4 + 4 * dim)


# ---- dimensions around the AVX cut-over (d < 32 scalar order; d % 32 != 0 tail), sparse ids, small ef ----------------
@pytest.mark.parametrize("dim", [3, 8, 31, 32, 33, 70, 100, 768])
@pytest.mark.parametrize("gm,om", METRICS[:2])
def test_dimension_sweep(dim, gm, om):
    n, nq = (600, 24) if dim < 768 else (400, 12)
    rng = np.random.default_rng(dim)
    rows = rng.standard_normal((n, dim)).astype(np.float32)
    ids = np.sort(rng.choice(10**12, size=n, replace=False).astype(np.uint64)) * 3 + 1     # sparse u64 ids
    queries = rng.standard_normal((nq, dim)).astype(np.float32)
    gpu, ora = build_pair(gm, om, rows, ids=ids, m=8, m0=16, efc=40)
    for ef, k in ((10, 10), (37, 5), (100, 10)):
        params = hx.SearchParams.strict(k, ef)
        gi, gs, gc = gpu.search_batch(queries, params)
        for q in range(nq):
            oi, os_ = ora.search(queries[q], k, ef=ef)
            assert_same(gi[q], gs[q], gc[q], oi, os_, f"dim={dim} ef={ef} q={q}")
    cand = ids[::3]
    gi, gs, gc = gpu.search_restricted_batch(queries, hx.SearchParams.strict(7), hx.RestrictedVectorCandidates.from_ids(cand))
    for q in range(nq):
        oi, os_ = ora.search_restricted(queries[q], 7, cand)
        assert_same(gi[q], gs[q], gc[q], oi, os_, f"restricted dim={dim} q={q}")


# ---- f64 tolerance of the device scores, as the reference states it for its own kernels ---------------------------------
def test_scores_within_reference_f64_tolerance():
    dim, n = 1536, 64
    rng = np.random.default_rng(5)
    for gm, om in METRICS:
        lim = hxo.component_limit(om, dim)
        scale = 1.0 if lim is None else min(float(lim), 1e3)
        rows = (rng.uniform(-1, 1, (n, dim)) * scale).astype(np.float32)
        q = (rng.uniform(-1, 1, dim) * scale).astype(np.float32)
        gpu = hx.VectorIndex(gm, hx.VectorIndexConfig("tol", "embedding", dim))
        gpu.load_vectors(np.arange(n, dtype=np.uint64), rows)
        gpu.load_graph(0, np.arange(n, dtype=np.uint64), np.zeros(n + 1, dtype=np.uint32), [])
        gpu.set_entry(0, 0)
        gi, gs, gc = gpu.search_restricted_batch(q.reshape(1, -1), hx.SearchParams.strict(n),
                                                 hx.RestrictedVectorCandidates.from_ids(np.arange(n)))
        r64, q64 = rows.astype(np.float64), q.astype(np.float64)
        if om == hxo.EUCLIDEAN:
            exact = ((r64 - q64) ** 2).sum(1)
        elif om == hxo.MANHATTAN:
            exact = np.abs(r64 - q64).sum(1)
        else:
            exact = (1.0 - (r64 @ q64) / (np.linalg.norm(r64, axis=1) * np.linalg.norm(q64))) / 2.0
        tol = max(dim * float(np.finfo(np.float32).eps), 1.0e-5)
        for j in range(int(gc[0])):
            e = exact[int(gi[0, j])]
            assert abs(float(gs[0, j]) - e) <= max(abs(e), 1.0) * tol


# ---- restricted exact scan: plan thresholds, clamps, errors, absent ids, per-query sets ---------------------------------------
@pytest.mark.parametrize("gm,om", METRICS)
def test_restricted_scan_edge_cases(gm, om):
    n, dim = 5000, 64
    rng = np.random.default_rng(11)
    rows = rng.standard_normal((n, dim)).astype(np.float32)
    ids = np.arange(10, 10 + 2 * n, 2, dtype=np.uint64)                 # even ids only: odd ids are absent
    ora = hxo.Index(om, dim)
    ora.put_vectors(ids, rows)
    ora.put_neighbors(0, int(ids[0]), [])
    ora.set_entry(int(ids[0]), 0)
    gpu = hx.VectorIndex(gm, hx.VectorIndexConfig("r", "embedding", dim))
    gpu.load_vectors(ids, rows)
    gpu.load_graph(0, ids[:1], [0, 0], [])
    gpu.set_entry(int(ids[0]), 0)
    queries = rng.standard_normal((9, dim)).astype(np.float32)
    for ncand, k in ((1, 10), (3, 10), (255, 10), (256, 10), (257, 10), (2000, 800), (5000, 1), (1500, 33)):
        cand = np.sort(rng.choice(np.arange(0, 10 + 2 * n + 50, dtype=np.uint64), size=ncand, replace=False))
        gi, gs, gc = gpu.search_restricted_batch(queries, hx.SearchParams.strict(k),
                                                 hx.RestrictedVectorCandidates.from_ids(cand))
        for q in range(len(queries)):
            oi, os_ = ora.search_restricted(queries[q], k, cand)
            assert_same(gi[q], gs[q], gc[q], oi, os_, f"|C|={ncand} k={k} q={q}")
            assert set(gi[q, :gc[q]].tolist()) <= set(cand.tolist())     # every result id is a candidate
    # empty candidate set -> Ok([]) ; k' = min(k,|C|) > 800 -> Query error
    assert gpu.search_restricted(queries[0], hx.SearchParams.strict(5), hx.RestrictedVectorCandidates.from_ids([])) == []
    with pytest.raises(hx.HelixDbError) as e:
        gpu.search_restricted(queries[0], hx.SearchParams.strict(801), hx.RestrictedVectorCandidates.from_ids(ids[:900]))
    assert e.value.variant == "Query"
    assert len(gpu.search_restricted(queries[0], hx.SearchParams.strict(801),
                                     hx.RestrictedVectorCandidates.from_ids(ids[:700]))) == 700
    # one candidate set per query
    offs, cands = [0], []
    for q in range(len(queries)):
        c = np.sort(rng.choice(ids, size=50 + 37 * q, replace=False))
        cands.append(c)
        offs.append(offs[-1] + len(c))
    gi, gs, gc = gpu.search_restricted_multi(queries, hx.SearchParams.strict(10), np.concatenate(cands), offs)
    for q in range(len(queries)):
        oi, os_ = ora.search_restricted(queries[q], 10, cands[q])
        assert_same(gi[q], gs[q], gc[q], oi, os_, f"multi q={q}")
    # the same sets resident on the device (uploaded and mapped once): identical answers, absent ids included
    with_absent = [np.sort(np.concatenate([c, np.array([1, 3, 10**9], dtype=np.uint64)])) for c in cands]
    dsets = [gpu.cache_candidates(hx.RestrictedVectorCandidates.from_ids(c)) for c in with_absent]
    assert len(dsets[0]) == len(with_absent[0])
    si, ss, scnt = gpu.search_restricted_sets(queries, hx.SearchParams.strict(10), dsets)
    assert si.tolist() == gi.tolist() and ss.tobytes() == gs.tobytes() and scnt.tolist() == gc.tolist()
    si, ss, scnt = gpu.search_restricted_sets(queries, hx.SearchParams.strict(10), dsets[3])     # one set for all queries
    for q in range(len(queries)):
        oi, os_ = ora.search_restricted(queries[q], 10, cands[3])
        assert_same(si[q], ss[q], scnt[q], oi, os_, f"shared device set q={q}")
    empty = gpu.cache_candidates(hx.RestrictedVectorCandidates.from_ids([]))
    assert gpu.search_restricted_sets(queries, hx.SearchParams.strict(10), empty)[2].tolist() == [0] * len(queries)
    big = gpu.cache_candidates(hx.RestrictedVectorCandidates.from_ids(ids[:900]))
    with pytest.raises(hx.HelixDbError) as e:
        gpu.search_restricted_sets(queries, hx.SearchParams.strict(801), big)
    assert e.value.variant == "Query"
    gpu.load_vectors(ids, rows)                                            # a reloaded image invalidates the sets
    gpu.load_graph(0, ids[:1], [0, 0], [])
    gpu.set_entry(int(ids[0]), 0)
    with pytest.raises(hx.HelixDbError) as e:
        gpu.search_restricted_sets(queries, hx.SearchParams.strict(10), dsets)
    assert e.value.variant == "InvariantViolation"


def test_restricted_full_million_candidate_bound():
    gpu = hx.VectorIndex(hx.Metric.Euclidean, hx.VectorIndexConfig("b", "embedding", 4))
    gpu.load_vectors([1, 2], [[0, 0, 0, 1], [0, 0, 1, 0]])
    gpu.load_graph(0, [1, 2], [0, 1, 2], [2, 1])
    gpu.set_entry(1, 0)
    big = np.arange(1_000_001, dtype=np.uint64)
    ids = np.zeros((1, 1), dtype=np.uint64)
    with pytest.raises(hx.HelixDbError) as e:
        gpu.search_restricted_batch(np.zeros((1, 4), np.float32) + 1, hx.SearchParams.strict(1),
                                    hx.RestrictedVectorCandidates(big))
    assert e.value.variant == "Query"
    gi, gs, gc = gpu.search_restricted_batch(np.array([[0, 0, 0, 1]], np.float32), hx.SearchParams.strict(2),
                                             hx.RestrictedVectorCandidates(big[:1_000_000]))
    assert gi[0, :gc[0]].tolist() == [1, 2] and gs[0, 0] == 0.0


# ---- persistent CTAs: more queries than CTAs, repeated launches across the stamp-epoch wrap ---------------------------
def test_many_queries_and_epoch_wrap():
    n, dim = 1500, 32
    rng = np.random.default_rng(3)
    rows = rng.standard_normal((n, dim)).astype(np.float32)
    gpu, ora = build_pair(hx.Metric.Euclidean, hxo.EUCLIDEAN, rows, m=8, m0=16, efc=60)
    queries = rng.standard_normal((1500, dim)).astype(np.float32)
    params = hx.SearchParams.strict(5, 20)
    gi, gs, gc = gpu.search_batch(queries, params)
    oi, os_, oc, _, _ = ora.search_batch(queries, 5, 20, threads=4)
    assert gc.tolist() == oc.tolist() and gi.tolist() == oi.tolist() and gs.tobytes() == os_.tobytes()
    for it in range(300):                                  # one CTA, > 255 consecutive epochs
        q = queries[it % 7: it % 7 + 1]
        a, b, c = gpu.search_batch(q, params)
        assert a[0].tolist() == oi[it % 7].tolist() and b[0].tobytes() == os_[it % 7].tobytes()


# ---- every launch shape of the traversal kernels answers with the same bits: default, tiny visited tables (every query
# ---- re-hashes into the overflow pool), few warps / shallow rings, every admission strategy of the CTA build, and the
# ---- dimension whose row does not fit a warp's share (d = 1600: the warp build reduces rows of 6.4 KB through 1-2 slots)
@pytest.mark.parametrize("gm,om,dim", [(hx.Metric.Euclidean, hxo.EUCLIDEAN, 70), (hx.Metric.Cosine, hxo.COSINE, 768),
                                       (hx.Metric.Cosine, hxo.COSINE, 40), (hx.Metric.Euclidean, hxo.EUCLIDEAN, 1600),
                                       (hx.Metric.Manhattan, hxo.MANHATTAN, 96)])
def test_traversal_builds_agree(gm, om, dim):
    n, nq = (1200, 320) if dim < 1000 else (500, 300)
    rng = np.random.default_rng(dim + 7)
    rows = rng.standard_normal((n, dim)).astype(np.float32)
    queries = rng.standard_normal((nq, dim)).astype(np.float32)
    gpu, ora = build_pair(gm, om, rows, m=8, m0=16, efc=60)
    k, ef = 10, 64
    oi, os_, oc, ost, _ = ora.search_batch(queries, k, ef, threads=4)
    params = hx.SearchParams.strict(k, ef)
    params.collect_stats = True
    variants = [{}, {"visited_log2": 6}, {"ring_warps": 5, "ring_rows": 2, "l2_hint": 0}, {"ring_rows": 1},
                {"ring_warps": 1, "prefetch_below": 0}, {"pipeline": 0}]
    for knobs in variants:
        gpu.tune(**knobs)
        st = hx.SearchStats()
        gi, gs, gc = gpu.search_batch(queries, params, st)
        assert gc.tolist() == oc.tolist(), knobs
        assert gi.tolist() == oi.tolist(), knobs
        assert gs.tobytes() == os_.tobytes(), knobs
        for f in ("expansion_steps", "neighbors_examined", "distance_computations"):
            assert getattr(st, f) == ost[f], (f, knobs)
    # small batches (B < #SMs) take the CTA-per-query build (visited set in shared memory, register beam up to ef = 128)
    nsmall = 40
    _, _, _, sst, _ = ora.search_batch(queries[:nsmall], k, ef, threads=4)
    small_stats = (sst["expansion_steps"], sst["neighbors_examined"], sst["distance_computations"])
    for knobs in [{}, {"visited_log2": 6}, {"ring_rows": 3}, {"lat_warps": 3, "l2_hint": 0}, {"lat_spec": 1}, {"lat_warps": 1},
                  {"lat_admit_seq": 1, "visited_log2": 7}]:
        gpu.tune(**knobs)
        st = hx.SearchStats()
        gi, gs, gc = gpu.search_batch(queries[:nsmall], params, st)
        assert gc.tolist() == oc[:nsmall].tolist(), knobs
        assert gi.tolist() == oi[:nsmall].tolist(), knobs
        assert gs.tobytes() == os_[:nsmall].tobytes(), knobs
        assert (st.expansion_steps, st.neighbors_examined, st.distance_computations) == small_stats, knobs
    gpu.tune()
    assert gpu.tuning()["visited_log2"] == -1
    # beams wider than 128 entries take the shared-memory beam of the latency build (the register beam holds 4 x 32)
    wi, ws, wc, _, _ = ora.search_batch(queries[:nsmall], k, 200, threads=4)
    gi, gs, gc = gpu.search_batch(queries[:nsmall], hx.SearchParams.strict(k, 200))
    assert gc.tolist() == wc.tolist() and gi.tolist() == wi.tolist() and gs.tobytes() == ws.tobytes()
    gi, gs, gc = gpu.search_batch(queries[:nsmall], hx.SearchParams.strict(k, 128))
    wi, ws, wc, _, _ = ora.search_batch(queries[:nsmall], k, 128, threads=4)
    assert gc.tolist() == wc.tolist() and gi.tolist() == wi.tolist() and gs.tobytes() == ws.tobytes()
    # a pool of zero overflow tables: the overflow is reported, never silently truncated
    gpu.tune(visited_log2=6, visited_pool=0)
    with pytest.raises(hx.HelixDbError) as e:
        gpu.search_batch(queries, params)
    assert e.value.variant == "InvariantViolation"
    gpu.tune()
    with pytest.raises(TypeError):
        gpu.tune(no_such_knob=1)


# ---- rows too large to stage (d = 12 288: 48 KB per row): the CTA build cannot hold a row next to its visited table and a
# ---- warp's share holds at most a few, down to none (ring_rows is capped by what fits) — results still bit-exact
@pytest.mark.parametrize("dim", [12288, 30016])      # 30016: not even one 120 KB row fits next to the 120 KB query -> R = 0
def test_very_large_dimension(dim):
    n, nq = 300, 160
    rng = np.random.default_rng(5)
    rows = rng.standard_normal((n, dim)).astype(np.float32)
    queries = rng.standard_normal((nq, dim)).astype(np.float32)
    gpu, ora = build_pair(hx.Metric.Cosine, hxo.COSINE, rows, m=6, m0=12, efc=30)
    oi, os_, oc, _, _ = ora.search_batch(queries, 5, 24, threads=4)
    params = hx.SearchParams.strict(5, 24)
    for b in (nq, 9, 1):
        gi, gs, gc = gpu.search_batch(queries[:b], params)
        assert gc.tolist() == oc[:b].tolist() and gi.tolist() == oi[:b].tolist() and gs.tobytes() == os_[:b].tobytes(), b


# ---- exact score ties at the beam boundary (duplicate vectors): the tie stack / `dropped` bookkeeping decides
# ---- expansion_steps, so ids, scores AND counters must match for every admission strategy ----------------------------------
@pytest.mark.parametrize("gm,om", METRICS[:2])
def test_exact_ties_at_beam_boundary(gm, om):
    rng = np.random.default_rng(99)
    n, dim, nq = 1000, 4, 200
    rows = rng.integers(0, 5, size=(n, dim)).astype(np.float32) + 1.0      # 625 grid positions: many identical vectors
    queries = (rng.random((nq, dim)) * 5.0 + 0.5).astype(np.float32)
    gpu, ora = build_pair(gm, om, rows, m=6, m0=12, efc=40)
    for ef, k in ((4, 4), (10, 10), (33, 10)):
        oi, os_, oc, _, _ = ora.search_batch(queries, k, ef, threads=4)
        per_q = [ora.search(queries[q], k, ef=ef, with_stats=True)[2] for q in range(24)]
        params = hx.SearchParams.strict(k, ef)
        for env in ({}, {"lat_admit_seq": 1}, {"ring_rows": 2, "lat_warps": 2}):
            gpu.tune(**env)
            gi, gs, gc = gpu.search_batch(queries, params)                     # warp-per-query builds
            assert gc.tolist() == oc.tolist() and gi.tolist() == oi.tolist() and gs.tobytes() == os_.tobytes(), (ef, env)
            gi, gs, gc = gpu.search_batch(queries[:100], params)               # CTA-per-query builds
            assert gc.tolist() == oc[:100].tolist() and gi.tolist() == oi[:100].tolist(), (ef, env)
            assert gs.tobytes() == os_[:100].tobytes(), (ef, env)
            params.collect_stats = True
            for q in range(24):
                st = hx.SearchStats()
                gpu.search_batch(queries[q:q + 1], params, st)
                for f in ("expansion_steps", "neighbors_examined", "distance_computations"):
                    assert getattr(st, f) == per_q[q][f], (f, q, ef, env)
            params.collect_stats = False


# ---- large host batches are pipelined: chunked H2D on a second stream, validation fused into the search kernel ----------
@pytest.mark.parametrize("gm,om", METRICS[:2])
def test_pipelined_host_search(gm, om):
    n, dim, nq = 1500, 40, 3000
    rng = np.random.default_rng(8)
    rows = rng.standard_normal((n, dim)).astype(np.float32)
    gpu, ora = build_pair(gm, om, rows, m=8, m0=16, efc=60)
    queries = rng.standard_normal((nq, dim)).astype(np.float32)
    params = hx.SearchParams.strict(5, 24)
    oi, os_, oc, ost, _ = ora.search_batch(queries, 5, 24, threads=4)
    for pipe in ("1", "0"):
        gpu.tune(pipeline=int(pipe))
        st = hx.SearchStats()
        params.collect_stats = True
        gi, gs, gc = gpu.search_batch(queries, params, st)
        assert gc.tolist() == oc.tolist() and gi.tolist() == oi.tolist() and gs.tobytes() == os_.tobytes(), pipe
        assert st.expansion_steps == ost["expansion_steps"] and st.distance_computations == ost["distance_computations"]
        assert st.kernel_launches == (1 if pipe == "1" else 2)            # no separate validation launch when pipelined
        bad = queries.copy()
        bad[2711, 7] = np.nan                                              # in the last chunk
        bad[2900, 3] = np.inf
        with pytest.raises(hx.HelixDbError) as e:
            gpu.search_batch(bad, params)
        assert e.value.variant == "InvalidVectorComponent" and e.value.index == 7
        if om == hxo.COSINE:
            bad = queries.copy()
            bad[17] = 0.0
            with pytest.raises(hx.HelixDbError) as e:
                gpu.search_batch(bad, params)
            assert e.value.variant == "ZeroNormCosineVector"
        else:
            lim = hxo.component_limit(om, dim)
            bad = queries.copy()
            bad[1234, 39] = float(np.nextafter(np.float32(lim), np.float32(np.inf)))
            with pytest.raises(hx.HelixDbError) as e:
                gpu.search_batch(bad, params)
            assert e.value.variant == "VectorComponentMagnitudeExceeded" and e.value.index == 39
        gi2, gs2, gc2 = gpu.search_batch(queries, params)                  # the handle is healthy after an error
        assert gi2.tolist() == oi.tolist()


# ---- wide beams: ef far above the register beam (128) and k in the hundreds, both batch regimes -------------------------
@pytest.mark.parametrize("gm,om", METRICS[:2])
def test_wide_beam_and_large_k(gm, om):
    n, dim = 4000, 64
    rng = np.random.default_rng(31)
    rows = rng.standard_normal((n, dim)).astype(np.float32)
    gpu, ora = build_pair(gm, om, rows, m=8, m0=16, efc=60)
    queries = rng.standard_normal((200, dim)).astype(np.float32)
    for k, ef in ((200, 1000), (64, 4096), (1, 129)):
        oi, os_, oc, ost, _ = ora.search_batch(queries, k, ef, threads=4)
        params = hx.SearchParams.strict(k, ef)
        params.collect_stats = True
        st = hx.SearchStats()
        gi, gs, gc = gpu.search_batch(queries, params, st)                 # warp-per-query build
        assert gc.tolist() == oc.tolist() and gi.tolist() == oi.tolist() and gs.tobytes() == os_.tobytes(), (k, ef)
        assert st.expansion_steps == ost["expansion_steps"] and st.distance_computations == ost["distance_computations"]
        gi, gs, gc = gpu.search_batch(queries[:12], params)                # CTA-per-query build, shared-memory beam
        assert gc.tolist() == oc[:12].tolist() and gi.tolist() == oi[:12].tolist() and gs.tobytes() == os_[:12].tobytes()
    with pytest.raises(hx.HelixDbError):
        gpu.search_batch(queries[:2], hx.SearchParams.strict(10, 5000))    # above the supported beam width


# ---- sharded path: per-shard top-k merged by (score, id) equals the unsharded exact answer ---------------------------------------
def test_merge_topk_matches_unsharded_scan():
    import torch
    n, dim, B, k, S = 4000, 48, 33, 10, 4
    rng = np.random.default_rng(21)
    rows = rng.integers(-3, 4, size=(n, dim)).astype(np.float32)        # many exact score ties across shards
    ids = np.arange(n, dtype=np.uint64)
    queries = rng.integers(-3, 4, size=(B, dim)).astype(np.float32)
    ora = hxo.Index(hxo.EUCLIDEAN, dim)
    ora.put_vectors(ids, rows)
    ora.set_entry(0, 0)
    all_ids = np.zeros((S, B, k), dtype=np.uint64)
    all_sc = np.zeros((S, B, k), dtype=np.float32)
    all_cnt = np.zeros((S, B), dtype=np.uint32)
    per = n // S
    for s in range(S):                                                   # contiguous id ranges (SURVEY §8e)
        lo, hi = s * per, (s + 1) * per if s < S - 1 else n
        g = hx.VectorIndex(hx.Metric.Euclidean, hx.VectorIndexConfig(f"s{s}", "embedding", dim))
        g.load_vectors(ids[lo:hi], rows[lo:hi])
        g.load_graph(0, ids[lo:lo + 1], [0, 0], [])
        g.set_entry(int(ids[lo]), 0)
        a, b, c = g.search_restricted_batch(queries, hx.SearchParams.strict(k), hx.RestrictedVectorCandidates(ids[lo:hi]))
        all_ids[s], all_sc[s], all_cnt[s] = a, b, c
        g.close()
    dev = torch.device("cuda:0")
    t_ids = torch.from_numpy(all_ids.view(np.int64)).to(dev)
    t_sc = torch.from_numpy(all_sc).to(dev)
    t_cnt = torch.from_numpy(all_cnt.view(np.int32)).to(dev)
    o_ids = torch.zeros((B, k), dtype=torch.int64, device=dev)
    o_sc = torch.zeros((B, k), dtype=torch.float32, device=dev)
    o_cnt = torch.zeros((B,), dtype=torch.int32, device=dev)
    hx.merge_topk_device(0, t_ids.data_ptr(), t_sc.data_ptr(), t_cnt.data_ptr(), S, B, k, o_ids.data_ptr(),
                         o_sc.data_ptr(), o_cnt.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    for q in range(B):
        ei, es = ora.search_exact(queries[q], k)
        assert o_cnt[q].item() == k
        assert o_ids[q].cpu().numpy().view(np.uint64).tolist() == ei.tolist()
        assert o_sc[q].cpu().numpy().tobytes() == es.tobytes()


# ---- device-buffer entry points (inputs resident in HBM) agree with the host-buffer calls ---------------------------------------
def test_device_buffer_entry_points():
    import torch
    n, dim, B, k = 2500, 96, 700, 10
    rng = np.random.default_rng(8)
    rows = rng.standard_normal((n, dim)).astype(np.float32)
    gpu, ora = build_pair(hx.Metric.Cosine, hxo.COSINE, rows, m=8, m0=16, efc=60)
    queries = rng.standard_normal((B, dim)).astype(np.float32)
    params = hx.SearchParams.strict(k, 40)
    hi, hs, hc = gpu.search_batch(queries, params)
    dev = torch.device("cuda:0")
    dq = torch.from_numpy(queries).to(dev)
    o_ids = torch.zeros((B, k), dtype=torch.int64, device=dev)
    o_sc = torch.zeros((B, k), dtype=torch.float32, device=dev)
    o_cnt = torch.zeros((B,), dtype=torch.int32, device=dev)
    stream = torch.cuda.current_stream().cuda_stream
    for _ in range(3):
        gpu.search_device(dq.data_ptr(), B, params, o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr(), stream)
    torch.cuda.synchronize()
    assert o_ids.cpu().numpy().view(np.uint64).tolist() == hi.tolist()
    assert o_sc.cpu().numpy().tobytes() == hs.tobytes()
    ms, launches = gpu.last_kernel_ms()
    assert launches == 3 and ms > 0.0
    # restricted: per-query candidate sets as device slots
    cand = np.arange(0, n, 5, dtype=np.uint64)
    d_c = torch.from_numpy(cand.view(np.int64)).to(dev)
    d_slots = torch.zeros((len(cand),), dtype=torch.int32, device=dev)
    gpu.map_candidates_device(d_c.data_ptr(), len(cand), d_slots.data_ptr(), stream)
    gpu.search_restricted_device(dq.data_ptr(), B, hx.SearchParams.strict(k), d_slots.data_ptr(), 0, len(cand), 0,
                                 o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr(), stream)
    torch.cuda.synchronize()
    ri, rs, rc = gpu.search_restricted_batch(queries, hx.SearchParams.strict(k), hx.RestrictedVectorCandidates(cand))
    assert o_ids.cpu().numpy().view(np.uint64).tolist() == ri.tolist()
    assert o_sc.cpu().numpy().tobytes() == rs.tobytes()


# ---- device build (SURVEY §8(f).1): reference invariants, recall, and oracle parity on the device-built graph ---------------
def _check_graph_invariants(g, lim0, m):
    n, s0, su = g["n"], g["layer0_stride"], g["upper_stride"]
    nbr0 = g["nbr0"].reshape(n, s0)
    deg0 = g["deg0"]
    assert deg0.max() <= lim0
    adj = [set(nbr0[i, :deg0[i]].tolist()) for i in range(n)]
    for i in range(n):
        row = nbr0[i, :deg0[i]]
        assert i not in adj[i]                                        # no self link
        assert np.all(row[1:] > row[:-1])                             # strictly ascending
    for i in range(n):
        for j in adj[i]:
            assert i in adj[j], f"layer-0 edge {i}->{j} is not bidirectional"
    rows = len(g["upper_node"])
    unbr = g["upper_nbr"].reshape(max(rows, 1), su) if rows else np.zeros((0, su), np.uint32)
    upper = {}
    for r in range(rows):
        key = (int(g["upper_layer"][r]), int(g["upper_node"][r]))
        d = int(g["upper_deg"][r])
        assert d <= m
        lst = unbr[r, :d]
        assert np.all(lst[1:] > lst[:-1]) and key[1] not in lst.tolist()
        upper[key] = set(lst.tolist())
    for (layer, node), s in upper.items():
        assert g["levels"][node] >= layer
        for w in s:
            assert node in upper[(layer, w)], f"layer-{layer} edge {node}->{w} is not bidirectional"
    top = int(g["levels"].max())
    assert g["max_layer"] == top and g["levels"][g["entry_slot"]] == top


@pytest.mark.parametrize("gm,om,n,dim,m", [(hx.Metric.Euclidean, hxo.EUCLIDEAN, 4000, 64, 16),
                                           (hx.Metric.Cosine, hxo.COSINE, 3000, 100, 8),
                                           (hx.Metric.Manhattan, hxo.MANHATTAN, 1500, 24, 16)])
def test_device_build(gm, om, n, dim, m):
    rng = np.random.default_rng(n)
    cent = rng.standard_normal((32, dim)).astype(np.float32)
    rows = (cent[rng.integers(0, 32, n)] + 0.5 * rng.standard_normal((n, dim))).astype(np.float32)
    ids = np.arange(100, 100 + n, dtype=np.uint64)
    gpu = hx.VectorIndex(gm, hx.VectorIndexConfig("b", "embedding", dim).with_m(m).with_m0(2 * m).with_ef_construction(100))
    gpu.load_vectors(ids, rows)
    gpu.build(seed=42)
    g = gpu.download_graph()
    g["entry_slot"] = int(g["entry_point"] - 100)
    _check_graph_invariants(g, 2 * m, m)
    # level law: about 1/m of the nodes reach layer >= 1 (select_layer, mod.rs:769-796)
    frac = float((g["levels"] >= 1).mean())
    assert 0.5 / m < frac < 2.0 / m
    # the oracle traverses the identical adjacency: results must agree bit for bit
    ora = hxo.Index(om, dim, m=m, m0=2 * m, ef_construction=100)
    ora.put_vectors(ids, rows)
    ora.import_graph(g["levels"], g["deg0"], g["nbr0"], g["layer0_stride"], g["upper_node"], g["upper_layer"],
                     g["upper_deg"], g["upper_nbr"], g["upper_stride"], g["entry_point"], g["max_layer"])
    queries = (cent[rng.integers(0, 32, 48)] + 0.5 * rng.standard_normal((48, dim))).astype(np.float32)
    gi, gs, gc = gpu.search_batch(queries, hx.SearchParams.strict(10))
    hit = 0
    for q in range(len(queries)):
        oi, os_ = ora.search(queries[q], 10)
        assert_same(gi[q], gs[q], gc[q], oi, os_, f"built graph q={q}")
        ex, _ = ora.search_exact(queries[q], 10)
        hit += len(set(oi.tolist()) & set(ex.tolist()))
    assert hit / (10.0 * len(queries)) >= 0.95
    # explicit levels are honoured (scripted layers [0,1,3] => entry = the level-3 node, index.rs:1919-1973)
    lv = np.zeros(n, dtype=np.uint16)
    lv[1], lv[2] = 1, 3
    gpu.build(levels=lv)
    gi2 = gpu.graph_info()
    assert gi2["entry_point"] == 102 and gi2["max_layer"] == 3


# ---- dense tensor-core path (wgmma bf16 contraction nominates, exact fp32 re-rank decides) -------------------------------------
@pytest.mark.parametrize("gm,om,n,dim,B", [(hx.Metric.Cosine, hxo.COSINE, 5000, 768, 300),
                                          (hx.Metric.Euclidean, hxo.EUCLIDEAN, 3000, 100, 130),
                                          (hx.Metric.Cosine, hxo.COSINE, 700, 64, 5),
                                          (hx.Metric.Cosine, hxo.COSINE, 60000, 128, 260)])
def test_dense_tensor_core_path(gm, om, n, dim, B):
    rng = np.random.default_rng(n + dim)
    lat = rng.standard_normal((n, 16)).astype(np.float32)
    proj = rng.standard_normal((16, dim)).astype(np.float32)
    rows = (lat @ proj + 0.05 * rng.standard_normal((n, dim))).astype(np.float32)
    queries = (rng.standard_normal((B, 16)).astype(np.float32) @ proj).astype(np.float32)
    if om == hxo.COSINE:
        rows /= np.linalg.norm(rows, axis=1, keepdims=True)
    ids = np.arange(n, dtype=np.uint64) + 7
    gpu = hx.VectorIndex(gm, hx.VectorIndexConfig("d", "embedding", dim), storage=1)
    gpu.load_vectors(ids, rows)
    gpu.load_graph(0, ids[:1], [0, 0], [])
    gpu.set_entry(int(ids[0]), 0)
    k = 10
    di, ds, dc = gpu.search_dense_batch(queries, hx.SearchParams.strict(k))
    ei, es, ec = gpu.search_restricted_batch(queries, hx.SearchParams.strict(k), hx.RestrictedVectorCandidates(ids))
    assert dc.tolist() == ec.tolist() == [k] * B
    hit = 0
    for q in range(B):
        exact = {int(i): es[q, j].tobytes() for j, i in enumerate(ei[q])}
        hit += len(set(di[q].tolist()) & set(exact))
        for j, i in enumerate(di[q]):                      # every returned score is the exact fp32 reference score
            if int(i) in exact:
                assert ds[q, j].tobytes() == exact[int(i)]
        keys = [(float(ds[q, j]), int(di[q, j])) for j in range(k)]
        assert keys == sorted(keys)                        # (score, id) order
    assert hit / float(B * k) >= 0.99
    # ... and against the ORACLE's exact scan (not only this repository's own scan kernel): same ids except where a true
    # neighbour was not nominated by its bf16 score, and every returned score is the oracle's score for that id, bit for bit
    ora = hxo.Index(om, dim)
    ora.put_vectors(ids, rows)
    nchk, ohit = min(B, 24), 0
    for q in range(nchk):
        oi, os_ = ora.search_exact(queries[q], k)
        exact = {int(i): os_[j].tobytes() for j, i in enumerate(oi)}
        ohit += len(set(di[q].tolist()) & set(exact))
        for j, i in enumerate(di[q]):
            if int(i) in exact:
                assert ds[q, j].tobytes() == exact[int(i)], (q, j)
        if len(set(di[q].tolist()) & set(exact)) == k:
            assert di[q].tolist() == oi.tolist(), q                      # complete answers come in the oracle's order
    assert ohit / float(nchk * k) >= 0.99
    storage0 = hx.VectorIndex(gm, hx.VectorIndexConfig("d0", "embedding", dim))
    storage0.load_vectors(ids[:10], rows[:10])
    with pytest.raises(hx.HelixDbError):
        storage0.search_dense_batch(queries[:1], hx.SearchParams.strict(1))


# ---- row-image import (SURVEY §8(f).2): hydrate from the reference's encoded rows, search, export ---------------------------
@pytest.mark.parametrize("gm,om", METRICS[:2])
def test_row_image_import_and_export(gm, om):
    n, dim = 800, 48
    rng = np.random.default_rng(17)
    rows = rng.standard_normal((n, dim)).astype(np.float32)
    ids = np.arange(n, dtype=np.uint64) * 5 + 3
    gpu_ref, ora = build_pair(gm, om, rows, ids=ids, m=8, m0=16, efc=40)
    # encode every row the way the reference stores it: [header f32][f32 x dim], native endian (mod.rs:866-871)
    item_rows = b"".join(struct.pack("<f", hxo.header(om, rows[i])) + rows[i].tobytes() for i in range(n))
    gpu = hx.VectorIndex(gm, hx.VectorIndexConfig("img", "embedding", dim).with_m(8).with_m0(16).with_ef_construction(40))
    gpu.load_vector_rows(ids, item_rows)
    graph, state = ora.export_graph()
    for layer, (nodes, offs, nbrs) in graph.items():
        enc = [hx.encode_neighbor_row(layer, nbrs[offs[i]:offs[i + 1]]) for i in range(len(nodes))]
        gpu.load_neighbor_rows(layer, nodes, enc)
    gpu.set_entry(*state)
    queries = rng.standard_normal((40, dim)).astype(np.float32)
    gi, gs, gc = gpu.search_batch(queries, hx.SearchParams.strict(10))
    for q in range(len(queries)):
        oi, os_ = ora.search(queries[q], 10)
        assert_same(gi[q], gs[q], gc[q], oi, os_, f"row image q={q}")
    # export: the device row encodes back to the reference's bytes
    some = int(ids[7])
    assert gpu.export_neighbor_row(0, some) == hx.encode_neighbor_row(0, ora.neighbors(0, some))
    # a stored header that does not match the recomputed one is a decode error (HeaderMismatch, mod.rs:942-945)
    bad = bytearray(item_rows)
    bad[0:4] = struct.pack("<f", 123.0)
    with pytest.raises(hx.HelixDbError) as e:
        gpu.load_vector_rows(ids, bytes(bad))
    assert e.value.variant == "InvariantViolation"


# ---- the handle is Send + Sync: concurrent searches from several host threads (one query batch per thread) -------------------
def test_concurrent_host_threads():
    import threading
    n, dim = 3000, 64
    rng = np.random.default_rng(23)
    rows = rng.standard_normal((n, dim)).astype(np.float32)
    gpu, ora = build_pair(hx.Metric.Euclidean, hxo.EUCLIDEAN, rows, m=8, m0=16, efc=60)
    queries = rng.standard_normal((6, 200, dim)).astype(np.float32)
    params = hx.SearchParams.strict(10, 50)
    expected = [gpu.search_batch(queries[t], params) for t in range(6)]
    cand = hx.RestrictedVectorCandidates(np.arange(0, n, 3, dtype=np.uint64))
    expected_r = [gpu.search_restricted_batch(queries[t][:20], params, cand) for t in range(6)]
    results, errors = [None] * 6, []

    def worker(t):
        try:
            for _ in range(5):
                a = gpu.search_batch(queries[t], params)
                b = gpu.search_restricted_batch(queries[t][:20], params, cand)
            results[t] = (a, b)
        except Exception as e:   # pragma: no cover
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(6)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for t in range(6):
        (ai, as_, ac), (bi, bs, bc) = results[t]
        assert ai.tolist() == expected[t][0].tolist() and as_.tobytes() == expected[t][1].tobytes()
        assert bi.tolist() == expected_r[t][0].tolist() and bs.tobytes() == expected_r[t][1].tobytes()
