"""Every scoring kernel held to the oracle across the float32 range (fixtures: tests/numeric_range.py).

Bit for bit (count, ids, score bits and, where the entry reports them, the SearchStats counters) through each entry point
whose kernels compute scores: the restricted exact scan (k_scan_topk, k_scan + k_select, device sets), strict HNSW search
(warp-per-query ring and CTA builds), the default SimHash mode, both query services, the ACORN walk, the sequential device
build and row-image import; each returned score is also checked against the float64 formula.  Validation at the component
limit is checked through each of its implementations, and the dense path's nomination through the float64 reference of
tests/test_dense_reference.py.
"""
import struct

import numpy as np
import pytest

import helix_db_b200 as hx
from oracle import hxo

import numeric_range as nr
from test_gpu_build_seq import _rows_of_device, _rows_of_oracle
from test_gpu_dense import check_against_reference, dense_index
from test_gpu_parity import build_pair, levels_for
from test_gpu_policy import compare as compare_policy
from test_gpu_policy import oracle_cfg

pytestmark = pytest.mark.gpu
EUC, COS, MAN = hxo.EUCLIDEAN, hxo.COSINE, hxo.MANHATTAN
GM = {EUC: hx.Metric.Euclidean, COS: hx.Metric.Cosine, MAN: hx.Metric.Manhattan}


def flat_pair(om, ids, rows):
    """Device index and oracle holding the same rows, populated (entry = first id), no graph edges."""
    gpu = hx.VectorIndex(GM[om], hx.VectorIndexConfig("range", "embedding", rows.shape[1]))
    gpu.load_vectors(ids, rows)
    gpu.load_graph(0, ids[:1], [0, 0], [])
    gpu.set_entry(int(ids[0]), 0)
    ora = hxo.Index(om, rows.shape[1])
    ora.put_vectors(ids, rows)
    ora.put_neighbors(0, int(ids[0]), [])
    ora.set_entry(int(ids[0]), 0)
    return gpu, ora


def assert_same(got, want, what):
    gi, gs, gc = got
    wi, ws, wc = want[:3]
    assert gc.tolist() == wc.tolist(), f"{what}: counts"
    for b in range(len(gc)):
        c = int(gc[b])
        assert gi[b, :c].tolist() == wi[b, :c].tolist(), f"{what}: ids of query {b}"
        assert gs[b, :c].view(np.uint32).tolist() == ws[b, :c].view(np.uint32).tolist(), f"{what}: score bits of query {b}"


def assert_results(res, oi, os_, what):
    assert [int(r.entity_id()) for r in res] == oi.tolist(), f"{what}: ids"
    assert np.array([r.score() for r in res], np.float32).view(np.uint32).tolist() == os_.view(np.uint32).tolist(), \
        f"{what}: score bits"


def restricted_oracle(ora, queries, k, sets):
    ids = np.concatenate(sets).astype(np.uint64)
    offs = np.concatenate([[0], np.cumsum([len(s) for s in sets])]).astype(np.uint64)
    return ora.search_restricted_batch(queries, k, ids, offs)


def simhash_bits(rng, ids, rows, queries):
    planes = rng.standard_normal((64, rows.shape[1])).astype(np.float32)
    return (np.array([hxo.simhash_from_planes(planes, r) for r in rows], dtype=np.uint64),
            np.array([hxo.simhash_from_planes(planes, q) for q in queries], dtype=np.uint64))


# ---- restricted exact scan ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", nr.DIMS)
@pytest.mark.parametrize("om", [EUC, COS, MAN])
def test_restricted_scan(om, d):
    ids, rows, queries = nr.corpus(om, d)
    gpu, ora = flat_pair(om, ids, rows)
    B = len(queries)
    every = [ids] * B
    for k, knobs, what in ((10, {}, "k_scan_topk"), (10, {"scan_fused": 0}, "k = 10 unfused"), (40, {}, "k_scan + k_select")):
        gpu.tune(**knobs)
        try:
            got = gpu.search_restricted_batch(queries, hx.SearchParams.strict(k), hx.RestrictedVectorCandidates(ids))
        finally:
            gpu.tune()
        assert_same(got, restricted_oracle(ora, queries, k, every), f"{what}")
        nr.assert_within_f64(om, queries, rows, ids, *got, what=what)
    rng = np.random.default_rng(d)
    sets = [np.sort(rng.choice(ids, size=len(ids) * 2 // 3, replace=False)) for _ in range(B)]
    got = gpu.search_restricted_multi(queries, hx.SearchParams.strict(10), np.concatenate(sets),
                                      np.concatenate([[0], np.cumsum([len(s) for s in sets])]).astype(np.uint64))
    assert_same(got, restricted_oracle(ora, queries, 10, sets), "search_restricted_multi")
    dc = gpu.cache_candidates(hx.RestrictedVectorCandidates(sets[0]))
    got = gpu.search_restricted_sets(queries, hx.SearchParams.strict(10), dc)
    assert_same(got, restricted_oracle(ora, queries, 10, [sets[0]] * B), "device candidate set")
    gpu.close()


# ---- strict HNSW: warp-per-query ring (B >= 132) and CTA build (B < 132) ---------------------------------------------------
@pytest.mark.parametrize("om,d", [(COS, 33), (COS, 768), (EUC, 33), (EUC, 768), (MAN, 70)])
def test_strict_hnsw(om, d):
    ids, rows, queries = nr.corpus(om, d, n_rows=100, n_queries=140)
    gpu, ora = build_pair(GM[om], om, rows, ids=ids, m=8, m0=16, efc=40)
    k, ef = 10, 40
    want = [ora.search(q, k, ef=ef, with_stats=True) for q in queries]
    for B in (140, 40):
        params = hx.SearchParams.strict(k, ef)
        params.collect_stats = True
        st = hx.SearchStats()
        gi, gs, gc = gpu.search_batch(queries[:B], params, st)
        for b in range(B):
            oi, os_, _ = want[b]
            assert int(gc[b]) == len(oi) and gi[b, :gc[b]].tolist() == oi.tolist(), f"B = {B}: ids of query {b}"
            assert gs[b, :gc[b]].view(np.uint32).tolist() == os_.view(np.uint32).tolist(), f"B = {B}: score bits of query {b}"
        for f in ("expansion_steps", "neighbors_examined", "distance_computations"):
            assert getattr(st, f) == sum(w[2][f] for w in want[:B]), f"B = {B}: {f}"
        nr.assert_within_f64(om, queries[:B], rows, ids, gi, gs, gc, what=f"B = {B}")
    gpu.close()


# ---- default mode (SimHash Adaptive) -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("om,d", [(COS, 33), (COS, 768), (EUC, 70)])
def test_default_mode(om, d):
    ids, rows, queries = nr.corpus(om, d, n_rows=100, n_queries=48)
    gpu, ora = build_pair(GM[om], om, rows, ids=ids, m=8, m0=16, efc=40)
    bits, qsim = simhash_bits(np.random.default_rng(d), ids, rows, queries)
    gpu.load_simhash(ids, bits)
    ora.put_simhash(ids, bits)
    params = hx.SearchParams.new(10).with_ef(32)
    gpu.set_simhash_config()
    compare_policy(gpu, ora, queries, qsim, params, oracle_cfg(params), f"default mode d={d}")
    gpu.close()


# ---- query services: one query per call, the query read from the host-mapped ring --------------------------------------------
@pytest.mark.parametrize("om,d", [(COS, 33), (COS, 768), (EUC, 70), (MAN, 31)])
def test_services(om, d):
    ids, rows, queries = nr.corpus(om, d, n_rows=100, n_queries=16)
    gpu, ora = build_pair(GM[om], om, rows, ids=ids, m=8, m0=16, efc=40)
    cand = ids[::2].copy()
    with gpu.service(10, 40) as svc:
        for b, q in enumerate(queries):
            oi, os_ = ora.search(q, 10, ef=40)
            assert_results(svc.search(q), oi, os_, f"service query {b}")
    with gpu.restricted_service(10) as rsvc:
        allowed = hx.RestrictedVectorCandidates(cand)
        for b, q in enumerate(queries):
            oi, os_ = ora.search_restricted(q, 10, cand)
            assert_results(rsvc.search(q, allowed), oi, os_, f"restricted service query {b}")
    gpu.close()


# ---- ACORN walk ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("om,d", [(COS, 33), (EUC, 70)])
def test_acorn_walk(om, d):
    ids, rows, queries = nr.corpus(om, d, n_rows=200, n_queries=24)
    gpu, ora = build_pair(GM[om], om, rows, ids=ids, m=8, m0=16, efc=40)
    bits, qsim = simhash_bits(np.random.default_rng(d + 1), ids, rows, queries)
    gpu.load_simhash(ids, bits)
    ora.put_simhash(ids, bits)
    cand = ids[::2].copy()
    st = hx.FilteredStats()
    gi, gs, gc = gpu.search_filtered_graph(queries, hx.SearchParams.new(10).with_ef(40), hx.RestrictedVectorCandidates(cand),
                                           qsim, stats=st)
    tot = dict(vector_payload_requests=0, distance_computations=0, routing_rows=0, bridge_rows=0, bridge_frontier_pushes=0)
    for b in range(len(queries)):
        oi, os_, ost = ora.search_filtered_graph(queries[b], 10, cand, int(qsim[b]), ef=40)
        assert int(gc[b]) == len(oi) and gi[b, :gc[b]].tolist() == oi.tolist(), f"query {b}: ids"
        assert gs[b, :gc[b]].view(np.uint32).tolist() == os_.view(np.uint32).tolist(), f"query {b}: score bits"
        for f in tot:
            tot[f] += ost[f]
    for f in tot:
        assert getattr(st, f) == tot[f], f
    gpu.close()


# ---- sequential device build: the fallback inside hxb_pair ---------------------------------------------------------------------
def test_sequential_build_on_mixed_scales():
    ids, rows, _ = nr.corpus(COS, 33, n_rows=160, n_queries=40)
    n, m, m0, efc = len(ids), 8, 16, 40
    lv = levels_for(n, m, 5)
    ora = hxo.Index(COS, 33, m=m, m0=m0, ef_construction=efc)
    for i in range(n):
        ora.insert(int(ids[i]), rows[i], lv[i])
    gpu = hx.VectorIndex(hx.Metric.Cosine, hx.VectorIndexConfig("seq", "embedding", 33).with_m(m).with_m0(m0)
                         .with_ef_construction(efc))
    gpu.load_vectors(ids, rows)
    gpu.build(levels=np.array(lv, dtype=np.uint16), sequential=True)
    want, wstate = _rows_of_oracle(ora)
    got, gstate = _rows_of_device(gpu, ids)
    assert (int(gstate[0]), int(gstate[1])) == (int(wstate[0]), int(wstate[1]))
    assert set(got) == set(want)
    diff = [key for key in want if want[key] != got[key]]
    assert not diff, f"{len(diff)} of {len(want)} rows differ, first: {diff[0]} want {want[diff[0]]} got {got[diff[0]]}"
    gpu.close()


# ---- row images: the device recomputes every header bit for bit ------------------------------------------------------------------
@pytest.mark.parametrize("om,d", [(COS, 33), (COS, 768), (EUC, 70)])
def test_row_images_of_extreme_rows(om, d):
    ids, rows, _ = nr.corpus(om, d, n_rows=60, n_queries=4)
    hdr = np.array([hxo.header(om, r) for r in rows], np.float32)

    def image(h):
        return b"".join(struct.pack("<f", float(h[i])) + rows[i].tobytes() for i in range(len(rows)))

    def fresh():
        return hx.VectorIndex(GM[om], hx.VectorIndexConfig("img", "embedding", d))

    gpu = fresh()
    gpu.load_vector_rows(ids, image(hdr))
    got_ids, got_rows = gpu.download_vectors(0, len(ids))
    assert got_ids.tolist() == ids.tolist() and got_rows.tobytes() == rows.tobytes()
    gpu.close()
    fmax = np.float32(nr.FLT_MAX)
    picks = [int(np.argmax(hdr)), int(np.argmin(np.where(hdr > 0, hdr, np.inf))) if om == COS else 0]
    for i in picks:
        bad = hdr.copy()
        bad[i] = np.nextafter(bad[i], np.float32(0) if bad[i] == fmax else fmax)
        gpu = fresh()
        with pytest.raises(hx.HelixDbError) as e:
            gpu.load_vector_rows(ids, image(bad))
        assert e.value.variant == "InvariantViolation", (i, float(hdr[i]))
        gpu.close()


# ---- validation at the component limit, through every implementation -----------------------------------------------------------
@pytest.mark.parametrize("d", [3, 70, 768])
@pytest.mark.parametrize("om", [EUC, MAN])
def test_component_limit_on_every_entry_point(om, d):
    ids, rows, queries = nr.corpus(om, d, n_rows=60, n_queries=20)
    gpu, ora = build_pair(GM[om], om, rows, ids=ids, m=8, m0=16, efc=40)
    lim = np.float32(hxo.component_limit(om, d))
    over = np.nextafter(lim, np.float32(np.inf))
    j = d - 1 if d > 3 else 1
    p = hx.SearchParams.strict(10, 40)

    def with_value(q, b, v):
        q = q.copy()
        q[b, j] = v
        return q

    def refused(call, what):
        with pytest.raises(hx.HelixDbError) as e:
            call()
        assert e.value.variant == "VectorComponentMagnitudeExceeded" and e.value.index == j, what

    big = np.ascontiguousarray(np.resize(queries, (1100, d)))
    for B, b, what in ((3, 2, "host validation"), (20, 13, "device validation"), (1100, 1099, "pipelined search")):
        q = big[:B]
        for sign in (1, -1):
            at = with_value(q, b, sign * lim)
            gi, gs, gc = gpu.search_batch(at, p)
            oi, os_ = ora.search(at[b], 10, ef=40)
            assert gi[b, :gc[b]].tolist() == oi.tolist() and gs[b, :gc[b]].tobytes() == os_.tobytes(), what
            refused(lambda: gpu.search_batch(with_value(q, b, sign * over), p), what)
    refused(lambda: gpu.search_restricted_batch(with_value(queries, 13, over), p, hx.RestrictedVectorCandidates(ids)),
            "restricted scan")
    at = with_value(queries, 0, lim)[0]
    with gpu.service(10, 40) as svc:
        assert_results(svc.search(at), *ora.search(at, 10, ef=40), "service at the limit")
        refused(lambda: svc.search(with_value(queries, 0, -over)[0]), "service")
    with gpu.restricted_service(10) as rsvc:
        allowed = hx.RestrictedVectorCandidates(ids)
        assert_results(rsvc.search(at, allowed), *ora.search_restricted(at, 10, ids), "restricted service at the limit")
        refused(lambda: rsvc.search(with_value(queries, 0, over)[0], allowed), "restricted service")
    gpu.close()
    if om == EUC:   # the dense path computes the limit itself
        dense = dense_index(EUC, ids, rows)
        got = dense.search_dense_batch(with_value(queries, 13, -lim), hx.SearchParams.strict(10))
        want = ora.search_exact_batch(with_value(queries, 13, -lim), 10)
        assert_same(got, want, "dense at the limit")
        refused(lambda: dense.search_dense_batch(with_value(queries, 13, over), hx.SearchParams.strict(10)), "dense")
        dense.close()


# ---- dense path: nomination over the float32 range -----------------------------------------------------------------------------
def _dense_check(om, ids, rows, queries, what, k=10, floor=0.5):
    gpu = dense_index(om, ids, rows)
    got = gpu.search_dense_batch(queries, hx.SearchParams.strict(k))
    gpu.close()
    covered = check_against_reference(om, ids, rows, queries, k, got)
    assert covered >= floor, f"{what}: only {covered:.2f} of the queries have their exact top-{min(k, 4)} rows sure"


@pytest.mark.parametrize("n_rows", [600, 100])   # 725 rows: tensor-core pass (>= 8 * 64); 225 rows: exact scan
def test_dense_cosine_fixture(n_rows):
    ids, rows, queries = nr.corpus(COS, 768, n_rows=n_rows, n_queries=40)
    _dense_check(COS, ids, rows, queries, f"cosine fixture, {len(ids)} rows")


def test_dense_extreme_queries_on_an_order_one_corpus():
    ids, rows, _ = nr.scaled_corpus(4000, 128, 0, 40)
    rng = np.random.default_rng(3)
    sel = rng.choice(len(ids), size=45, replace=False)
    e = np.resize(np.array(nr.EXPONENTS, np.float64), 45)
    queries = (rows[sel].astype(np.float64) * np.exp2(e)[:, None]).astype(np.float32)   # its own row is the nearest
    queries = np.concatenate([queries, nr.cosine_queries(5, 128)])
    _dense_check(COS, ids, rows, queries, "extreme queries")


def test_dense_order_one_queries_on_an_extreme_corpus():
    ids, rows, queries = nr.scaled_corpus(4000, 128, 0, 40)
    rng = np.random.default_rng(4)
    e = rng.choice(nr.EXPONENTS, size=len(rows)).astype(np.float64)
    rows = (rows.astype(np.float64) * np.exp2(e)[:, None]).astype(np.float32)
    rows = np.ascontiguousarray(np.where(rows.any(axis=1, keepdims=True), rows, np.float32(nr.TINY)))
    rows[:3] = nr._cosine_specials(rng, 128)[[0, 2, 3]]
    _dense_check(COS, ids, rows, queries, "extreme corpus")


def test_dense_euclidean_at_two_to_the_minus_70():
    ids, rows, queries = nr.scaled_corpus(4000, 128, -70, 40, metric=EUC)
    _dense_check(EUC, ids, rows, queries, "euclidean at 2^-70")
