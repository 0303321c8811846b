"""hx_search_dense_restricted[_set]: the tensor-core path over one candidate set shared by the B queries.

The contract is hx_search_dense's over the sub-corpus C ∩ live rows: the answer for a set C must pass what
check_against_reference demands of an index that holds only the present rows of C (exact score bits, (score, id) order,
count min(k, present), every sure row returned).  Below 8 * min(max(4k, 64), 800) present rows the call runs the exact scan
and must return hx_search_restricted's answer bit for bit.
"""
import threading

import numpy as np
import pytest

import helix_db_b200 as hx
from oracle import hxo
from test_dense_reference import tie_fixture
from test_gpu_dense import GPU_METRIC, assert_same, check_against_reference, dense_index, oracle_of

import numeric_range as nr

pytestmark = pytest.mark.gpu
EUC, COS = hxo.EUCLIDEAN, hxo.COSINE
Cands = hx.RestrictedVectorCandidates


def min_rows(k):
    return 8 * min(max(4 * k, 64), 800)


def present_of(ids, rows, cand):
    """The rows of the candidate ids the index holds (ids ascending)."""
    keep = np.isin(ids, cand)
    return ids[keep], rows[keep]


def dense_restricted(gpu, queries, k, cand):
    st = hx.SearchStats()
    got = gpu.search_dense_restricted_batch(queries, hx.SearchParams.strict(k), Cands(cand), stats=st)
    return got, st


def make_set(kind, ids, rng):
    n = len(ids)
    if kind == "random10":
        return np.sort(rng.choice(ids, size=n // 10, replace=False))
    if kind == "range":
        a = n // 5
        return ids[a:a + n // 3].copy()
    if kind == "all":
        return ids.copy()
    # a random 30 % mixed with as many ids the index does not hold (ids are 3 i + 11: ids + 1 are never rows)
    part = rng.choice(ids, size=3 * n // 10, replace=False)
    return np.unique(np.concatenate([part, part + np.uint64(1)]))


# ---- nomination against the float64 reference, on the sub-corpus ---------------------------------------------------------------
# dims 8 / 65 / 768 / 1536, B across one and several 128-query tiles and above 1024, k up to 800; n off the tile size
CASES = [(EUC, 20011, 8, 129, 10, "random10"), (COS, 30007, 65, 1500, 1, "range"), (EUC, 9001, 768, 1, 10, "all"),
         (COS, 12007, 1536, 129, 10, "mixed"), (EUC, 80021, 64, 8, 800, "random10"), (COS, 20077, 768, 300, 10, "random10"),
         (EUC, 30011, 65, 129, 800, "range"), (COS, 4001, 8, 1500, 1, "all")]


@pytest.mark.parametrize("om,n,dim,B,k,kind", CASES)
def test_dense_restricted_nominates_every_sure_row(om, n, dim, B, k, kind):
    rng = np.random.default_rng(n * 7 + dim + B)
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    queries = rng.standard_normal((B, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64) * 3 + 11
    cand = make_set(kind, ids, rng)
    pid, prow = present_of(ids, rows, cand)
    assert len(pid) >= min_rows(k), "the case must reach the tensor-core pass"
    gpu = dense_index(om, ids, rows)
    got, st = dense_restricted(gpu, queries, k, cand)
    assert st.reserved > 0 and st.distance_computations == B * len(pid), "the tensor-core pass ran over the present rows"
    covered = check_against_reference(om, pid, prow, queries, k, got)
    assert covered >= 0.75, f"only {covered:.2f} of the queries have their exact top-{min(k, 4)} rows sure"
    gpu.close()


# ---- small sets: the exact scan, hx_search_restricted's answer ------------------------------------------------------------------
@pytest.mark.parametrize("om,k,present", [(EUC, 10, 511), (COS, 10, 512), (COS, 10, 1), (EUC, 10, 7), (EUC, 1000, 500),
                                          (COS, 200, 6399), (EUC, 200, 6400)])
def test_small_sets_follow_the_exact_scan(om, k, present):
    rng = np.random.default_rng(present + k)
    n, dim, B = 9000, 24, 33
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    queries = rng.standard_normal((B, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64) * 2 + 1
    pick = np.sort(rng.choice(ids, size=present, replace=False))
    cand = np.unique(np.concatenate([pick, pick[: present // 2] + np.uint64(1)]))   # absent ids do not count as present
    gpu = dense_index(om, ids, rows)
    got, st = dense_restricted(gpu, queries, k, cand)
    assert got[2].tolist() == [min(k, present)] * B
    if present < min_rows(k):
        assert st.reserved == 0
        assert_same(got, gpu.search_restricted_batch(queries, hx.SearchParams.strict(k), Cands(cand)), f"{present} present")
    else:
        assert st.reserved > 0
        check_against_reference(om, *present_of(ids, rows, cand), queries, k, got)
    gpu.close()


# ---- the set entry, and storage 0 -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("om", [EUC, COS])
def test_set_entry_and_storage_zero_return_the_same_bits(om):
    rng = np.random.default_rng(31 + om)
    n, dim, B, k = 25000, 96, 200, 10
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    queries = rng.standard_normal((B, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64) * 3 + 11
    for kind in ("random10", "mixed"):
        cand = make_set(kind, ids, rng)
        gpu = dense_index(om, ids, rows)
        want, _ = dense_restricted(gpu, queries, k, cand)
        s = gpu.cache_candidates(Cands(cand))
        assert_same(gpu.search_dense_restricted_sets(queries, hx.SearchParams.strict(k), s), want, f"{kind}: set entry")
        s.close()
        gpu.close()
        plain = hx.VectorIndex(GPU_METRIC[om], hx.VectorIndexConfig("s0", "embedding", dim), storage=0)
        plain.load_vectors(ids, rows)
        plain.load_graph(0, ids[:1], [0, 0], [])
        plain.set_entry(int(ids[0]), 0)
        assert_same(dense_restricted(plain, queries, k, cand)[0], want, f"{kind}: storage 0")
        s0 = plain.cache_candidates(Cands(cand))
        assert_same(plain.search_dense_restricted_sets(queries, hx.SearchParams.strict(k), s0), want, f"{kind}: storage 0 set")
        s0.close()
        plain.close()


# ---- absent and deleted rows ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("om", [EUC, COS])
def test_deleted_and_absent_rows_are_never_returned(om):
    rng = np.random.default_rng(41 + om)
    n, dim, B, k = 30000, 16, 64, 10
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    queries = rng.standard_normal((B, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64) * 3 + 5
    cand = make_set("mixed", ids, rng)
    gpu = dense_index(om, ids, rows)
    old = gpu.cache_candidates(Cands(cand))
    dense_restricted(gpu, queries, k, cand)
    pid, prow = present_of(ids, rows, cand)
    nn, _, _, _ = oracle_of(om, pid, prow).search_exact_batch(queries, 1, threads=8)
    dead = set(nn[:, 0].tolist()) | set(rng.choice(pid, size=len(pid) // 3, replace=False).tolist())
    dead.discard(int(ids[0]))
    dead = np.array(sorted(dead), dtype=np.uint64)
    gpu.delete_vectors(dead)
    with pytest.raises(hx.HelixDbError) as e:   # the set was mapped before the deletion
        gpu.search_dense_restricted_sets(queries, hx.SearchParams.strict(k), old)
    assert e.value.code == hx.HX_ERR_INVARIANT_VIOLATION
    old.close()
    live = ~np.isin(pid, dead)
    got, st = dense_restricted(gpu, queries, k, cand)
    assert st.reserved > 0
    assert not set(got[0][:, :k].ravel().tolist()) & set(dead.tolist()), "a deleted row was returned"
    assert not set(got[0][:, :k].ravel().tolist()) - set(pid.tolist()) - {0}, "an absent id was returned"
    check_against_reference(om, pid[live], prow[live], queries, k, got)
    fresh = gpu.cache_candidates(Cands(cand))
    assert_same(gpu.search_dense_restricted_sets(queries, hx.SearchParams.strict(k), fresh), got, "fresh set after deletes")
    fresh.close()
    gpu.close()


def test_mostly_deleted_set_keeps_its_count():
    """A set of 20 000 ids of which 600 survive, all packed into the first tiles of the gathered tile: the count is
    min(k, survivors) and the answer the exact scan's."""
    rng = np.random.default_rng(6)
    n, dim, B, k = 40000, 32, 17, 100
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    queries = rng.standard_normal((B, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64)
    cand = ids[10000:30000]
    keep = np.sort(rng.choice(cand, size=600, replace=False))
    gpu = dense_index(EUC, ids, rows)
    dead = cand[~np.isin(cand, keep)]
    gpu.delete_vectors(dead)
    got, _ = dense_restricted(gpu, queries, k, cand)
    assert got[2].tolist() == [k] * B
    oi, os_, oc, _ = oracle_of(EUC, keep, rows[keep.astype(np.int64)]).search_exact_batch(queries, k, threads=8)
    assert_same(got, (oi, os_, oc), "survivors of a mostly deleted set")
    # ... and at k = 10 the 600 survivors reach the tensor-core pass
    got, st = dense_restricted(gpu, queries, 10, cand)
    assert st.reserved > 0 and got[2].tolist() == [10] * B
    check_against_reference(EUC, keep, rows[keep.astype(np.int64)], queries, 10, got)
    gpu.close()


# ---- exact ties -------------------------------------------------------------------------------------------------------------
def test_exact_ties_resolve_by_id_inside_a_set():
    ids, rows, q, tied = tie_fixture()
    k = 10
    rng = np.random.default_rng(12)
    cand = np.unique(np.concatenate([tied, rng.choice(ids, size=1500, replace=False)]))
    gpu = dense_index(EUC, ids, rows)
    (di, ds, dc), st = dense_restricted(gpu, q[None, :], k, cand)
    assert st.reserved > 0
    oi, os_ = oracle_of(EUC, *present_of(ids, rows, cand)).search_exact(q, k)
    assert oi.tolist() == tied[:k].tolist()
    assert int(dc[0]) == k
    assert di[0].tolist() == tied[:k].tolist(), "tied rows must come in id order, and the smallest ids must make the cut"
    assert ds[0].view(np.uint32).tolist() == os_.view(np.uint32).tolist()
    gpu.close()


# ---- neighbours clustered by candidate rank -----------------------------------------------------------------------------------
def test_rank_clustered_neighbours_are_all_returned():
    """40 near-duplicates of each query sit at consecutive ranks of the set (interleaved with non-candidates in id space).
    The tile placement spreads consecutive ranks over the four column quarters (at most 3 of the 10 nearest in any
    bucket), so every sure row comes back and the top 10 are the exact scan's; placed in rank order, one bucket would hold
    all 10 and keep 8."""
    rng = np.random.default_rng(77)
    n, dim, k, nh = 60000, 64, 10, 8
    rows = rng.standard_normal((n, dim)).astype(np.float32)
    hq = rng.standard_normal((nh, dim)).astype(np.float32)
    ids = np.arange(n, dtype=np.uint64)
    cand = ids[::2].copy()                           # candidate rank r is id 2 r
    for h in range(nh):
        r0 = 3000 * h + 100                          # ranks r0 .. r0 + 39
        for i in range(40):
            rows[2 * (r0 + i)] = hq[h] + np.float32(0.01 * (i + 1)) * rng.standard_normal(dim).astype(np.float32)
    gpu = dense_index(EUC, ids, rows)
    got, st = dense_restricted(gpu, hq, k, cand)
    assert st.reserved > 0
    pid, prow = present_of(ids, rows, cand)
    oi, os_, oc, _ = oracle_of(EUC, pid, prow).search_exact_batch(hq, k)
    for h in range(nh):
        assert set(oi[h].tolist()) <= {2 * (3000 * h + 100 + i) for i in range(40)}   # the fixture is what it claims
    check_against_reference(EUC, pid, prow, hq, k, got)
    assert_same(got, (oi, os_, oc), "rank-clustered neighbours")
    gpu.close()


# ---- the float32 range ------------------------------------------------------------------------------------------------------
def _range_check(om, ids, rows, queries, cand, what, k=10, floor=0.5):
    gpu = dense_index(om, ids, rows)
    got, st = dense_restricted(gpu, queries, k, cand)
    gpu.close()
    pid, prow = present_of(ids, rows, cand)
    if len(pid) >= min_rows(k):
        assert st.reserved > 0
    covered = check_against_reference(om, pid, prow, queries, k, got)
    assert covered >= floor, f"{what}: only {covered:.2f} of the queries have their exact top-{min(k, 4)} rows sure"


def test_extreme_scale_cosine_fixture_on_a_subset():
    ids, rows, queries = nr.corpus(COS, 768, n_rows=1400, n_queries=40)
    rng = np.random.default_rng(5)
    cand = np.sort(rng.choice(ids, size=len(ids) // 2, replace=False))
    _range_check(COS, ids, rows, queries, cand, "cosine fixture subset")


def test_extreme_queries_on_an_order_one_subset():
    ids, rows, _ = nr.scaled_corpus(8000, 128, 0, 40)
    rng = np.random.default_rng(3)
    cand = np.sort(rng.choice(ids, size=4000, replace=False))
    sel = rng.choice(np.searchsorted(ids, cand), size=45, replace=False)
    e = np.resize(np.array(nr.EXPONENTS, np.float64), 45)
    queries = (rows[sel].astype(np.float64) * np.exp2(e)[:, None]).astype(np.float32)   # its own row is the nearest
    queries = np.concatenate([queries, nr.cosine_queries(5, 128)])
    _range_check(COS, ids, rows, queries, cand, "extreme queries")


def test_order_one_queries_on_an_extreme_subset():
    ids, rows, queries = nr.scaled_corpus(8000, 128, 0, 40)
    rng = np.random.default_rng(4)
    e = rng.choice(nr.EXPONENTS, size=len(rows)).astype(np.float64)
    rows = (rows.astype(np.float64) * np.exp2(e)[:, None]).astype(np.float32)
    rows = np.ascontiguousarray(np.where(rows.any(axis=1, keepdims=True), rows, np.float32(nr.TINY)))
    rows[:3] = nr._cosine_specials(rng, 128)[[0, 2, 3]]
    cand = np.union1d(np.sort(rng.choice(ids, size=4000, replace=False)), ids[:3])
    _range_check(COS, ids, rows, queries, cand, "extreme corpus")


def test_euclidean_at_two_to_the_minus_70_on_a_subset():
    ids, rows, queries = nr.scaled_corpus(8000, 128, -70, 40, metric=EUC)
    rng = np.random.default_rng(70)
    cand = np.sort(rng.choice(ids, size=5000, replace=False))
    _range_check(EUC, ids, rows, queries, cand, "euclidean at 2^-70")


# ---- admission --------------------------------------------------------------------------------------------------------------
def _code(fn):
    try:
        fn()
    except hx.HelixDbError as e:
        return e.code
    return hx.HX_OK


def test_admission_order():
    rng = np.random.default_rng(3)
    n, dim, k = 3000, 32, 10
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64) * 2
    gpu = dense_index(COS, ids, rows)
    q = rng.standard_normal((3, dim), dtype=np.float32)
    nan = q.copy()
    nan[1, 7] = np.nan
    p = hx.SearchParams.strict(k)
    empty = Cands(np.zeros(0, np.uint64))
    # B = 0
    got = gpu.search_dense_restricted_batch(np.zeros((0, dim), np.float32), p, Cands(ids[:10]))
    assert got[2].size == 0
    # an empty set: counts 0 without validating the queries
    got = gpu.search_dense_restricted_batch(nan, p, empty)
    assert got[2].tolist() == [0, 0, 0]
    # |C| > 1e6 is Query
    assert _code(lambda: gpu.search_dense_restricted_batch(q, p, Cands(np.arange(1_000_001, dtype=np.uint64)))) == hx.HX_ERR_QUERY
    # min(k, |C|) > 800 is Query; k is clamped to |C|
    assert _code(lambda: gpu.search_dense_restricted_batch(q, hx.SearchParams.strict(900), Cands(ids[:1000]))) == hx.HX_ERR_QUERY
    got = gpu.search_dense_restricted_batch(q, hx.SearchParams.strict(1000), Cands(ids[:500]))
    assert got[0].shape == (3, 1000) and got[2].tolist() == [500] * 3
    # not ascending / not unique
    assert _code(lambda: gpu.search_dense_restricted_batch(q, p, Cands(ids[[5, 3, 9]]))) == hx.HX_ERR_INVALID_PARAMETER
    assert _code(lambda: gpu.search_dense_restricted_batch(q, p, Cands(ids[[3, 3, 9]]))) == hx.HX_ERR_INVALID_PARAMETER
    # ... checked before the queries
    assert _code(lambda: gpu.search_dense_restricted_batch(nan, p, Cands(ids[[5, 3, 9]]))) == hx.HX_ERR_INVALID_PARAMETER
    # a NaN query with a non-empty set, on both paths (small set / tensor-core pass), and with only absent ids
    for cand in (ids[:10], ids[::2], ids[:10] + np.uint64(1)):
        assert _code(lambda: gpu.search_dense_restricted_batch(nan, p, Cands(cand))) == hx.HX_ERR_INVALID_VECTOR_COMPONENT
        big = np.tile(nan, (5, 1))   # B > 8: validated on the device
        assert _code(lambda: gpu.search_dense_restricted_batch(big, p, Cands(cand))) == hx.HX_ERR_INVALID_VECTOR_COMPONENT
    zero = q.copy()
    zero[2] = 0
    assert _code(lambda: gpu.search_dense_restricted_batch(zero, p, Cands(ids[::2]))) == hx.HX_ERR_ZERO_NORM_COSINE
    # dimension
    p16 = hx.SearchParams.strict(k)
    p16.query_dimension = 16
    assert _code(lambda: gpu.search_dense_restricted_batch(q[:, :16].copy(), p16, Cands(ids[:10]))) == hx.HX_ERR_INVALID_DIMENSION
    # a set of another index, or of an older generation
    other = dense_index(COS, ids, rows, "other")
    foreign = other.cache_candidates(Cands(ids[:100]))
    assert _code(lambda: gpu.search_dense_restricted_sets(q, p, foreign)) == hx.HX_ERR_INVARIANT_VIOLATION
    foreign.close()
    other.close()
    # an unpopulated index (vectors, no entry point) and an empty index: counts 0 after validation
    bare = hx.VectorIndex(hx.Metric.Cosine, hx.VectorIndexConfig("bare", "embedding", dim))
    bare.load_vectors(ids, rows)
    assert bare.search_dense_restricted_batch(q, p, Cands(ids[::2]))[2].tolist() == [0, 0, 0]
    assert _code(lambda: bare.search_dense_restricted_batch(nan, p, Cands(ids[::2]))) == hx.HX_ERR_INVALID_VECTOR_COMPONENT
    bare.close()
    none = hx.VectorIndex(hx.Metric.Cosine, hx.VectorIndexConfig("none", "embedding", dim))
    assert none.search_dense_restricted_batch(q, p, Cands(ids[::2]))[2].tolist() == [0, 0, 0]
    assert _code(lambda: none.search_dense_restricted_batch(nan, p, Cands(ids[::2]))) == hx.HX_ERR_INVALID_VECTOR_COMPONENT
    none.close()
    gpu.close()
    # Manhattan: unsupported, even with an empty set
    l1 = hx.VectorIndex(hx.Metric.Manhattan, hx.VectorIndexConfig("l1", "embedding", dim))
    l1.load_vectors(ids, rows)
    l1.load_graph(0, ids[:1], [0, 0], [])
    l1.set_entry(int(ids[0]), 0)
    assert _code(lambda: l1.search_dense_restricted_batch(q, p, empty)) == hx.HX_ERR_UNSUPPORTED
    assert _code(lambda: l1.search_dense_restricted_batch(nan, p, Cands(ids[:10]))) == hx.HX_ERR_UNSUPPORTED
    assert _code(lambda: l1.search_dense_restricted_batch(q, p, Cands(np.arange(1_000_001, dtype=np.uint64)))) == \
        hx.HX_ERR_UNSUPPORTED
    l1.close()


# ---- sharing one handle -----------------------------------------------------------------------------------------------------
def test_alternating_entries_and_concurrent_callers():
    rng = np.random.default_rng(90)
    n, dim, B, k = 40000, 128, 150, 10
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    queries = rng.standard_normal((B, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64) * 3 + 1
    small = np.sort(rng.choice(ids, size=3000, replace=False))
    large = np.sort(rng.choice(ids, size=20000, replace=False))
    p = hx.SearchParams.strict(k)
    ref = dense_index(EUC, ids, rows, "ref")
    want = {"dense": ref.search_dense_batch(queries, p), "small": dense_restricted(ref, queries, k, small)[0],
            "large": dense_restricted(ref, queries, k, large)[0],
            "exact": ref.search_restricted_batch(queries, p, Cands(large))}
    ref.close()
    check_against_reference(EUC, *present_of(ids, rows, large), queries, k, want["large"])
    gpu = dense_index(EUC, ids, rows)
    calls = {"dense": lambda: gpu.search_dense_batch(queries, p), "small": lambda: dense_restricted(gpu, queries, k, small)[0],
             "large": lambda: dense_restricted(gpu, queries, k, large)[0],
             "exact": lambda: gpu.search_restricted_batch(queries, p, Cands(large))}
    for name in ["large", "dense", "small", "exact", "large", "small", "dense", "large"]:
        assert_same(calls[name](), want[name], f"alternating: {name}")
    results, errors = [None] * 8, []

    def worker(t):
        try:
            results[t] = dense_restricted(gpu, queries, k, large if t % 2 else small)[0]
        except Exception as e:   # reported below
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(8)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for t in range(8):
        assert_same(results[t], want["large" if t % 2 else "small"], f"thread {t}")
    gpu.close()
