"""Resident candidate sets (hx_candidates_make_resident) and the stream-ordered entry hx_search_dense_restricted_set_device.

A resident set keeps its present slots, bf16 tile, row terms and view word across calls.  Its answers must be the answers of
the same ids through a non-resident set bit for bit (ids, order, score bits, counts, and `how` for the exact entry), on every
shape, metric and set kind, after row writes, and from the stream-ordered entry.
"""
import threading
import time

import numpy as np
import pytest

import helix_db_b200 as hx
from oracle import hxo
from test_gpu_dense import assert_same, dense_index
from test_gpu_dense_exact import hazard_fixture
from test_gpu_dense_restricted import make_set

import numeric_range as nr

pytestmark = pytest.mark.gpu
EUC, COS = hxo.EUCLIDEAN, hxo.COSINE
Cands = hx.RestrictedVectorCandidates


def min_rows(k):
    return 8 * min(max(4 * k, 64), 800)


def resident_bytes(present, dim):
    ldb = (dim + 63) // 64 * 64
    n_pad = (present + 255) // 256 * 256
    return 0 if present == 0 else n_pad * (2 * ldb + 4) + 4 * present + 4


def sets_of(gpu, cand):
    """(plain, resident) device sets over the same ids."""
    return gpu.cache_candidates(Cands(cand)), gpu.cache_candidates(Cands(cand)).make_resident()


def check_resident(gpu, queries, k, cand, what):
    """The resident set entry equals a non-resident set over the same ids; the resident exact entry equals
    search_restricted_sets, with the non-resident exact entry's `how`.  Returns that `how`."""
    p = hx.SearchParams.strict(k)
    plain, res = sets_of(gpu, cand)
    assert_same(gpu.search_dense_restricted_sets(queries, p, res), gpu.search_dense_restricted_sets(queries, p, plain),
                what + ": plain entry")
    got = gpu.search_dense_restricted_exact_sets(queries, p, res)
    assert_same(got[:3], gpu.search_restricted_sets(queries, p, plain), what + ": exact entry")
    assert got[3].tolist() == gpu.search_dense_restricted_exact_sets(queries, p, plain)[3].tolist(), what + ": how"
    plain.close()
    res.close()
    return got[3]


def device_search(gpu, queries, k, dset, stream=None):
    """hx_search_dense_restricted_set_device on a torch side stream: (ids, scores, counts, how)."""
    import torch
    B = len(queries)
    dq = torch.from_numpy(np.ascontiguousarray(queries)).cuda()
    di = torch.zeros((B, k), dtype=torch.int64, device="cuda")
    ds = torch.zeros((B, k), dtype=torch.float32, device="cuda")
    dc = torch.zeros(B, dtype=torch.int32, device="cuda")
    dh = torch.full((B,), 255, dtype=torch.uint8, device="cuda")
    s = stream if stream is not None else torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        gpu.search_dense_restricted_set_device(dq.data_ptr(), B, hx.SearchParams.strict(k), dset, di.data_ptr(), ds.data_ptr(),
                                               dc.data_ptr(), dh.data_ptr(), s.cuda_stream)
    s.synchronize()
    return di.cpu().numpy().view(np.uint64), ds.cpu().numpy(), dc.cpu().numpy().view(np.uint32), dh.cpu().numpy()


# ---- bit-identity: d 8 / 65 / 768 / 1536, B 1 / 129 / 1500, k 1 / 10 / 800, every set kind, both metrics ------------------------
CASES = [(EUC, 20011, 8, 129, 10, "random10"), (COS, 30007, 65, 1500, 1, "range"), (EUC, 9001, 768, 1, 10, "all"),
         (COS, 12007, 1536, 129, 10, "mixed"), (EUC, 80021, 64, 8, 800, "random10"), (COS, 30011, 65, 129, 800, "range"),
         (COS, 20077, 768, 1500, 10, "random10"), (EUC, 4001, 8, 1500, 1, "all"), (EUC, 12007, 1536, 1, 1, "mixed"),
         (COS, 9001, 8, 1, 800, "all")]


@pytest.mark.parametrize("om,n,dim,B,k,kind", CASES)
def test_resident_set_returns_the_same_bits(om, n, dim, B, k, kind):
    rng = np.random.default_rng(n * 7 + dim + B)
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    queries = rng.standard_normal((B, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64) * 3 + 11
    cand = make_set(kind, ids, rng)
    gpu = dense_index(om, ids, rows)
    how = check_resident(gpu, queries, k, cand, f"case {om, n, dim, B, k, kind}")
    assert set(how.tolist()) <= ({0, 1} if np.isin(ids, cand).sum() >= min_rows(k) else {2})
    gpu.close()


@pytest.mark.parametrize("om,k,present", [(EUC, 10, 511), (COS, 10, 512), (COS, 800, 6399), (EUC, 800, 6400)])
def test_sets_at_the_dense_minimum(om, k, present):
    rng = np.random.default_rng(present + k)
    n, dim, B = 9000, 24, 33
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    queries = rng.standard_normal((B, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64) * 2 + 1
    pick = np.sort(rng.choice(ids, size=present, replace=False))
    cand = np.unique(np.concatenate([pick, pick[: present // 2] + np.uint64(1)]))   # absent ids do not count as present
    gpu = dense_index(om, ids, rows)
    how = check_resident(gpu, queries, k, cand, f"{present} present, k = {k}")
    assert (how == 2).all() == (present < min_rows(k))
    gpu.close()


@pytest.mark.parametrize("om", [EUC, COS])
def test_storage_zero(om):
    rng = np.random.default_rng(31 + om)
    n, dim, B, k = 25000, 96, 200, 10
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    queries = rng.standard_normal((B, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64) * 3 + 11
    plain = hx.VectorIndex(hx.Metric.Euclidean if om == EUC else hx.Metric.Cosine,
                           hx.VectorIndexConfig("s0", "embedding", dim), storage=0)
    plain.load_vectors(ids, rows)
    plain.load_graph(0, ids[:1], [0, 0], [])
    plain.set_entry(int(ids[0]), 0)
    for kind in ("random10", "mixed"):
        check_resident(plain, queries, k, make_set(kind, ids, rng), f"storage 0, {kind}")
    plain.close()


# ---- the certificate and the hazards ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["stride4", "run48"])
@pytest.mark.parametrize("om", [COS, EUC])
def test_hazards_through_a_resident_set(kind, om):
    pytest.importorskip("torch")
    ids, rows, queries, nh = hazard_fixture(kind, om)
    gpu = dense_index(om, ids, rows)
    k = 10
    how = check_resident(gpu, queries, k, ids, f"{kind} {om}")
    assert (how[:nh] == 1).all(), how[:nh]
    res = gpu.cache_candidates(Cands(ids)).make_resident()
    got = device_search(gpu, queries, k, res)
    assert got[3].tolist() == how.tolist(), "the device entry marks the queries the exact entry rescans"
    assert_same(got[:3], gpu.search_dense_restricted_sets(queries, hx.SearchParams.strict(k), res), "device = host entry")
    res.close()
    gpu.close()


# ---- stats ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("om", [EUC, COS])
def test_stats_drop_exactly_the_per_call_view_work(om):
    rng = np.random.default_rng(5 + om)
    n, dim, B, k = 30000, 96, 200, 10
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    queries = rng.standard_normal((B, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64) * 2 + 1
    cand = make_set("mixed", ids, rng)
    present = int(np.isin(ids, cand).sum())
    ldb = (dim + 63) // 64 * 64
    gather = present * (4 * dim + 2 * ldb + 4)
    gpu = dense_index(om, ids, rows)
    plain, res = sets_of(gpu, cand)
    p = hx.SearchParams.strict(k)
    sp, sr = hx.SearchStats(), hx.SearchStats()
    assert_same(gpu.search_dense_restricted_sets(queries, p, res, stats=sr),
                gpu.search_dense_restricted_sets(queries, p, plain, stats=sp), "plain")
    assert sp.kernel_launches - sr.kernel_launches == 3   # k_compact_count, k_compact_scatter, k_to_bf16
    assert sr.algorithmic_bytes == present * 2 * ldb and sp.algorithmic_bytes == gather + present * 2 * ldb
    assert (sr.distance_computations, sr.reserved) == (sp.distance_computations, sp.reserved)
    sp, sr = hx.SearchStats(), hx.SearchStats()
    hr = gpu.search_dense_restricted_exact_sets(queries, p, res, stats=sr)[3]
    hp = gpu.search_dense_restricted_exact_sets(queries, p, plain, stats=sp)[3]
    assert hr.tolist() == hp.tolist()
    assert sp.kernel_launches - sr.kernel_launches == 4   # ... and k_dense_view_bound
    rescans = int((hr == 1).sum()) * present * (4 * dim + (4 if om == COS else 0))
    assert sr.algorithmic_bytes == present * 2 * ldb + rescans and sp.algorithmic_bytes == gather + sr.algorithmic_bytes
    plain.close()
    res.close()
    gpu.close()


# ---- staleness ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("om", [EUC, COS])
def test_row_writes_refresh_the_view(om):
    rng = np.random.default_rng(11 + om)
    n, dim, B, k = 20000, 64, 64, 10
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    queries = rng.standard_normal((B, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64) * 2 + 1
    cand = make_set("random10", ids, rng)
    gpu = dense_index(om, ids, rows)
    p = hx.SearchParams.strict(k)
    res = gpu.cache_candidates(Cands(cand)).make_resident()
    before = gpu.search_dense_restricted_sets(queries, p, res)
    # a row outside the set, made query 0's twin: the answer does not move
    outside = ids[~np.isin(ids, cand)][:1]
    gpu.upsert_vectors(outside, queries[:1])
    assert_same(gpu.search_dense_restricted_sets(queries, p, res), before, "upsert outside the set")
    # a row of the set, made query 0's twin: it is the next call's nearest row
    inside = cand[len(cand) // 2:len(cand) // 2 + 1]
    gpu.upsert_vectors(inside, queries[:1])
    got = gpu.search_dense_restricted_sets(queries, p, res)
    assert int(got[0][0, 0]) == int(inside[0])
    fresh = gpu.cache_candidates(Cands(cand))
    assert_same(got, gpu.search_dense_restricted_sets(queries, p, fresh), "upsert inside the set")
    assert_same(gpu.search_dense_restricted_exact_sets(queries, p, res)[:3], gpu.search_restricted_sets(queries, p, fresh),
                "exact entry after the upsert")
    # delete, then reload: both sets are refused
    gpu.delete_vectors(ids[-1:])
    for _ in range(2):
        for s in (res, fresh):
            for fn in (gpu.search_dense_restricted_sets, gpu.search_dense_restricted_exact_sets):
                with pytest.raises(hx.HelixDbError) as e:
                    fn(queries, p, s)
                assert e.value.code == hx.HX_ERR_INVARIANT_VIOLATION
        gpu.load_vectors(ids, rows)
    res.close()
    fresh.close()
    gpu.close()


def test_concurrent_first_calls_after_an_upsert():
    rng = np.random.default_rng(8)
    n, dim, B, k = 40000, 128, 150, 10
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    queries = rng.standard_normal((B, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64) * 3 + 1
    cand = make_set("random10", ids, rng)
    gpu = dense_index(EUC, ids, rows)
    p = hx.SearchParams.strict(k)
    res = gpu.cache_candidates(Cands(cand)).make_resident()
    gpu.search_dense_restricted_sets(queries, p, res)
    twins = np.sort(rng.choice(cand, size=B, replace=False))
    gpu.upsert_vectors(twins, queries + np.float32(1e-3))
    fresh = gpu.cache_candidates(Cands(cand))
    want = gpu.search_dense_restricted_sets(queries, p, fresh)
    results, errors = [None] * 8, []

    def worker(t):
        try:
            results[t] = gpu.search_dense_restricted_sets(queries, p, res)
        except Exception as e:   # reported below
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(8)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for t in range(8):
        assert_same(results[t], want, f"thread {t}")
    res.close()
    fresh.close()
    gpu.close()


# ---- the stream-ordered entry ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("om", [EUC, COS])
def test_device_entry_matches_the_host_entry(om):
    pytest.importorskip("torch")
    rng = np.random.default_rng(21 + om)
    n, dim, B, k = 30000, 96, 129, 10
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    queries = rng.standard_normal((B, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64) * 3 + 11
    gpu = dense_index(om, ids, rows)
    p = hx.SearchParams.strict(k)
    for cand, small in ((make_set("mixed", ids, rng), False), (np.sort(rng.choice(ids, size=300, replace=False)), True)):
        plain, res = sets_of(gpu, cand)
        got = device_search(gpu, queries, k, res)
        assert_same(got[:3], gpu.search_dense_restricted_sets(queries, p, res), f"small={small}")
        if small:
            assert (got[3] == 2).all()
        else:
            assert set(got[3].tolist()) <= {0, 1} and (got[3] == 0).mean() >= 0.5
            assert got[3].tolist() == gpu.search_dense_restricted_exact_sets(queries, p, res)[3].tolist()
        exact = gpu.search_restricted_sets(queries, p, plain)   # a certified query's answer is the exact scan's
        c = np.flatnonzero(got[3] != 1)
        assert_same((got[0][c], got[1][c], got[2][c]), (exact[0][c], exact[1][c], exact[2][c]), "certified = exact")
        plain.close()
        res.close()
    gpu.close()


def test_device_entry_does_not_synchronise():
    """After a warm call, ~200 ms of device work is queued on the stream in front of the call: the call must return to the
    host long before that work ends."""
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(9)
    n, dim, B, k = 20000, 64, 64, 10
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    queries = rng.standard_normal((B, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64)
    gpu = dense_index(COS, ids, rows)
    res = gpu.cache_candidates(Cands(ids[::3])).make_resident()
    s = torch.cuda.Stream()
    want = device_search(gpu, queries, k, res, s)   # warm: scratch, tensor maps, kernel attributes
    dq = torch.from_numpy(queries).cuda()
    di = torch.zeros((B, k), dtype=torch.int64, device="cuda")
    ds = torch.zeros((B, k), dtype=torch.float32, device="cuda")
    dc = torch.zeros(B, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(400_000_000)   # a bounded spin of ~0.2 s at H100 clocks
        t0 = time.perf_counter()
        gpu.search_dense_restricted_set_device(dq.data_ptr(), B, hx.SearchParams.strict(k), res, di.data_ptr(),
                                               ds.data_ptr(), dc.data_ptr(), None, s.cuda_stream)
        t_call = time.perf_counter() - t0
    s.synchronize()
    t_all = time.perf_counter() - t0
    assert t_all > 0.1, t_all
    assert t_call < 0.25 * t_all, (t_call, t_all)
    got = (di.cpu().numpy().view(np.uint64), ds.cpu().numpy(), dc.cpu().numpy().view(np.uint32))
    assert_same(got, want[:3], "after the spin")
    res.close()
    gpu.close()


# ---- the float32 range --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("om", [COS, EUC])
def test_float32_range_through_a_resident_set(om):
    for d in nr.DIMS:
        ids, rows, queries = nr.corpus(om, d, n_rows=1400, n_queries=40)
        rng = np.random.default_rng(d)
        cand = np.union1d(np.sort(rng.choice(ids, size=len(ids) * 3 // 4, replace=False)), ids[-3 * len(queries):])
        gpu = dense_index(om, ids, rows)
        for k in (1, 5):
            check_resident(gpu, queries, k, cand, f"range {om} d={d} k={k}")
        gpu.close()


# ---- admission, memory ----------------------------------------------------------------------------------------------------------
def _code(fn):
    try:
        fn()
    except hx.HelixDbError as e:
        return e.code
    return hx.HX_OK


def test_make_resident_admission_and_bytes():
    rng = np.random.default_rng(3)
    n, dim = 3000, 40
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64) * 2
    L = hx.load_library()
    gpu = dense_index(COS, ids, rows)
    s = gpu.cache_candidates(Cands(np.union1d(ids[::2], ids[:40] + np.uint64(1))))   # 1500 present, 40 absent
    assert L.hx_candidates_make_resident(None, s.h) == hx.HX_ERR_INVALID_PARAMETER
    assert L.hx_candidates_make_resident(gpu.h, None) == hx.HX_ERR_INVALID_PARAMETER
    assert L.hx_candidates_resident_bytes(None) == 0
    assert s.resident_bytes == 0
    s.make_resident()
    assert s.resident_bytes == resident_bytes(1500, dim)
    s.make_resident()   # a no-op
    assert s.resident_bytes == resident_bytes(1500, dim)
    for cand in (np.zeros(0, np.uint64), ids[:10] + np.uint64(1)):   # empty, and nothing present
        e = gpu.cache_candidates(Cands(cand)).make_resident()
        assert e.resident_bytes == 0
        e.close()
    # Manhattan before anything about the set, then a set of another index or of an older generation
    l1 = hx.VectorIndex(hx.Metric.Manhattan, hx.VectorIndexConfig("l1", "embedding", dim))
    l1.load_vectors(ids, rows)
    mine = l1.cache_candidates(Cands(ids[:10]))
    assert _code(mine.make_resident) == hx.HX_ERR_UNSUPPORTED
    assert L.hx_candidates_make_resident(l1.h, s.h) == hx.HX_ERR_UNSUPPORTED
    mine.close()
    l1.close()
    other = dense_index(COS, ids, rows, "other")
    foreign = other.cache_candidates(Cands(ids[:100]))
    assert L.hx_candidates_make_resident(gpu.h, foreign.h) == hx.HX_ERR_INVARIANT_VIOLATION
    foreign.close()
    other.close()
    stale = gpu.cache_candidates(Cands(ids[:600]))
    gpu.delete_vectors(ids[-1:])
    assert _code(stale.make_resident) == hx.HX_ERR_INVARIANT_VIOLATION
    stale.close()
    s.close()
    gpu.close()


def test_device_entry_admission_order():
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(4)
    n, dim, B = 3000, 32, 3
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64) * 2
    gpu = dense_index(COS, ids, rows)
    dq = torch.from_numpy(rng.standard_normal((B, dim), dtype=np.float32)).cuda()
    di = torch.zeros((B, 1000), dtype=torch.int64, device="cuda")
    ds = torch.zeros((B, 1000), dtype=torch.float32, device="cuda")
    dc = torch.full((B,), 7, dtype=torch.int32, device="cuda")
    dh = torch.zeros(B, dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()

    def call(ix, dset, k=10, b=B, q=dq.data_ptr()):
        def run():
            ix.search_dense_restricted_set_device(q, b, hx.SearchParams.strict(k), dset, di.data_ptr(), ds.data_ptr(),
                                                  dc.data_ptr(), dh.data_ptr(), s.cuda_stream)
            s.synchronize()
        return _code(run)

    plain = gpu.cache_candidates(Cands(ids[::2]))
    res = gpu.cache_candidates(Cands(ids[::2])).make_resident()
    empty = gpu.cache_candidates(Cands(np.zeros(0, np.uint64)))
    assert call(gpu, plain, k=0) == hx.HX_ERR_INVALID_PARAMETER     # params first
    assert call(gpu, plain, b=0) == hx.HX_OK                        # B = 0
    assert call(gpu, plain, q=None) == hx.HX_ERR_INVALID_PARAMETER  # null pointers
    assert call(gpu, empty) == hx.HX_OK                             # an empty set: counts 0, resident or not
    assert dc.cpu().tolist() == [0] * B and dh.cpu().tolist() == [2] * B
    assert call(gpu, plain, k=900) == hx.HX_ERR_QUERY               # min(k, |C|) > 800
    other = dense_index(COS, ids, rows, "other")
    foreign = other.cache_candidates(Cands(ids[:1000])).make_resident()
    assert call(gpu, foreign) == hx.HX_ERR_INVARIANT_VIOLATION      # a set of another index ...
    assert call(gpu, plain) == hx.HX_ERR_INVALID_PARAMETER          # ... then not resident
    assert call(gpu, res) == hx.HX_OK
    assert dc.cpu().tolist() == [10] * B
    foreign.close()
    other.close()
    l1 = hx.VectorIndex(hx.Metric.Manhattan, hx.VectorIndexConfig("l1", "embedding", dim))
    l1.load_vectors(ids, rows)
    l1_set = l1.cache_candidates(Cands(np.zeros(0, np.uint64)))
    assert call(l1, l1_set) == hx.HX_ERR_UNSUPPORTED                # Manhattan before anything about the set
    l1_set.close()
    l1.close()
    gpu.delete_vectors(ids[-1:])
    assert call(gpu, res) == hx.HX_ERR_INVARIANT_VIOLATION          # an older generation
    for x in (plain, res, empty):
        x.close()
    gpu.close()
