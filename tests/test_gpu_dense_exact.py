"""hx_search_dense_exact / hx_search_dense_restricted_exact[_set]: the tensor-core path made exact by the certificate.

Every answer must be hx_search_restricted's over every live id (or over the set), bit for bit: ids, order, score bits and
count.  `how` says how each query was answered: 0 certified, 1 rescanned by the exact scan, 2 the view is below
hx_dense_min_rows(k) and the exact scan answered every query.  The hazards of DESIGN §8 (a full bucket holding more than
HXD_T true neighbours) must come back rescanned with the exact answer, where the plain entry loses neighbours.
"""
import numpy as np
import pytest

import helix_db_b200 as hx
from oracle import hxo
from test_dense_reference import tie_fixture
from test_gpu_dense import CASES, assert_same, dense_index

import numeric_range as nr

pytestmark = pytest.mark.gpu
EUC, COS = hxo.EUCLIDEAN, hxo.COSINE
Cands = hx.RestrictedVectorCandidates


def min_rows(k):
    return 8 * min(max(4 * k, 64), 800)


def exact_all(gpu, queries, k, live_ids):
    """The reference answer: the restricted exact scan over every live id."""
    return gpu.search_restricted_batch(queries, hx.SearchParams.strict(k), Cands(np.asarray(live_ids, np.uint64)))


def check_exact(gpu, queries, k, live_ids, what, n_slots=None):
    """n_slots: rows the index has ever held, deleted ones included (the plain entry's distance count is B * n_slots)."""
    st = hx.SearchStats()
    ids, sc, cnt, how = gpu.search_dense_exact_batch(queries, hx.SearchParams.strict(k), stats=st)
    assert_same((ids, sc, cnt), exact_all(gpu, queries, k, live_ids), what)
    small = len(live_ids) < min_rows(k)
    assert set(how.tolist()) <= ({2} if small else {0, 1}), (what, np.unique(how))
    if not small:   # a certified query's answer is the plain entry's
        pi, ps, pc = gpu.search_dense_batch(queries, hx.SearchParams.strict(k))
        c0 = np.flatnonzero(how == 0)
        assert_same((ids[c0], sc[c0], cnt[c0]), (pi[c0], ps[c0], pc[c0]), what + " (certified = plain)")
        assert st.kernel_launches > 0
        n_slots = len(live_ids) if n_slots is None else n_slots
        assert st.distance_computations == len(queries) * n_slots + int((how == 1).sum()) * len(live_ids)
    return how


# ---- random corpora of the plain path's shapes ---------------------------------------------------------------------------
@pytest.mark.parametrize("om,n,dim,B,k", CASES)
def test_exact_entry_is_the_exact_scan(om, n, dim, B, k):
    rng = np.random.default_rng(n * 7 + dim)
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    queries = rng.standard_normal((B, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64) * 3 + 11
    gpu = dense_index(om, ids, rows)
    how = check_exact(gpu, queries, k, ids, f"case {om, n, dim, B, k}")
    if n >= min_rows(k) and 4 * k <= 800:   # k' = 4k nominees: the cut lies well behind the k-th row
        assert (how == 0).mean() >= 0.5, f"only {(how == 0).mean():.2f} certified"
    if k == 800 and n >= min_rows(k):        # k' = k: the cut is the k-th row itself, nothing can be certified
        assert (how == 1).all()
    gpu.close()


# ---- the hazards: more than HXD_T true neighbours in one bucket --------------------------------------------------------------
def hazard_fixture(kind, metric):
    rng = np.random.default_rng(77)
    n, dim, nh, nr_ = 40_000, 64, 16, 48
    rows = rng.standard_normal((n, dim)).astype(np.float32)
    hq = rng.standard_normal((nh, dim)).astype(np.float32)
    for h in range(nh):
        base = 2048 * h + 192
        if kind == "stride4":   # 11 nearest at ids congruent mod 4 inside one tile: one column quarter
            for i in range(11):
                rows[base + 4 * i] = hq[h] + np.float32(0.01 * (i + 1)) * rng.standard_normal(dim).astype(np.float32)
        else:                   # 48 consecutive near-duplicates, all at about the same distance: 12 per quarter
            rows[base:base + 48] = hq[h] + np.float32(0.01) * rng.standard_normal((48, dim)).astype(np.float32)
    queries = np.concatenate([hq, rng.standard_normal((nr_, dim)).astype(np.float32)])
    return np.arange(n, dtype=np.uint64), rows, queries, nh


@pytest.mark.parametrize("kind", ["stride4", "run48"])
@pytest.mark.parametrize("om", [COS, EUC])
def test_hazard_queries_are_rescanned(kind, om):
    ids, rows, queries, nh = hazard_fixture(kind, om)
    gpu = dense_index(om, ids, rows)
    k = 10
    how = check_exact(gpu, queries, k, ids, f"{kind} {om}")
    assert (how[:nh] == 1).all(), how[:nh]
    if kind == "stride4":   # the plain entry does lose neighbours here: the certificate is what makes the answer exact
        pi, _, _ = gpu.search_dense_batch(queries[:nh], hx.SearchParams.strict(k))
        wi, _, _ = exact_all(gpu, queries[:nh], k, ids)
        assert any(set(pi[b].tolist()) != set(wi[b].tolist()) for b in range(nh))
    gpu.close()


# ---- ties, deleted rows, upserts, small corpora ----------------------------------------------------------------------------
def test_ties_deletes_upsert_and_small_corpora():
    ids, rows, q, tied = tie_fixture()
    gpu = dense_index(EUC, ids, rows)
    qs = np.stack([q, q + np.float32(1e-3)])
    for k in (1, 5, 10, 20, 25):
        check_exact(gpu, qs, k, ids, f"ties k={k}")
    # delete tied rows and every 7th row (not the entry point: the index stays populated); then bring one back by upsert
    gone = np.union1d(tied[:3], ids[1::7])
    gpu.delete_vectors(gone)
    live = np.setdiff1d(ids, gone)
    for k in (5, 20):
        check_exact(gpu, qs, k, live, f"deleted k={k}", n_slots=len(ids))
    back = np.array([tied[1]], np.uint64)
    gpu.upsert_vectors(back, rows[np.searchsorted(ids, back)])
    live = np.union1d(live, back)
    check_exact(gpu, qs, 5, live, "upserted", n_slots=len(ids))
    # below hx_dense_min_rows: every query how == 2
    how = check_exact(gpu, qs, 800, live, "small corpus, k = 800", n_slots=len(ids))
    assert (how == 2).all()
    gpu.close()


# ---- the float32 range ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("om", [COS, EUC])
def test_float32_range(om):
    for d in nr.DIMS:
        _, rows, queries = nr.corpus(om, d, n_rows=700)
        ids = np.arange(len(rows), dtype=np.uint64) + 5
        gpu = dense_index(om, ids, rows)
        for k in (1, 5):
            check_exact(gpu, queries, k, ids, f"range {om} d={d} k={k}")
        gpu.close()
    # Euclidean at 2^-70: products in the fp32 subnormal range
    rng = np.random.default_rng(70)
    rows = (rng.standard_normal((1500, 31)) * 2.0 ** -70).astype(np.float32)
    queries = (rng.standard_normal((20, 31)) * 2.0 ** -70).astype(np.float32)
    ids = np.arange(1500, dtype=np.uint64)
    gpu = dense_index(EUC, ids, rows)
    check_exact(gpu, queries, 10, ids, "euclidean 2^-70")
    gpu.close()


# ---- restricted -----------------------------------------------------------------------------------------------------------------
def check_restricted(gpu, queries, k, cand, what):
    p = hx.SearchParams.strict(k)
    want = gpu.search_restricted_batch(queries, p, Cands(cand))
    got = gpu.search_dense_restricted_exact_batch(queries, p, Cands(cand))
    assert_same(got[:3], want, what + " (host ids)")
    dev = gpu.cache_candidates(Cands(cand))
    got2 = gpu.search_dense_restricted_exact_sets(queries, p, dev)
    dev.close()
    assert_same(got2[:3], want, what + " (device set)")
    assert got[3].tolist() == got2[3].tolist()
    return got[3]


@pytest.mark.parametrize("om", [COS, EUC])
def test_restricted_exact(om):
    rng = np.random.default_rng(31 + om)
    n, dim = 30_000, 96
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64) * 2 + 1
    queries = rng.standard_normal((300, dim), dtype=np.float32)
    gpu = dense_index(om, ids, rows)
    gpu.delete_vectors(ids[5::11])
    cand = np.union1d(ids[::3], np.arange(0, 2 * n, 17, dtype=np.uint64) * 2)   # present, deleted and absent ids
    for k in (1, 10, 64):
        how = check_restricted(gpu, queries, k, cand, f"restricted k={k}")
        assert (how == 0).mean() >= 0.5
    how = check_restricted(gpu, queries, 10, cand[:400], "small set")
    assert (how == 2).all()
    # a rank-clustered set: 11 near rows of each hazard query at ranks congruent mod 4 inside one tile of the set's
    # present rows (the tile is laid out over present rank)
    hq = queries[:8]
    c = ids[:20_000][~np.isin(ids[:20_000], ids[5::11])]
    near = []
    for h in range(8):
        for i in range(11):
            near.append(c[2048 * h + 192 + 4 * i])
            rows[np.searchsorted(ids, near[-1])] = hq[h] + np.float32(0.01 * (i + 1)) * rng.standard_normal(dim).astype(np.float32)
    near = np.array(near, np.uint64)
    gpu.upsert_vectors(near, rows[np.searchsorted(ids, near)])
    how = check_restricted(gpu, hq, 10, c, "rank-clustered set")
    assert (how == 1).all(), how
    gpu.close()


# ---- admission: the exact entries answer every refusal as the plain ones --------------------------------------------------------
def _outcome(fn):
    try:
        r = fn()
        return ("ok", r[2].tolist())
    except hx.HelixDbError as e:
        return ("err", e.code)


def test_admission_order_matches_the_plain_entries():
    rng = np.random.default_rng(3)
    n, dim, k = 3000, 32, 10
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64) * 2
    gpu = dense_index(COS, ids, rows)
    q = rng.standard_normal((3, dim), dtype=np.float32)
    nan = q.copy()
    nan[1, 7] = np.nan
    zero = q.copy()
    zero[2] = 0
    p = hx.SearchParams.strict(k)
    p16 = hx.SearchParams.strict(k)
    p16.query_dimension = 16
    cases = [(np.zeros((0, dim), np.float32), p, ids[:10]), (nan, p, np.zeros(0, np.uint64)),
             (q, p, np.arange(1_000_001, dtype=np.uint64)), (q, hx.SearchParams.strict(900), ids[:1000]),
             (q, hx.SearchParams.strict(1000), ids[:500]), (q, p, ids[[5, 3, 9]]), (q, p, ids[[3, 3, 9]]),
             (nan, p, ids[[5, 3, 9]]), (nan, p, ids[:10]), (nan, p, ids[::2]), (np.tile(nan, (5, 1)), p, ids[::2]),
             (nan, p, ids[:10] + np.uint64(1)), (zero, p, ids[::2]), (q[:, :16].copy(), p16, ids[:10]), (q, p, ids[::2])]
    for qq, pp, cand in cases:
        plain = _outcome(lambda: gpu.search_dense_restricted_batch(qq, pp, Cands(cand)))
        exact = _outcome(lambda: gpu.search_dense_restricted_exact_batch(qq, pp, Cands(cand)))
        assert plain == exact, (len(cand), plain, exact)
    for qq, pp in [(q, p), (nan, p), (zero, p), (np.tile(nan, (5, 1)), p), (q[:, :16].copy(), p16),
                   (q, hx.SearchParams.strict(900)), (np.zeros((0, dim), np.float32), p)]:
        plain = _outcome(lambda: gpu.search_dense_batch(qq, pp))
        exact = _outcome(lambda: gpu.search_dense_exact_batch(qq, pp))
        assert plain == exact, (plain, exact)
    other = dense_index(COS, ids, rows, "other")
    foreign = other.cache_candidates(Cands(ids[:100]))
    assert _outcome(lambda: gpu.search_dense_restricted_sets(q, p, foreign)) == \
        _outcome(lambda: gpu.search_dense_restricted_exact_sets(q, p, foreign)) == ("err", hx.HX_ERR_INVARIANT_VIOLATION)
    foreign.close()
    other.close()
    # an index without the bf16 copy, an unpopulated and an empty index
    s0 = hx.VectorIndex(hx.Metric.Cosine, hx.VectorIndexConfig("s0", "embedding", dim))
    s0.load_vectors(ids, rows)
    s0.load_graph(0, ids[:1], [0, 0], [])
    s0.set_entry(int(ids[0]), 0)
    assert _outcome(lambda: s0.search_dense_batch(q, p)) == _outcome(lambda: s0.search_dense_exact_batch(q, p))
    s0.close()
    for name, load in (("bare", True), ("none", False)):
        ix = hx.VectorIndex(hx.Metric.Cosine, hx.VectorIndexConfig(name, "embedding", dim), storage=1)
        if load:
            ix.load_vectors(ids, rows)
        for qq in (q, nan):
            assert _outcome(lambda: ix.search_dense_restricted_batch(qq, p, Cands(ids[::2]))) == \
                _outcome(lambda: ix.search_dense_restricted_exact_batch(qq, p, Cands(ids[::2])))
            assert _outcome(lambda: ix.search_dense_batch(qq, p)) == _outcome(lambda: ix.search_dense_exact_batch(qq, p))
        got = ix.search_dense_exact_batch(q, p)
        assert got[2].tolist() == [0, 0, 0] and got[3].tolist() == [2, 2, 2]
        ix.close()
    gpu.close()
    l1 = hx.VectorIndex(hx.Metric.Manhattan, hx.VectorIndexConfig("l1", "embedding", dim), storage=1)
    l1.load_vectors(ids, rows)
    l1.load_graph(0, ids[:1], [0, 0], [])
    l1.set_entry(int(ids[0]), 0)
    for fn in (lambda: l1.search_dense_restricted_exact_batch(q, p, Cands(np.zeros(0, np.uint64))),
               lambda: l1.search_dense_exact_batch(q, p)):
        assert _outcome(fn) == ("err", hx.HX_ERR_UNSUPPORTED)
    l1.close()


# ---- non-vacuity on the bench recipe ---------------------------------------------------------------------------------------------
# CPU prediction (scripts/dense_exact_sweep.py --predict-cpu 200000: the margin study's corpus at 200k x 768, nominee cut
# only): every one of 256 queries certified for both metrics; the smallest gap L_q - S_k is 5.5x the bound E_q at L_q
# (cosine 0.0217 vs 0.0039, euclidean 0.087 vs 0.0157).  The bucket tails can only lower L_q.
CERTIFIED_SHARE = 0.99


@pytest.mark.parametrize("om", [COS, EUC])
def test_bench_recipe_is_mostly_certified(om):
    n, dim, B = 200_000, 768, 512
    seed, ncent, sigma, kind = 0x0DB9ED1A, 1024, 1.0, 32   # bench.py's "embedding" recipe
    gpu = hx.VectorIndex(hx.Metric.Cosine if om == COS else hx.Metric.Euclidean,
                         hx.VectorIndexConfig("bench", "embedding", dim), storage=1)
    gpu.generate_vectors(0, n, seed, ncent, sigma, kind)
    ids = np.arange(n, dtype=np.uint64)
    gpu.load_graph(0, ids[:1], [0, 0], [])
    gpu.set_entry(0, 0)
    queries = gpu.generate_queries(seed, B, first_query=30_000_000, n_centroids=ncent, sigma=sigma, kind=kind)
    how = check_exact(gpu, queries, 10, ids, "bench recipe")
    share = float((how == 0).mean())
    print(f"certified share {share:.4f} ({'cosine' if om == COS else 'euclidean'})")
    assert share >= CERTIFIED_SHARE, share
    gpu.close()
