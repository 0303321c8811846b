"""hx_search_dense held to the exact scan.

The tensor-core pass (csrc/k_dense.cu) only nominates candidates; after it the path promises: every returned score is the
reference's fp32 score, the order is (score, id) — ties included —, the count is min(k, live rows), and deleted rows are
never returned.  The nomination itself is checked against the float64 reference of tests/test_dense_reference.py: a row
that is sure for a query (fewer than HXD_T rows can come within epsilon of beating its bf16 score) must be nominated,
whatever the tile and bucket layout.
"""
import threading

import numpy as np
import pytest

import helix_db_b200 as hx
from helix_db_b200 import sharding as sh
from oracle import hxo
from test_dense_reference import emulate, sure_rows, tie_fixture

pytestmark = pytest.mark.gpu
EUC, COS = hxo.EUCLIDEAN, hxo.COSINE
GPU_METRIC = {EUC: hx.Metric.Euclidean, COS: hx.Metric.Cosine}


def dense_index(om, ids, rows, name="dense"):
    gpu = hx.VectorIndex(GPU_METRIC[om], hx.VectorIndexConfig(name, "embedding", rows.shape[1]), storage=1)
    gpu.load_vectors(ids, rows)
    gpu.load_graph(0, ids[:1], [0, 0], [])
    gpu.set_entry(int(ids[0]), 0)
    return gpu


def oracle_of(om, ids, rows):
    ora = hxo.Index(om, rows.shape[1])
    ora.put_vectors(ids, rows)
    ora.set_entry(int(ids[0]), 0)   # populated: the restricted scan answers (an unpopulated index answers nothing)
    return ora


def exact_score_bits(ora, query, cand):
    """The oracle's exact score bits of the ids `cand` (restricted scan in chunks of <= 256: the exact branch)."""
    out = {}
    cand = np.unique(np.asarray(cand, dtype=np.uint64))
    for i in range(0, len(cand), 256):
        c = cand[i:i + 256]
        ri, rs = ora.search_restricted(query, len(c), c)
        out.update(zip(ri.tolist(), rs.view(np.uint32).tolist()))
    return out


def assert_same(got, want, what):
    gi, gs, gc = got
    wi, ws, wc = want
    assert gc.tolist() == wc.tolist(), f"{what}: counts"
    for b in range(len(gc)):
        c = int(gc[b])
        assert gi[b, :c].tolist() == wi[b, :c].tolist(), f"{what}: ids of query {b}"
        assert gs[b, :c].view(np.uint32).tolist() == ws[b, :c].view(np.uint32).tolist(), f"{what}: score bits of query {b}"


def check_against_reference(om, ids, rows, queries, k, got):
    """Count, exact score bits, (score, id) order, sure rows nominated, and the answer's sure prefix equal to the oracle.
    Returns the fraction of queries whose exact top-min(k, 4) rows are all sure (the checks below are not vacuous)."""
    di, ds, dc = got
    n = len(ids)
    ora = oracle_of(om, ids, rows)
    oi, os_, oc, _ = ora.search_exact_batch(queries, k, threads=8)
    approx, eps = emulate(om, queries, rows)
    covered = 0
    for b in range(len(queries)):
        c = int(dc[b])
        assert c == min(k, n) == int(oc[b]), f"query {b}: count {c}, want {min(k, n)}"
        got_ids = di[b, :c].tolist()
        got_bits = ds[b, :c].view(np.uint32).tolist()
        assert len(set(got_ids)) == c, f"query {b}: repeated ids"
        assert [(s, i) for s, i in zip(got_bits, got_ids)] == sorted(zip(got_bits, got_ids)), f"query {b}: (score, id) order"
        want = dict(zip(oi[b].tolist(), os_[b].view(np.uint32).tolist()))
        extra = [i for i in got_ids if i not in want]
        if extra:
            want.update(exact_score_bits(ora, queries[b], extra))
        assert got_bits == [want[i] for i in got_ids], f"query {b}: score bits differ from the oracle"
        pos = np.searchsorted(ids, oi[b])
        sure = sure_rows(approx[b], eps[b], pos)
        missing = [int(i) for i, s in zip(oi[b], sure) if s and int(i) not in set(got_ids)]
        assert not missing, f"query {b}: sure rows {missing} of the exact top-{k} were not returned"
        m = int(np.argmin(sure)) if not sure.all() else len(sure)
        assert got_ids[:m] == oi[b, :m].tolist() and got_bits[:m] == os_[b, :m].view(np.uint32).tolist(), \
            f"query {b}: the first {m} rows are sure but differ from the oracle"
        if m == len(sure):
            assert got_ids == oi[b].tolist(), f"query {b}: every exact row is sure, the answer must be the oracle's"
        covered += m >= min(k, 4)
    return covered / len(queries)


# ---- nomination against the float64 reference -----------------------------------------------------------------------------
# dim 8 / 65 / 100: one padded k-block, a nearly empty last k-block; 768 / 1536: 12 / 24 k-blocks.  n off the 256-row tile;
# B across one / several 128-query tiles and above 1024; k' = 800 on ~200 k rows.  n = 200 is below 8 * k' (exact scan).
CASES = [(EUC, 1000, 8, 127, 1), (COS, 4999, 65, 128, 33), (EUC, 3001, 100, 129, 10), (COS, 20077, 768, 300, 10),
         (EUC, 2503, 1536, 1, 1), (COS, 9003, 64, 1500, 10), (EUC, 200_013, 64, 8, 800), (COS, 200, 100, 5, 10)]


@pytest.mark.parametrize("om,n,dim,B,k", CASES)
def test_dense_nominates_every_sure_row(om, n, dim, B, k):
    rng = np.random.default_rng(n * 7 + dim)
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    queries = rng.standard_normal((B, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64) * 3 + 11
    gpu = dense_index(om, ids, rows)
    got = gpu.search_dense_batch(queries, hx.SearchParams.strict(k))
    covered = check_against_reference(om, ids, rows, queries, k, got)
    assert covered >= 0.75, f"only {covered:.2f} of the queries have their exact top-{min(k, 4)} rows sure"
    gpu.close()


def test_sharded_dense_entries_match_the_host_path():
    """The same answer through hx_search_sharded (host buffers) and hx_search_sharded_device on a torch stream."""
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(41)
    n, dim, B, k = 3001, 100, 129, 10
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    queries = rng.standard_normal((B, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64) + 1000
    host = dense_index(EUC, ids, rows)
    want = host.search_dense_batch(queries, hx.SearchParams.strict(k))
    check_against_reference(EUC, ids, rows, queries, k, want)
    gpu = dense_index(EUC, ids, rows, "sharded")
    g = sh.ShardGroup(gpu, 1, 0, None)
    assert_same(g.search(sh.DENSE, queries, hx.SearchParams.strict(k), k), want, "sharded host entry")
    gpu2 = dense_index(EUC, ids, rows, "sharded-device")   # first dense call on the torch stream builds the bf16 copy
    g2 = sh.ShardGroup(gpu2, 1, 0, None)
    dq = torch.from_numpy(queries).cuda()
    di = torch.zeros((B, k), dtype=torch.int64, device="cuda")
    ds = torch.zeros((B, k), dtype=torch.float32, device="cuda")
    dc = torch.zeros(B, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g2.search_device(sh.DENSE, dq.data_ptr(), B, hx.SearchParams.strict(k), k, di.data_ptr(), ds.data_ptr(), dc.data_ptr(),
                         s.cuda_stream)
    s.synchronize()
    got = (di.cpu().numpy().view(np.uint64), ds.cpu().numpy(), dc.cpu().numpy().view(np.uint32))
    assert_same(got, want, "sharded device entry")
    for x in (g, g2):
        x.close()
    for x in (host, gpu, gpu2):
        x.close()


# ---- exact ties ------------------------------------------------------------------------------------------------------------
def test_exact_ties_resolve_by_id():
    """20 rows at one exact fp32 distance, whose bf16 scores rank them in reverse id order: k = 10 returns the 10 smallest
    ids, ascending, at the oracle's score bits — on the host path and the sharded dense path."""
    ids, rows, q, tied = tie_fixture()
    k = 10
    ora = oracle_of(EUC, ids, rows)
    oi, os_ = ora.search_exact(q, k)
    assert oi.tolist() == tied[:k].tolist()
    gpu = dense_index(EUC, ids, rows)
    di, ds, dc = gpu.search_dense_batch(q[None, :], hx.SearchParams.strict(k))
    assert int(dc[0]) == k
    assert di[0].tolist() == tied[:k].tolist(), "tied rows must come in id order, and the smallest ids must make the cut"
    assert ds[0].view(np.uint32).tolist() == os_.view(np.uint32).tolist()
    g = sh.ShardGroup(gpu, 1, 0, None)
    si, ss, sc = g.search(sh.DENSE, q[None, :], hx.SearchParams.strict(k), k)
    assert int(sc[0]) == k and si[0].tolist() == tied[:k].tolist()
    assert ss[0].view(np.uint32).tolist() == os_.view(np.uint32).tolist()
    g.close()
    gpu.close()


# ---- deleted rows ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("om", [EUC, COS])
def test_deleted_rows_are_never_returned(om):
    rng = np.random.default_rng(21 + om)
    n, dim, B, k = 6000, 16, 64, 10
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    queries = rng.standard_normal((B, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64) * 3 + 5
    gpu = dense_index(om, ids, rows)
    gpu.search_dense_batch(queries, hx.SearchParams.strict(k))          # the bf16 copy exists before the deletion
    nn, _, _, _ = oracle_of(om, ids, rows).search_exact_batch(queries, 1, threads=8)
    dead = set(nn[:, 0].tolist()) | set(rng.choice(ids[1:], size=int(0.3 * n), replace=False).tolist())
    dead.discard(int(ids[0]))                                             # the entry point stays (deleting it unpopulates)
    dead = np.array(sorted(dead), dtype=np.uint64)
    gpu.delete_vectors(dead)
    alive = ~np.isin(ids, dead)
    live_ids, live_rows = ids[alive], rows[alive]
    got = gpu.search_dense_batch(queries, hx.SearchParams.strict(k))
    assert not set(got[0][got[0] != 0].tolist()) & set(dead.tolist()), "a deleted row was returned"
    oi, os_, oc, _ = oracle_of(om, live_ids, live_rows).search_exact_batch(queries, k, threads=8)
    assert_same(got, (oi, os_, oc), "dense after deletes vs an oracle of the live rows")
    assert_same(got, gpu.search_restricted_batch(queries, hx.SearchParams.strict(k), hx.RestrictedVectorCandidates(live_ids)),
                "dense after deletes vs the restricted scan over every live id")
    # an upsert brings a deleted id back
    back = int(nn[0, 0])
    j = int(np.searchsorted(ids, back))
    gpu.upsert_vectors(np.array([back], np.uint64), rows[j:j + 1])
    alive[j] = True
    got = gpu.search_dense_batch(queries, hx.SearchParams.strict(k))
    oi, os_, oc, _ = oracle_of(om, ids[alive], rows[alive]).search_exact_batch(queries, k, threads=8)
    assert int(got[0][0, 0]) == back
    assert_same(got, (oi, os_, oc), "dense after re-inserting a deleted id")
    gpu.close()


def test_packed_survivors_keep_their_count():
    """12 rows survive in one tile, all with ids = 0 (mod 4): one column quarter, one bucket of 8 in the tensor-core pass."""
    rng = np.random.default_rng(4)
    n, dim, B, k = 256, 32, 5, 10
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    queries = rng.standard_normal((B, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64)
    keep = ids[::4][:12]
    gpu = dense_index(EUC, ids, rows)
    gpu.delete_vectors(ids[~np.isin(ids, keep)])
    got = gpu.search_dense_batch(queries, hx.SearchParams.strict(k))
    assert got[2].tolist() == [k] * B
    oi, os_, oc, _ = oracle_of(EUC, keep, rows[::4][:12]).search_exact_batch(queries, k)
    assert_same(got, (oi, os_, oc), "packed survivors")
    gpu.close()


# ---- small corpora ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 7, 255, 257, 700, 1000])
def test_small_corpus_counts(n):
    om = EUC if n % 2 == 0 else COS
    rng = np.random.default_rng(1000 + n)
    dim, B = 24, 33
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    queries = rng.standard_normal((B, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64) * 2 + 1
    gpu = dense_index(om, ids, rows)
    for k in (1, 10, 100, 200, 800):
        got = gpu.search_dense_batch(queries, hx.SearchParams.strict(k))
        assert got[2].tolist() == [min(k, n)] * B, f"k = {k}"
        if n < min(max(32 * k, 512), 6400):   # answered by the exact scan over every live row (DESIGN.md, dense path)
            oi, os_, oc, _ = oracle_of(om, ids, rows).search_exact_batch(queries, k)
            assert_same(got, (oi, os_, oc), f"n = {n}, k = {k}")
        else:
            check_against_reference(om, ids, rows, queries, k, got)
    gpu.close()


# ---- first call after every rebuild of the bf16 copy -----------------------------------------------------------------------
def test_first_call_after_every_rebuild():
    """The first dense call after load / upsert / delete, and from 8 threads at once on a fresh index, reads a complete
    bf16 copy: each answer equals the exact scan.  Each point runs once (a correctness check, not a race hunt)."""
    n, dim, B, k = 1 << 18, 768, 256, 1
    rng = np.random.default_rng(18)
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint64)
    plant = np.unique(np.concatenate([np.linspace(1, n - 1, B - 16).astype(np.int64), np.arange(n - 16, n)]))
    p = hx.SearchParams.strict(k)

    def queries_at(r):
        return (r + 0.01 * rng.standard_normal(r.shape, dtype=np.float32)).astype(np.float32)

    def exact(gpu, q, live):
        return gpu.search_restricted_batch(q, p, hx.RestrictedVectorCandidates(live))

    gpu = dense_index(EUC, ids, rows)
    q = queries_at(rows[plant])
    got = gpu.search_dense_batch(q, p)                                  # first call after load_vectors
    assert got[0][:, 0].tolist() == ids[plant].tolist()
    assert_same(got, exact(gpu, q, ids), "first call after load")
    new = rng.standard_normal((len(plant), dim), dtype=np.float32)
    gpu.upsert_vectors(ids[plant], new)
    q = queries_at(new)
    got = gpu.search_dense_batch(q, p)                                  # first call after upsert_vectors
    assert got[0][:, 0].tolist() == ids[plant].tolist()
    assert_same(got, exact(gpu, q, ids), "first call after upsert")
    dead = ids[plant[1::2]]
    gpu.delete_vectors(dead)
    got = gpu.search_dense_batch(q, p)                                  # first call after delete_vectors
    live = ids[~np.isin(ids, dead)]
    assert_same(got, exact(gpu, q, live), "first call after delete")
    rows[plant] = new
    gpu.close()

    fresh = dense_index(EUC, ids, rows, "fresh")
    results, errors = [None] * 8, []

    def worker(t):
        try:
            results[t] = fresh.search_dense_batch(q, p)
        except Exception as e:   # reported below
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(8)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    want = exact(fresh, q, ids)
    for t in range(8):
        assert_same(results[t], want, f"thread {t} of the first concurrent calls")
    fresh.close()
