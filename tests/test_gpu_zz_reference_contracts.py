"""Reference contracts added at the end of round 2, on the device (the file sorts last on purpose: the driver runs the GPU
suite with `-x`, and everything above has a longer green history):
  * the reference's layer-0 search-mode contracts (V/index.rs:2414-2557) through hx_search_ex, bit-exact vs the oracle;
  * VectorIndex::delete (V/mutation.rs:1606-2050) restated in the oracle and applied to the device mirror as row patches,
    including a write that deletes the entry point and the whole top layer;
  * the C++ host mirror (helix-db_b200/host/vector_index.hpp) linked and executed: phase-0 KAT on the device.
V/ = helix-db/crates/db/src/search/vector/ (cited, never read at run time)."""
import numpy as np
import pytest

import helix_db_b200 as hx
from oracle import hxo
from hx_testutil import mirror_from_oracle
from test_gpu_mirror import _apply_diff, _graph_rows
from test_gpu_parity import build_pair, levels_for
from test_gpu_policy import compare, oracle_cfg

pytestmark = pytest.mark.gpu


def test_reference_layer0_search_mode_contracts_on_the_device():
    """V/index.rs:2414-2557 (`test_layer0_search_modes_cover_sampling_filtering_and_adaptive_bypass`) through the C ABI:
    Cosine d=2, m=8, m0=16, ef_construction=32, index threshold 0 / sampling ratio 0.5, 32 points on the unit circle with
    ids 1..=32.  The reference asserts relations between the four searches (its insertion layers come from `rand::rng()`);
    here the same relations are asserted on the DEVICE's answers and counters, and every answer is also compared with the
    oracle bit for bit (tests/test_oracle_kat.py replays the same contract on the oracle alone)."""
    import math
    planes = np.random.default_rng(42).standard_normal((64, 2)).astype(np.float32)
    ang = (np.arange(32, dtype=np.float32) * np.float32(2.0 * math.pi) / np.float32(32.0)).astype(np.float32)
    rows = np.stack([np.cos(ang, dtype=np.float32), np.sin(ang, dtype=np.float32)], axis=1).astype(np.float32)
    ids = np.arange(1, 33, dtype=np.uint64)
    gpu, ora = build_pair(hx.Metric.Cosine, hxo.COSINE, rows, ids=ids, m=8, m0=16, efc=32, seed=4)
    bits = np.array([hxo.simhash_from_planes(planes, r) for r in rows], dtype=np.uint64)
    gpu.set_simhash_planes(planes)
    gpu.compute_simhash()
    assert gpu.download_simhash(0, 32).tolist() == bits.tolist()
    ora.put_simhash(ids, bits)
    qang = (np.arange(48, dtype=np.float32) * np.float32(2.0 * math.pi) / np.float32(48.0) + np.float32(0.01))
    queries = np.stack([np.cos(qang), np.sin(qang)], axis=1).astype(np.float32)
    queries[0], queries[1] = (1.0, 0.0), (0.0, 1.0)            # the reference's two queries
    qsim = np.array([hxo.simhash_from_planes(planes, q) for q in queries], dtype=np.uint64)
    gpu.set_simhash_config(threshold=0, sampling_ratio=0.5)

    def run(params):
        st, ps = hx.SearchStats(), hx.PolicyStats()
        params.collect_stats = True
        gi, gs, gc = gpu.search_ex(queries[:2], params, query_simhash=qsim[:2], stats=st, policy_stats=ps)
        compare(gpu, ora, queries, qsim, params, oracle_cfg(params, threshold=0, sampling_ratio=0.5), "circle contract")
        return gi, gc, st, ps.as_dict()

    def base():                                                # the builders mutate in place: a fresh object per search
        return hx.SearchParams.new(5).with_ef(16)

    off_i, off_c, off_st, off_ps = run(base().with_simhash_mode(hx.SimHashMode.Off).with_pre_simhash_sampling_ratio(1.0))
    assert off_c[0] > 0 and off_st.expansion_steps > 0
    assert off_ps["simhash_examined"] == 0 and off_ps["simhash_filtered"] == 0
    al_i, al_c, _, al_ps = run(base().with_simhash_mode(hx.SimHashMode.Always).with_pre_simhash_sampling_ratio(1.0)
                               .with_simhash_sampling_ratio(0.0))
    assert al_c[0] > 0 and al_ps["simhash_examined"] > 0 and al_ps["simhash_passed_before_sampling"] > 0
    fx_i, fx_c, _, fx_ps = run(base().with_simhash_mode(hx.SimHashMode.Always).with_pre_simhash_sampling_ratio(1.0)
                               .with_simhash_sampling_ratio(1.0))
    assert fx_i[0, :fx_c[0]].tolist() == off_i[0, :off_c[0]].tolist() and fx_ps["simhash_filtered"] == 0
    ad_i, ad_c, ad_st, ad_ps = run(base().with_simhash_mode(hx.SimHashMode.Adaptive).with_pre_simhash_sampling_ratio(0.25)
                                   .with_simhash_sampling_ratio(0.5).with_simhash_failure_prob(0.5)
                                   .with_simhash_bypass_tuning(1, 1, 1.0, 1))
    assert ad_c[1] > 0 and ad_st.expansion_steps > 0 and ad_ps["simhash_bypass_expansions"] > 0
    gpu.close()


@pytest.mark.parametrize("gm,om", [(hx.Metric.Euclidean, hxo.EUCLIDEAN), (hx.Metric.Cosine, hxo.COSINE)])
def test_reference_delete_as_row_patches(gm, om):
    """VectorIndex::delete (mutation.rs:1606-1773: delete_from_layer + relink_neighbor + entry-candidate promotion) runs on
    the oracle; the rows it dirtied reach the device as patches (hx_index_delete_vectors, hx_index_upsert_neighbor_rows,
    hx_index_set_entry).  After every committed write the mirror must answer exactly like the oracle — the first write
    deletes the entry point and every other node of the top layer, so the graph loses a layer."""
    rng = np.random.default_rng(23)
    n, dim, k, ef = 1200, 32, 10, 50
    rows = rng.standard_normal((n, dim)).astype(np.float32)
    ids = np.arange(100, 100 + n, dtype=np.uint64)
    lv = levels_for(n, 8, 11)
    ora = hxo.Index(om, dim, m=8, m0=16, ef_construction=60)
    for i in range(n):
        ora.insert(int(ids[i]), rows[i], lv[i])
    gpu = hx.VectorIndex(gm, hx.VectorIndexConfig("del", "embedding", dim).with_m(8).with_m0(16).with_ef_construction(60))
    mirror_from_oracle(gpu, ora)
    entry0, top0 = ora.export_graph()[1]
    top_nodes = [int(ids[i]) for i in range(n) if lv[i] == top0]
    assert entry0 in top_nodes and top0 >= 2
    order = [int(x) for x in rng.permutation(ids) if int(x) not in top_nodes]
    writes = [top_nodes + order[:20], order[20:60], order[60:100], order[100:140]]
    q_small = rng.standard_normal((120, dim)).astype(np.float32)   # B < #SMs: the CTA-per-query build
    q_big = rng.standard_normal((400, dim)).astype(np.float32)     # the warp-per-query build
    p = hx.SearchParams.strict(k, ef)
    gone = set()
    for w, victims in enumerate(writes):
        before, _ = _graph_rows(ora)
        for v in victims:
            assert ora.delete(v) is True
        gone.update(victims)
        after, state = _graph_rows(ora)
        assert not (set(node for _, node in after) & gone)
        gpu.delete_vectors(victims)
        assert _apply_diff(gpu, before, after, state) > 0
        gpu.set_version(3, 10 + w)
        if w == 0:
            assert state[1] < top0                             # the top layer is gone, the entry moved down
        for q in (q_small, q_big):
            gi, gs, gc = gpu.search_batch(q, p)
            oi, os_, oc, _, _ = ora.search_batch(q, k, ef, threads=4)
            assert gc.tolist() == oc.tolist() and gi.tolist() == oi.tolist() and gs.tobytes() == os_.tobytes(), w
            assert not (set(gi.flatten().tolist()) & gone)
    # the exact restricted scan skips deleted ids like absent ones
    cand = np.array(sorted(set(int(x) for x in ids[::5]) | set(list(gone)[:40])), dtype=np.uint64)
    ri, rs, rc = gpu.search_restricted_batch(q_small[:8], hx.SearchParams.strict(6), hx.RestrictedVectorCandidates(cand))
    live = np.array([c for c in cand.tolist() if c not in gone], dtype=np.uint64)
    for b in range(8):
        ei, es = ora.search_restricted(q_small[b], 6, live)
        assert ri[b, :rc[b]].tolist() == ei.tolist() and rs[b, :rc[b]].tobytes() == es.tobytes()
    # a fresh hydration of the final oracle state answers identically
    fresh = hx.VectorIndex(gm, hx.VectorIndexConfig("fresh", "embedding", dim).with_m(8).with_m0(16).with_ef_construction(60))
    mirror_from_oracle(fresh, ora)
    a, b = gpu.search_batch(q_big, p), fresh.search_batch(q_big, p)
    assert a[0].tolist() == b[0].tolist() and a[1].tobytes() == b[1].tobytes() and a[2].tolist() == b[2].tolist()
    gpu.close()
    fresh.close()


def test_cpp_host_mirror_runs_the_phase0_kat_on_the_device(tmp_path):
    """helix-db_b200/host/vector_index.hpp as a TESTED host binding: a C++ program linked against libhelix_b200.so runs the
    reference's phase-0 known-answer test (index.rs:2318-2411), the validation-order KAT and a prefiltered scan through
    helix::VectorIndex on the device (tests/cpp/host_mirror_selftest.cpp)."""
    import shutil
    from hx_testutil import build_and_run_cpp_selftest
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    rc, out = build_and_run_cpp_selftest(tmp_path)
    assert rc == 0 and "passed on the device" in out, out


@pytest.mark.parametrize("gm,om", [(hx.Metric.Cosine, hxo.COSINE), (hx.Metric.Euclidean, hxo.EUCLIDEAN)])
def test_dense_path_keeps_id_clustered_neighbours(gm, om):
    """hx_search_dense nominates by bucket — (query, run of tiles, 64-column quarter), best HXD_T = 8 rows each.  With rows
    placed in id order a bucket holds 64 CONSECUTIVE ids per tile, so a query whose 11 nearest rows are consecutive ids (chunks
    of one document inserted back to back) would keep only 8 of them (recall 0.8 on exactly this fixture).  The interleaved placement (HXD_INTERLEAVE, csrc/k_dense.cu) spreads consecutive
    ids over the four quarters: every true neighbour must come back, with the oracle's exact scan as the ground truth."""
    rng = np.random.default_rng(77)
    n, dim, k, nh = 40_000, 64, 10, 16
    rows = rng.standard_normal((n, dim)).astype(np.float32)
    hq = rng.standard_normal((nh, dim)).astype(np.float32)
    for h in range(nh):
        base = 2048 * h + 192                                  # tile rows 192..202: inside the fourth 64-row stripe of a tile
        for i in range(11):
            rows[base + i] = hq[h] + np.float32(0.01 * (i + 1)) * rng.standard_normal(dim).astype(np.float32)
    ids = np.arange(n, dtype=np.uint64)
    gpu = hx.VectorIndex(gm, hx.VectorIndexConfig("hz", "embedding", dim), storage=1)
    gpu.load_vectors(ids, rows)
    gpu.load_graph(0, ids[:1], [0, 0], [])
    gpu.set_entry(int(ids[0]), 0)
    ora = hxo.Index(om, dim)
    ora.put_vectors(ids, rows)
    di, ds, dc = gpu.search_dense_batch(hq, hx.SearchParams.strict(k))
    for h in range(nh):
        oi, os_ = ora.search_exact(hq[h], k)
        assert set(oi.tolist()) <= set(range(2048 * h + 192, 2048 * h + 203))      # the fixture is what it claims to be
        assert di[h, :dc[h]].tolist() == oi.tolist() and ds[h, :dc[h]].tobytes() == os_.tobytes(), h
    gpu.close()
