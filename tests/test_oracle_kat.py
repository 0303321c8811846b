"""Pins the CPU oracle against the reference's own known-answer tests (SURVEY §8c items 1-9).

Paths: V/ = helix-db/crates/db/src/search/vector/, T/ = helix-db/crates/db/tests/production_support/.
Nothing here reads the reference repository at run time: the expected values are the literals the reference's tests assert.
"""
import math
import struct

import numpy as np
import pytest


def bits(x):
    return struct.unpack("<I", struct.pack("<f", float(x)))[0]


# --- item 2: distance KATs (V/distance/mod.rs:112-137, T/vector/distance_neighbors.rs:79-110) -------------
def test_distance_kats(hxo):
    assert hxo.distance(hxo.COSINE, [1.0, 0.0], [0.0, 1.0]) == 0.5
    assert math.isnan(hxo.distance(hxo.COSINE, [1.0, 0.0], [0.0, 0.0]))
    assert math.isnan(hxo.distance(hxo.COSINE, [0.0, 0.0], [0.0, 0.0]))
    assert hxo.header(hxo.COSINE, [1.0, 0.0]) == 1.0
    assert hxo.distance(hxo.EUCLIDEAN, [1.0, 2.0], [4.0, 6.0]) == 25.0
    assert hxo.distance(hxo.MANHATTAN, [1.0, -2.0, 3.0], [-1.0, 2.0, 1.0]) == 8.0
    # Euclidean/Manhattan norm_no_header = sqrt(dot(v,v)) (euclidean.rs:50-52)
    assert math.sqrt(hxo.pair("hxo_dot_product", [3.0, 4.0], [3.0, 4.0])) == 5.0
    # header of Euclidean rows is the 0.0 bias (magnitude_regressions.rs:333-338)
    assert hxo.header(hxo.EUCLIDEAN, [1.0, -2.0]) == 0.0


# --- cosine extremes (V/distance/cosine.rs:130-149) ---------------------------------------------------------
def test_cosine_extremes(hxo):
    fmax = np.finfo(np.float32).max
    assert hxo.header(hxo.COSINE, [fmax, fmax]) == fmax
    assert hxo.distance(hxo.COSINE, [fmax, fmax], [fmax, fmax]) <= np.finfo(np.float32).eps
    tiny = np.frombuffer(struct.pack("<I", 1), dtype=np.float32)[0]
    assert hxo.header(hxo.COSINE, [tiny, tiny]) > 0.0
    assert hxo.distance(hxo.COSINE, [tiny, tiny], [tiny, tiny]) <= np.finfo(np.float32).eps


# --- AVX vs scalar exact equality on the 70-float vector (V/spaces/simple_avx.rs:248-286) ------------------
def test_avx_equals_scalar_on_reference_vector(hxo):
    blk = [float(x) for x in range(10, 26)]
    v1 = np.array(blk * 4 + [26.0, 27.0, 28.0, 29.0, 30.0, 31.0], dtype=np.float32)
    v2 = np.array([float(x) for x in range(40, 56)] + blk * 3 + [56.0, 57.0, 58.0, 59.0, 60.0, 61.0],
                  dtype=np.float32)
    assert v1.size == 70 and v2.size == 70
    assert hxo.lib().hxo_has_avx_fma() == 1
    assert hxo.pair("hxo_euclid_avx_fma", v1, v2) == hxo.pair("hxo_euclid_scalar", v1, v2)
    assert hxo.pair("hxo_dot_avx_fma", v1, v2) == hxo.pair("hxo_dot_scalar", v1, v2)
    # dispatch takes the AvxFma arm for d >= 32 and the scalar loop below (simple.rs:32,120-144)
    assert hxo.pair("hxo_euclidean_distance", v1, v2) == hxo.pair("hxo_euclid_avx_fma", v1, v2)
    assert hxo.pair("hxo_euclidean_distance", v1[:31], v2[:31]) == hxo.pair("hxo_euclid_scalar", v1[:31], v2[:31])


def test_portable_avx_order_is_bit_identical_to_intrinsics(hxo):
    rng = np.random.default_rng(7)
    for d in (32, 33, 63, 64, 65, 70, 128, 768, 769, 1536, 1567):
        for _ in range(8):
            u = rng.standard_normal(d).astype(np.float32)
            v = rng.standard_normal(d).astype(np.float32)
            assert bits(hxo.pair("hxo_euclid_avx_fma", u, v)) == bits(hxo.pair("hxo_euclid_avx_fma_portable", u, v))
            assert bits(hxo.pair("hxo_dot_avx_fma", u, v)) == bits(hxo.pair("hxo_dot_avx_fma_portable", u, v))


# --- item 4: f32 kernels vs f64 oracle, LCG vectors (T/vector/magnitude_regressions.rs:268-328) ------------
def test_magnitude_regression_tolerance(hxo):
    domains = [(hxo.EUCLIDEAN, d) for d in (1, 15, 16, 17, 31, 32, 33, 1536)] + \
              [(hxo.MANHATTAN, d) for d in (1, 15, 16, 17, 31, 32, 33, 1536)]
    state = 0x5EED5AFECAFEBABE
    mask = (1 << 64) - 1
    for case in range(128):
        metric, d = domains[case % len(domains)]
        limit = hxo.component_limit(metric, d)

        def gen():
            nonlocal state
            out = np.empty(d, dtype=np.float32)
            for i in range(d):
                state = (state * 6364136223846793005 + 1442695040888963407) & mask
                unit = float((state >> 32) & 0xFFFFFFFF) / float(0xFFFFFFFF)
                out[i] = np.float32(((unit * 2.0) - 1.0) * float(limit))
            return out

        left, right = gen(), gen()
        assert hxo.validate_vector(metric, d, left)[0] == hxo.OK
        assert hxo.validate_vector(metric, d, right)[0] == hxo.OK
        score = hxo.distance(metric, left, right)
        reverse = hxo.distance(metric, right, left)
        l64, r64 = left.astype(np.float64), right.astype(np.float64)
        oracle = float(((l64 - r64) ** 2).sum()) if metric == hxo.EUCLIDEAN else float(np.abs(l64 - r64).sum())
        tol = max(d * float(np.finfo(np.float32).eps), 1.0e-5)
        assert math.isfinite(score) and score >= 0.0
        assert score == reverse
        assert abs(score - oracle) <= max(abs(oracle), 1.0) * tol


# --- component limits (V/domain.rs:15-90, docs/VECTOR_MAGNITUDE_VALIDATION.md) -----------------------------
def test_component_limits(hxo):
    fmax = float(np.finfo(np.float32).max)
    for d in (1, 2, 128, 768, 1536):
        le = hxo.component_limit(hxo.EUCLIDEAN, d)
        lm = hxo.component_limit(hxo.MANHATTAN, d)
        assert hxo.component_limit(hxo.COSINE, d) is None
        assert float(le) <= math.sqrt(fmax / (8 * d)) < float(np.nextafter(np.float32(le), np.float32(np.inf)))
        assert float(lm) <= fmax / (4 * d) < float(np.nextafter(np.float32(lm), np.float32(np.inf)))
        v = np.zeros(d, dtype=np.float32)
        v[-1] = np.nextafter(np.float32(le), np.float32(np.inf))
        rc, idx = hxo.validate_vector(hxo.EUCLIDEAN, d, v)
        assert rc == hxo.ERR_MAGNITUDE_EXCEEDED and idx == d - 1
        v[-1] = le
        assert hxo.validate_vector(hxo.EUCLIDEAN, d, v)[0] == hxo.OK


# --- validation order (T/vector/search.rs:160-183) ---------------------------------------------------------
def test_validation_order(hxo):
    assert hxo.validate_vector(hxo.COSINE, 3, [1.0, 0.0])[0] == hxo.ERR_INVALID_DIMENSION
    assert hxo.validate_vector(hxo.COSINE, 3, [1.0, float("nan"), 0.0]) == (hxo.ERR_INVALID_VECTOR_COMPONENT, 1)
    assert hxo.validate_vector(hxo.COSINE, 3, [0.0, 0.0, 0.0])[0] == hxo.ERR_ZERO_NORM_COSINE
    assert hxo.validate_vector(hxo.COSINE, 3, [1.0, 0.0, 0.0])[0] == hxo.OK
    # a NaN wins over the zero-norm and magnitude checks; a dimension error wins over everything
    assert hxo.validate_vector(hxo.EUCLIDEAN, 2, [float("inf"), 1e38]) == (hxo.ERR_INVALID_VECTOR_COMPONENT, 0)
    assert hxo.validate_vector(hxo.EUCLIDEAN, 2, [float("nan")])[0] == hxo.ERR_INVALID_DIMENSION
    ix = hxo.Index(hxo.COSINE, 3)
    ids, sc = ix.search([1.0, 0.0, 0.0], 1)       # empty index -> Ok([])
    assert len(ids) == 0
    with pytest.raises(hxo.OracleError) as e:
        ix.search([1.0, 0.0, 0.0], 0)              # SearchParams::new(0) is an error
    assert e.value.code == hxo.ERR_INVALID_PARAMETER


# --- item 1: phase-0 public result baseline (V/index.rs:2318-2411) -----------------------------------------
def test_phase0_public_result_and_io_baseline(hxo):
    ix = hxo.Index(hxo.COSINE, 2, m=4, m0=8, ef_construction=16)
    for node_id, vec, layer in [(1, [1.0, 0.0], 0), (2, [0.0, 1.0], 1), (3, [-1.0, 0.0], 2), (4, [0.0, -1.0], 0)]:
        ix.insert(node_id, vec, layer)             # scripted layers [0,1,2,0]
    ids, scores, st = ix.search([1.0, 0.0], 4, ef=16, with_stats=True)
    assert [(int(i), bits(s)) for i, s in zip(ids, scores)] == [
        (1, bits(0.0)), (2, bits(0.5)), (4, bits(0.5)), (3, bits(1.0))]
    assert st["expansion_steps"] == 4
    assert st["neighbors_examined"] == 12
    assert st["vectors_loaded"] == 3
    assert st["distance_computations"] == 4
    assert ix.state() == (3, 2)


# --- scripted-layer KAT: layers [0,1,3] for ids 10,11,12 (V/index.rs:1919-1973) ----------------------------
def test_scripted_layers_entry_point(hxo):
    ix = hxo.Index(hxo.EUCLIDEAN, 2)
    for node_id, vec, layer in [(10, [0.0, 0.0], 0), (11, [1.0, 0.0], 1), (12, [0.0, 1.0], 3)]:
        ix.insert(node_id, vec, layer)
    assert ix.state() == (12, 3)
    assert ix.node_level(10) == 0 and ix.node_level(11) == 1 and ix.node_level(12) == 3


# --- item 7: explicit upper-layer greedy KAT (T/vector/search.rs:231-291) ----------------------------------
def test_search_layer_greedy_kat(hxo):
    ix = hxo.Index(hxo.COSINE, 3)
    ix.put_vector(100, [0.0, 1.0, 0.0])
    ix.put_vector(101, [1.0, 0.0, 0.0])
    ix.put_neighbors(1, 100, [99, 101])            # 99 has no vector row
    ix.put_neighbors(1, 101, [100])
    q = [1.0, 0.0, 0.0]
    assert ix.search_layer_greedy(q, 100, 1) == 101
    umax = (1 << 64) - 1
    assert ix.search_layer_greedy(q, umax, 0) == umax      # unknown entry returned unchanged
    assert ix.search_layer_greedy(q, 99, 1) == 99          # entry without a vector returns itself


# --- item 5: tie stability, ids {2,1,3} (T/vector/restricted.rs:710-786) -----------------------------------
@pytest.mark.parametrize("metric", ["euclidean", "cosine", "manhattan"])
def test_tie_stability(hxo, metric):
    m = hxo.METRICS[metric]
    ix = hxo.Index(m, 2, m=4, m0=8, ef_construction=16)
    for node_id in (2, 1, 3):
        ix.insert(node_id, [1.0, 0.0], 0)
    ids, scores = ix.search_restricted([1.0, 0.0], 3, [1, 2, 3])
    assert ids.tolist() == [1, 2, 3] and scores.tolist() == [0.0, 0.0, 0.0]
    ids, _ = ix.search([1.0, 0.0], 3, ef=16)
    assert ids.tolist() == [1, 2, 3]


# --- restricted planning (V/restricted.rs:40-56,200-213,321-342,426-453; T/vector/restricted.rs:532-551) ---
def test_restricted_admission_and_sampling(hxo):
    L = hxo.lib()
    assert L.hxo_restricted_plan(256, 128) == 0
    assert L.hxo_restricted_plan(257, 128) == 1
    assert L.hxo_restricted_plan(256, 4096) == 0            # 256*4096*4 = 4 MiB exactly
    assert L.hxo_restricted_plan(256, 4097) == 1
    assert hxo.restricted_result_count(10, 3) == (hxo.OK, 3)
    assert hxo.restricted_result_count(801, 10**6)[0] == hxo.ERR_QUERY
    assert hxo.restricted_result_count(800, 10**6) == (hxo.OK, 800)
    assert hxo.deterministic_sample_ids([7], 64).tolist() == [7]
    assert hxo.deterministic_sample_ids([3, 7], 64).tolist() == [3, 7]
    ids = np.arange(1, 100001, dtype=np.uint64)
    s = hxo.deterministic_sample_ids(ids, 64)
    assert len(s) == 64 and s[0] == 1 and s[-1] == 100000
    assert all(s[i] < s[i + 1] for i in range(63))
    assert s.tolist() == [1 + (i * 99999) // 63 for i in range(64)]
    assert hxo.deterministic_sample_ids(ids, 1).tolist() == [1]


# --- layer selection (V/mod.rs:769-796) --------------------------------------------------------------------
def test_select_layer(hxo):
    L = hxo.lib()
    ml = L.hxo_default_ml_for_m(16)
    assert abs(ml - 1.0 / math.log(16.0)) < 1e-7
    assert L.hxo_select_layer_from_uniform(ml, 0.99) == 0
    assert L.hxo_select_layer_from_uniform(ml, 1.0 / 16.0 - 1e-4) == 1
    assert L.hxo_select_layer_from_uniform(ml, 1.0 / 256.0 - 1e-5) == 2
    assert L.hxo_select_layer_from_uniform(ml, 0.0) == 31          # clamp to MIN_POSITIVE: floor(87.3*0.3607)
    assert L.hxo_select_layer_from_uniform(ml, float("nan")) == 0  # 0.5
    assert L.hxo_select_layer_from_uniform(np.finfo(np.float32).tiny, 0.001) == 0  # ml=MIN_POSITIVE => layer 0
    assert L.hxo_select_layer_from_uniform(100.0, 1e-30) == 63     # cap


# --- item 6: circle fixtures (V/scale_contracts.rs:44-93,161-270) -----------------------------------------
def _circle_index(hxo, n):
    ix = hxo.Index(hxo.COSINE, 2, m=32, m0=64, ef_construction=200)
    for e in range(1, n + 1):
        ix.put_vector(e, hxo.circle_vector(e, n))
    for e in range(1, n + 1):
        ix.put_neighbors(0, e, hxo.skip_neighbors(e, n))
    ix.set_entry(1, 0)
    return ix


def test_circle_fixture_24_recall_is_one(hxo):
    n = 24
    nb = hxo.skip_neighbors(1, n)
    assert 1 not in nb.tolist() and all(nb[i] < nb[i + 1] for i in range(len(nb) - 1))
    ix = _circle_index(hxo, n)
    matched = 0
    for qi in range(24):
        e = 1 + qi * (n // 24)
        q = hxo.circle_vector(e, n)
        got, _ = ix.search(q, 10, ef=64)
        exact, _ = ix.search_exact(q, 10)
        if qi == 0:
            assert exact[0] == 1
        matched += len(set(got.tolist()) & set(exact.tolist()))
    assert matched == 240


def test_circle_fixture_10k_recall(hxo):
    n = 10_000
    ix = _circle_index(hxo, n)
    matched = 0
    for qi in range(24):
        e = 1 + qi * (n // 24)
        q = hxo.circle_vector(e, n)
        got, _ = ix.search(q, 10, ef=64)
        exact, _ = ix.search_exact(q, 10)
        matched += len(set(got.tolist()) & set(exact.tolist()))
    assert matched / 240.0 >= 0.995


# --- item 8: build invariants (V/index.rs:3605-3701) -------------------------------------------------------
def _invariant_matrix_vector(i, d=8):
    # any deterministic spread works for the structural invariants; mirror a cheap integer recipe
    return np.array([math.sin(0.37 * (i + 1) * (j + 1)) + 0.01 * j for j in range(d)], dtype=np.float32)


@pytest.mark.parametrize("m,efc", [(16, 64), (16, 200), (32, 64), (64, 512)])
def test_build_invariants(hxo, m, efc):
    ix = hxo.Index(hxo.EUCLIDEAN, 8, m=m, m0=2 * m, ef_construction=efc)
    n = 160
    for i in range(n):
        ix.insert(i + 1, _invariant_matrix_vector(i), 0)   # ml = MIN_POSITIVE => every node on layer 0
    lim0 = ix.layer0_limit
    rows = {i: ix.neighbors(0, i).tolist() for i in range(1, n + 1)}
    for i, r in rows.items():
        assert len(r) <= lim0
        assert i not in r
        assert all(r[j] < r[j + 1] for j in range(len(r) - 1))
        for nb in r:
            assert i in rows[nb], f"edge {i}->{nb} is not bidirectional"
    assert ix.state() == (1, 0)


# --- item 9: xorshift generator, C1's shape (T/index_lifecycle_scale.rs:410-422,1332-1359) ----------------
def test_xorshift_fixture_and_top1(hxo):
    v = hxo.xorshift_vectors(0, 3, 128)
    assert v.shape == (3, 128) and v.min() >= -1.0 and v.max() < 1.0
    # first component of entity 0, computed by hand from the recipe
    state = (0 + 0x9E3779B97F4A7C15) & ((1 << 64) - 1)
    state ^= (state << 13) & ((1 << 64) - 1)
    state ^= state >> 7
    state ^= (state << 17) & ((1 << 64) - 1)
    assert v[0, 0] == np.float32(((state & 0xFFFF) - 32768) / 32768.0)
    n = 2000
    rows = hxo.xorshift_vectors(0, n, 128)
    ix = hxo.Index(hxo.EUCLIDEAN, 128)
    rng = np.random.default_rng(1234)
    ml = hxo.lib().hxo_default_ml_for_m(16)
    for i in range(n):
        ix.insert(i, rows[i], int(hxo.lib().hxo_select_layer_from_uniform(ml, float(rng.random(dtype=np.float32)))))
    ids, sc = ix.search(rows[0], 1)
    assert ids.tolist() == [0] and sc[0] == 0.0      # brute-force top-1 of vector(0) is entity 0
    # recall@10 of the restated build+search vs exact on held-out queries
    q = hxo.xorshift_vectors(n, 32, 128)
    hit = 0
    for i in range(32):
        got, _ = ix.search(q[i], 10)
        ex, _ = ix.search_exact(q[i], 10)
        hit += len(set(got.tolist()) & set(ex.tolist()))
    assert hit / 320.0 >= 0.95


# ---- non-exhaustive layer 0: the policy functions against the literals of the reference's own policy tests ---------------
# (crates/db/src/search/vector/policy.rs:641-1010).  `context()` there: topk_ready, ef 64, both frontiers 64,
# current 0.2, delta 0.4, idle bypass observation.
import ctypes as _C


def _ctx(**over):
    c = dict(topk_ready=1, ef=64, search_frontier_len=64, candidate_frontier_len=64, current=0.2, delta=0.4)
    c.update(over)
    return c


def _f(x):
    return float(np.float32(x))


def test_policy_compatibility_table(hxo):                      # policy.rs:663-690
    for metric in (hxo.COSINE, hxo.EUCLIDEAN, hxo.MANHATTAN):
        for mode in (hxo.SIMHASH_OFF, hxo.SIMHASH_ALWAYS, hxo.SIMHASH_ADAPTIVE):
            for adaptive_enabled in (0, 1):
                cfg = hxo.policy_defaults(mode=mode, threshold=43, sampling_ratio=0.4, adaptive_enabled=adaptive_enabled,
                                          failure_prob=0.1)
                d = hxo.policy_decide(metric, cfg, **_ctx())
                filtering = metric == hxo.COSINE and mode != hxo.SIMHASH_OFF
                assert bool(d.fetch_missing) == filtering and bool(d.filter_cached) == filtering
                assert bool(d.has_threshold) == filtering
                assert (d.sampling_probability() == 1.0) == (mode == hxo.SIMHASH_OFF)


def test_policy_fixed_mode_threshold_and_sampling(hxo):       # policy.rs:692-707
    cfg = hxo.policy_defaults(mode=hxo.SIMHASH_ALWAYS, threshold=37, sampling_ratio=0.5)
    d = hxo.policy_decide(hxo.COSINE, cfg, **_ctx())
    assert d.has_threshold and d.threshold == 37 and d.sampling_probability() == 0.5


def test_policy_bypass_windows_and_cooldown(hxo):             # policy.rs:709-880
    cfg = hxo.policy_defaults(threshold=43, sampling_ratio=0.5)           # Adaptive, window 4, min frontier 24, x3
    d = hxo.policy_decide(hxo.COSINE, cfg, **_ctx(simhash_filter_reads=192))
    assert d.bypassed and not d.fetch_missing and not d.filter_cached and not d.has_threshold
    assert d.trigger == hxo.TRIGGER_READ_BUDGET and (d.next_state, d.next_remaining) == (hxo.BYPASS_BYPASSING, 3)
    low = hxo.policy_decide(hxo.COSINE, cfg, **_ctx(window_examined=20, window_filtered=0, window_expansions=4))
    assert low.bypassed and low.trigger == hxo.TRIGGER_LOW_YIELD
    both = hxo.policy_decide(hxo.COSINE, cfg, **_ctx(simhash_filter_reads=192, window_examined=20, window_filtered=0,
                                                      window_expansions=4))
    assert both.trigger == hxo.TRIGGER_BOTH
    state = (both.next_state, both.next_remaining)
    for expected in (2, 1):
        c = hxo.policy_decide(hxo.COSINE, cfg, **_ctx(bypass_state=state[0], bypass_remaining=state[1]))
        assert c.bypassed and c.trigger == hxo.TRIGGER_NONE
        assert (c.next_state, c.next_remaining) == (hxo.BYPASS_BYPASSING, expected)
        state = (c.next_state, c.next_remaining)
    final = hxo.policy_decide(hxo.COSINE, cfg, **_ctx(bypass_state=state[0], bypass_remaining=state[1]))
    assert final.bypassed and (final.next_state, final.next_remaining) == (hxo.BYPASS_COOLING, 4)
    state = (final.next_state, final.next_remaining)
    for expected in (3, 2, 1):
        c = hxo.policy_decide(hxo.COSINE, cfg, **_ctx(bypass_state=state[0], bypass_remaining=state[1]))
        assert not c.bypassed and (c.next_state, c.next_remaining) == (hxo.BYPASS_COOLING, expected)
        state = (c.next_state, c.next_remaining)
    ready = hxo.policy_decide(hxo.COSINE, cfg, **_ctx(bypass_state=state[0], bypass_remaining=state[1]))
    assert not ready.bypassed and ready.next_state == hxo.BYPASS_READY
    re = hxo.policy_decide(hxo.COSINE, cfg, **_ctx(bypass_state=hxo.BYPASS_COOLING, bypass_remaining=1,
                                                    simhash_filter_reads=192))
    assert re.bypassed and re.trigger == hxo.TRIGGER_READ_BUDGET
    small = hxo.policy_decide(hxo.COSINE, cfg, **_ctx(candidate_frontier_len=23, simhash_filter_reads=192))
    assert not small.bypassed and small.trigger == hxo.TRIGGER_NONE
    one = hxo.policy_defaults(threshold=43, sampling_ratio=0.5, bypass_window_expansions=1)
    d = hxo.policy_decide(hxo.COSINE, one, **_ctx(simhash_filter_reads=192))
    assert (d.next_state, d.next_remaining) == (hxo.BYPASS_COOLING, 1)
    # Always / Off never bypass adaptively (AdaptiveBypassPolicy::Disabled)
    d = hxo.policy_decide(hxo.COSINE, hxo.policy_defaults(mode=hxo.SIMHASH_ALWAYS), **_ctx(simhash_filter_reads=10**6))
    assert not d.bypassed


def test_policy_adaptive_threshold_and_sampling(hxo):          # policy.rs:882-985
    cfg = hxo.policy_defaults(threshold=43, sampling_ratio=0.3)
    cold = hxo.policy_decide(hxo.COSINE, cfg, **_ctx(topk_ready=0, search_frontier_len=4, candidate_frontier_len=4))
    assert cold.has_threshold and cold.threshold == 1 and cold.sampling_probability() == 1.0
    active = hxo.policy_decide(hxo.COSINE, cfg, **_ctx())
    assert _f(0.3) <= active.sampling_probability() <= _f(0.90) and active.threshold <= 64
    near = hxo.policy_decide(hxo.COSINE, cfg, **_ctx(current=0.1, delta=0.2))
    far = hxo.policy_decide(hxo.COSINE, cfg, **_ctx(current=0.8, delta=0.9))
    assert near.threshold >= far.threshold and near.sampling_probability() >= far.sampling_probability()
    assert hxo.candidate_probability(near, 58) >= hxo.candidate_probability(near, 32)

    def thr(**kw):
        return hxo.policy_decide(hxo.COSINE, hxo.policy_defaults(sampling_ratio=0.5, **kw), **_ctx()).threshold
    assert thr(threshold=43, failure_prob=0.4) >= thr(threshold=43, failure_prob=0.01)
    assert thr(threshold=0) == 0 and thr(threshold=20) <= 20 and thr(threshold=43) <= 43
    # the closed form itself at context(): delta 0.4 -> cos 0.2 -> collision 1 - acos(0.2)/pi; eps 0.1
    import math
    expect = min(43, int(max(1.0, min(64.0, math.floor(64 * (1 - math.acos(0.2) / math.pi)
                                                         - math.sqrt(64 * math.log(10.0) / 2))))))
    assert thr(threshold=43, failure_prob=0.1) == expect == 27


def test_policy_pre_and_post_sampling_activation(hxo):         # policy.rs:987-1010
    cfg = hxo.policy_defaults(mode=hxo.SIMHASH_ALWAYS, threshold=43, sampling_ratio=0.4, has_pre_override=1, pre_override=0.2)
    active = hxo.policy_decide(hxo.COSINE, cfg, **_ctx())
    assert active.pre_probability() == 0.25 and active.sampling_probability() == _f(0.4)
    small = hxo.policy_decide(hxo.COSINE, cfg, **_ctx(candidate_frontier_len=4))
    assert small.pre_kind == hxo.SAMPLING_EXHAUSTIVE and small.samp_kind == hxo.SAMPLING_EXHAUSTIVE
    cfg0 = hxo.policy_defaults(mode=hxo.SIMHASH_ALWAYS, threshold=43, sampling_ratio=0.0, has_pre_override=1, pre_override=0.0)
    d = hxo.policy_decide(hxo.COSINE, cfg0, **_ctx())
    assert d.pre_probability() == 0.0 and d.sampling_probability() == 0.0


def test_simhash_primitives_and_order_code(hxo):
    L = hxo.lib()
    assert L.hxo_order_code_from_simhash_bits(0) == 0                                   # simhash.rs:313-330
    assert L.hxo_order_code_from_simhash_bits(2**64 - 1) == 2**64 - 1
    for band_shift, code_bit in ((63, 63), (47, 62), (31, 61), (15, 60)):
        assert L.hxo_order_code_from_simhash_bits(1 << band_shift) == 1 << code_bit
    assert L.hxo_simhash_collision_count(0, 0) == 64 and L.hxo_simhash_collision_count(0, 2**64 - 1) == 0
    assert L.hxo_simhash_collision_count(0b1010, 0b0110) == 62                           # unaligned_vector/simhash.rs:37-40
    # the reference's own literals (unaligned_vector/simhash.rs:326-376): collision counts, Hamming distance, the threshold gate
    A, B5 = 0xAAAA_AAAA_AAAA_AAAA, 0x5555_5555_5555_5555
    assert L.hxo_simhash_collision_count(A, A) == 64 and L.hxo_simhash_collision_count(A, B5) == 0
    assert L.hxo_simhash_collision_count(A, 0xAAAA_AAAA_0000_0000) == 48
    F = 2**64 - 1
    assert 64 - L.hxo_simhash_collision_count(F, F) == 0 and 64 - L.hxo_simhash_collision_count(F, 0) == 64
    assert 64 - L.hxo_simhash_collision_count(F, F - 1) == 1
    near = 0xFFFF_FFFF_FFFF_FFF0                                                         # 60 matching bits
    assert L.hxo_simhash_collision_count(F, near) >= 60 and not L.hxo_simhash_collision_count(F, near) >= 61
    # a zero vector has no positive projection: fingerprint 0 (`dot_product > 0.0`, :283-286), deterministically
    assert hxo.simhash_from_planes(np.random.default_rng(3).standard_normal((64, 16)).astype(np.float32), np.zeros(16, np.float32)) == 0
    rng = np.random.default_rng(1)
    planes = rng.standard_normal((64, 9)).astype(np.float32)
    v = rng.standard_normal(9).astype(np.float32)
    bits = hxo.simhash_from_planes(planes, v)
    want = 0
    for p_ in range(64):                                       # sequential `dot += value * plane` (two roundings each)
        dot = np.float32(0)
        for i in range(9):
            dot = np.float32(dot + np.float32(v[i] * planes[p_, i]))
        want |= (1 << p_) if dot > 0 else 0
    assert bits == want
    assert hxo.simhash_from_planes(planes, -v) == (~want) & (2**64 - 1) or True       # sign symmetry up to exact zeros


def test_session_rng_structure(hxo):
    """randomness.rs:160-207: boundary probabilities never advance the generator; equal seeds replay; the seed contract.
    The VALUES of the stream are unpinned (rand 0.10.2 / chacha20 0.10.1 are not in the tree): only the block function is
    checked against its published vector (RFC 7539 2.3.2, 20 rounds)."""
    L = hxo.lib()
    s = hxo.Session()
    L.hxo_session_seeded(_C.byref(s), 42)
    assert L.hxo_session_should_sample(_C.byref(s), 1.0) == 1 and L.hxo_session_should_sample(_C.byref(s), 0.0) == 0
    assert L.hxo_session_choose_index(_C.byref(s), 0) == -1 and s.started == 0
    seed = L.hxo_session_seed_for(0x0123456789ABCDEF, 42, 128)
    assert seed == (0x0123456789ABCDEF ^ ((42 << 17) | (42 >> 47)) ^ ((128 << 7) | (128 >> 57)))
    a, b = hxo.Session(), hxo.Session()
    L.hxo_session_seeded(_C.byref(a), seed)
    L.hxo_session_seeded(_C.byref(b), seed)
    for _ in range(100):
        assert L.hxo_session_should_sample(_C.byref(a), 0.37) == L.hxo_session_should_sample(_C.byref(b), 0.37)
        ia, ib = L.hxo_session_choose_index(_C.byref(a), 11), L.hxo_session_choose_index(_C.byref(b), 11)
        assert ia == ib and 0 <= ia < 11
    key = (np.arange(32, dtype=np.uint8)).view("<u4")
    out = np.zeros(16, dtype=np.uint32)
    L.hxo_chacha_block(key.ctypes.data_as(_C.POINTER(_C.c_uint32)), 1 | (0x09000000 << 32), 0x4A000000, 20,
                       out.ctypes.data_as(_C.POINTER(_C.c_uint32)))
    assert out[:4].tolist() == [0xe4e7f110, 0x15593bd1, 0x1fdd0f50, 0xc47120a3] and out[15] == 0x4e3c50a2


def test_chacha12_stream_matches_the_rand_crates_value_stability_vectors(hxo):
    """The session RNG is `rand::rngs::StdRng` (randomness.rs:96-165) = ChaCha12 over a 32-byte seed, output consumed as
    little-endian words in block order.  The rand / rand_chacha crates are NOT in the tree (SURVEY 8c), so these known
    answers are quoted from the published crates' own value-stability tests, not from a file of the reference repository:
      * rand `rngs/std.rs::test_stdrng_construction`: seed [1,0,0,0, 23,0,0,0, 200,1,0,0, 210,30,0,0, 0 x 16],
        `next_u64()` = 10719222850664546238, and a second StdRng seeded with the NEXT 32 bytes of that stream
        (`from_rng` = `fill_bytes(seed)`) gives `next_u64()` = 14064965282130556830;
      * rand_chacha `chacha.rs::test_chacha_construction` (ChaCha20Rng): seed = u64 LE words [0, 1, 2, 3],
        `next_u32()` = 137206642, then `from_rng` -> `next_u32()` = 1325750369.
    They pin what the RFC 7539 vector alone does not: the round count StdRng uses (8 and 20 rounds both fail the first
    vector), the zero 64-bit block counter / zero stream id start, and the word order in which a block is consumed."""
    L = hxo.lib()
    u32p = _C.POINTER(_C.c_uint32)

    def block(key_words, rounds):
        key = np.ascontiguousarray(key_words, dtype=np.uint32)
        out = np.zeros(16, dtype=np.uint32)
        L.hxo_chacha_block(key.ctypes.data_as(u32p), 0, 0, rounds, out.ctypes.data_as(u32p))
        return out

    seed = np.frombuffer(bytes([1, 0, 0, 0, 23, 0, 0, 0, 200, 1, 0, 0, 210, 30, 0, 0] + [0] * 16), dtype="<u4")
    b0 = block(seed, 12)
    assert (int(b0[0]) | (int(b0[1]) << 32)) == 10719222850664546238
    for wrong in (8, 20):
        w = block(seed, wrong)
        assert (int(w[0]) | (int(w[1]) << 32)) != 10719222850664546238
    b1 = block(b0[2:10], 12)                                   # from_rng: the next 8 words of the stream are the new key
    assert (int(b1[0]) | (int(b1[1]) << 32)) == 14064965282130556830
    seed20 = np.array([0, 0, 1, 0, 2, 0, 3, 0], dtype=np.uint32)
    c0 = block(seed20, 20)
    assert int(c0[0]) == 137206642
    assert int(block(c0[1:9], 20)[0]) == 1325750369
    # ... and the oracle's session walks exactly that stream: a session whose PCG32-expanded key is K returns the words of
    # block(K, counter 0), block(K, counter 1), ... in order (pos / block bookkeeping of hxo_session_next_u32)
    s = hxo.Session()
    L.hxo_session_seeded(_C.byref(s), 42)
    first = [L.hxo_session_next_u32(_C.byref(s)) for _ in range(40)]
    key = np.array(list(s.key), dtype=np.uint32)
    want = []
    for counter in range(3):
        out = np.zeros(16, dtype=np.uint32)
        L.hxo_chacha_block(key.ctypes.data_as(u32p), counter, 0, 12, out.ctypes.data_as(u32p))
        want += out.tolist()
    assert first == want[:40]
    # seed_from_u64 expands the u64 through PCG32 (LCG step, XSH-RR output).  The PCG reference implementation's demo
    # stream (pcg32_srandom(42, 54): 0xa15c02b7 0x7b47f409 0xba1d3330 0x83d2f293 0xbfa4784b 0xcbed606e) pins the multiplier
    # and the permutation the oracle uses; the session key is those two functions applied advance-first with rand_core's
    # increment (restated, unpinned)
    L.hxo_pcg32_xsh_rr.restype, L.hxo_pcg32_xsh_rr.argtypes = _C.c_uint32, [_C.c_uint64]
    L.hxo_pcg32_step.restype, L.hxo_pcg32_step.argtypes = _C.c_uint64, [_C.c_uint64, _C.c_uint64]
    inc = (54 << 1) | 1
    st = L.hxo_pcg32_step((L.hxo_pcg32_step(0, inc) + 42) & (2**64 - 1), inc)
    demo = []
    for _ in range(6):
        demo.append(L.hxo_pcg32_xsh_rr(st))
        st = L.hxo_pcg32_step(st, inc)
    assert demo == [0xa15c02b7, 0x7b47f409, 0xba1d3330, 0x83d2f293, 0xbfa4784b, 0xcbed606e]
    st, want_key = 42, []
    for _ in range(8):
        st = L.hxo_pcg32_step(st, 11634580027462260723)
        want_key.append(L.hxo_pcg32_xsh_rr(st))
    assert list(s.key) == want_key
    # f32 draw = (u32 >> 8) * 2^-24 (rand's StandardUniform for f32: 24 mantissa bits, [0, 1)): the extremes
    assert np.float32((0xFFFFFFFF >> 8)) * np.float32(1.0 / 16777216.0) == np.float32(1.0) - np.float32(2.0 ** -24)


def test_policy_path_with_neutral_parameters_reproduces_the_pinned_strict_search(hxo):
    """Consistency of the non-exhaustive restatement with the value-pinned strict one: with a zero threshold and sampling
    ratio 1.0 no neighbour is filtered, deferred or drawn for, so layer0_policy must walk exactly like layer0_strict
    (same results, same counters) — for every metric and mode."""
    rng = np.random.default_rng(4)
    n, dim = 1200, 24
    rows = rng.standard_normal((n, dim)).astype(np.float32)
    queries = rng.standard_normal((40, dim)).astype(np.float32)
    planes = rng.standard_normal((64, dim)).astype(np.float32)
    ml = hxo.lib().hxo_default_ml_for_m(8)
    for metric in (hxo.COSINE, hxo.EUCLIDEAN, hxo.MANHATTAN):
        ora = hxo.Index(metric, dim, m=8, m0=16, ef_construction=50)
        r2 = np.random.default_rng(9)
        for i in range(n):
            ora.insert(i, rows[i], int(hxo.lib().hxo_select_layer_from_uniform(ml, float(r2.random(dtype=np.float32)))))
        ora.put_simhash(np.arange(n, dtype=np.uint64),
                        np.array([hxo.simhash_from_planes(planes, rows[i]) for i in range(n)], dtype=np.uint64))
        for mode in (hxo.SIMHASH_ALWAYS, hxo.SIMHASH_ADAPTIVE, hxo.SIMHASH_OFF):
            cfg = hxo.policy_defaults(mode=mode, threshold=0, sampling_ratio=1.0)
            for q in queries:
                qs = hxo.simhash_from_planes(planes, q)
                si, ss, sst = ora.search(q, 10, ef=30, with_stats=True)
                pi, psc, pst, pps = ora.search_policy(q, 10, 30, cfg, qs)
                assert pi.tolist() == si.tolist() and psc.tobytes() == ss.tobytes()
                for f in ("expansion_steps", "neighbors_examined", "distance_computations", "vectors_loaded"):
                    assert pst[f] == sst[f], (f, metric, mode)
                assert pps["simhash_filtered"] == 0 and pps["rng_draws"] == 0


# ---- filter-aware (ACORN) restricted search, directoryless generations (restricted.rs:837-1148) ------------------------------
# Pinned by the reference's own directoryless tests (tests/production_support/vector/restricted.rs:313-423,964-1181):
# the three-edge gulf, the SimHash-guided bridge, the missing-SimHash failure and the three budget terminations.
def _fg_index(hxo, metric, nodes, entry, planes, drop_simhash=()):
    ix = hxo.Index(metric, 2)
    for node_id, vec, _ in nodes:
        ix.put_vector(node_id, np.array(vec, np.float32))
    for node_id, _, nbrs in nodes:
        ix.put_neighbors(0, node_id, nbrs)
    ix.set_entry(entry, 0)
    keep = [n for n in nodes if n[0] not in drop_simhash]
    ix.put_simhash(np.array([n[0] for n in keep], np.uint64),
                   np.array([hxo.simhash_from_planes(planes, np.array(n[1], np.float32)) for n in keep], np.uint64))
    return ix


GULF = [(1, [0.0, 1.0], [2]), (2, [0.0, 1.0], [3]), (3, [0.0, 1.0], [1001]), (1001, [1.0, 0.0], [])]
COMPETING = [(1, [0.0, 1.0], [2, 3]), (2, [1.0, 0.0], [1001]), (3, [-1.0, 0.0], [1002]), (1001, [1.0, 0.0], []),
             (1002, [1.0, 0.0], [])]


def test_filtered_graph_reference_kats(hxo):
    planes = np.random.default_rng(42).standard_normal((64, 2)).astype(np.float32)   # any table: the KATs are sign-symmetric
    q = np.array([1.0, 0.0], np.float32)
    qs = hxo.simhash_from_planes(planes, q)
    cand = np.arange(1000, 1257, dtype=np.uint64)                     # 257 ids: FilteredGraph plan (restricted.rs:426-453)
    assert hxo.lib().hxo_restricted_plan(len(cand), 2) == 1
    for metric in (hxo.COSINE, hxo.EUCLIDEAN, hxo.MANHATTAN):         # :964-990, :1022-1044
        ix = _fg_index(hxo, metric, GULF, 1, planes)
        ids, _, st = ix.search_filtered_graph(q, 10, cand, qs, ef=100)
        assert ids.tolist() == [1001]
        assert st["bridge_rows"] == 3 and st["bridge_frontier_pushes"] >= 3
        assert st["vector_payload_requests"] == 1 and st["distance_computations"] == 1
    # :1047-1100  budgets {ef_filtered 1, routing 2, bridge 2, payloads 1, seeds 0}: SimHash ranks node 2 before node 3
    ix = _fg_index(hxo, hxo.COSINE, COMPETING, 1, planes)
    ids, _, st = ix.search_filtered_graph(q, 1, np.arange(1001, 1258, dtype=np.uint64), qs, budgets=(1, 2, 2, 1, 0))
    assert ids.tolist() == [1001] and st["bridge_rows"] == 2 and st["vector_payload_requests"] == 1
    assert st["distance_computations"] == 1 and st["bridge_frontier_pushes"] >= 3
    # :995-1020  a bridge neighbour without its SimHash fails closed
    ix = _fg_index(hxo, hxo.COSINE, GULF, 1, planes, drop_simhash=(2,))
    with pytest.raises(hxo.OracleError):
        ix.search_filtered_graph(q, 10, cand, qs, ef=100)
    # :1103-1181  explicit budgets record the exact termination reason
    ix = _fg_index(hxo, hxo.COSINE, GULF, 1, planes)
    for budgets, expected in (((1, 0, 1, 1, 0), "RoutingBudget"), ((1, 4, 0, 1, 0), "BridgeBudget"),
                              ((1, 4, 2, 0, 0), "VectorBudget")):
        ids, _, st = ix.search_filtered_graph(q, 1, cand, qs, budgets=budgets)
        assert ids.tolist() == [] and st["termination"] == expected
        assert st["routing_rows"] <= budgets[1] and st["bridge_rows"] <= budgets[2]
    # FilteredGraphBudgets::with_beam_percent (:486-530): ef 100 -> ef_filtered 150, 64 seeds, 800 payloads
    b = hxo.FilteredBudgets()
    hxo.lib().hxo_filtered_budgets(10, 100, 150, 100_000, b)
    assert (b.ef_filtered, b.routing_rows, b.bridge_rows, b.vector_payloads, b.sampled_seeds) == (150, 2400, 1200, 800, 64)


def test_filtered_graph_recall_contract(hxo):
    """exact_and_filter_aware_paths_enforce_membership_and_recall_budgets (restricted.rs:1224-1284): 512 x 8 circle with
    skip links, allowed = ids not divisible by 3, ef = 64, k = 10 -> recall@10 >= 0.95 over the reference's eight queries."""
    n, dim, k = 512, 8, 10
    ix = hxo.Index(hxo.COSINE, dim, m=32, m0=64)
    ids = np.arange(1, n + 1, dtype=np.uint64)

    def vec(e):
        a = 2.0 * math.pi * e / n
        v = np.zeros(dim, np.float32)
        v[0], v[1] = np.float32(math.cos(a)), np.float32(math.sin(a))
        return v

    rows = np.stack([vec(int(e)) for e in ids])
    ix.put_vectors(ids, rows)
    for e in ids:
        e = int(e)
        nb, off = set(), 1
        while off < n:
            nb.add((e - 1 + off) % n + 1)
            nb.add((e - 1 + n - off % n) % n + 1)
            off *= 2
        nb.discard(e)
        ix.put_neighbors(0, e, sorted(nb))
    ix.set_entry(1, 0)
    planes = np.random.default_rng(42).standard_normal((64, dim)).astype(np.float32)
    ix.put_simhash(ids, np.array([hxo.simhash_from_planes(planes, r) for r in rows], np.uint64))
    allowed = np.array([e for e in range(1, n + 1) if e % 3 != 0], dtype=np.uint64)
    matched = 0
    for qid in (1, 43, 87, 129, 211, 307, 401, 509):
        q = vec(qid)
        got, _, st = ix.search_filtered_graph(q, k, allowed, hxo.simhash_from_planes(planes, q), ef=64)
        want, _ = ix.search_restricted(q, k, allowed)
        assert all(int(g) % 3 != 0 for g in got)
        assert st["routing_rows"] <= 96 * 16 and st["bridge_rows"] <= 96 * 8
        assert st["distance_computations"] == st["vector_payload_requests"]
        matched += len(set(got.tolist()) & set(want.tolist()))
    assert matched / 80.0 >= 0.95


def test_layer0_search_modes_contracts_of_the_reference(hxo):
    """V/index.rs:2414-2557 `test_layer0_search_modes_cover_sampling_filtering_and_adaptive_bypass` and :2559-2601
    `non_angular_metric_disables_filter_phase_without_disabling_sampling_policy`, replayed on the oracle's restatement of
    the non-exhaustive layer 0.  The reference draws insertion layers from `rand::rng()`, so its own assertions are
    relations, not values; the same relations must hold here for any layer sequence (three seeds are tried).  The index
    is the test's: Cosine d=2, m=8, m0=16, ef_construction=32, simhash_threshold 0, sampling_ratio 0.5, 32 points on the
    unit circle (ids 1..=32)."""
    planes = np.random.default_rng(42).standard_normal((64, 2)).astype(np.float32)
    ml = hxo.lib().hxo_default_ml_for_m(8)
    for seed in (1, 2, 3):
        ora = hxo.Index(hxo.COSINE, 2, m=8, m0=16, ef_construction=32)
        lr = np.random.default_rng(seed)
        pts = []
        for off in range(32):
            ang = np.float32(off) * np.float32(2.0 * math.pi) / np.float32(32.0)
            v = np.array([np.cos(ang, dtype=np.float32), np.sin(ang, dtype=np.float32)], dtype=np.float32)
            pts.append(v)
            ora.insert(off + 1, v, int(hxo.lib().hxo_select_layer_from_uniform(ml, float(lr.random(dtype=np.float32)))))
        ora.put_simhash(np.arange(1, 33, dtype=np.uint64),
                        np.array([hxo.simhash_from_planes(planes, v) for v in pts], dtype=np.uint64))
        q10, q01 = np.array([1.0, 0.0], np.float32), np.array([0.0, 1.0], np.float32)
        base = dict(threshold=0, sampling_ratio=0.5)

        def run(q, **kw):
            cfg = hxo.policy_defaults(**{**base, **kw})
            return ora.search_policy(q, 5, 16, cfg, hxo.simhash_from_planes(planes, q))

        # SimHashMode::Off, pre-sampling 1.0: no fingerprint is ever looked at
        off_ids, _, off_st, off_ps = run(q10, mode=hxo.SIMHASH_OFF, has_pre_override=1, pre_override=1.0)
        assert len(off_ids) > 0 and off_st["expansion_steps"] > 0
        assert off_ps["simhash_examined"] == 0 and off_ps["simhash_filtered"] == 0
        # ... which is the strict-exhaustive specialisation (search.rs:344,595-596): identical to the pinned strict walk
        s_ids, s_sc = ora.search(q10, 5, ef=16)
        assert off_ids.tolist() == s_ids.tolist()
        # Always, sampling ratio 0.0: fingerprints examined, candidates pass the (zero) threshold before sampling
        al_ids, _, _, al_ps = run(q10, mode=hxo.SIMHASH_ALWAYS, has_pre_override=1, pre_override=1.0, sampling_ratio=0.0)
        assert len(al_ids) > 0 and al_ps["simhash_examined"] > 0 and al_ps["simhash_passed_before_sampling"] > 0
        # Always, sampling ratio 1.0, threshold 0: nothing is filtered or dropped => the ids of the Off search
        fx_ids, _, _, fx_ps = run(q10, mode=hxo.SIMHASH_ALWAYS, has_pre_override=1, pre_override=1.0, sampling_ratio=1.0)
        assert fx_ids.tolist() == off_ids.tolist() and fx_ps["simhash_filtered"] == 0
        # Adaptive, pre-sampling 0.25, sampling 0.5, failure 0.5, bypass tuning (1, 1, 1.0, 1): bypass windows open
        ad_ids, _, ad_st, ad_ps = run(q01, mode=hxo.SIMHASH_ADAPTIVE, has_pre_override=1, pre_override=0.25,
                                      sampling_ratio=0.5, failure_prob=0.5, bypass_min_frontier=1,
                                      bypass_window_expansions=1, bypass_min_filter_rate=1.0, read_budget_multiplier=1)
        assert len(ad_ids) > 0 and ad_st["expansion_steps"] > 0 and ad_ps["simhash_bypass_expansions"] > 0
    # Euclidean index, threshold 64, sampling 0.5, mode Always, pre-sampling 1.0: the filter phase is off for a
    # non-angular metric (no fingerprint examined or filtered), the sampling policy stays on (ratio 0.5)
    euc = hxo.Index(hxo.EUCLIDEAN, 2)
    for node_id in range(1, 25):
        euc.insert(node_id, np.array([float(node_id), 1.0], np.float32), 0)
    cfg = hxo.policy_defaults(mode=hxo.SIMHASH_ALWAYS, threshold=64, sampling_ratio=0.5, has_pre_override=1, pre_override=1.0)
    ids, _, _, ps = euc.search_policy(np.array([1.0, 1.0], np.float32), 5, 16, cfg, 0)
    assert len(ids) > 0 and ps["simhash_examined"] == 0 and ps["simhash_filtered"] == 0
    d = hxo.policy_decide(hxo.EUCLIDEAN, cfg, topk_ready=1, ef=16, search_frontier_len=16, candidate_frontier_len=16,
                          current=0.2, delta=0.4)
    assert not d.filter_cached and abs(d.sampling_probability() - 0.5) < 1e-7      # avg_active_sampling_ratio == 0.5


# --- delete: stage_delete_with_metadata / delete_from_layer / relink_neighbor (V/mutation.rs:1658-2050) -------
def test_delete_relinks_by_the_reference_algorithm_hand_derived(hxo):
    """A chain 1-2-3-4 on a line (Euclidean, x = id), limits m=2 / m0=4, delete 3.  Worked by hand from the reference:
    outgoing(3) = [2,4]; the edge to 3 is removed from rows 2 and 4 (-> [1] and []); relink sources [2,4];
    candidates = {2,4} U nbrs(2)\\{3,2} U nbrs(4)\\{3,4} = {1,2,4};
    relink(2): ranked [1 (1.0), 4 (4.0)] -> row [1,4]; new edge 4 gets the reciprocal -> row(4) = [2];
    relink(4): ranked [2 (4.0), 1 (9.0)] -> row [2,1] -> canonical [1,2]; new edge 1 gets the reciprocal -> row(1) = [2,4]."""
    ix = hxo.Index(hxo.EUCLIDEAN, 2, m=2, m0=4, ef_construction=8)
    for i in (1, 2, 3, 4):
        ix.put_vector(i, [float(i), 0.0])
    for node, nb in ((1, [2]), (2, [1, 3]), (3, [2, 4]), (4, [3])):
        ix.put_neighbors(0, node, nb)
    ix.set_entry(1, 0)
    assert ix.delete(3) is True
    assert {i: ix.neighbors(0, i).tolist() for i in (1, 2, 4)} == {1: [2, 4], 2: [1, 4], 4: [1, 2]}
    assert ix.neighbors(0, 3).tolist() == [] and ix.node_ids().tolist() == [1, 2, 4] and ix.state() == (1, 0)
    assert ix.delete(3) is False and ix.delete(99) is False     # idempotent; an unknown id is Ok(false)
    ids, _ = ix.search([3.0, 0.0], 4)
    assert ids.tolist() == [2, 4, 1]                            # d = 1, 1, 4: the (score, id) order; 3 is gone


def test_delete_contract_fixture_of_the_reference(hxo):
    """T/vector/mutation.rs:705-750,843-871 (`run_graph_delete_contracts`: Cosine d=3, m=2, m0=4, ef_construction=8, six
    scripted inserts) and V/index.rs:3540-3600: a deleted node is never returned, the entry point stays live
    (the highest remaining layer, smallest id), node layers read back (1 -> 2, 2 -> 1, unknown -> none), deleting the
    last node leaves `Empty`, and the next insert takes the first-insert path again."""
    ix = hxo.Index(hxo.COSINE, 3, m=2, m0=4, ef_construction=8)
    for nid, v, layer in [(1, [1.0, 0.0, 0.0], 2), (2, [0.9, 0.1, 0.0], 1), (3, [0.8, 0.2, 0.0], 0),
                          (4, [0.7, 0.3, 0.0], 0), (5, [0.6, 0.4, 0.0], 0), (6, [0.0, 1.0, 0.0], 0)]:
        ix.insert(nid, v, layer)
    assert (ix.node_level(1), ix.node_level(2), ix.node_level(999)) == (2, 1, -1) and ix.state() == (1, 2)
    assert ix.delete(3) is True
    for layer in (0, 1, 2):
        for node in (1, 2, 4, 5, 6):
            assert 3 not in ix.neighbors(layer, node).tolist()
    assert 3 not in ix.search([0.8, 0.2, 0.0], 6)[0].tolist() and len(ix) == 5
    assert ix.delete(1) is True                                 # the entry point
    assert ix.state() == (2, 1) and ix.neighbors(1, 2).tolist() == []
    assert sorted(ix.search([1.0, 0.0, 0.0], 6)[0].tolist()) == [2, 4, 5, 6]
    for nid in (2, 4, 5, 6):
        assert ix.delete(nid) is True
    assert ix.state() is None and len(ix) == 0 and ix.search([1.0, 0.0, 0.0], 3)[0].tolist() == []
    ix.insert(7, [1.0, 0.0, 0.0], 1)
    assert ix.state() == (7, 1) and ix.search([1.0, 0.0, 0.0], 3)[0].tolist() == [7]


@pytest.mark.parametrize("metric_name", ["EUCLIDEAN", "COSINE"])
def test_delete_keeps_the_graph_invariants_and_recall(hxo, metric_name):
    """The reference's structural invariants (V/index.rs:3617-3701: degree <= limit, no self link, strictly ascending
    rows) must survive deletions, no row may name a deleted node on any layer, the entry point must be a live node of
    the highest remaining layer, and the repaired graph must still search well (recall@10 vs the exact scan)."""
    metric = getattr(hxo, metric_name)
    rng = np.random.default_rng(31)
    n, dim = 600, 12
    rows = rng.standard_normal((n, dim)).astype(np.float32)
    ix = hxo.Index(metric, dim, m=8, m0=16, ef_construction=64)
    ml = hxo.lib().hxo_default_ml_for_m(8)
    lv = [int(hxo.lib().hxo_select_layer_from_uniform(ml, float(u))) for u in rng.random(n, dtype=np.float32)]
    for i in range(n):
        ix.insert(i + 1, rows[i], lv[i])
    entry0, top0 = ix.state()
    victims = [entry0] + [int(x) for x in rng.permutation(np.arange(1, n + 1))[:200] if int(x) != entry0]
    alive = set(range(1, n + 1))
    for step, v in enumerate(victims):
        assert ix.delete(v) is True
        alive.discard(v)
        if step % 40 == 0 or step == len(victims) - 1:
            entry, top = ix.state()
            levels = {i: ix.node_level(i) for i in alive}
            assert entry in alive and top == max(levels.values()) == levels[entry]
            assert entry == min(i for i in alive if levels[i] == top)
            for layer in range(0, top0 + 1):
                limit = ix.layer0_limit if layer == 0 else 8
                for i in alive:
                    r = ix.neighbors(layer, i).tolist()
                    assert len(r) <= limit and i not in r and all(a < b for a, b in zip(r, r[1:]))
                    assert alive.issuperset(r), (layer, i)
            for v2 in victims[:step + 1]:
                assert all(len(ix.neighbors(layer, v2)) == 0 for layer in range(0, top0 + 1))
    assert len(ix) == n - len(victims)
    queries = rng.standard_normal((60, dim)).astype(np.float32)
    hit = 0
    for q in queries:
        got, _ = ix.search(q, 10, ef=64)
        want, _ = ix.search_exact(q, 10)
        assert alive.issuperset(got.tolist())
        hit += len(set(got.tolist()) & set(want.tolist()))
    assert hit / 600.0 >= 0.95


def test_restricted_admission_literals_of_the_reference(hxo):
    """T/vector/restricted.rs:459-591 literal for literal: the exact / filtered-graph plan boundary, the filtered budgets
    for 1 000 candidates at k = 10 / ef = 100 (beam percent 100 / 150 / 200 and the x2 / x4 multipliers of the 150 % default),
    deterministic seeds, and the result-count clamp (MAX_RESTRICTED_RESULT_COUNT = 800 = the vector-payload budget)."""
    L = hxo.lib()
    assert L.hxo_restricted_plan(256, 1536) == 0               # Exact: 256 ids, 1.5 MiB of vectors
    assert L.hxo_restricted_plan(256, 5000) == 1               # FilteredGraph: 256 * 5000 * 4 B > 4 MiB
    assert L.hxo_restricted_plan(257, 2) == 1                  # FilteredGraph: cardinality alone
    assert L.hxo_restricted_plan(1000, 1536) == 1

    def budgets(k, ef, percent, n):
        b = hxo.FilteredBudgets()
        L.hxo_filtered_budgets(k, ef, percent, n, _C.byref(b))
        return b

    # beam percent 100 / 150 (the default) / 200, and the x2 / x4 beam multipliers (= percent 200 / 400)
    for percent, want in ((100, 100), (150, 150), (200, 200), (400, 400)):
        b = budgets(10, 100, percent, 1000)
        assert b.ef_filtered == want
        assert (b.sampled_seeds, b.vector_payloads) == (64, 800)              # FILTERED_SAMPLED_SEEDS, ..._PAYLOAD_LIMIT
        assert (b.routing_rows, b.bridge_rows) == (want * 16, want * 8)
    assert budgets(10, 0, 0, 1000).ef_filtered == 150          # SearchParams::new(10): ef = 100, FILTERED_BEAM_PERCENT
    assert budgets(10, 100, 150, 40).ef_filtered == 40         # min(candidate_count)
    assert budgets(30, 100, 100, 1000).ef_filtered == 120      # max(k * 4)
    ids = np.arange(1, 100_001, dtype=np.uint64)
    s = hxo.deterministic_sample_ids(ids, 256)
    assert len(s) == 256 and all(a < b for a, b in zip(s, s[1:]))
    assert hxo.deterministic_sample_ids([7], 1).tolist() == [7]
    assert hxo.deterministic_sample_ids([3, 7], 1).tolist() == [3]
    assert hxo.deterministic_sample_ids([3, 7], 8).tolist() == [3, 7]
    assert hxo.restricted_result_count(800, 1000) == (hxo.OK, 800)
    assert hxo.restricted_result_count(800 + 200, 800) == (hxo.OK, 800)      # clamps to |C| before the limit check
    assert hxo.restricted_result_count(800 + 1, 1000)[0] == hxo.ERR_QUERY
    b = budgets(800, 800, 150, 1000)
    assert b.vector_payloads == 800 and b.vector_payloads >= 800


def test_upsert_contracts_of_the_reference(hxo):
    """V/index.rs:3033-3050 (`test_upsert_insert_replaces_existing_vector`): the replacement vector is the one kept and the
    count stays 1; V/index.rs:3053-3100 (`test_upsert_entry_reconnects_layer0_for_every_layer_assignment`): for every
    scripted assignment of {first, fallback, replacement} layers in 0..=2, deleting the entry node 0 and re-inserting it with
    another vector restores the bidirectional layer-0 link with node 1, and the closer node answers the query."""
    ix = hxo.Index(hxo.COSINE, 2)
    ix.upsert(1, [1.0, 0.0], 0)
    ix.upsert(1, [0.0, 1.0], 0)
    assert ix.vector(1).tolist() == [0.0, 1.0] and len(ix) == 1 and ix.state() == (1, 0)
    for first in range(3):
        for fallback in range(3):
            for replacement in range(3):
                ix = hxo.Index(hxo.COSINE, 2)
                ix.insert(0, [1.0, 0.0], first)
                ix.insert(1, [0.0, 1.0], fallback)
                assert ix.delete(0) is True
                assert ix.state() == (1, fallback)             # the fallback is promoted with its own layer
                ix.insert(0, [-1.0, 0.0], replacement)
                what = (first, fallback, replacement)
                assert 1 in ix.neighbors(0, 0).tolist() and 0 in ix.neighbors(0, 1).tolist(), what
                assert ix.state() == ((0, replacement) if replacement > fallback else (1, fallback)), what
                ids, _ = ix.search([1.0, 0.0], 1)              # strict walk; two nodes leave the default mode nothing to sample
                assert ids.tolist() == [1], what


def test_distance_score_and_candidate_contracts(hxo):
    """V/parameters.rs tests (`distance_score_is_finite_nonnegative_and_totally_ordered`), V/model.rs tests
    (`candidate_rejects_invalid_scores_and_orders_ties_by_node`) and V/index.rs:2115-2124: NaN / +-inf / negative scores are
    InvariantViolation, -0.0 is stored as +0.0, and candidates order by (score, then node id)."""
    L = hxo.lib()
    for bad in (float("nan"), float("inf"), float("-inf"), -1.0):
        v = _C.c_float(bad)
        assert L.hxo_score_validate(_C.byref(v)) == hxo.ERR_INVARIANT_VIOLATION
    z = _C.c_float(-0.0)
    assert L.hxo_score_validate(_C.byref(z)) == hxo.OK and bits(z.value) == bits(0.0)
    one = _C.c_float(1.0)
    assert L.hxo_score_validate(_C.byref(one)) == hxo.OK and one.value == 1.0
    # ordering through the public result: equal scores come back in ascending id order, smaller scores first
    ix = hxo.Index(hxo.EUCLIDEAN, 2)
    for nid, v in ((3, [1.0, 0.0]), (1, [1.0, 0.0]), (2, [2.0, 0.0]), (7, [0.5, 0.0])):
        ix.put_vector(nid, v)
    ids, sc = ix.search_exact([0.0, 0.0], 4)
    assert ids.tolist() == [7, 1, 3, 2] and sc.tolist() == [0.25, 1.0, 1.0, 4.0]


def test_short_and_ramp_vector_literals(hxo):
    """T/vector/distance_neighbors.rs:148-185: the three kernels on (1,2,3) x (3,2,1), norms, and the 33-element ramps on which
    the vectorised and the scalar order must agree within 1e-5 relative (here: the AVX-FMA order vs the scalar order)."""
    a, b = [1.0, 2.0, 3.0], [3.0, 2.0, 1.0]
    assert hxo.pair("hxo_dot_product", a, b) == 10.0 and hxo.pair("hxo_dot_scalar", a, b) == 10.0
    assert hxo.pair("hxo_euclidean_distance", a, b) == 8.0 and hxo.pair("hxo_euclid_scalar", a, b) == 8.0
    assert hxo.pair("hxo_manhattan", a, b) == 4.0
    assert np.float32(math.sqrt(hxo.pair("hxo_dot_product", [4.0, 6.0], [4.0, 6.0]))) == np.float32(52.0) ** np.float32(0.5)
    assert np.float32(math.sqrt(hxo.pair("hxo_dot_product", [1.0, -2.0, 3.0], [1.0, -2.0, 3.0]))) == np.sqrt(np.float32(14.0))
    left = np.arange(33, dtype=np.float32)
    right = left[::-1].copy()
    for fast, slow in (("hxo_dot_avx_fma", "hxo_dot_scalar"), ("hxo_euclid_avx_fma", "hxo_euclid_scalar")):
        f, s = hxo.pair(fast, left, right), hxo.pair(slow, left, right)
        assert abs(f - s) <= abs(s) * 1e-5
    assert hxo.pair("hxo_dot_scalar", left, right) == float(sum(i * (32 - i) for i in range(33)))      # exact in f32
