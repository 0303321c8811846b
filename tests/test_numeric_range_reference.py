"""The oracle on the full float32 range (tests/numeric_range.py), against an independent float64 evaluation.

The GPU tests of tests/test_gpu_numeric_range.py compare the device with the oracle bit for bit on these fixtures; this file
checks the checker there: its scores and headers agree with float64 within the reference's own tolerance, its fallback is
the one that runs where the fast path cannot, and its validation accepts every fixture vector and refuses one ulp more.
"""
import numpy as np
import pytest

from oracle import hxo

import numeric_range as nr

METRICS = [hxo.EUCLIDEAN, hxo.COSINE, hxo.MANHATTAN]


@pytest.mark.parametrize("d", nr.DIMS)
@pytest.mark.parametrize("metric", METRICS)
def test_oracle_scores_agree_with_float64(metric, d):
    ids, rows, queries = nr.corpus(metric, d)
    n_q = 8 if d == 768 else len(queries)
    exact = nr.exact_f64(metric, queries[:n_q], rows)
    tol = nr.tolerance(metric, queries[:n_q], rows, exact)
    got = np.array([[hxo.distance(metric, rows[j], queries[b]) for j in range(len(rows))] for b in range(n_q)])
    assert np.isfinite(got).all() and (got >= 0).all()
    bad = np.argwhere(np.abs(got - exact) > tol)
    assert not len(bad), f"query {bad[0][0]} row {bad[0][1]}: oracle {got[tuple(bad[0])]!r}, float64 {exact[tuple(bad[0])]!r}"
    # the batch entry (the one the GPU tests compare with) gives the same bits as the pairwise one
    ora = hxo.Index(metric, d)
    ora.put_vectors(ids, rows)
    oi, os_, oc, _ = ora.search_exact_batch(queries[:n_q], len(ids))
    pos = np.searchsorted(ids, oi)
    assert (oc == len(ids)).all()
    assert os_.view(np.uint32).tolist() == np.take_along_axis(got, pos.astype(np.int64), 1).astype(np.float32).view(np.uint32).tolist()


@pytest.mark.parametrize("d", nr.DIMS)
def test_cosine_headers_and_fallback_coverage(d):
    """Headers equal the float64 norm clamped to FLT_MAX; the fixture reaches every branch of the cosine finish."""
    ids, rows, queries = nr.corpus(hxo.COSINE, d)
    r64 = rows.astype(np.float64)
    norms = np.sqrt((r64 * r64).sum(1))
    h = np.array([hxo.header(hxo.COSINE, r) for r in rows])
    want = np.minimum(norms, nr.FLT_MAX).astype(np.float32)
    rel = np.abs(h - want.astype(np.float64)) / want.astype(np.float64)
    assert (rel <= max(d * 2.0 ** -23, 1e-5)).all()
    assert (h == np.float32(nr.FLT_MAX)).sum() >= 3, "clamped / FLT_MAX headers"
    assert (h == np.float32(nr.TINY)).any(), "a row of norm 2^-149"
    # pairings: fast path, FLT_MAX header, norm product not normal (overflow and underflow), dot product overflow
    qh = np.array([hxo.header(hxo.COSINE, q) for q in queries], np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        pnqn = qh[:, None] * h.astype(np.float32)[None, :]
        dot = (queries[:, None, :].astype(np.float32) * rows[None, :, :]).sum(-1, dtype=np.float32)
    fmax = np.float32(nr.FLT_MAX)
    header_max = (qh[:, None] == fmax) | (h.astype(np.float32)[None, :] == fmax)
    normal = (np.abs(pnqn) >= np.finfo(np.float32).tiny) & np.isfinite(pnqn)
    fast = ~header_max & normal & np.isfinite(dot)
    assert fast.any() and header_max.any()
    assert (~np.isfinite(pnqn)).any() and ((pnqn != 0) & (np.abs(pnqn) < np.finfo(np.float32).tiny) | (pnqn == 0)).any()
    assert (~np.isfinite(dot) & ~header_max).any(), "a dot product that overflows without a FLT_MAX header"


@pytest.mark.parametrize("d", nr.DIMS)
@pytest.mark.parametrize("metric", METRICS)
def test_fixture_is_valid_and_one_ulp_more_is_refused(metric, d):
    ids, rows, queries = nr.corpus(metric, d)
    assert len(np.unique(ids)) == len(ids) and (np.diff(ids.astype(np.int64)) > 0).all()
    for v in np.concatenate([rows, queries]):
        assert hxo.validate_vector(metric, d, v) == (hxo.OK, 0)
    lim = hxo.component_limit(metric, d)
    if lim is None:
        assert metric == hxo.COSINE
        return
    lim = np.float32(lim)
    at = np.abs(rows) == lim
    assert at.any() and (np.abs(rows) == np.nextafter(lim, np.float32(0))).any()
    assert ((np.abs(rows) > 0) & (np.abs(rows) < np.finfo(np.float32).tiny)).any(), "subnormal components"
    assert (np.signbit(rows) & (rows == 0)).any(), "-0 components"
    # every row holding the limit: push the first such component one ulp out, either sign
    for i in np.flatnonzero(at.any(axis=1))[:10]:
        j = int(np.flatnonzero(at[i])[0])
        v = rows[i].copy()
        v[j] = np.nextafter(v[j], np.float32(np.copysign(np.inf, v[j])))
        assert hxo.validate_vector(metric, d, v) == (hxo.ERR_MAGNITUDE_EXCEEDED, j)
    # the limit is the largest float32 the reference's bound admits
    bound = np.sqrt(nr.FLT_MAX / (8.0 * d)) if metric == hxo.EUCLIDEAN else nr.FLT_MAX / (4.0 * d)
    assert float(lim) <= bound < float(np.nextafter(lim, np.float32(np.inf)))
