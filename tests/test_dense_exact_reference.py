"""The certificate of the exact dense entries (hx_search_dense_exact, csrc/k_dense.cu: hxd_exact_floor), restated in float64
and held to the oracle on the CPU.

The certificate clears query q when floor(L_q) > S_k: every row the tensor-core pass dropped has an approximate score
>= L_q, and floor(L) bounds from below the reference's fp32 score of any row whose approximate score is >= L.  The kernel's
approximate score differs from the float64 value of emulate() (bf16 operands, exact arithmetic) by at most kernel_error();
so the statement checked here, for every (query, row) pair, is
    oracle fp32 score >= floor(emulate() + kernel_error())
i.e. the worst approximate score the kernel could have produced for that row still lower-bounds the exact one.  A floor
that is not a number never certifies (the kernel flags the query), and neither does a cosine query or row whose fp32 norm
is below FLT_MIN: the reference divides by that norm, and its rounding there is not relative.
"""
import numpy as np
import pytest

from oracle import hxo
from test_dense_reference import emulate, bf16_round, pow2_normalize

U, UB, SUB, TINY = 2.0 ** -24, 2.0 ** -8, 2.0 ** -150, 2.0 ** -126


def gamma(n):
    return n * U / (1.0 - n * U)


def ldb_of(dim):
    return (dim + 63) // 64 * 64


def kernel_error(metric, dim, q_aux=None, r2=None):
    """Bound (a) of the derivation: |the kernel's approximate score - emulate()'s|."""
    ldb = ldb_of(dim)
    c_acc, g_sq = (ldb + 16.0) * 4.0 * U, gamma(ldb // 32 + 5.0)
    if metric == hxo.COSINE:
        psi = 1.01 * (g_sq + ldb * SUB + 4.0 * U)
        big_psi = 1.01 * (2.0 * psi + U)
        return 0.5 * (c_acc + 1.01 * big_psi) + 1.6 * U + 2.0 ** -100
    q, x = np.sqrt((q_aux + ldb * SUB) / (1.0 - g_sq)), np.sqrt((r2 + ldb * SUB) / (1.0 - g_sq))
    m = (q + x) ** 2
    a_acc = 2.0 * (ldb + 16.0) * TINY + TINY * np.sqrt(ldb) * (q + x)
    return (g_sq + c_acc + 3.0 * U) * m + 2.0 * ldb * SUB + 2.0 * a_acc + SUB


def exact_floor(metric, dim, L, q_aux=None, r2=None):
    """hxd_exact_floor: lower bound on the reference's fp32 score of any row whose kernel score is >= L."""
    ldb = ldb_of(dim)
    sd, n_ref = np.sqrt(ldb), 2.0 * dim + 10.0
    err = kernel_error(metric, dim, q_aux, r2)
    if metric == hxo.COSINE:
        eta = UB + sd * 2.0 ** -133
        eta1 = 1.01 * eta / (1.0 - eta)
        h = np.maximum(np.sqrt(np.maximum(L - err, 0.0)) - eta1, 0.0)
        return h * h - (1.01 * (gamma(n_ref) + 3.0 * U) + 2.0 * U)
    g_sq = gamma(ldb // 32 + 5.0)
    q, x = np.sqrt((q_aux + ldb * SUB) / (1.0 - g_sq)), np.sqrt((r2 + ldb * SUB) / (1.0 - g_sq))
    a = sd * 2.0 ** -134
    beta = UB * (q + x + 2.0 * a) / (1.0 - UB) + 2.0 * a
    d = np.maximum(np.sqrt(np.maximum(L - err, 0.0)) - beta, 0.0)
    return (1.0 - gamma(n_ref)) * d * d - n_ref * SUB


def terms(metric, queries, rows):
    """The pass's fp32 query terms and the view's largest row term (euclidean |v^|^2; unused for cosine)."""
    if metric == hxo.COSINE:
        return None, None
    q = bf16_round(queries).astype(np.float64)
    x = bf16_round(rows).astype(np.float64)
    return (q * q).sum(1).astype(np.float32).astype(np.float64), float(np.float32((x * x).sum(1).max()))


def oracle_scores(metric, queries, rows):
    """[B, n] the oracle's exact fp32 scores, columns in row order."""
    n, d = rows.shape
    ids = np.arange(n, dtype=np.uint64)
    ora = hxo.Index(metric, d)
    ora.put_vectors(ids, rows)
    out = np.empty((len(queries), n), np.float64)
    for b, q in enumerate(queries):
        oi, os_ = ora.search_exact(q, n)
        out[b, oi.astype(np.int64)] = os_.astype(np.float64)
    return out


def check_floor(metric, queries, rows):
    """Asserts the floor under every pair; returns (floor, approx, exact) for the callers' non-vacuity checks."""
    d = rows.shape[1]
    approx, _ = emulate(metric, queries, rows)
    q_aux, r2 = terms(metric, queries, rows)
    qa = None if q_aux is None else q_aux[:, None]
    worst = approx + kernel_error(metric, d, qa, r2)
    with np.errstate(invalid="ignore", over="ignore"):
        fl = exact_floor(metric, d, worst, qa, r2)
    exact = oracle_scores(metric, queries, rows)
    ok = np.isnan(fl) | (exact >= fl)
    if metric == hxo.COSINE:   # pairs the kernel flags: a norm below FLT_MIN
        fmin = float(np.finfo(np.float32).tiny)
        with np.errstate(over="ignore"):   # norms above FLT_MAX: inf, not below FLT_MIN either way
            qn = np.linalg.norm(queries.astype(np.float64), axis=1).astype(np.float32)
            xn = np.linalg.norm(rows.astype(np.float64), axis=1).astype(np.float32)
        ok |= (qn < fmin)[:, None] | (xn < fmin)[None, :]
    bad = np.argwhere(~ok)
    assert not len(bad), (f"metric {metric} d {d}: floor above the exact score at {bad[:5].tolist()}: "
                          f"{[(exact[i, j], fl[i, j], approx[i, j]) for i, j in bad[:5]]}")
    return fl, approx, exact


@pytest.mark.parametrize("metric", [hxo.COSINE, hxo.EUCLIDEAN])
@pytest.mark.parametrize("d", [8, 65, 768, 1536])
def test_floor_bounds_the_exact_score_on_random_data(metric, d):
    rng = np.random.default_rng(d * 3 + metric)
    rows = rng.standard_normal((400, d)).astype(np.float32)
    queries = rng.standard_normal((6, d)).astype(np.float32)
    rows[:20] = queries[rng.integers(0, 6, 20)] + np.float32(0.05) * rng.standard_normal((20, d)).astype(np.float32)
    fl, approx, exact = check_floor(metric, queries, rows)
    # not vacuous: the floor sits within a few bf16 steps of the score (relative to the scale of the scores)
    scale = exact.max()
    assert np.isfinite(fl).all()
    assert ((exact - fl) / scale).max() < 0.05, ((exact - fl) / scale).max()
    assert (fl > 0.5 * exact).mean() > 0.9


@pytest.mark.parametrize("metric", [hxo.COSINE, hxo.EUCLIDEAN])
def test_floor_bounds_the_exact_score_over_the_float32_range(metric):
    import numeric_range as nr
    for d in nr.DIMS:
        _, rows, queries = nr.corpus(metric, d)
        check_floor(metric, queries, rows)


def test_floor_is_monotone_and_scale_free_for_cosine():
    L = np.linspace(0.0, 1.0, 1001)
    fl = exact_floor(hxo.COSINE, 768, L)
    assert (np.diff(fl) >= 0).all()
    assert (fl < L).all() and (fl[L > 0.01] > 0).all()
    # euclidean: monotone in L, and scaling the data by 2^e scales the bound's relative terms alike
    q2, r2 = 1.0, 1.0
    fe = exact_floor(hxo.EUCLIDEAN, 768, L * 4.0, q2, r2)
    assert (np.diff(fe) >= 0).all() and (fe < L * 4.0).all()
    fs = exact_floor(hxo.EUCLIDEAN, 768, L * 4.0 * 2.0 ** 40, q2 * 2.0 ** 40, r2 * 2.0 ** 40)
    assert np.allclose(fs, fe * 2.0 ** 40, rtol=1e-9, atol=1e-30 * 2.0 ** 40)


def test_tiny_euclidean_corpus_is_held_by_the_absolute_terms():
    """At 2^-70 the squared distances are ~2^-134, far below the flush terms of the bound (~2^-119): relative error
    bounds alone would be false there.  The floor still holds, and a kernel score near the true value floors at <= 0, so
    such queries are rescanned rather than certified on a relative bound."""
    rng = np.random.default_rng(5)
    rows = (rng.standard_normal((50, 31)) * 2.0 ** -70).astype(np.float32)
    queries = (rng.standard_normal((4, 31)) * 2.0 ** -70).astype(np.float32)
    _, approx, exact = check_floor(hxo.EUCLIDEAN, queries, rows)
    q_aux, r2 = terms(hxo.EUCLIDEAN, queries, rows)
    err = kernel_error(hxo.EUCLIDEAN, 31, q_aux[:, None], r2)
    assert (err > 1e3 * approx.max()).all()
    assert (exact_floor(hxo.EUCLIDEAN, 31, approx, q_aux[:, None], r2) <= 0).all()


def test_pow2_normalize_keeps_cosine_operands_at_least_one():
    """The cosine bound treats its absolute terms as relative because every nonzero operand has |v^| >= 1."""
    rng = np.random.default_rng(2)
    x = (rng.standard_normal((100, 40)) * np.exp2(rng.integers(-140, 120, 100))[:, None]).astype(np.float32)
    v = bf16_round(pow2_normalize(x)).astype(np.float64)
    assert (np.sqrt((v * v).sum(1)) >= 1.0).all()
