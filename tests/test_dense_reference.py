"""Float64 reference of the dense path's nomination step (hx_search_dense, csrc/k_dense.cu), and CPU checks of it.

The tensor-core pass scores every row with bf16 operands and fp32 accumulation and only NOMINATES candidates: per
(query, run of tiles, 64-column quarter) bucket it keeps the HXD_T = 8 best rows, and the k' best nominees go to the exact
fp32 re-rank.  This module restates the approximate score in float64 from bf16-rounded operands, with no dependence on
the tile or bucket layout, and bounds the kernel's own fp32 error by a per-(query, row) epsilon.

A row is SURE for a query when fewer than HXD_T other rows can come within epsilon of beating its approximate score: it
survives its bucket whatever the layout, and is inside k' >= 64.  tests/test_gpu_dense.py holds the kernel to that.
"""
import numpy as np
import pytest

from oracle import hxo

HXD_T = 8
EPS_REL = 2.0 ** -14   # far above the fp32 accumulation / epilogue error, far below bf16's 2^-8


def bf16_round(x):
    """float32 -> bf16 -> float32, round to nearest even, by bit operations (no torch)."""
    a = np.ascontiguousarray(x, dtype=np.float32)
    u = a.view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000).astype(np.uint32)
    nan = np.isnan(a)
    r[nan] = (u[nan].astype(np.uint32) | 0x00400000) & 0xFFFF0000   # NaN stays NaN (quiet)
    return r.view(np.float32).reshape(a.shape)


def pow2_normalize(a):
    """Each row times the power of two that brings its largest |component| into [1, 2) (k_to_bf16 does this for cosine
    before rounding); all-zero rows are left alone.  One rounding at most (a result below 2^-126), as ldexpf."""
    a = np.asarray(a, dtype=np.float32)
    m = np.abs(a).max(axis=1)
    _, e = np.frexp(m)
    shift = np.where(m > 0, 1 - e, 0)
    return np.ldexp(a.astype(np.float64), shift[:, None]).astype(np.float32)


def emulate(metric, queries, rows):
    """Approximate scores of k_dense_scores in float64, [B, n], and the per-(query, row) epsilon bounding its fp32 error.

    cosine:    0.5 - 0.5 <q^, x^> / (|q^| |x^|)            euclidean: |q^|^2 + |x^|^2 - 2 <q^, x^>        (both clamped at 0)
    epsilon:   2^-14 (cosine)                              2^-14 (sum_j |q^_j x^_j| + |q^|^2 + |x^|^2)
    q^, x^ are the bf16-rounded operands; for cosine, of the rows after pow2_normalize, as in k_to_bf16.
    """
    if metric == hxo.COSINE:
        queries, rows = pow2_normalize(queries), pow2_normalize(rows)
    q = bf16_round(queries).astype(np.float64)
    x = bf16_round(rows).astype(np.float64)
    dot = q @ x.T
    qn = (q * q).sum(1)
    xn = (x * x).sum(1)
    if metric == hxo.COSINE:
        approx = 0.5 - 0.5 * dot / np.sqrt(qn)[:, None] / np.sqrt(xn)[None, :]
        eps = np.full_like(approx, EPS_REL)
    else:
        approx = qn[:, None] + xn[None, :] - 2.0 * dot
        eps = EPS_REL * (np.abs(q) @ np.abs(x).T + qn[:, None] + xn[None, :])
    return np.maximum(approx, 0.0), eps


def sure_rows(approx, eps, cols):
    """For one query (1-d approx / eps over all rows): which of the rows `cols` are sure (see the module docstring)."""
    lo = np.sort(approx - eps)
    hi = approx[cols] + eps[cols]
    rivals = np.searchsorted(lo, hi, side="right") - 1   # rows j != i with approx_j - eps_j <= approx_i + eps_i
    return rivals < HXD_T


def tie_fixture(n=4000, dim=64, n_tied=20, seed=11):
    """Euclidean rows whose exact fp32 distances to one query tie, while their bf16 scores order them in REVERSE id order.

    The query is zero except at one coordinate c_i per tied row, where it holds f_i (a multiple of 2^-16, exact in bf16,
    in [-2^-9, 2^-8)); tied row i is the query plus 1.0 at c_i.  In fp32 every tied row is at squared distance exactly 1
    (1 + f_i is exact and (1 + f_i) - f_i = 1).  In bf16, 1 + f_i rounds to 1, so the approximate score is (1 - f_i)^2:
    f_i rising with the id puts the largest id first.  The rest of the corpus is far away.
    Returns (ids, rows, query, tied_ids ascending)."""
    rng = np.random.default_rng(seed)
    ids = np.sort(rng.choice(np.arange(10, 50 * n, dtype=np.uint64), size=n, replace=False))
    rows = (rng.standard_normal((n, dim)) * 3.0 + 4.0).astype(np.float32)   # squared distance to the query ~ dim * 25
    pos = np.sort(rng.choice(np.arange(n), size=n_tied, replace=False))     # scattered ids
    coords = rng.permutation(dim)[:n_tied]
    f = np.round(np.linspace(-2.0 ** -9, 2.0 ** -8 - 2.0 ** -12, n_tied) * 2.0 ** 16) / 2.0 ** 16
    q = np.zeros(dim, np.float32)
    q[coords] = f
    for i, p in enumerate(pos):
        rows[p] = q
        rows[p, coords[i]] = np.float32(1.0) + np.float32(f[i])
    return ids, rows, q, ids[pos]


# ---- CPU checks ---------------------------------------------------------------------------------------------------------
def test_bf16_round_matches_torch_on_edge_values():
    torch = pytest.importorskip("torch")
    f32 = np.float32
    vals = [0.0, -0.0, 1.0, -1.0, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, 1.0 + 2.0 ** -8 + 2.0 ** -20, 1.0 - 2.0 ** -9,
            1.0 + 2.0 ** -7, 3.0e38, -3.0e38, 3.3895314e38, 3.4028235e38, float("inf"), float("-inf"),
            1e-40, -1e-40, 2.0 ** -133, 3 * 2.0 ** -134, 1.17549435e-38, 1.1754942e-38, 2.0 ** -126 + 2.0 ** -134,
            0.1, -0.1, 65504.0, 1.0 / 3.0]
    # ties to even at both parities of the kept bit, and a sweep over the low 16 bits
    base = np.array([0x3F800000, 0x3F810000, 0x00010000, 0x7F7F0000, 0x80018000], dtype=np.uint32)
    low = np.array([0x0000, 0x0001, 0x7FFF, 0x8000, 0x8001, 0xFFFF], dtype=np.uint32)
    swept = (base[:, None] | low[None, :]).ravel().view(np.float32)
    rng = np.random.default_rng(3)
    rand = rng.integers(0, 2 ** 32, size=20000, dtype=np.uint64).astype(np.uint32).view(np.float32)
    a = np.concatenate([np.array(vals, dtype=f32), swept, rand[np.isfinite(rand)]])
    want = torch.from_numpy(a.copy()).to(torch.bfloat16).to(torch.float32).numpy()
    got = bf16_round(a)
    assert got.view(np.uint32).tolist() == want.view(np.uint32).tolist()
    # the sign of zero survives, NaN stays NaN
    assert bf16_round(np.array([-0.0], f32)).view(np.uint32)[0] == 0x80000000
    assert np.isnan(bf16_round(np.array([np.nan], f32)))[0]


def test_emulated_scores_follow_the_metric_definitions():
    rng = np.random.default_rng(8)
    q = rng.standard_normal((3, 40)).astype(np.float32)
    x = rng.standard_normal((50, 40)).astype(np.float32)
    qb, xb = bf16_round(q).astype(np.float64), bf16_round(x).astype(np.float64)
    a_e, e_e = emulate(hxo.EUCLIDEAN, q, x)
    assert np.allclose(a_e, ((qb[:, None, :] - xb[None, :, :]) ** 2).sum(-1), rtol=1e-12, atol=1e-12)
    a_c, e_c = emulate(hxo.COSINE, q, x)
    cos = (qb @ xb.T) / np.linalg.norm(qb, axis=1)[:, None] / np.linalg.norm(xb, axis=1)[None, :]
    assert np.allclose(a_c, 0.5 - 0.5 * cos, rtol=1e-12, atol=1e-12)
    assert (e_c == EPS_REL).all() and (e_e > 0).all()
    # rows equal to the query clamp at 0 instead of going negative
    a0, _ = emulate(hxo.EUCLIDEAN, x[:2], x)
    assert a0[0, 0] == 0.0 and a0[1, 1] == 0.0 and (a0 >= 0).all()


def test_sure_rows_counts_rivals_within_epsilon():
    approx = np.array([0.0, 1.0, 1.0 + 1e-9, 5.0] + [10.0] * 20)
    eps = np.full_like(approx, 1e-6)
    # row 0: no rival; rows 1, 2: each other (1 rival besides row 0); row 3: 3 rivals; the 20 tied rows: 23 each
    assert sure_rows(approx, eps, np.arange(len(approx))).tolist() == [True, True, True, True] + [False] * 20
    # 8 tied rows: 7 rivals each (a bucket of 8 keeps them all); the row behind them has 8
    tied = np.array([0.0] * 8 + [1.0])
    assert sure_rows(tied, np.full_like(tied, 1e-6), np.arange(9)).tolist() == [True] * 8 + [False]
    assert sure_rows(np.zeros(9), np.full(9, 1e-6), np.arange(9)).tolist() == [False] * 9


def test_tie_fixture_is_an_exact_tie_in_reversed_bf16_order():
    ids, rows, q, tied = tie_fixture()
    ora = hxo.Index(hxo.EUCLIDEAN, rows.shape[1])
    ora.put_vectors(ids, rows)
    oi, os_ = ora.search_exact(q, len(tied) + 5)
    # the exact scan: all tied rows first, at one score, in id order; the rest far behind
    assert oi[:len(tied)].tolist() == tied.tolist()
    assert set(os_[:len(tied)].view(np.uint32).tolist()) == {np.float32(1.0).view(np.uint32)}
    assert os_[len(tied)] > 100.0
    oi10, os10 = ora.search_exact(q, 10)
    assert oi10.tolist() == tied[:10].tolist()
    # the emulated bf16 scores of the tied rows fall strictly as the id rises, with gaps well beyond the kernel's error.
    # (bf16 rounding moves a score by at most ~2^-7 of the magnitudes epsilon is 2^-14 of, so 20 rows span at most
    # ~2^7 epsilon: gaps of 4x the two epsilons are what this geometry allows.)
    pos = np.searchsorted(ids, tied)
    approx, eps = emulate(hxo.EUCLIDEAN, q[None, :], rows[pos])
    a, e = approx[0], eps[0]
    assert (np.diff(a) < 0).all()
    gap = -np.diff(a)
    assert (gap >= 4.0 * (e[:-1] + e[1:])).all(), (gap.min(), e.max())
    # ... and far rows never come near
    far, _ = emulate(hxo.EUCLIDEAN, q[None, :], np.delete(rows, pos, axis=0))
    assert far.min() > 100.0


# ---- the emulation over the full float32 range (tests/numeric_range.py) -------------------------------------------------------
def test_emulate_is_finite_over_the_float32_range():
    import numeric_range as nr
    for metric in (hxo.COSINE, hxo.EUCLIDEAN):
        for d in nr.DIMS:
            ids, rows, queries = nr.corpus(metric, d)
            approx, eps = emulate(metric, queries, rows)
            assert np.isfinite(approx).all() and np.isfinite(eps).all(), (metric, d)
            assert (approx >= 0).all() and (eps >= 0).all()
    # FLT_MAX rows and the 2^-149 row score like any other direction: a row against itself is 0, its negation 1
    f = np.float32(np.finfo(np.float32).max)
    x = np.array([[f, -f, f], [0.0, 2.0 ** -149, 0.0], [3e-39, 1e-45, 0.0]], np.float32)
    a, _ = emulate(hxo.COSINE, np.concatenate([x, -x]), x)
    assert np.allclose(np.diag(a[:3]), 0.0, atol=1e-6) and np.allclose(np.diag(a[3:]), 1.0, atol=1e-6)


def test_pow2_normalize_is_exact_and_lands_in_one_to_two():
    rng = np.random.default_rng(9)
    x = (rng.standard_normal((50, 33)) * np.exp2(rng.integers(-100, 100, 50))[:, None]).astype(np.float32)
    y = pow2_normalize(x)
    m = np.abs(y).max(1)
    assert ((m >= 1.0) & (m < 2.0)).all()
    assert (np.abs(pow2_normalize(x * np.float32(2.0 ** -20)) - y) == 0).all()
    f = np.float32(np.finfo(np.float32).max)
    assert pow2_normalize(np.array([[f, 0.0]], np.float32)).tolist() == [[float(np.nextafter(np.float32(2), np.float32(0))), 0.0]]
    assert pow2_normalize(np.array([[2.0 ** -149, 0.0]], np.float32)).tolist() == [[1.0, 0.0]]


@pytest.mark.parametrize("e", [-100, -70, -1, 1, 60, 100])
def test_cosine_emulation_is_unchanged_by_a_power_of_two(e):
    """Scaling one row, or one query, by 2^e leaves every cosine score and epsilon as they were (the scaled values are
    exact in float32 here: normal, below FLT_MAX)."""
    rng = np.random.default_rng(e + 500)
    q = rng.standard_normal((6, 70)).astype(np.float32)
    x = rng.standard_normal((40, 70)).astype(np.float32)
    a0, e0 = emulate(hxo.COSINE, q, x)
    s = np.float32(2.0 ** e)
    x2, q2 = x.copy(), q.copy()
    x2[7] *= s
    q2[2] *= s
    assert (x2[7].astype(np.float64) == x[7].astype(np.float64) * 2.0 ** e).all()
    a1, e1 = emulate(hxo.COSINE, q2, x2)
    assert a1.tobytes() == a0.tobytes() and e1.tobytes() == e0.tobytes()


@pytest.mark.parametrize("e", [-60, -20, 20, 40])
def test_euclidean_emulation_scales_by_four_to_the_e(e):
    rng = np.random.default_rng(e + 900)
    q = rng.standard_normal((6, 70)).astype(np.float32)
    x = rng.standard_normal((40, 70)).astype(np.float32)
    a0, e0 = emulate(hxo.EUCLIDEAN, q, x)
    s = np.float32(2.0 ** e)
    a1, e1 = emulate(hxo.EUCLIDEAN, q * s, x * s)
    assert (a1 == a0 * 2.0 ** (2 * e)).all() and (e1 == e0 * 2.0 ** (2 * e)).all()
