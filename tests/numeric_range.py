"""Seeded corpora and queries that cover the float32 range each metric accepts (plain module, no device).

The score kernels (csrc/hx_common.cuh: the octet kernel, the ring's warp rows, hx_manhattan_seq and the cosine finish with
its f64 fallback) are bit-exact on order-1 data; these fixtures put them where float32 arithmetic gets hard:

* cosine has no component limit, so rows and queries are random directions times 2^e for e from -140 (subnormal
  components) to 126, plus rows of +-FLT_MAX components (the header clamps to FLT_MAX, so the f64 fallback runs) and a row
  whose only non-zero component is 2^-149.  Queries are drawn the same way: every pairing of the fast path with the
  fallback, an overflowing dot product and a norm product that is not a normal float occurs.
* Euclidean and Manhattan mix components exactly at component_limit(metric, d), one ulp below it, subnormal
  (2^-149 .. 2^-127), +-0 and order 1, within rows and across rows.

Every query gets NEAR rows (small perturbations of it at its own scale), so the top-k is not decided by ties alone.
"""
import numpy as np

from oracle import hxo

DIMS = (3, 31, 33, 70, 768)
EXPONENTS = (-140, -100, -70, -64, 0, 64, 70, 100, 126)
FLT_MAX = float(np.finfo(np.float32).max)
TINY = 2.0 ** -149
NEAR = 3   # near rows per query


def _directions(rng, n, d):
    """Gaussian directions clipped to |z| <= 3.9, so that 2^126 * z stays finite."""
    return np.clip(rng.standard_normal((n, d)), -3.9, 3.9)


def _nonzero(rows, rng):
    """A cosine row must have a non-zero component: rows that rounded to all zeros get +-2^-149 at one position."""
    for i in np.flatnonzero(~rows.any(axis=1)):
        rows[i, rng.integers(rows.shape[1])] = np.float32(TINY if rng.random() < 0.5 else -TINY)
    return rows


def _cosine_draw(rng, n, d):
    e = rng.choice(EXPONENTS, size=n)
    return _nonzero((_directions(rng, n, d) * np.exp2(e.astype(np.float64))[:, None]).astype(np.float32), rng)


def _cosine_specials(rng, d):
    """Rows that take the f64 fallback from their own header, or sit at the bottom of the range."""
    signs = np.where(rng.random((2, d)) < 0.5, -1.0, 1.0)
    out = [signs[0] * FLT_MAX]                                          # every component +-FLT_MAX: header clamped
    r = _directions(rng, 1, d)[0] * 2.0 ** 100
    r[rng.integers(d)] = -FLT_MAX                                        # one FLT_MAX component among 2^100 ones
    out.append(r)
    one = np.zeros(d)
    one[rng.integers(d)] = FLT_MAX                                       # header exactly FLT_MAX, not clamped
    out.append(one)
    t = np.zeros(d)
    t[rng.integers(d)] = TINY                                            # only 2^-149
    out.append(t)
    out.append(signs[1] * TINY)                                          # every component +-2^-149
    return np.array(out, dtype=np.float32)


def _limit_values(metric, d):
    lim = np.float32(hxo.component_limit(metric, d))
    return lim, np.nextafter(lim, np.float32(0))


def _lp_draw(rng, metric, n, d):
    """Euclidean / Manhattan rows: each row is one of six kinds, the last mixing every kind within the row."""
    lim, below = _limit_values(metric, d)
    sign = np.where(rng.random((n, d)) < 0.5, -1.0, 1.0)
    at = sign * np.where(rng.random((n, d)) < 0.5, float(lim), float(below))
    sub = sign * np.exp2(rng.integers(-149, -126, size=(n, d)).astype(np.float64))
    zero = sign * 0.0
    one = _directions(rng, n, d)
    kind = rng.integers(0, 6, size=n)
    mixed = np.choose(rng.integers(0, 4, size=(n, d)), [at, sub, zero, one])
    out = np.choose(kind[:, None], [at, sub, zero, one, one * np.float64(below) / 4.0, mixed])
    return out.astype(np.float32)


def _near(rng, q, m):
    """m rows close to q at its own scale: every component shrunk toward 0 by up to 2%, so no limit is crossed."""
    f = 1.0 - 0.02 * rng.random((m, q.size))
    return (q.astype(np.float64)[None, :] * f).astype(np.float32)


def corpus(metric, d, n_rows=120, n_queries=24, seed=0):
    """(ids, rows, queries): ids ascending and sparse, rows float32 [n, d] (n = n_rows + the special rows + NEAR per query),
    queries float32 [n_queries, d].  Rows and queries are valid for the metric (hxo.validate_vector)."""
    rng = np.random.default_rng([seed, metric, d])
    if metric == hxo.COSINE:
        base = _cosine_draw(rng, n_rows, d)
        specials = _cosine_specials(rng, d)
        rows = np.concatenate([base, specials])
        queries = np.concatenate([specials[[0, 3]], _cosine_draw(rng, n_queries - 2, d)])[:n_queries]
    else:
        rows = _lp_draw(rng, metric, n_rows, d)
        queries = _lp_draw(rng, metric, n_queries, d)
    near = np.concatenate([_near(rng, q, NEAR) for q in queries])
    if metric == hxo.COSINE:
        near = _nonzero(near, rng)
    rows = np.concatenate([rows, near])
    rows = rows[rng.permutation(len(rows))]                              # near rows are not id-adjacent to their query
    ids = np.sort(rng.choice(np.arange(1, 40 * len(rows), dtype=np.uint64), size=len(rows), replace=False))
    return ids, np.ascontiguousarray(rows), np.ascontiguousarray(queries)


def scaled_corpus(n, d, exponent, n_queries, seed=0, metric=hxo.COSINE):
    """Random directions times 2^exponent with NEAR rows per query, for the dense path's scale checks."""
    rng = np.random.default_rng([seed, n, d, exponent + 1000])
    s = 2.0 ** exponent
    queries = (_directions(rng, n_queries, d) * s).astype(np.float32)
    near = np.concatenate([_near(rng, q, NEAR) for q in queries])
    rows = np.concatenate([(_directions(rng, n - len(near), d) * s).astype(np.float32), near])
    rows = rows[rng.permutation(n)]
    if metric == hxo.COSINE:
        rows, queries = _nonzero(rows, rng), _nonzero(queries, rng)
    return np.arange(n, dtype=np.uint64) * 3 + 2, np.ascontiguousarray(rows), np.ascontiguousarray(queries)


def cosine_queries(n, d, seed=0):
    """Cosine queries at every exponent of EXPONENTS plus the FLT_MAX and 2^-149 specials."""
    rng = np.random.default_rng([seed, d, 77])
    return np.ascontiguousarray(np.concatenate([_cosine_specials(rng, d)[[0, 2, 3]], _cosine_draw(rng, n - 3, d)]))


# ---- float64 restatement of the three metrics --------------------------------------------------------------------------
def exact_f64(metric, queries, rows):
    """Scores [B, n] in float64 from the float32 inputs: squared L2, L1, or (1 - cos) / 2 (no float32 step anywhere)."""
    q = np.asarray(queries, np.float64)
    x = np.asarray(rows, np.float64)
    if metric == hxo.EUCLIDEAN:
        return ((q[:, None, :] - x[None, :, :]) ** 2).sum(-1)
    if metric == hxo.MANHATTAN:
        return np.abs(q[:, None, :] - x[None, :, :]).sum(-1)
    # FLT_MAX^2 * 768 and 2^-298 are both inside float64's range: the plain formula is exact enough
    qn = np.sqrt((q * q).sum(1))
    xn = np.sqrt((x * x).sum(1))
    c = np.clip((q @ x.T) / qn[:, None] / xn[None, :], -1.0, 1.0)
    return (1.0 - c) / 2.0


def tolerance(metric, queries, rows, exact):
    """The reference's tolerance for its own kernels, max(d * 2^-23, 1e-5) * max(|e|, 1), plus an absolute term for what
    float32 cannot hold below 2^-126: for L2 and L1, 4 d * 2^-149 (every term and partial sum is rounded to the subnormal
    spacing); for cosine, 2^-149 / |v| per vector (the header, a float32 norm, is rounded to that spacing when subnormal)."""
    d = rows.shape[1]
    t = max(d * 2.0 ** -23, 1e-5) * np.maximum(np.abs(exact), 1.0)
    if metric != hxo.COSINE:
        return t + 4.0 * d * TINY
    qn = np.sqrt((np.asarray(queries, np.float64) ** 2).sum(1))
    xn = np.sqrt((np.asarray(rows, np.float64) ** 2).sum(1))
    return t + TINY / qn[:, None] + TINY / xn[None, :]


def assert_within_f64(metric, queries, rows, ids, got_ids, got_scores, counts, what=""):
    """Every returned score within tolerance() of the float64 score of its (query, row)."""
    pos = {int(i): j for j, i in enumerate(ids)}
    for b in range(len(counts)):
        c = int(counts[b])
        if c == 0:
            continue
        cols = [pos[int(i)] for i in got_ids[b, :c]]
        e = exact_f64(metric, queries[b:b + 1], rows[cols])
        err = np.abs(got_scores[b, :c].astype(np.float64) - e[0])
        bad = np.flatnonzero(err > tolerance(metric, queries[b:b + 1], rows[cols], e)[0])
        e = e[0]
        assert not len(bad), f"{what} query {b}: score {got_scores[b, bad[0]]!r} vs float64 {e[bad[0]]!r}"
