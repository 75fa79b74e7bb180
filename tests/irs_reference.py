"""fp64 numpy restatement of IRS, shared by tests/test_irs_score_cpu.py and tests/test_irs_score_gpu.py (numpy only, so
the GPU tests can use it), and a line-by-line float32 restatement of disentanglement_lib's irs.py.

The definition, under the conventions of include/disvae_b200.h (INTEGRATION.md states it in full):
- `edges` / `bins`: np.histogram(v, 20)'s fp64 edges of an integer factor column and each value's bin (0 .. 19);
- `quantile`: np.percentile(a, diff_quantile * 100) by numpy's linear rule, each operation rounded in fp64;
- `fit`: the kernel's tables (max deviations, active latents, group deviations and counts, the IRS matrix) of drawn
  fp32 codes and the scored factors' values;
- `score`: the host finish (per-latent maxima, parents, the weighted mean).
`library_irs` is irs.py's compute_irs after its draw: make_discretizer (the 20-bin histogram of every factor),
_drop_constant_dims and scalable_disentanglement_score, in float32 on the codes as the library computes them.
"""
import numpy as np

BINS = 20


def edges(v):
    """np.histogram's 21 fp64 edges of the integer column v: lo, hi = min, max (lo - 0.5, hi + 0.5 when equal),
    step = (hi - lo) / 20, edge_j = j * step + lo (each operation rounded), edge_20 = hi."""
    v = np.asarray(v, np.int64)
    lo, hi = float(v.min()), float(v.max())
    if lo == hi:
        lo, hi = lo - 0.5, hi + 0.5
    step = (hi - lo) / BINS
    return np.array([j * step + lo for j in range(BINS)] + [hi], np.float64)


def bins(v, e):
    """The bin of every value of v (0 .. 19): the number of e[0] .. e[19] at or below it, less one."""
    v = np.asarray(v, np.float64)
    return (e[None, :BINS] <= v[:, None]).sum(1) - 1


def quantile(a, diff_quantile):
    """np.percentile(a, diff_quantile * 100, axis=0) of a non-empty fp64 array by numpy's linear rule: q = (dq * 100) /
    100, h = (m - 1) q, lo = floor(h), hi = min(lo + 1, m - 1), t = h - lo, then a_lo + (a_hi - a_lo) t for t < 0.5,
    else a_hi - (a_hi - a_lo)(1 - t), on the ascending order statistics of every column."""
    s = np.sort(np.asarray(a, np.float64), axis=0)
    m = s.shape[0]
    q = (float(diff_quantile) * 100.0) / 100.0
    h = (m - 1) * q
    lo = int(np.floor(h))
    hi = min(lo + 1, m - 1)
    t = h - lo
    x_lo, x_hi = s[lo], s[hi]
    diff = x_hi - x_lo
    return x_lo + diff * t if t < 0.5 else x_hi - diff * (1.0 - t)


def fit(x, values, diff_quantile):
    """The tables of `dv_irs_fit` for drawn fp32 codes x [n, D] and the scored factors' values [K, n] -> dict of
    max_deviation [D], active [D], irs_matrix [D, K], group_deviation [K, 20, D], group_count [K, 20], edges [K, 21]."""
    x = np.asarray(x, np.float32).astype(np.float64)
    values = np.asarray(values, np.int64)
    n, D = x.shape
    K = values.shape[0]
    max_dev = np.abs(x - x.mean(0)).max(0)
    active = np.array([not np.all(x[:, d] == x[0, d]) for d in range(D)])
    e = np.stack([edges(values[k]) for k in range(K)])
    group_dev = np.full((K, BINS, D), np.nan)
    group_count = np.zeros((K, BINS), np.int64)
    irs = np.full((D, K), np.nan)
    for k in range(K):
        b = bins(values[k], e[k])
        cum = np.zeros(D)
        groups = 0
        for j in range(BINS):
            g = x[b == j]
            group_count[k, j] = len(g)
            if not len(g):
                continue
            groups += 1
            group_dev[k, j] = quantile(np.abs(g - g.mean(0)), diff_quantile)
            cum += group_dev[k, j]
        cum /= groups
        irs[active, k] = 1.0 - cum[active] / max_dev[active]
    return dict(max_deviation=max_dev, active=active, irs_matrix=irs, group_deviation=group_dev,
                group_count=group_count, edges=e)


def score(irs, max_dev, active):
    """(IRS, per-latent scores [D] (NaN inactive), parents [D] (-1 inactive)): the rows' maxima and first argmaxima,
    and their mean weighted by max_dev over the active latents, added in latent order; 0.0 with none active."""
    D = irs.shape[0]
    per, parents = np.full(D, np.nan), np.full(D, -1, np.int64)
    num = den = 0.0
    for d in range(D):
        if not active[d]:
            continue
        parents[d] = int(np.argmax(irs[d]))
        per[d] = irs[d, parents[d]]
        num += max_dev[d] * per[d]
        den += max_dev[d]
    return (num / den if den > 0 else 0.0), per, parents


def draw_values(lat_sizes, rows):
    """(scored factor indices, their values [K', n] of the C-order grid rows)."""
    factors = [k for k, s in enumerate(lat_sizes) if s > 1]
    v = np.stack(np.unravel_index(np.asarray(rows, np.int64), lat_sizes))
    return factors, v[factors]


# ---- disentanglement_lib's irs.py, line by line, in float32 ------------------------------------------------------
def _histogram_discretize(target, num_bins=BINS):
    discretized = np.zeros_like(target)
    for i in range(target.shape[0]):
        discretized[i, :] = np.digitize(target[i, :], np.histogram(target[i, :], num_bins)[1][:-1])
    return discretized


def _drop_constant_dims(ys):
    ys = np.asarray(ys)
    variances = ys.var(axis=1)
    active_mask = variances > 0.
    return ys[active_mask, :]


def scalable_disentanglement_score(gen_factors, latents, diff_quantile=0.99):
    num_gen = gen_factors.shape[1]
    num_lat = latents.shape[1]
    max_deviations = np.max(np.abs(latents - latents.mean(axis=0)), axis=0)
    cum_deviations = np.zeros([num_lat, num_gen])
    for i in range(num_gen):
        unique_factors = np.unique(gen_factors[:, i], axis=0)
        num_distinct_factors = unique_factors.shape[0]
        for k in range(num_distinct_factors):
            match = gen_factors[:, i] == unique_factors[k]
            e_loc = np.mean(latents[match, :], axis=0)
            diffs = np.abs(latents[match, :] - e_loc)
            max_diffs = np.percentile(diffs, q=diff_quantile * 100, axis=0)
            cum_deviations[:, i] += max_diffs
        cum_deviations[:, i] /= num_distinct_factors
    normalized_deviations = cum_deviations / max_deviations[:, np.newaxis]
    irs_matrix = 1.0 - normalized_deviations
    disentanglement_scores = irs_matrix.max(axis=1)
    if np.sum(max_deviations) > 0.0:
        avg_score = np.average(disentanglement_scores, weights=max_deviations)
    else:
        avg_score = np.mean(disentanglement_scores)
    parents = irs_matrix.argmax(axis=1)
    return {"disentanglement_scores": disentanglement_scores, "avg_score": avg_score, "parents": parents,
            "IRS": irs_matrix, "max_deviations": max_deviations}


def library_irs(mus, ys, diff_quantile=0.99):
    """compute_irs after its draw: mus float32 [D, n] codes, ys int [K, n] factor values -> {"IRS",
    "num_active_dims"}."""
    mus = np.asarray(mus, np.float32)
    ys_discrete = _histogram_discretize(np.asarray(ys, np.int64))
    active_mus = _drop_constant_dims(mus)
    if not active_mus.any():
        irs_score = 0.0
    else:
        irs_score = scalable_disentanglement_score(ys_discrete.T, active_mus.T, diff_quantile)["avg_score"]
    return {"IRS": irs_score, "num_active_dims": np.sum(active_mus)}
