"""fp64 numpy restatement of the DCI score's fits, shared by tests/test_dci_score_cpu.py and tests/test_dci_score_gpu.py
(numpy only, so the GPU tests can use it).

`fit` grows, for one factor, the gradient-boosted trees of sklearn's GradientBoostingClassifier() at its defaults (100
stages of depth-3 friedman_mse regression trees on the log-loss residuals, learning rate 0.1) under the rules
`dv_dci_fit` states in include/disvae_b200.h: the split proxy is summed exactly over residuals rounded to 2^-40, an
exact tie goes to the lowest latent and then the lowest threshold, impurities (in the centred form) and leaf values are
fp64 sums, and every score update is a rounded product and a rounded sum (no fused multiply-add).  `fit_factors` runs
`fit` on what the kernel reads (the rows, the labels of `sap_labels`), and `dci_restated` restates disentanglement_lib's
dci.py line by line on an importance matrix.
"""
import numpy as np

EPS32 = float(np.finfo(np.float32).eps)      # the clip of the prior probabilities
DBL_EPSILON = float(np.finfo(np.float64).eps)
FEATURE_THRESHOLD = 1e-7
FIX = 2.0 ** 40                              # the fixed point of the split proxy's sums
MAX_DEPTH = 3
NODES = 15                                   # heap-ordered nodes of a depth-3 tree
LEARNING_RATE = 0.1
LEAF, ABSENT = -1, -2                        # tree feature of a leaf, of a node the tree does not have


def init_raw(counts, n):
    """Initial raw scores [cols] of a factor with training class counts `counts` [nc] (nc >= 2) over n rows."""
    p = np.clip(np.asarray(counts, np.float64) / n, EPS32, 1 - EPS32)
    if len(p) == 2:
        return np.array([np.log(p[1] / (1 - p[1]))])
    return np.log(p / np.exp(np.mean(np.log(p))))


def residuals(raw, y, nc):
    """(residuals [cols, n], targets [cols, n]) at the raw scores [cols, n] of rows with classes y [n]."""
    if nc == 2:
        t = (y == 1).astype(np.float64)
        z = raw[0]
        e = np.exp(-np.abs(z))
        g = np.where(z < 0, ((1 - t) * e - t) / (1 + e), ((1 - t) - t * e) / (1 + e))    # sigmoid(z) - t
        return -g[None], t[None]
    m = raw.max(0)
    e = np.exp(raw - m)
    t = (y[None] == np.arange(nc)[:, None]).astype(np.float64)
    return t - e / e.sum(0), t


def _best_split(xT, order, rows, q):
    """(latent, threshold) of the best split of the rows `rows` (bool [n]), or None: the largest proxy over every
    latent and every gap x_b > x_a + 1e-7 between consecutive sorted values, the lowest latent and then the lowest
    threshold on an exact tie."""
    D = xT.shape[0]
    cnt = int(rows.sum())
    o = order[rows[order]].reshape(D, cnt)                   # the node's rows, sorted by each latent
    v = np.take_along_axis(xT, o, 1)
    Q = np.cumsum(q[o], axis=1)
    nl = np.arange(1, cnt, dtype=np.float64)
    nr = cnt - nl
    Sl = Q[:, :-1].astype(np.float64) / FIX
    Sr = (Q[:, -1:] - Q[:, :-1]).astype(np.float64) / FIX
    diff = nr * Sl - nl * Sr
    proxy = np.where(v[:, 1:] > v[:, :-1] + FEATURE_THRESHOLD, diff * diff / (nl * nr), -np.inf)
    if proxy.shape[1] == 0:
        return None
    pos = proxy.argmax(1)
    best = proxy[np.arange(D), pos]
    d = int(best.argmax())
    if best[d] == -np.inf:
        return None
    a, b = v[d, pos[d]], v[d, pos[d] + 1]
    t = a / 2 + b / 2
    return d, (a if t == b else t)


def grow(xT, order, r, t, nc):
    """One tree on the residuals r [n] (targets t [n]) -> (feature int32 [15], threshold [15], value [15], leaf of
    every training row [n], importance contributions {node: (latent, n imp - n_l imp_l - n_r imp_r)})."""
    n = r.shape[0]
    q = np.rint(r * FIX).astype(np.int64)
    h = (t - r) * (1 - (t - r))
    feature = np.full(NODES, ABSENT, np.int32)
    threshold = np.full(NODES, np.nan)
    value = np.full(NODES, np.nan)
    node = np.zeros(n, np.int64)
    size, imp = {}, {}
    for depth in range(MAX_DEPTH + 1):
        for m in range(2 ** depth - 1, 2 ** (depth + 1) - 1):
            if m > 0 and feature[(m - 1) // 2] < 0:
                continue
            rows = node == m
            cnt = int(rows.sum())
            s = r[rows].sum()
            size[m] = cnt
            e = r[rows] - s / cnt
            imp[m] = (e * e).sum() / cnt                       # the centred form of sum r^2/n - (sum r/n)^2
            split = None
            if depth < MAX_DEPTH and cnt >= 2 and imp[m] > DBL_EPSILON:
                split = _best_split(xT, order, rows, q)
            if split is None:
                feature[m] = LEAF
                num = s * ((nc - 1) / nc) if nc > 2 else s
                den = h[rows].sum()
                value[m] = 0.0 if abs(den) < 1e-150 else num / den
            else:
                feature[m], threshold[m] = split
                left = rows & (xT[split[0]] <= split[1])
                node[left] = 2 * m + 1
                node[rows & ~left] = 2 * m + 2
    contrib = {m: (int(feature[m]), size[m] * imp[m] - size[2 * m + 1] * imp[2 * m + 1] - size[2 * m + 2]
                   * imp[2 * m + 2]) for m in range(7) if feature[m] >= 0}
    return feature, threshold, value, node, contrib


def apply(feature, threshold, xT):
    """The leaf of every row of xT [D, n] (x <= threshold goes left)."""
    node = np.zeros(xT.shape[1], np.int64)
    for _ in range(MAX_DEPTH):
        f = feature[node]
        inner = f >= 0
        go_left = xT[np.maximum(f, 0), np.arange(xT.shape[1])] <= threshold[node]
        node = np.where(inner, np.where(go_left, 2 * node + 1, 2 * node + 2), node)
    return node


def predict(raw, nc):
    if nc == 1:
        return np.zeros(raw.shape[1], np.int64)
    if nc == 2:
        return (raw[0] >= 0).astype(np.int64)
    return raw.argmax(0)


def fit(x_train, y, nc, x_test, stages=100):
    """The boosted fit of one factor: x_train [n, D] and x_test [m, D] fp32 values, y [n] classes 0 .. nc-1 (every
    class present) -> dict(importance [D] fp64, pred_train [n], pred_test [m], feature int32 [cols, stages, 15],
    threshold, value [cols, stages, 15], raw_train [cols, n]).  cols = nc above two classes, 1 for two, 0 for one."""
    xT = np.asarray(x_train, np.float32).astype(np.float64).T.copy()
    xe = np.asarray(x_test, np.float32).astype(np.float64).T.copy()
    y = np.asarray(y, np.int64)
    D, n = xT.shape
    cols = nc if nc > 2 else nc - 1
    order = np.argsort(xT, axis=1, kind="stable")
    out = dict(feature=np.full((cols, stages, NODES), ABSENT, np.int32),
               threshold=np.full((cols, stages, NODES), np.nan), value=np.full((cols, stages, NODES), np.nan))
    if nc == 1:
        out.update(importance=np.zeros(D), pred_train=np.zeros(n, np.int64), pred_test=np.zeros(xe.shape[1], np.int64),
                   raw_train=np.zeros((0, n)))
        return out
    init = init_raw(np.bincount(y, minlength=nc), n)
    raw = np.repeat(init[:, None], n, 1)
    raw_test = np.repeat(init[:, None], xe.shape[1], 1)
    acc = np.zeros((cols, D))
    relevant = 0
    for s in range(stages):
        r, t = residuals(raw, y, nc)
        for c in range(cols):
            feature, threshold, value, leaf, contrib = grow(xT, order, r[c], t[c], nc)
            out["feature"][c, s], out["threshold"][c, s], out["value"][c, s] = feature, threshold, value
            for m in sorted(contrib):
                d, v = contrib[m]
                acc[c, d] += v / n
            relevant += int(feature[0] >= 0)
            raw[c] = raw[c] + LEARNING_RATE * value[leaf]
            raw_test[c] = raw_test[c] + LEARNING_RATE * value[apply(feature, threshold, xe)]
    importance = np.zeros(D)
    if relevant:
        total = np.zeros(D)
        for c in range(cols):
            total = total + acc[c]
        mean = total / relevant
        norm = mean.sum()
        if norm != 0:
            importance = np.abs(mean / norm)
    out.update(importance=importance, pred_train=predict(raw, nc), pred_test=predict(raw_test, nc), raw_train=raw)
    return out


def fit_factors(mu, train_rows, test_rows, train_cls, test_cls, n_classes, stages=100):
    """What `dv_dci_fit` computes, from its own inputs (numpy): mu [N, D] fp32, the rows, and `sap_labels`' classes
    -> (importance [D, K'], pred [K', num_train + num_test] (class indices), fits (one `fit` dict per factor))."""
    mu = np.asarray(mu, np.float32)
    K = len(n_classes)
    fits = [fit(mu[train_rows], train_cls[k], int(n_classes[k]), mu[test_rows], stages) for k in range(K)]
    importance = np.stack([f["importance"] for f in fits], 1)
    pred = np.stack([np.concatenate([f["pred_train"], f["pred_test"]]) for f in fits])
    return importance, pred, fits


# ---- disentanglement_lib's dci.py, restated line by line --------------------------------------------------------------
def dci_restated(importance_matrix):
    """disentanglement(importance_matrix), completeness(importance_matrix) as dci.py computes them."""
    import scipy.stats

    def disentanglement_per_code(m):
        return 1. - scipy.stats.entropy(m.T + 1e-11, base=m.shape[1])

    def disentanglement(m):
        per_code = disentanglement_per_code(m)
        if m.sum() == 0.:
            m = np.ones_like(m)
        code_importance = m.sum(axis=1) / m.sum()
        return np.sum(per_code * code_importance)

    def completeness_per_factor(m):
        return 1. - scipy.stats.entropy(m + 1e-11, base=m.shape[0])

    def completeness(m):
        per_factor = completeness_per_factor(m)
        if m.sum() == 0.:
            m = np.ones_like(m)
        factor_importance = m.sum(axis=0) / m.sum()
        return np.sum(per_factor * factor_importance)

    return float(disentanglement(importance_matrix)), float(completeness(importance_matrix))
