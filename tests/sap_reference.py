"""fp64 numpy restatement of the SAP score's fits, shared by tests/test_sap_score_cpu.py and tests/test_sap_score_gpu.py
(numpy only, so the GPU tests can use it).

`solve` is the exact minimiser of the objective LinearSVC(C, class_weight="balanced") hands liblinear for one binary
problem on 1-D data (squared hinge, L2, the intercept a regularised feature of scale 1):
    f(w, b) = 1/2 (w^2 + b^2) + sum_i c_i max(0, 1 - s_i (w x_i + b))^2,
by semismooth Newton with a backtracking line search, many problems at once.  `problems` builds a factor's problems the
way the SAP score defines them, `predict` applies the fitted lines, and `score_matrix` computes from the kernel's own
inputs what `dv_sap_score_matrix` computes.
"""
import numpy as np


def _parts(z, x, s, c):
    """f, gradient [P, 2], generalised Hessian [P, 2, 2] and the stationarity scale [P] at z [P, 2]."""
    m = 1.0 - s * (z[:, :1] * x + z[:, 1:])
    cm = np.where(m > 0, c * m, 0.0)
    ca = np.where(m > 0, c, 0.0)
    f = 0.5 * (z * z).sum(1) + (cm * m).sum(1)
    g = z - 2.0 * np.stack([(cm * s * x).sum(1), (cm * s).sum(1)], 1)
    hxx, hx, h1 = (ca * x * x).sum(1), (ca * x).sum(1), ca.sum(1)
    H = np.stack([np.stack([1 + 2 * hxx, 2 * hx], 1), np.stack([2 * hx, 1 + 2 * h1], 1)], 1)
    scale = np.abs(z).sum(1) + 2.0 * (cm * (np.abs(x) + 1.0)).sum(1)
    return f, g, H, scale


def gradient(z, x, s, c):
    """(gradient [P, 2], scale [P]) of f at z [P, 2]: the KKT residual of a solution and what it is measured against."""
    _, g, _, scale = _parts(np.asarray(z, np.float64).reshape(-1, 2), x, s, c)
    return g, scale


def solve(x, s, c, tol=1e-11, max_iter=100):
    """argmin f for every row of x, s, c [P, n] (fp64) -> (z [P, 2] = (w, b), Newton steps [P], -1 where not
    converged to |gradient|_inf <= tol * scale)."""
    x, s, c = (np.asarray(a, np.float64) for a in (x, s, c))
    P = x.shape[0]
    z = np.zeros((P, 2))
    steps = np.full(P, -1)
    f, g, H, scale = _parts(z, x, s, c)
    todo = np.arange(P)
    for it in range(max_iter + 1):
        conv = np.abs(g[todo]).max(1) <= tol * scale[todo]
        steps[todo[conv]] = it
        todo = todo[~conv]
        if not len(todo) or it == max_iter:
            break
        p = -np.linalg.solve(H[todo], g[todo][..., None])[..., 0]
        slope = (g[todo] * p).sum(1)
        t = np.ones(len(todo))
        pend = np.arange(len(todo))
        for _ in range(60):
            j = todo[pend]
            zt = z[j] + t[pend, None] * p[pend]
            ft, gt, Ht, st = _parts(zt, x[j], s[j], c[j])
            ok = ft - f[j] <= 1e-4 * t[pend] * slope[pend] + 1e-15 * np.abs(f[j])
            a = j[ok]
            z[a], f[a], g[a], H[a], scale[a] = zt[ok], ft[ok], gt[ok], Ht[ok], st[ok]
            pend = pend[~ok]
            t[pend] *= 0.5
            if not len(pend):
                break
        todo = np.setdiff1d(todo, todo[pend])     # a problem whose line search failed stays unconverged
    return z, steps


def problems(y, nc, C, num_train):
    """(s, c, positive classes) of one factor's training labels y [n] (class indices 0 .. nc-1), s and c
    [n_problems, n]: one-vs-rest per class above two classes (the positives weighted C * cw_c, the negatives plain
    C), one problem with positive class 1 and every row weighted C * cw_{y_i} for two, none for one.
    cw_c = num_train / (nc * count_c)."""
    counts = np.bincount(y, minlength=nc).astype(np.float64)
    cw = num_train / (nc * counts)
    if nc == 1:
        return np.zeros((0, len(y))), np.zeros((0, len(y))), []
    pos = list(range(nc)) if nc > 2 else [1]
    s = np.stack([np.where(y == p, 1.0, -1.0) for p in pos])
    if nc > 2:
        c = np.stack([np.where(y == p, C * cw[p], C) for p in pos])
    else:
        c = (C * cw[y])[None, :]
    return s, c, pos


def decisions(lines, x):
    """w_c x + b_c [n, n_problems] in fp64, the product and the sum rounded separately."""
    x = np.asarray(x, np.float64)[:, None]
    return np.add(np.multiply(lines[:, 0][None, :], x), lines[:, 1][None, :])


def predict(lines, nc, x):
    """Class indices predicted for x [n] by a factor's fitted lines [n_problems, 2], and the gap between the two
    deciding values of every row (the top two decisions, or |w x + b| for two classes; inf for one class)."""
    n = len(x)
    if nc == 1:
        return np.zeros(n, np.int64), np.full(n, np.inf)
    v = decisions(lines, x)
    if nc == 2:
        return (v[:, 0] > 0).astype(np.int64), np.abs(v[:, 0])
    top = np.sort(v, axis=1)
    return np.argmax(v, axis=1), top[:, -1] - top[:, -2]


def score_matrix(mu, train_rows, test_rows, train_cls, test_cls, n_classes, counts, C):
    """What dv_sap_score_matrix computes, in fp64 from the same inputs (numpy arrays; mu [N, D] fp32) -> (score fp32
    [D, K], coef [D, K, S, 2] NaN beyond a factor's problems, steps [D, K, S] 0 beyond, gap [D, K, num_test] the
    deciding gap of each test row)."""
    x_train = np.asarray(mu, np.float32)[train_rows].astype(np.float64)         # [n, D]
    x_test = np.asarray(mu, np.float32)[test_rows].astype(np.float64)
    n, D = x_train.shape
    K, S = counts.shape
    score = np.zeros((D, K), np.float32)
    coef = np.full((D, K, S, 2), np.nan)
    steps = np.zeros((D, K, S), np.int64)
    gap = np.zeros((D, K, len(test_rows)))
    for k in range(K):
        nc = int(n_classes[k])
        y = np.asarray(train_cls[k], np.int64)
        s, c, pos = problems(y, nc, C, n)
        npb = len(pos)
        if npb:
            z, st = solve(np.repeat(x_train.T, npb, axis=0), np.tile(s, (D, 1)), np.tile(c, (D, 1)))
            coef[:, k, :npb] = z.reshape(D, npb, 2)
            steps[:, k, :npb] = st.reshape(D, npb)
        for d in range(D):
            pred, gap[d, k] = predict(coef[d, k, :npb], nc, x_test[:, d])
            score[d, k] = np.float32((pred == np.asarray(test_cls[k])).sum() / len(test_rows))
    return score, coef, steps, gap


def sap(score):
    """Mean over columns of the largest minus the second largest entry, in fp64."""
    m = np.sort(np.asarray(score, np.float64), axis=0)
    return float(np.mean(m[-1] - m[-2]))
