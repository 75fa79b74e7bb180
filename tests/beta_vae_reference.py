"""fp64 numpy restatement of the beta-VAE score's features, fit and predictions, shared by
tests/test_beta_vae_score_cpu.py and tests/test_beta_vae_score_gpu.py (numpy only, so the GPU tests can use it).

`fit` is the exact minimiser of what sklearn's LogisticRegression(C=1) minimises (L2 on the weights, the intercept
unpenalised): multinomial above two classes, reported with the intercepts summing to zero; one binary model with
positive class 1 for two; nothing for one.  It is dense Newton with a backtracking line search on features centred on
their mean (an exact change of variables, since the intercept is free), with the multinomial Hessian's null direction
(the same constant on every intercept) removed by a rank-one term.
"""
import numpy as np


def features(mu, rows_a, rows_b):
    """x [V, D] fp64: the mean over l of |mu[rows_a[v, l]] - mu[rows_b[v, l]]|, the fp32 values differenced in fp64 and
    added in ascending l, then divided by L."""
    mu = np.asarray(mu, np.float32).astype(np.float64)
    rows_a, rows_b = np.asarray(rows_a), np.asarray(rows_b)
    s = np.zeros((rows_a.shape[0], mu.shape[1]))
    for l in range(rows_a.shape[1]):
        s = s + np.abs(mu[rows_a[:, l]] - mu[rows_b[:, l]])
    return s / rows_a.shape[1]


def _rows(x, theta, R, multi):
    """(loss [n] pieces' sum, p [n, R], logits [n, R]) at theta [R, D + 1] on augmented x [n, D + 1]."""
    z = x @ theta.T
    if multi:
        m = z.max(1, keepdims=True)
        e = np.exp(z - m)
        se = e.sum(1, keepdims=True)
        return m[:, 0] + np.log(se[:, 0]), e / se, z
    lse = np.maximum(z[:, 0], 0) + np.log1p(np.exp(-np.abs(z[:, 0])))
    return lse, (1.0 / (1.0 + np.exp(-z))), z


def objective(x, y, nc, W, b):
    """(f, gradient [rows, D + 1], scale [rows, D + 1]) of the fit's objective at (W [rows, D], b [rows]) on the raw
    features x [n, D]: the KKT residual of a solution and the scale of its parts (|weight| + sum_i |q_i x_i|)."""
    x = np.asarray(x, np.float64)
    xa = np.c_[x, np.ones(len(x))]
    theta = np.c_[W, b]
    multi = nc > 2
    lse, p, z = _rows(xa, theta, theta.shape[0], multi)
    if multi:
        t = np.eye(nc)[y]
        f = 0.5 * (W * W).sum() + (lse - z[np.arange(len(y)), y]).sum()
    else:
        t = (y == 1).astype(np.float64)[:, None]
        f = 0.5 * (W * W).sum() + (lse - np.where(y == 1, z[:, 0], 0.0)).sum()
    q = p - t
    reg = np.c_[W, np.zeros(len(b))]
    return f, reg + q.T @ xa, np.abs(reg) + np.abs(q).T @ np.abs(xa)


def fit(x, y, nc, tol=1e-12, max_iter=100):
    """(W [rows, D], b [rows], Newton steps or -1) for features x [n, D] and class indices y [n] in 0 .. nc-1."""
    x = np.asarray(x, np.float64)
    y = np.asarray(y, np.int64)
    n, D = x.shape
    if nc == 1:
        return np.zeros((0, D)), np.zeros(0), 0
    multi = nc > 2
    R = nc if multi else 1
    m = x.mean(0)
    xa = np.c_[x - m, np.ones(n)]
    Dp = D + 1
    t = np.eye(nc)[y] if multi else (y == 1).astype(np.float64)[:, None]
    reg = np.tile(np.r_[np.ones(D), 0.0], R)
    u = np.zeros(R * Dp)
    if multi:
        u[D::Dp] = 1.0 / np.sqrt(R)

    def parts(theta):
        th = theta.reshape(R, Dp)
        lse, p, z = _rows(xa, th, R, multi)
        loss = lse - ((z * t).sum(1) if multi else np.where(y == 1, z[:, 0], 0.0))
        f = 0.5 * (reg * theta * theta).sum() + loss.sum()
        q = p - t
        g = reg * theta + (q.T @ xa).ravel()
        sc = np.abs(reg * theta) + (np.abs(q).T @ np.abs(xa)).ravel()
        return f, g, sc, p

    theta = np.zeros(R * Dp)
    f, g, sc, p = parts(theta)
    steps = -1
    for it in range(max_iter + 1):
        if np.abs(g).max() <= tol * sc.max():
            steps = it
            break
        if it == max_iter:
            break
        # H = diag(reg) + sum_i (diag(p_i) - p_i p_i^T) (x) x_i x_i^T  (binary: p_i (1 - p_i) x_i x_i^T)
        H = np.diag(reg)
        if multi:
            for c in range(R):
                sl = slice(c * Dp, (c + 1) * Dp)
                H[sl, sl] += (xa * p[:, c:c + 1]).T @ xa
            M = (p[:, :, None] * xa[:, None, :]).reshape(n, R * Dp)
            H -= M.T @ M
            H += np.outer(u, u)
        else:
            H += (xa * (p * (1 - p))).T @ xa
        d = -np.linalg.solve(H, g)
        slope = g @ d
        step = 1.0
        for _ in range(60):
            ft, gt, st, pt = parts(theta + step * d)
            if ft - f <= 1e-4 * step * slope + 1e-15 * abs(f):
                break
            step *= 0.5
        else:
            break
        theta, f, g, sc, p = theta + step * d, ft, gt, st, pt
    th = theta.reshape(R, Dp)
    W = th[:, :D].copy()
    b = th[:, D] - W @ m
    if multi:
        b = b - b.mean()
    return W, b, steps


def decisions(W, b, x):
    """W x + b [n, rows] in fp64."""
    return np.asarray(x, np.float64) @ np.asarray(W).T + np.asarray(b)[None, :]


def predict(W, b, nc, x):
    """(class indices [n], the gap between the two deciding values of each row: the top two decisions, |w x + b| for
    two classes, inf for one)."""
    n = len(x)
    if nc == 1:
        return np.zeros(n, np.int64), np.full(n, np.inf)
    v = decisions(W, b, x)
    if nc == 2:
        return (v[:, 0] > 0).astype(np.int64), np.abs(v[:, 0])
    top = np.sort(v, axis=1)
    return np.argmax(v, axis=1), top[:, -1] - top[:, -2]
