"""fp64 numpy restatement of the UDR score (Duan et al. 2020, as disentanglement_lib's udr.py computes it with
compute_udr_sklearn), steps 2 to 6 of its definition in INTEGRATION.md, with this project's deviations: the Lasso is
solved to its exact minimiser, a constant column's Spearman correlation is 0, and a pair where either model has no
informative latent scores 0.  Shared by the CPU and GPU tests; needs no GPU."""
import numpy as np

KL_THRESHOLD = 0.01
ALPHA = 0.1
GAP_TOL = 1e-12
MAX_SWEEPS = 10000


def kl(mu, logvar):
    """Mean over the points of 0.5 (mu^2 + exp(logvar) - logvar - 1) of every latent, fp64 from the fp32 values."""
    mu, logvar = np.asarray(mu, np.float64), np.asarray(logvar, np.float64)
    return (0.5 * (mu * mu + np.exp(logvar) - logvar - 1.0)).mean(0)


def standardise(x):
    """StandardScaler().fit_transform in fp64: mean, std with ddof 0, a std of 0 divided by 1."""
    x = np.asarray(x, np.float64)
    mean = x.mean(0)
    sd = np.sqrt(((x - mean) ** 2).mean(0))
    return (x - mean) / np.where(sd == 0, 1.0, sd)


def average_ranks(x):
    """scipy.stats.rankdata(x, "average") of every column (1-based, ties averaged)."""
    x = np.asarray(x)
    out = np.empty(x.shape, np.float64)
    for d in range(x.shape[1]):
        v = x[:, d]
        order = np.argsort(v, kind="stable")
        s = v[order]
        lo = np.searchsorted(s, s, "left")
        hi = np.searchsorted(s, s, "right")
        out[order, d] = 0.5 * (lo + hi + 1)
    return out


def features(mu, informative, correlation):
    """The feature columns of one model: standardised latents (or, for Spearman, standardised average ranks) times
    the informative mask."""
    f = standardise(average_ranks(mu) if correlation == "spearman" else mu)
    return f * np.asarray(informative, np.float64)


def lasso(G, C, q, alpha=ALPHA, tol=GAP_TOL, max_sweeps=MAX_SWEEPS):
    """min_w 1/2 (q_b - 2 C[:, b]^T w + w^T G w) + alpha |w|_1 for every target b at once, by cyclic coordinate
    descent from 0 until every target's duality gap is at most tol q_b -> (W [D_in, D_out], sweeps [D_out], -1 at the
    cap).  A target with q_b = 0 keeps w = 0."""
    Din, Dout = C.shape
    W = np.zeros((Din, Dout))
    sweeps = np.full(Dout, -1)
    live = q > 0
    sweeps[~live] = 0
    for s in range(max_sweeps + 1):
        g = C - G @ W
        cw = (C * W).sum(0)
        wg = (W * g).sum(0)
        r2, ry = q - cw - wg, q - cw
        gmax = np.abs(g).max(0) if Din else np.zeros(Dout)
        cst = np.where(gmax > alpha, alpha / np.where(gmax > 0, gmax, 1.0), 1.0)
        gap = np.where(gmax > alpha, 0.5 * r2 * (1 + cst * cst), r2) + alpha * np.abs(W).sum(0) - cst * ry
        done = live & (sweeps < 0) & (gap <= tol * q)
        sweeps[done] = s
        if not (live & (sweeps < 0)).any() or s == max_sweeps:
            break
        act = live & (sweeps < 0)                               # a converged target stops where it is
        for a in range(Din):
            if G[a, a] == 0:
                continue
            rho = C[a, act] - G[a] @ W[:, act] + G[a, a] * W[a, act]
            W[a, act] = np.sign(rho) * np.maximum(np.abs(rho) - alpha, 0.0) / G[a, a]
    return W, sweeps


def similarity(Zi, Zj, correlation):
    """R_ij [D_i, D_j] of the feature columns Zi (inputs) and Zj (targets), and the Lasso's sweeps [D_j] (None for
    Spearman)."""
    n = Zi.shape[0]
    C = Zi.T @ Zj / n
    if correlation == "spearman":
        return np.abs(C), None
    G = Zi.T @ Zi / n
    q = (Zj * Zj).sum(0) / n
    W, sweeps = lasso(G, C, q)
    return np.abs(W), sweeps


def pair_score(R, informative_i, informative_j):
    """The pair score: R's rows filtered by i's informative latents and its columns by j's; the mean over columns of
    max^2 / sum and over rows of max^2 / sum (0 / 0 counted 0), averaged; 0 when either filter is empty."""
    M = R[np.asarray(informative_i, bool)][:, np.asarray(informative_j, bool)]
    if M.size == 0:
        return 0.0
    with np.errstate(invalid="ignore", divide="ignore"):
        sx = np.nan_to_num(M.max(0) ** 2 / M.sum(0))
        sy = np.nan_to_num(M.max(1) ** 2 / M.sum(1))
    return (sx.mean() + sy.mean()) / 2


def model_scores(pair, groups):
    """UDR_k = np.median over the others j of k's group of pair[j, k]."""
    out = np.zeros(pair.shape[0])
    for g in groups:
        for k in g:
            out[k] = np.median([pair[j, k] for j in g if j != k])
    return out


def udr(mu, logvar, correlation="lasso", groups=None):
    """The whole score of mu, logvar [K, n, D] -> dict(kl, informative, features, raw, pair, sweeps, model_scores)."""
    mu, logvar = np.asarray(mu, np.float32), np.asarray(logvar, np.float32)
    K, n, D = mu.shape
    groups = [list(range(K))] if groups is None else groups
    k_l = np.stack([kl(mu[k], logvar[k]) for k in range(K)])
    inf = k_l > KL_THRESHOLD
    Z = [features(mu[k], inf[k], correlation) for k in range(K)]
    raw = np.full((K, K, D, D), np.nan)
    pair = np.full((K, K), np.nan)
    sweeps = np.zeros((K, K), np.int64)
    for i in range(K):
        for j in range(K):
            if i == j:
                continue
            raw[i, j], s = similarity(Z[i], Z[j], correlation)
            if s is not None:
                sweeps[i, j] = -1 if (s < 0).any() else s.max()
            pair[i, j] = pair_score(raw[i, j], inf[i], inf[j])
    return dict(kl=k_l, informative=inf, features=Z, raw=raw, pair=pair, sweeps=sweeps,
                model_scores=model_scores(pair, groups))
