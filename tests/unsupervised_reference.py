"""fp64 numpy restatement of the unsupervised scores, shared by tests/test_unsupervised_cpu.py and
tests/test_unsupervised_gpu.py (numpy only, so the GPU tests can use it).

The definition is disentanglement_lib's unsupervised_metrics.py under the conventions of include/disvae_b200.h:
- `sampled`: mu + exp(logvar / 2) eps in fp64 (the kernel rounds it once more, in fp32, with expf and fmaf);
- `cov`: np.cov of the codes (ddof 1) in fp64;
- `total_correlation`: -1/2 sum log eig(R), R the correlation matrix with a unit row and column for a constant
  latent, +inf when eig_min(R) <= D DBL_EPSILON eig_max(R);
- `wasserstein`: 2 trace(C) - 2 sum sqrt(max(eig(S), 0)), S = diag(c)^1/2 C diag(c)^1/2, and its norm (0 when
  trace(C) = 0);
- `mutual_info_matrix` / `mutual_info_score`: m[i][j] = sklearn's mutual_info_score(bins_j, bins_i) over the 20-bin
  histogram bins of tests/modularity_reference.py, the diagonal zeroed, sum / (D^2 - D).
"""
import numpy as np

import modularity_reference as MR

EPS = np.finfo(np.float64).eps
KEYS = ("gaussian_total_correlation", "gaussian_wasserstein_correlation", "gaussian_wasserstein_correlation_norm",
        "mutual_info_score")


def sampled(mu, logvar, eps):
    mu, logvar, eps = (np.asarray(a, np.float64) for a in (mu, logvar, eps))
    return mu + np.exp(logvar / 2) * eps


def cov(x):
    return np.cov(np.asarray(x, np.float64).T, ddof=1)


def correlation(C):
    c = np.diag(C).copy()
    s = np.sqrt(c)
    with np.errstate(divide="ignore", invalid="ignore"):
        R = C / np.outer(s, s)
    dead = c == 0
    R[dead, :] = 0.0
    R[:, dead] = 0.0
    np.fill_diagonal(R, 1.0)
    return R


def s_matrix(C):
    s = np.sqrt(np.diag(C))
    return s[:, None] * C * s[None, :]


def eigenvalues(C):
    """(eig(R), eig(S)), each ascending."""
    return np.linalg.eigvalsh(correlation(C)), np.linalg.eigvalsh(s_matrix(C))


def total_correlation(lam_r):
    lam_r = np.asarray(lam_r, np.float64)
    if lam_r[0] <= len(lam_r) * EPS * lam_r[-1]:
        return np.inf
    return -0.5 * np.log(lam_r).sum()


def wasserstein(C, lam_s):
    trace = np.trace(C)
    w = 2 * trace - 2 * np.sqrt(np.maximum(np.asarray(lam_s, np.float64), 0)).sum()
    return w, (w / trace if trace != 0 else 0.0)


def bins(x):
    """int [D, n]: the 20-bin histogram bin (1 .. 20) of every fp32 latent of x [n, D]."""
    x = np.asarray(x, np.float32)
    return np.stack([MR.bins(x[:, d], MR.edges(x[:, d])) for d in range(x.shape[1])])


def mutual_info_matrix(x):
    b = bins(x)
    D = b.shape[0]
    return np.array([[MR.mutual_info(b[j], b[i]) for j in range(D)] for i in range(D)])


def mutual_info_score(m):
    m = np.array(m, np.float64)
    D = m.shape[0]
    np.fill_diagonal(m, 0.0)
    return m.sum() / (D * D - D)


def scores_from(C, lam_r, lam_s, m):
    w, wn = wasserstein(C, lam_s)
    return dict(zip(KEYS, (total_correlation(lam_r), w, wn, mutual_info_score(m))))


def scores(x):
    """The four scores of the fp32 codes x [n, D]."""
    C = cov(x)
    return scores_from(C, *eigenvalues(C), mutual_info_matrix(x))
