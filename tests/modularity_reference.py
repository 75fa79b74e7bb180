"""fp64 numpy restatement of modularity and explicitness, shared by tests/test_modularity_score_cpu.py and
tests/test_modularity_score_gpu.py (numpy only, so the GPU tests can use it).

The definition is disentanglement_lib's compute_modularity_explicitness with num_bins = 20, under the conventions of
include/disvae_b200.h:
- `edges` / `bins`: np.digitize(x, np.histogram(x, 20)[1][:-1]) of an fp32 column, the edges built in fp32 as numpy's
  linspace builds them, and the same rule where numpy refuses the range;
- `mutual_info`: sklearn's mutual_info_score, term by term in its form;
- `modularity`: modularity_explicitness.py's modularity(), line by line;
- `standardise`, `probabilities`, `auc`, `explicitness`: the explicitness half, with the fit of
  tests/beta_vae_reference.py (the exact minimiser of LogisticRegression(C=1)).
"""
import numpy as np

import beta_vae_reference as BR

BINS = 20
EPS = np.finfo(np.float64).eps


def edges(x):
    """The 21 fp32 edges of the fp32 column x: lo, hi = min, max (lo - 0.5, hi + 0.5 when equal), step = (hi - lo) / 20,
    edge_j = j * step + lo (each operation rounded to fp32), edge_20 = hi."""
    x = np.asarray(x, np.float32)
    lo, hi = np.float32(x.min()), np.float32(x.max())
    if lo == hi:
        lo, hi = np.float32(lo - np.float32(0.5)), np.float32(hi + np.float32(0.5))
    step = np.float32(np.float32(hi - lo) / np.float32(BINS))
    e = np.array([np.float32(np.float32(np.float32(j) * step) + lo) for j in range(BINS)] + [hi], np.float32)
    return e


def bins(x, e):
    """The bin of every value of x (1 .. 20): the number of e[0] .. e[19] at or below it (np.digitize's answer where
    the edges increase)."""
    x = np.asarray(x, np.float32)
    return (e[None, :BINS] <= x[:, None]).sum(1)


def mutual_info(cls, b):
    """sklearn's mutual_info_score(cls, b) over the non-zero cells of the contingency table, in its term form, the bins
    of a class in order, then the classes in order."""
    cls, b = np.asarray(cls), np.asarray(b)
    n = len(cls)
    ci, bi = np.unique(cls, return_inverse=True)[1], np.unique(b, return_inverse=True)[1]
    nc, nb = ci.max() + 1, bi.max() + 1
    if nc == 1 or nb == 1:
        return 0.0
    table = np.zeros((nc, nb), np.int64)
    np.add.at(table, (ci, bi), 1)
    a, bb = table.sum(1), table.sum(0)
    ln = np.log(float(n))
    s = 0.0
    for c in range(nc):
        for j in range(nb):
            v = table[c, j]
            if v == 0:
                continue
            cn = v / n
            term = cn * (np.log(float(v)) - ln) + cn * (-np.log(float(a[c] * bb[j])) + ln + ln)
            s += 0.0 if abs(term) < EPS else term
    return max(s, 0.0)


def mutual_information(x, cls):
    """(mi [D, K], edges [D, 21]) of fp32 training latents x [n, D] and class labels cls [K, n]."""
    x = np.asarray(x, np.float32)
    E = np.stack([edges(x[:, d]) for d in range(x.shape[1])])
    mi = np.array([[mutual_info(c, bins(x[:, d], E[d])) for c in cls] for d in range(x.shape[1])])
    return mi, E


def modularity(mutual_information):
    """modularity_explicitness.py's modularity(), line by line -> (score, per-latent scores)."""
    squared_mi = np.square(mutual_information)
    max_squared_mi = np.max(squared_mi, axis=1)
    numerator = np.sum(squared_mi, axis=1) - max_squared_mi
    denominator = max_squared_mi * (squared_mi.shape[1] - 1.)
    with np.errstate(divide="ignore", invalid="ignore"):
        delta = numerator / denominator
    modularity_score = 1. - delta
    index = (max_squared_mi == 0.)
    modularity_score[index] = 0.
    return np.mean(modularity_score), modularity_score


def standardise(x_train, x_test):
    """(train features, test features, mean, std): fp64 mean and std (ddof 0) of the fp32 training latents, a std of 0
    replaced by 1."""
    xt = np.asarray(x_train, np.float32).astype(np.float64)
    xe = np.asarray(x_test, np.float32).astype(np.float64)
    mean = xt.mean(0)
    std = np.sqrt(((xt - mean) ** 2).mean(0))
    std = np.where(std == 0, 1.0, std)
    return (xt - mean) / std, (xe - mean) / std, mean, std


def probabilities(W, b, nc, x):
    """[rows, columns] class probabilities: softmax of W x + b for nc > 2, (1 - p_1, p_1) with p_1 = 1 / (1 + exp(-z))
    for nc = 2."""
    z = BR.decisions(W, b, x)
    if nc == 2:
        p1 = 1.0 / (1.0 + np.exp(-z[:, 0]))
        return np.stack([1.0 - p1, p1], 1)
    e = np.exp(z - z.max(1, keepdims=True))
    return e / e.sum(1, keepdims=True)


def auc(p, labels, c):
    """ROC AUC of column c: positives the rows labelled c, negatives the others; (2 #{p_pos > p_neg} + #{p_pos =
    p_neg}) / (2 n_pos n_neg) with exact integer pair counts; NaN without positives or negatives."""
    p, labels = np.asarray(p, np.float64), np.asarray(labels)
    pos, neg = np.sort(p[labels == c]), p[labels != c]
    if len(pos) == 0 or len(neg) == 0:
        return float("nan")
    lo = np.searchsorted(pos, neg, side="left")
    hi = np.searchsorted(pos, neg, side="right")
    gt = int((len(pos) - hi).sum())
    eq = int((hi - lo).sum())
    return (2 * gt + eq) / (2.0 * len(pos) * len(neg))


def columns(nc):
    return nc if nc > 2 else (2 if nc == 2 else 0)


def explicitness(f_train, y_train, f_test, y_test, nc):
    """(W, b, steps, train AUCs [columns], test AUCs [columns], train probabilities, test probabilities) of one factor
    with nc training classes (labels 0 .. nc-1; test labels -1 for unseen values)."""
    W, b, steps = BR.fit(f_train, y_train, nc)
    if nc < 2:
        return W, b, steps, np.zeros(0), np.zeros(0), None, None
    pt, pe = probabilities(W, b, nc, f_train), probabilities(W, b, nc, f_test)
    cols = columns(nc)
    return (W, b, steps, np.array([auc(pt[:, c], y_train, c) for c in range(cols)]),
            np.array([auc(pe[:, c], y_test, c) for c in range(cols)]), pt, pe)


def mean_defined(a):
    a = np.asarray(a, np.float64)
    a = a[~np.isnan(a)]
    return float(a.mean()) if a.size else float("nan")
