"""fp64 numpy restatement of the downstream-task score, shared by tests/test_downstream_task_cpu.py and
tests/test_downstream_task_gpu.py (numpy only, so the GPU tests can use it).

The definition is disentanglement_lib's downstream_task.py with LogisticRegressionCV(Cs=10, cv=KFold(5)) or
GradientBoostingClassifier(), under the conventions of include/disvae_b200.h:
- `fit`: the exact minimiser of C sum_i loss_i + 1/2 |W|^2 (intercepts unpenalised).  It is tests/beta_vae_reference.py's
  fit at C = 1 on the features scaled by sqrt(C): with V = W / sqrt(C), V (sqrt(C) x) = W x and 1/2 |V|^2 =
  1/2 |W|^2 / C, so that objective is this one over C.  A two-class multinomial fit is the binary fit at 2C split
  symmetrically: the rows +-(w, b) / 2.
- `fold_bounds`, `logistic_cv`: KFold without shuffling, each fold fitted over the classes its training part has
  (multinomial whenever the factor has more than two classes), the fold accuracies summed in fold order, the first
  maximum, the refit and its predictions;
- `boosted_trees`: tests/dci_reference.py's GradientBoostingClassifier().
"""
import numpy as np

import beta_vae_reference as BR
import dci_reference as DR

CS = np.logspace(-4, 4, 10)
FOLDS = 5
MAX_NEWTON = 300


def fold_bounds(n):
    """[(start, end)] of KFold(5)'s contiguous folds of n rows, the first n % 5 one row longer."""
    q, r = divmod(n, FOLDS)
    out, s = [], 0
    for f in range(FOLDS):
        e = s + q + (1 if f < r else 0)
        out.append((s, e))
        s = e
    return out


def fit(x, y, p, multi, C):
    """(W [rows, D], b [rows], Newton steps) of the minimiser over p classes (labels 0 .. p-1): multinomial over p
    rows when `multi`, one binary row otherwise; no rows for p < 2."""
    x = np.asarray(x, np.float64)
    if p < 2:
        return np.zeros((0, x.shape[1])), np.zeros(0), 0
    if multi and p == 2:
        w, b, steps = fit(x, y, 2, False, 2.0 * C)
        return np.r_[-w, w] / 2.0, np.r_[-b, b] / 2.0, steps
    s = np.sqrt(C)
    V, b, steps = BR.fit(x * s, y, p, max_iter=MAX_NEWTON)
    return V * s, b, steps


def kkt(x, y, multi, C, W, b):
    """(gradient, scale) of C sum_i loss_i + 1/2 |W|^2 at (W, b): the KKT residual of a fit and the scale of its parts
    (|weight| + C sum_i |q_i x_i|)."""
    x = np.asarray(x, np.float64)
    xa = np.c_[x, np.ones(len(x))]
    z = xa @ np.c_[W, b].T
    y = np.asarray(y)
    if multi:
        e = np.exp(z - z.max(1, keepdims=True))
        q = e / e.sum(1, keepdims=True) - np.eye(len(b))[y]
    else:
        q = 1.0 / (1.0 + np.exp(-z)) - (y == 1)[:, None]
    reg = np.c_[W, np.zeros(len(b))]
    return reg + C * (q.T @ xa), np.abs(reg) + C * (np.abs(q).T @ np.abs(xa))


def predict(W, b, multi, classes, x):
    """(classes of the rows of x, gap of their deciding values): argmax over the model rows mapped through `classes`
    (the lowest on a tie), class 1 when w x + b > 0 for a binary model, classes[0] without a model."""
    n = len(x)
    if len(b) == 0:
        return np.full(n, classes[0], np.int64), np.full(n, np.inf)
    v = BR.decisions(W, b, x)
    if not multi:
        return (v[:, 0] > 0).astype(np.int64), np.abs(v[:, 0])
    top = np.sort(v, axis=1)
    return np.asarray(classes)[np.argmax(v, axis=1)], top[:, -1] - top[:, -2]


def fold_fit(x, cls, nc, f, C):
    """Fold f's fit at C on training features x [n, D] with classes cls [n] of nc -> (W, b, steps, classes present,
    multi), the model rows those of the present classes in order."""
    s0, s1 = fold_bounds(len(x))[f]
    keep = np.r_[0:s0, s1:len(x)]
    present = np.unique(cls[keep])
    place = np.full(max(nc, 1), -1)
    place[present] = np.arange(len(present))
    multi = nc > 2
    W, b, steps = fit(x[keep], place[cls[keep]], len(present), multi, C)
    return W, b, steps, present, multi


def logistic_cv(x_train, cls, nc, x_eval, Cs=CS):
    """LogisticRegressionCV(Cs, cv=KFold(5)) of one factor: x_train [n, D] fp64, cls [n] classes 0 .. nc-1 (every
    class present), x_eval [m, D] -> dict(fold_acc [5, nC], fold_pred [nC, n], fold_steps [5, nC], chosen, W, b,
    steps, pred [n + m], gap [n + m], fold_gap [nC, n])."""
    x_train, cls = np.asarray(x_train, np.float64), np.asarray(cls, np.int64)
    n = len(x_train)
    out = dict(fold_acc=np.zeros((FOLDS, len(Cs))), fold_pred=np.zeros((len(Cs), n), np.int64),
               fold_gap=np.zeros((len(Cs), n)), fold_steps=np.zeros((FOLDS, len(Cs)), np.int64))
    for f, (s0, s1) in enumerate(fold_bounds(n)):
        for c, C in enumerate(Cs):
            W, b, steps, present, multi = fold_fit(x_train, cls, nc, f, C)
            p, gap = predict(W, b, multi, present, x_train[s0:s1])
            out["fold_pred"][c, s0:s1], out["fold_gap"][c, s0:s1] = p, gap
            out["fold_acc"][f, c] = (p == cls[s0:s1]).sum() / (s1 - s0)
            out["fold_steps"][f, c] = steps
    total = out["fold_acc"][0]
    for f in range(1, FOLDS):
        total = total + out["fold_acc"][f]
    chosen = int(np.argmax(total))
    multi = nc > 2
    W, b, steps = fit(x_train, cls, nc, multi, Cs[chosen])
    pred, gap = predict(W, b, multi, np.arange(max(nc, 1)), np.r_[x_train, np.asarray(x_eval, np.float64)])
    out.update(chosen=chosen, W=W, b=b, steps=steps, pred=pred, gap=gap)
    return out


def boosted_trees(x_train, cls, nc, x_eval):
    """GradientBoostingClassifier()'s predictions [n + m] of one factor (tests/dci_reference.py's fit)."""
    f = DR.fit(x_train, cls, nc, x_eval)
    return np.r_[f["pred_train"], f["pred_test"]]


def labels(lat_sizes, train_rows, test_rows):
    """sap_labels' classes of the scored factors, in numpy -> (factors, train_cls [K', n], test_cls [K', m],
    n_classes [K'])."""
    values_tr = np.stack(np.unravel_index(np.asarray(train_rows), lat_sizes))
    values_te = np.stack(np.unravel_index(np.asarray(test_rows), lat_sizes))
    factors = [k for k, s in enumerate(lat_sizes) if s > 1]
    tr, te, ncl = [], [], []
    for k in factors:
        seen = np.unique(values_tr[k])
        place = np.full(lat_sizes[k], -1)
        place[seen] = np.arange(len(seen))
        tr.append(place[values_tr[k]])
        te.append(place[values_te[k]])
        ncl.append(len(seen))
    return factors, np.stack(tr), np.stack(te), np.array(ncl)


def accuracies(pred, train_cls, test_cls):
    """(train accuracies [K'], test accuracies [K']) of predictions [K', n + m]."""
    n = train_cls.shape[1]
    return (pred[:, :n] == train_cls).mean(1), (pred[:, n:] == test_cls).mean(1)


def score_keys(size, train_acc, test_acc):
    """downstream_task.py's entries for one training size."""
    s = str(size)
    out = {s + ":mean_train_accuracy": np.mean(train_acc), s + ":mean_test_accuracy": np.mean(test_acc),
           s + ":min_train_accuracy": np.min(train_acc), s + ":min_test_accuracy": np.min(test_acc)}
    for i in range(len(train_acc)):
        out[s + ":train_accuracy_factor_{}".format(i)] = train_acc[i]
        out[s + ":test_accuracy_factor_{}".format(i)] = test_acc[i]
    return out
