"""The DCI score on the host (no GPU, no kernel): every refusal happens before any GPU work, the draws and labels are
SAP's, the fp64 restatement of the boosted fit in tests/dci_reference.py equals sklearn's GradientBoostingClassifier()
where no split is tied, `dci_from_importance` equals disentanglement_lib's dci.py, and the host path of `dci_score`
(with `dci_fit` replaced by the restatement) equals a direct evaluation of the definition."""
import numpy as np
import pytest
import torch

import dci_reference as R
from disvae import evaluate
from score_stubs import _evaluator, _Grid, no_gpu  # noqa: F401

# (dataset, latent_dim, settings, message) of every refusal
REFUSALS = [
    (_Grid([4, 5], factors=False), 10, {}, "no lat_sizes / lat_names"),
    (_Grid([4, 5], n=21), 10, {}, "has 21 items, not the 20 of the full grid"),
    (_Grid([1, 1, 1]), 10, {}, "has 0 factors of more than one value"),
    (_Grid([1, 7, 1]), 10, {}, "has 1 factors of more than one value"),
    (_Grid([2, 257]), 10, {}, "more than the kernel's limit of 256 values"),
    (_Grid([4, 5]), 1, {}, "latent_dim must be at least 2 .*, got 1"),
    (_Grid([4, 5]), 1025, {}, "latent_dim 1025 is above the kernel's limit of 1024"),
    (_Grid([4, 5]), 10, {"num_train": 0}, "num_train must be at least 1, got 0"),
    (_Grid([4, 5]), 10, {"num_train": 32769}, "num_train 32769 is above the kernel's limit of 32768"),
    (_Grid([4, 5]), 10, {"num_test": 0}, "num_test must be at least 1, got 0"),
]


@pytest.mark.parametrize("case", range(len(REFUSALS)))
def test_refusals_before_gpu_work(tmp_path, no_gpu, case):
    ds, latent_dim, settings, msg = REFUSALS[case]
    loader = torch.utils.data.DataLoader(ds, batch_size=10)
    with pytest.raises(ValueError, match=msg):
        _evaluator(tmp_path, latent_dim).compute_dci_score(loader, **settings)
    with pytest.raises(ValueError, match=msg):
        evaluate.check_dci_score(ds, latent_dim, **settings)
    if hasattr(ds, "lat_sizes"):
        with pytest.raises(ValueError, match=msg):
            evaluate.dci_score(torch.zeros(len(ds), latent_dim), ds.lat_sizes, **settings)
    assert not list(tmp_path.iterdir())


# ---- the host path with the fp64 restatement standing in for the kernel --------------------------------------------
class _Fp64Fit:
    """Stands in for `dci_fit` on the host: records its inputs, computes with tests/dci_reference.py."""

    def __init__(self):
        self.calls = []

    def __call__(self, mu, train_rows, test_rows, train_cls, n_classes, counts, stages=evaluate.DCI_STAGES,
                 trees=False):
        args = [t.clone() for t in (train_rows, test_rows, train_cls, n_classes, counts)]
        self.calls.append(args + [stages])
        importance, pred, fits = R.fit_factors(mu.numpy(), train_rows.numpy(), test_rows.numpy(), train_cls.numpy(),
                                               None, n_classes.numpy(), stages)
        for k, f in enumerate(fits):                            # sap_labels' counts are the fit's class counts
            nc = int(n_classes[k])
            assert np.array_equal(np.bincount(train_cls[k].numpy(), minlength=nc), counts[k, :nc].numpy())
        return torch.from_numpy(importance), torch.from_numpy(pred).int(), None


@pytest.fixture
def host_fit(monkeypatch):
    f = _Fp64Fit()
    monkeypatch.setattr(evaluate, "dci_fit", f)
    monkeypatch.setattr(evaluate.N, "require_cuda_f32", lambda *t: None)
    return f


def test_draws_and_labels_are_saps(host_fit, monkeypatch):
    lat_sizes, seed = [3, 1, 40, 2, 5], 31
    n = int(np.prod(lat_sizes))
    mu = torch.randn(n, 4, generator=torch.Generator().manual_seed(1))
    evaluate.dci_score(mu, lat_sizes, num_train=60, num_test=200, seed=seed)
    sap_calls = []

    def sap_matrix(mu, *args, **kw):
        sap_calls.append([t.clone() for t in args[:6]])
        args[8].zero_()                                         # every fit converged
        return torch.zeros(mu.shape[1], args[5].shape[0])
    monkeypatch.setattr(evaluate, "sap_score_matrix", sap_matrix)
    evaluate.sap_score(mu, lat_sizes, num_train=60, num_test=200, seed=seed)
    train_rows, test_rows, train_cls, n_classes, counts, stages = host_fit.calls[0]
    s_train, s_test, s_train_cls, _, s_n_classes, s_counts = sap_calls[0]
    assert stages == 100 and len(host_fit.calls) == 1
    for a, b in ((train_rows, s_train), (test_rows, s_test), (train_cls, s_train_cls), (n_classes, s_n_classes),
                 (counts, s_counts)):
        assert torch.equal(a, b)
    g = torch.Generator().manual_seed(seed)
    assert torch.equal(train_rows, torch.randint(n, (60,), generator=g))
    assert torch.equal(test_rows, torch.randint(n, (200,), generator=g))


def _restated(mu, lat_sizes, num_train, num_test, seed):
    """The definition, evaluated directly: the draws, each scored factor's values as classes, one fit per factor,
    accuracies against the factor values and dci.py's formulas."""
    n, D = mu.shape
    g = torch.Generator().manual_seed(seed)
    tr = torch.randint(n, (num_train,), generator=g).numpy()
    te = torch.randint(n, (num_test,), generator=g).numpy()
    vt, ve = np.unravel_index(tr, lat_sizes), np.unravel_index(te, lat_sizes)
    x = mu.numpy()
    cols, train_acc, test_acc = [], [], []
    for k, s in enumerate(lat_sizes):
        if s == 1:
            continue
        classes = np.unique(vt[k])
        f = R.fit(x[tr], np.searchsorted(classes, vt[k]), len(classes), x[te])
        cols.append(f["importance"])
        train_acc.append(np.mean(classes[f["pred_train"]] == vt[k]))
        test_acc.append(np.mean(classes[f["pred_test"]] == ve[k]))
    importance = np.stack(cols, 1)
    dis, com = R.dci_restated(importance)
    return importance, {"disentanglement": dis, "completeness": com, "informativeness_train": np.mean(train_acc),
                        "informativeness_test": np.mean(test_acc)}, train_acc, test_acc


def test_host_path_equals_the_definition(host_fit):
    """Factors of 4, 1, 2 and 6 values, with test values unseen in training; aligned, noise and constant latents."""
    lat_sizes = [4, 1, 2, 6]
    n = int(np.prod(lat_sizes))
    values = np.stack(np.unravel_index(np.arange(n), lat_sizes), 1).astype(np.float64)
    rng = np.random.default_rng(0)
    mu = np.stack([values[:, 3] + 0.3 * rng.standard_normal(n), values[:, 2] + 0.2 * rng.standard_normal(n),
                   rng.standard_normal(n), np.full(n, 0.5), values[:, 0]], 1)
    mu = torch.from_numpy(mu).float()
    score, helpers = evaluate.dci_score(mu, lat_sizes, num_train=30, num_test=300, seed=5)
    importance, want, train_acc, test_acc = _restated(mu, lat_sizes, 30, 300, 5)
    assert np.array_equal(helpers["importance_matrix"].numpy(), importance)
    assert score.keys() == want.keys()
    for key in want:
        assert score[key] == pytest.approx(want[key], rel=1e-12, abs=1e-12), key
    assert np.array_equal(helpers["train_accuracy"].numpy(), train_acc)
    assert np.array_equal(helpers["test_accuracy"].numpy(), test_acc)
    assert helpers["factors"].tolist() == [0, 2, 3]
    assert (np.asarray(test_acc) < 1).any()                       # 30 training rows miss some of the 24 cells
    tr = torch.randint(n, (30,), generator=torch.Generator().manual_seed(5)).numpy()
    for j, k in enumerate([0, 2, 3]):
        seen = np.unique(np.unravel_index(tr, lat_sizes)[k])
        assert helpers["classes"][j, :len(seen)].tolist() == seen.tolist()
        assert (helpers["classes"][j, len(seen):] == -1).all()


def test_one_value_factor_has_no_trees(host_fit):
    """A factor seen with one value in training: zero importance, every row predicted as that value."""
    lat_sizes, num_train = [2, 3], 2
    n = 6
    seed = next(s for s in range(100) if len(set(np.unravel_index(
        torch.randint(n, (num_train,), generator=torch.Generator().manual_seed(s)).numpy(), lat_sizes)[0])) == 1)
    mu = torch.randn(n, 3, generator=torch.Generator().manual_seed(2))
    score, helpers = evaluate.dci_score(mu, lat_sizes, num_train=num_train, num_test=50, seed=seed)
    assert (helpers["importance_matrix"][:, 0] == 0).all()
    assert helpers["train_accuracy"][0] == 1.0
    _, want, _, _ = _restated(mu, lat_sizes, num_train, 50, seed)
    assert score == pytest.approx(want, rel=1e-12, abs=1e-12)


# ---- dci.py's formulas ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["random", "diagonal", "one_hot_rows", "zeros", "sparse", "tall", "wide"])
def test_dci_from_importance_equals_dci_py(case):
    pytest.importorskip("scipy")
    rng = np.random.default_rng(3)
    m = {"random": rng.random((10, 5)), "diagonal": np.eye(6), "one_hot_rows": np.eye(4)[[0, 1, 1, 3, 2, 0]],
         "zeros": np.zeros((10, 5)), "sparse": rng.random((8, 3)) * (rng.random((8, 3)) < 0.3),
         "tall": rng.random((1024, 2)), "wide": rng.random((2, 40))}[case]
    got = evaluate.dci_from_importance(torch.from_numpy(m))
    want = R.dci_restated(m)
    assert got == pytest.approx(want, rel=1e-12, abs=1e-14)


# ---- the restated fit is GradientBoostingClassifier()'s -----------------------------------------------------------
def _grid_fixture(nc, n, D, levels, seed):
    """Latents on a grid of `levels` values each, classes drawn from a softmax of the grid cell: every node of a tree
    is a box of non-empty cells, so no two latents split one the same way and no split is tied."""
    rng = np.random.default_rng(seed)
    lv = np.sort(rng.standard_normal((D, levels)), 1).astype(np.float32)
    cell = rng.integers(0, levels, (n, D))
    w = rng.standard_normal((D, nc))
    logits = 1.5 * (cell - levels / 2) @ w / np.sqrt(D)
    p = np.exp(logits - logits.max(1, keepdims=True))
    p /= p.sum(1, keepdims=True)
    y = (p.cumsum(1) < rng.random((n, 1))).sum(1)
    return lv[np.arange(D), cell], np.minimum(y, nc - 1)


@pytest.mark.parametrize("nc, n, D, levels, stages", [(2, 3000, 4, 5, 100), (3, 3000, 5, 4, 100),
                                                      (40, 3000, 3, 6, 20)])
def test_restatement_equals_sklearn(nc, n, D, levels, stages):
    ensemble = pytest.importorskip("sklearn.ensemble")
    x, y = _grid_fixture(nc, n, D, levels, nc)
    classes = np.unique(y)
    y = np.searchsorted(classes, y)
    x_test, _ = _grid_fixture(nc, 700, D, levels, nc + 100)
    f = R.fit(x, y, len(classes), x_test, stages)
    clf = ensemble.GradientBoostingClassifier(random_state=0, n_estimators=stages).fit(x, y)
    assert np.array_equal(clf.predict(x), f["pred_train"])
    assert np.array_equal(clf.predict(x_test), f["pred_test"])
    assert np.abs(clf.feature_importances_ - f["importance"]).max() <= 1e-9
    assert len(classes) >= min(nc, 30)
    for s in (0, stages - 1):                                    # the trees themselves: first and last stage
        for c in range(clf.estimators_.shape[1]):
            _same_tree(clf.estimators_[s, c].tree_, f["feature"][c, s], f["threshold"][c, s], f["value"][c, s])


def _same_tree(tree, feature, threshold, value, i=0, h=0):
    """sklearn's tree node i against heap node h of the restatement's.  sklearn takes a child's impurity as the
    parent's minus the other child's sums, so a node whose residuals are all equal can carry an impurity of a few
    DBL_EPSILON and be split; the restatement computes it from the node's rows (about 0) and stops.  Such a node's
    subtree only splits equal residuals and predicts the same values."""
    if tree.children_left[i] < 0 or (feature[h] == R.LEAF and tree.impurity[i] < 1e-12):
        assert feature[h] == R.LEAF
        leaves = [j for j in range(tree.node_count) if tree.children_left[j] < 0 and _under(tree, i, j)]
        for j in leaves:
            assert value[h] == pytest.approx(tree.value[j].ravel()[0], rel=1e-9, abs=1e-12)
        return
    assert feature[h] == tree.feature[i] and threshold[h] == tree.threshold[i]
    _same_tree(tree, feature, threshold, value, tree.children_left[i], 2 * h + 1)
    _same_tree(tree, feature, threshold, value, tree.children_right[i], 2 * h + 2)


def _under(tree, i, j):
    """Whether sklearn's node j is node i or below it."""
    stack = [i]
    while stack:
        k = stack.pop()
        if k == j:
            return True
        if tree.children_left[k] >= 0:
            stack += [tree.children_left[k], tree.children_right[k]]
    return False


def test_factors_with_unseen_test_values_equal_sklearn():
    """fit_factors on SAP's labels against one GradientBoostingClassifier() per factor on the factor values: the
    same accuracies, with test values that no training row has counted wrong."""
    ensemble = pytest.importorskip("sklearn.ensemble")
    lat_sizes = [2, 5, 3]
    n = int(np.prod(lat_sizes))
    values = np.stack(np.unravel_index(np.arange(n), lat_sizes), 1)
    mu = (values[:, [2, 0, 1]] * np.array([1.0, 0.7, 0.4]) + np.arange(3)).astype(np.float32)
    g = torch.Generator().manual_seed(4)
    tr, te = torch.randint(n, (12,), generator=g), torch.randint(n, (400,), generator=g)
    # each latent follows one factor, so a node is a box of grid cells and no two latents split one the same way
    factors, train_cls, test_cls, n_classes, counts, _ = evaluate.sap_labels(lat_sizes, tr, te)
    importance, pred, _ = R.fit_factors(mu, tr.numpy(), te.numpy(), train_cls.numpy(), None, n_classes.numpy(), 100)
    unseen = 0
    for j, k in enumerate(factors):
        vt, ve = values[tr.numpy(), k], values[te.numpy(), k]
        clf = ensemble.GradientBoostingClassifier(random_state=0).fit(mu[tr.numpy()], vt)
        right = pred[j] == np.concatenate([train_cls[j].numpy(), test_cls[j].numpy()])
        assert right[:12].mean() == np.mean(clf.predict(mu[tr.numpy()]) == vt)
        assert right[12:].mean() == np.mean(clf.predict(mu[te.numpy()]) == ve)
        assert np.abs(importance[:, j] - clf.feature_importances_).max() <= 1e-9
        unseen += int((~np.isin(ve, vt)).sum())
    assert unseen > 0
