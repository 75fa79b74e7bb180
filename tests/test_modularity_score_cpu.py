"""Modularity and explicitness on the host (no GPU, no kernel): every refusal happens before any GPU work, the draws
and labels are SAP's, the fp64 restatement of tests/modularity_reference.py equals numpy's histogram bins, sklearn's
mutual_info_score, disentanglement_lib's modularity(), sklearn's roc_auc_score and LogisticRegression, and the host
path of `modularity_explicitness` (with the two kernels replaced by the restatement) equals a direct evaluation of the
definition and, where they agree by construction, disentanglement_lib's steps with sklearn at its defaults."""
import warnings

import numpy as np
import pytest
import torch

import modularity_reference as R
from disvae import evaluate
from score_stubs import _evaluator, _Grid, no_gpu  # noqa: F401

# (dataset, latent_dim, settings, message) of every refusal
REFUSALS = [
    (_Grid([4, 5], factors=False), 10, {}, "no lat_sizes / lat_names"),
    (_Grid([4, 5], n=21), 10, {}, "has 21 items, not the 20 of the full grid"),
    (_Grid([1, 1, 1]), 10, {}, "has 0 factors of more than one value"),
    (_Grid([1, 7, 1]), 10, {}, "has 1 factors of more than one value"),
    (_Grid([2, 257]), 10, {}, "more than the kernel's limit of 256 values"),
    (_Grid([4, 5]), 0, {}, r"latent_dim must be in \[1, 128\], got 0"),
    (_Grid([4, 5]), 129, {}, r"latent_dim must be in \[1, 128\], got 129"),
    (_Grid([4, 5]), 10, {"num_train": 0}, r"num_train must be in \[1, 32768\], got 0"),
    (_Grid([4, 5]), 10, {"num_train": 32769}, r"num_train must be in \[1, 32768\], got 32769"),
    (_Grid([4, 5]), 10, {"num_test": 0}, "num_test must be at least 1, got 0"),
]


@pytest.mark.parametrize("case", range(len(REFUSALS)))
def test_refusals_before_gpu_work(tmp_path, no_gpu, case):
    ds, latent_dim, settings, msg = REFUSALS[case]
    loader = torch.utils.data.DataLoader(ds, batch_size=10)
    with pytest.raises(ValueError, match=msg):
        _evaluator(tmp_path, latent_dim).compute_modularity_explicitness(loader, **settings)
    with pytest.raises(ValueError, match=msg):
        evaluate.check_modularity_explicitness(ds, latent_dim, **settings)
    if hasattr(ds, "lat_sizes"):
        with pytest.raises(ValueError, match=msg):
            evaluate.modularity_explicitness(torch.zeros(len(ds), latent_dim), ds.lat_sizes, **settings)
    assert not list(tmp_path.iterdir())


# ---- the host path with the fp64 restatement standing in for the kernels -------------------------------------------
class _Host:
    """Stands in for `discrete_mutual_info` and `explicitness_fit` on the host: records their inputs, computes with
    tests/modularity_reference.py."""

    def __init__(self):
        self.calls = []

    def mutual_info(self, mu, train_rows, train_cls, n_classes, class_stride):
        self.calls.append(("mi", [t.clone() for t in (train_rows, train_cls, n_classes)], class_stride))
        mi, edges = R.mutual_information(mu.numpy()[train_rows.numpy()], train_cls.numpy())
        return torch.from_numpy(mi), torch.from_numpy(edges)

    def explicitness(self, mu, train_rows, test_rows, train_cls, test_cls, n_classes, class_stride, proba=False):
        self.calls.append(("fit", [t.clone() for t in (train_rows, test_rows, train_cls, test_cls, n_classes)],
                           class_stride))
        x = mu.numpy()
        ft, fe, mean, std = R.standardise(x[train_rows.numpy()], x[test_rows.numpy()])
        K, S, D = len(n_classes), class_stride, x.shape[1]
        coef = np.full((K, S, D + 1), np.nan)
        auc = np.full((2, K, S), np.nan)
        iters = np.zeros(K, np.int32)
        for k in range(K):
            nc = int(n_classes[k])
            W, b, steps, at, ae, _, _ = R.explicitness(ft, train_cls[k].numpy(), fe, test_cls[k].numpy(), nc)
            coef[k, :len(b)] = np.c_[W, b]
            auc[0, k, :len(at)], auc[1, k, :len(ae)] = at, ae
            iters[k] = steps
        return (torch.from_numpy(coef), torch.from_numpy(auc), torch.from_numpy(iters), torch.from_numpy(mean),
                torch.from_numpy(std), None)


@pytest.fixture
def host(monkeypatch):
    h = _Host()
    monkeypatch.setattr(evaluate, "discrete_mutual_info", h.mutual_info)
    monkeypatch.setattr(evaluate, "explicitness_fit", h.explicitness)
    monkeypatch.setattr(evaluate.N, "require_cuda_f32", lambda *t: None)
    return h


def test_draws_and_labels_are_saps(host, monkeypatch):
    lat_sizes, seed = [3, 1, 40, 2, 5], 31
    n = int(np.prod(lat_sizes))
    mu = torch.randn(n, 4, generator=torch.Generator().manual_seed(1))
    evaluate.modularity_explicitness(mu, lat_sizes, num_train=300, num_test=200, seed=seed)
    sap_calls = []

    def sap_matrix(mu, *args, **kw):
        sap_calls.append([t.clone() for t in args[:6]])
        args[8].zero_()
        return torch.zeros(mu.shape[1], args[5].shape[0])
    monkeypatch.setattr(evaluate, "sap_score_matrix", sap_matrix)
    evaluate.sap_score(mu, lat_sizes, num_train=300, num_test=200, seed=seed)
    s_train, s_test, s_train_cls, s_test_cls, s_n_classes, s_counts = sap_calls[0]
    (_, (tr, cls, ncl), S1), (_, (tr2, te, cls2, te_cls, ncl2), S2) = host.calls
    assert S1 == S2 == s_counts.shape[1]
    for a, b in ((tr, s_train), (tr2, s_train), (te, s_test), (cls, s_train_cls), (cls2, s_train_cls),
                 (te_cls, s_test_cls), (ncl, s_n_classes), (ncl2, s_n_classes)):
        assert torch.equal(a, b)
    g = torch.Generator().manual_seed(seed)
    assert torch.equal(tr, torch.randint(n, (300,), generator=g))
    assert torch.equal(te, torch.randint(n, (200,), generator=g))


def _restated(mu, lat_sizes, num_train, num_test, seed):
    """The definition, evaluated directly on the factor values: the draws, the bins, mutual_info_score, modularity(),
    one fit per factor and the AUCs of its class columns."""
    n, D = mu.shape
    g = torch.Generator().manual_seed(seed)
    tr = torch.randint(n, (num_train,), generator=g).numpy()
    te = torch.randint(n, (num_test,), generator=g).numpy()
    vt, ve = np.unravel_index(tr, lat_sizes), np.unravel_index(te, lat_sizes)
    x = mu.numpy()
    mi, _ = R.mutual_information(x[tr], np.stack([vt[k] for k, s in enumerate(lat_sizes) if s > 1]))
    ft, fe, _, _ = R.standardise(x[tr], x[te])
    et, ee = [], []
    for k, s in enumerate(lat_sizes):
        if s == 1:
            continue
        classes = np.unique(vt[k])
        yt = np.searchsorted(classes, vt[k])
        ye = np.where(np.isin(ve[k], classes), np.searchsorted(classes, ve[k]), -1)
        _, _, _, at, ae, _, _ = R.explicitness(ft, yt, fe, ye, len(classes))
        et.append(R.mean_defined(at))
        ee.append(R.mean_defined(ae))
    return {"modularity_score": R.modularity(mi)[0], "explicitness_score_train": R.mean_defined(et),
            "explicitness_score_test": R.mean_defined(ee)}, mi, et, ee


def test_host_path_equals_the_definition(host):
    """Factors of 4, 1, 2 and 6 values with test values unseen in training; aligned, noise, constant and duplicated
    latents."""
    lat_sizes = [4, 1, 2, 6]
    n = int(np.prod(lat_sizes))
    values = np.stack(np.unravel_index(np.arange(n), lat_sizes), 1).astype(np.float64)
    rng = np.random.default_rng(0)
    mu = np.stack([values[:, 3] + 0.3 * rng.standard_normal(n), values[:, 2] + 0.2 * rng.standard_normal(n),
                   rng.standard_normal(n), np.full(n, 0.5), values[:, 0], values[:, 0]], 1)
    mu = torch.from_numpy(mu).float()
    score, helpers = evaluate.modularity_explicitness(mu, lat_sizes, num_train=30, num_test=300, seed=5)
    want, mi, et, ee = _restated(mu, lat_sizes, 30, 300, 5)
    assert np.array_equal(helpers["mutual_information"].numpy(), mi)
    assert score.keys() == want.keys()
    for key in want:
        assert score[key] == pytest.approx(want[key], rel=1e-12, abs=1e-12), key
    assert np.allclose(helpers["explicitness_train"].numpy(), et, rtol=1e-12, atol=1e-12, equal_nan=True)
    assert np.allclose(helpers["explicitness_test"].numpy(), ee, rtol=1e-12, atol=1e-12, equal_nan=True)
    assert helpers["factors"].tolist() == [0, 2, 3]
    assert helpers["feature_std"][3] == 1.0                      # the constant latent
    assert helpers["modularity_per_latent"][3] == 0.0            # it has no mutual information
    assert set(helpers) == {"mutual_information", "bin_edges", "modularity_per_latent", "factors", "classes",
                            "feature_mean", "feature_std", "coef", "train_auc", "test_auc", "explicitness_train",
                            "explicitness_test", "solver_iterations"}


def test_one_class_factor_and_no_value(host):
    """A factor seen with one value in training has no fit and no explicitness; when no factor has a value the scores
    are NaN with a RuntimeWarning."""
    lat_sizes, n = [2, 3], 6
    mu = torch.randn(n, 3, generator=torch.Generator().manual_seed(2))
    seed = next(s for s in range(200) if len(set(np.unravel_index(
        torch.randint(n, (2,), generator=torch.Generator().manual_seed(s)).numpy(), lat_sizes)[0])) == 1)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        score, helpers = evaluate.modularity_explicitness(mu, lat_sizes, num_train=2, num_test=50, seed=seed)
    assert torch.isnan(helpers["explicitness_train"][0]) and torch.isnan(helpers["train_auc"][0]).all()
    assert int(helpers["solver_iterations"][0]) == 0
    seed = next(s for s in range(200) if (lambda v: len(set(v[0])) == 1 and len(set(v[1])) == 1)(np.unravel_index(
        torch.randint(n, (1,), generator=torch.Generator().manual_seed(s)).numpy(), lat_sizes)))
    with pytest.warns(RuntimeWarning, match="no factor has an explicitness value"):
        score, _ = evaluate.modularity_explicitness(mu, lat_sizes, num_train=1, num_test=50, seed=seed)
    assert np.isnan(score["explicitness_score_train"]) and np.isnan(score["explicitness_score_test"])


# ---- the restatement against numpy and sklearn ---------------------------------------------------------------------
def _columns():
    rng = np.random.default_rng(7)
    cols = []
    for i in range(400):
        n = int(rng.integers(1, 300))
        scale = 10.0 ** rng.integers(-6, 7)
        cols.append((rng.standard_normal(n) * scale + rng.standard_normal() * scale * rng.integers(0, 50))
                    .astype(np.float32))
    cols.append(np.full(17, 3.25, np.float32))                              # constant
    cols.append(np.full(5, -0.0, np.float32))
    cols.append(np.r_[np.float32(1e-30), np.float32(1e6), rng.standard_normal(40).astype(np.float32)])   # magnitudes
    e = R.edges(np.r_[np.float32(0), np.float32(1)])
    cols.append(np.r_[e, e, np.float32(0.5)])                               # every value on an edge
    cols.append(np.r_[np.float32(-7.5), np.float32(12.0), R.edges(np.array([-7.5, 12.0], np.float32))[3:9]])
    return cols


def test_bins_equal_numpys_histogram():
    for x in _columns():
        e = np.histogram(x, R.BINS)[1]
        assert e.dtype == np.float32
        assert np.array_equal(R.edges(x), e)
        assert np.array_equal(R.bins(x, R.edges(x)), np.digitize(x, e[:-1]))


def test_numpy_refused_ranges_are_binned_with_the_same_edges():
    """Columns spanning a few ulps: numpy refuses them ("Too many bins for data range"); the rule still gives 21
    edges, not strictly increasing, and each value's bin is the count of the first 20 at or below it."""
    for base in (np.float32(1.0), np.float32(-3.0e5), np.float32(7.0e-20)):
        x = (base + np.arange(4, dtype=np.float32) * np.spacing(base)).astype(np.float32)
        with pytest.raises(ValueError, match="Too many bins"):
            np.histogram(x, 20)
        e = R.edges(x)
        assert e[0] == x.min() and e[-1] == x.max() and (np.diff(e) <= 0).any()
        b = R.bins(x, e)
        assert np.array_equal(b, [(e[:20] <= v).sum() for v in x]) and b.min() >= 1 and b.max() <= 20


@pytest.mark.parametrize("nc, nb, n", [(2, 20, 1000), (5, 3, 40), (40, 20, 10000), (256, 20, 5000), (3, 1, 50),
                                       (1, 20, 50), (7, 20, 7)])
def test_mutual_info_equals_sklearn(nc, nb, n):
    metrics = pytest.importorskip("sklearn.metrics")
    rng = np.random.default_rng(nc * 1000 + nb)
    c = rng.integers(0, nc, n)
    b = np.where(rng.random(n) < 0.5, c % nb, rng.integers(0, nb, n))       # some dependence
    assert R.mutual_info(c, b) == pytest.approx(metrics.mutual_info_score(c, b), rel=1e-12, abs=1e-12)


def _modularity_line_by_line(mutual_information):
    """modularity_explicitness.py's modularity(), as written there."""
    squared_mi = np.square(mutual_information)
    max_squared_mi = np.max(squared_mi, axis=1)
    numerator = np.sum(squared_mi, axis=1) - max_squared_mi
    denominator = max_squared_mi * (squared_mi.shape[1] - 1.)
    with np.errstate(divide="ignore", invalid="ignore"):
        delta = numerator / denominator
    modularity_score = 1. - delta
    index = (max_squared_mi == 0.)
    modularity_score[index] = 0.
    return np.mean(modularity_score)


@pytest.mark.parametrize("case", ["random", "zero_rows", "one_hot", "two_factors", "all_zero"])
def test_modularity_equals_disentanglement_lib(case):
    rng = np.random.default_rng(11)
    m = {"random": rng.random((10, 5)), "zero_rows": rng.random((6, 3)) * (np.arange(6) % 2)[:, None],
         "one_hot": np.eye(5)[[0, 1, 2, 2, 4, 3]] * 0.7, "two_factors": rng.random((128, 2)),
         "all_zero": np.zeros((4, 3))}[case]
    got, per = evaluate.modularity_from_mutual_info(torch.from_numpy(m))
    want = _modularity_line_by_line(m)
    assert got == pytest.approx(want, rel=1e-14, abs=1e-15)
    assert np.allclose(per.numpy(), R.modularity(m)[1], rtol=1e-14, atol=1e-15)
    assert (per.numpy()[np.square(m).max(1) == 0] == 0).all()


@pytest.mark.parametrize("nc, ties", [(2, False), (2, True), (3, False), (5, True), (40, False)])
def test_auc_equals_roc_auc_score(nc, ties):
    metrics = pytest.importorskip("sklearn.metrics")
    preprocessing = pytest.importorskip("sklearn.preprocessing")
    rng = np.random.default_rng(nc + 10 * ties)
    n = 2000
    y = rng.integers(0, nc, n)
    y[:nc] = np.arange(nc)
    z = rng.standard_normal((n, nc)) + 1.5 * np.eye(nc)[y]
    if ties:
        z = np.round(z * 2) / 2                                  # many equal probabilities
    if nc == 2:
        p1 = 1.0 / (1.0 + np.exp(-(z[:, 1] - z[:, 0])))
        p = np.stack([1.0 - p1, p1], 1)
    else:
        e = np.exp(z - z.max(1, keepdims=True))
        p = e / e.sum(1, keepdims=True)
    want = metrics.roc_auc_score(preprocessing.MultiLabelBinarizer().fit_transform(y[:, None]), p)
    got = np.mean([R.auc(p[:, c], y, c) for c in range(R.columns(nc))])
    assert got == pytest.approx(want, rel=1e-12, abs=1e-12)
    if ties:
        assert len(np.unique(p[:, 0])) < 0.6 * n                 # ties across rows


@pytest.mark.parametrize("nc, D, n", [(2, 3, 500), (3, 4, 800), (6, 10, 2000), (40, 10, 3000)])
def test_fit_equals_sklearn(nc, D, n):
    linear_model = pytest.importorskip("sklearn.linear_model")
    rng = np.random.default_rng(nc + D)
    y = rng.integers(0, nc, n)
    y[:nc] = np.arange(nc)
    x = rng.standard_normal((n, D)) + 0.8 * rng.standard_normal((nc, D))[y]
    ft, _, _, _ = R.standardise(x.astype(np.float32), x[:1].astype(np.float32))
    W, b, steps = R.BR.fit(ft, y, nc)
    assert steps >= 0
    clf = linear_model.LogisticRegression(solver="newton-cholesky", tol=1e-12, max_iter=1000).fit(ft, y)
    assert np.abs(clf.coef_ - W).max() <= 1e-6 * max(1.0, np.abs(W).max())
    b_sk = clf.intercept_ - (clf.intercept_.mean() if nc > 2 else 0.0)   # sklearn's intercepts up to a common shift
    assert np.abs(b_sk - b).max() <= 1e-6 * max(1.0, np.abs(b).max())
    p = R.probabilities(W, b, nc, ft)
    assert np.abs(clf.predict_proba(ft) - p).max() <= 1e-6


def test_whole_score_against_disentanglement_libs_steps(host):
    """disentanglement_lib's compute_modularity_explicitness steps with sklearn at its defaults (lbfgs, its float32
    normalisation) on the same draws, against the host path: modularity equal to 1e-12 (the same bins and mutual
    information), explicitness within 1e-4 (lbfgs stops at its tolerance; the restatement is the exact minimiser)."""
    pytest.importorskip("sklearn")
    from sklearn import linear_model, metrics, preprocessing
    lat_sizes = [3, 6, 8, 8]
    n = int(np.prod(lat_sizes))
    values = np.stack(np.unravel_index(np.arange(n), lat_sizes), 1).astype(np.float64)
    rng = np.random.default_rng(3)
    mu = values[:, [0, 1, 2, 3, 2]] / np.array(lat_sizes)[[0, 1, 2, 3, 2]] + 0.15 * rng.standard_normal((n, 5))
    mu = torch.from_numpy(mu).float()
    score, helpers = evaluate.modularity_explicitness(mu, lat_sizes, num_train=2000, num_test=1000, seed=9)
    g = torch.Generator().manual_seed(9)
    tr, te = torch.randint(n, (2000,), generator=g).numpy(), torch.randint(n, (1000,), generator=g).numpy()
    mus_train, mus_test = mu.numpy()[tr].T, mu.numpy()[te].T                # [D, n] as disentanglement_lib holds them
    ys_train, ys_test = values[tr].T.astype(np.int64), values[te].T.astype(np.int64)
    discretized = np.zeros_like(mus_train, dtype=np.int64)
    for i in range(mus_train.shape[0]):
        discretized[i] = np.digitize(mus_train[i], np.histogram(mus_train[i], 20)[1][:-1])
    mi = np.array([[metrics.mutual_info_score(ys_train[j], discretized[i]) for j in range(4)] for i in range(5)])
    mean, std = mus_train.mean(1), mus_train.std(1)
    xt, xe = ((mus_train - mean[:, None]) / std[:, None]).T, ((mus_test - mean[:, None]) / std[:, None]).T
    et, ee = [], []
    for j in range(4):
        clf = linear_model.LogisticRegression().fit(xt, ys_train[j])
        mlb = preprocessing.MultiLabelBinarizer()
        et.append(metrics.roc_auc_score(mlb.fit_transform(ys_train[j][:, None]), clf.predict_proba(xt)))
        ee.append(metrics.roc_auc_score(mlb.fit_transform(ys_test[j][:, None]), clf.predict_proba(xe)))
    assert np.abs(helpers["mutual_information"].numpy() - mi).max() <= 1e-12
    assert score["modularity_score"] == pytest.approx(_modularity_line_by_line(mi), rel=1e-12, abs=1e-12)
    d_train = abs(score["explicitness_score_train"] - np.mean(et))
    d_test = abs(score["explicitness_score_test"] - np.mean(ee))
    print("explicitness against disentanglement_lib's steps: |train diff| %.2e, |test diff| %.2e" % (d_train, d_test))
    assert d_train <= 1e-4 and d_test <= 1e-4
