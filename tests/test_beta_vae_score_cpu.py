"""The beta-VAE score on the host (no GPU, no kernel): every refusal happens before any GPU work, the documented draw
order reproduces the rows, the host path of `beta_vae_score` (with `pair_abs_diff_mean` and `logistic_fit` replaced
by the fp64 numpy stand-ins of tests/beta_vae_reference.py) equals a line-by-line restatement of the definition, and
the stand-in's fit equals sklearn's LogisticRegression(C=1), which pins the objective to disentanglement_lib's
classifier."""
import numpy as np
import pytest
import torch

import beta_vae_reference as R
from disvae import evaluate
from score_stubs import _evaluator, _Grid, no_gpu  # noqa: F401


# (dataset, latent_dim, settings, message) of every refusal
REFUSALS = [
    (_Grid([4, 5], factors=False), 10, {}, "no lat_sizes / lat_names"),
    (_Grid([4, 5], n=21), 10, {}, "has 21 items, not the 20 of the full grid"),
    (_Grid([1, 1, 1]), 10, {}, "has 0 factors of more than one value; the score needs at least 2"),
    (_Grid([1, 7, 1]), 10, {}, "has 1 factors of more than one value; the score needs at least 2"),
    (_Grid([2] * 33), 10, {}, "has 33 factors of more than one value, above the kernel's limit of 32"),
    (_Grid([4, 5]), 129, {}, "latent_dim 129 is above the kernel's limit of 128"),
    (_Grid([4, 5]), 10, {"batch_size": 0}, "batch_size must be at least 1, got 0"),
    (_Grid([4, 5]), 10, {"num_train": 0}, "num_train must be at least 1, got 0"),
    (_Grid([4, 5]), 10, {"num_eval": 0}, "num_eval must be at least 1, got 0"),
]


@pytest.mark.parametrize("case", range(len(REFUSALS)))
def test_evaluator_refusals_before_gpu_work(tmp_path, no_gpu, case):
    ds, latent_dim, settings, msg = REFUSALS[case]
    loader = torch.utils.data.DataLoader(ds, batch_size=10)
    with pytest.raises(ValueError, match=msg):
        _evaluator(tmp_path, latent_dim).compute_beta_vae_score(loader, **settings)
    if not settings:
        for is_metrics in (False, True):
            with pytest.raises(ValueError, match=msg):
                _evaluator(tmp_path, latent_dim)(loader, is_metrics=is_metrics, is_beta_vae_score=True)
    assert not list(tmp_path.iterdir())


@pytest.mark.parametrize("case", range(len(REFUSALS)))
def test_score_function_refusals_before_gpu_work(no_gpu, case):
    ds, latent_dim, settings, msg = REFUSALS[case]
    if not hasattr(ds, "lat_sizes"):
        return
    with pytest.raises(ValueError, match=msg):
        evaluate.check_beta_vae_score(ds, latent_dim, **settings)
    if len(ds) <= 10 ** 6:                          # not the 2^33-item grid
        with pytest.raises(ValueError, match=msg):
            evaluate.beta_vae_score(torch.zeros(len(ds), latent_dim), ds.lat_sizes, **settings)


# ---- the draw order -----------------------------------------------------------------------------------------------
def _hand_points(lat_sizes, count, L, g):
    """The draw order of INTEGRATION.md, restated with numpy's grid indexing: (label, rows_a, rows_b)."""
    scored = [k for k, s in enumerate(lat_sizes) if s > 1]
    label = torch.randint(len(scored), (count,), generator=g).numpy()
    a_vals, b_vals = [], []
    for k, s in enumerate(lat_sizes):
        a = torch.randint(s, (count, L), generator=g).numpy()
        b = torch.randint(s, (count, L), generator=g).numpy()
        on_k = np.array([scored[j] == k for j in label])
        b = np.where(on_k[:, None], a, b)
        a_vals.append(a)
        b_vals.append(b)
    return label, np.ravel_multi_index(a_vals, lat_sizes), np.ravel_multi_index(b_vals, lat_sizes)


def _hand_draws(lat_sizes, seed, num_train, num_eval, L):
    g = torch.Generator().manual_seed(seed)
    return _hand_points(lat_sizes, num_train, L, g), _hand_points(lat_sizes, num_eval, L, g)


@pytest.mark.parametrize("lat_sizes", [[1, 3, 6, 40, 32, 32], [2, 1, 5], [7, 3]])
def test_points_are_grid_indices_with_the_scored_factor_shared(lat_sizes):
    g = torch.Generator().manual_seed(3)
    label, a, b = evaluate.beta_vae_points(lat_sizes, 300, 16, g)
    scored = [k for k, s in enumerate(lat_sizes) if s > 1]
    va, vb = np.unravel_index(a.numpy(), lat_sizes), np.unravel_index(b.numpy(), lat_sizes)
    for v, j in enumerate(label.tolist()):
        k = scored[j]
        assert np.array_equal(va[k][v], vb[k][v])
    assert (a < int(np.prod(lat_sizes))).all() and (b < int(np.prod(lat_sizes))).all()
    assert set(label.tolist()) == set(range(len(scored)))


# ---- the host path with fp64 stand-ins for the kernels ------------------------------------------------------------
class _Fp64Kernels:
    """Stand in for `pair_abs_diff_mean` and `logistic_fit` on the host: record their inputs, compute with
    tests/beta_vae_reference.py."""

    def __init__(self):
        self.pairs, self.fits = [], []

    def pair(self, mu, rows_a, rows_b):
        self.pairs.append((rows_a.clone(), rows_b.clone()))
        return torch.from_numpy(R.features(mu.numpy(), rows_a.numpy(), rows_b.numpy()))

    def fit(self, x, labels, n_classes, K, num_train):
        self.fits.append((x.clone(), labels.clone(), n_classes.clone(), K, num_train))
        nc = int(n_classes[0])
        W, b, steps = R.fit(x[:num_train].numpy(), labels.numpy(), nc)
        assert steps >= 0
        coef = torch.full((K, x.shape[1] + 1), float("nan"), dtype=torch.float64)
        coef[:len(b)] = torch.from_numpy(np.c_[W, b])
        pred = torch.from_numpy(R.predict(W, b, nc, x.numpy())[0]).int()
        return coef, pred, torch.tensor([steps], dtype=torch.int32)


@pytest.fixture
def host_kernels(monkeypatch):
    k = _Fp64Kernels()
    monkeypatch.setattr(evaluate, "pair_abs_diff_mean", k.pair)
    monkeypatch.setattr(evaluate, "logistic_fit", k.fit)
    monkeypatch.setattr(evaluate.N, "require_cuda_f32", lambda *t: None)
    return k


def test_documented_draw_order_reproduces_the_rows(host_kernels):
    lat_sizes, seed = [3, 1, 40, 2, 5], 31
    n = int(np.prod(lat_sizes))
    mu = torch.randn(n, 4, generator=torch.Generator().manual_seed(1))
    evaluate.beta_vae_score(mu, lat_sizes, batch_size=7, num_train=60, num_eval=200, seed=seed)
    (lt, at, bt), (le, ae, be) = _hand_draws(lat_sizes, seed, 60, 200, 7)
    rows_a, rows_b = host_kernels.pairs[0]
    assert len(host_kernels.pairs) == 1 and len(host_kernels.fits) == 1
    assert np.array_equal(rows_a.numpy(), np.r_[at, ae]) and np.array_equal(rows_b.numpy(), np.r_[bt, be])
    x, labels, n_classes, K, num_train = host_kernels.fits[0]
    classes = np.unique(lt)
    assert K == 4 and num_train == 60 and labels.dtype == n_classes.dtype == torch.int32
    assert int(n_classes[0]) == len(classes) and np.array_equal(classes[labels.numpy()], lt)


def _restated(mu, lat_sizes, L, num_train, num_eval, seed):
    """Steps 1-3 of the definition, line by line: (score, classes, W, b, train confusion, eval confusion)."""
    (lt, at, bt), (le, ae, be) = _hand_draws(lat_sizes, seed, num_train, num_eval, L)
    x = R.features(mu.numpy(), np.r_[at, ae], np.r_[bt, be])
    K = sum(s > 1 for s in lat_sizes)
    classes = np.unique(lt)
    W, b, steps = R.fit(x[:num_train], np.searchsorted(classes, lt), len(classes))
    assert steps >= 0
    pred = classes[R.predict(W, b, len(classes), x)[0]]
    conf = []
    for truth, p in ((lt, pred[:num_train]), (le, pred[num_train:])):
        c = np.zeros((K, K), np.int64)
        np.add.at(c, (truth, p), 1)
        conf.append(c)
    score = {"train_accuracy": int(np.trace(conf[0])) / num_train, "eval_accuracy": int(np.trace(conf[1])) / num_eval}
    return score, classes, W, b, conf[0], conf[1]


def _check_against_restatement(mu, lat_sizes, L, num_train, num_eval, seed):
    got, helpers = evaluate.beta_vae_score(mu, lat_sizes, batch_size=L, num_train=num_train, num_eval=num_eval,
                                           seed=seed)
    score, classes, W, b, train_conf, eval_conf = _restated(mu, lat_sizes, L, num_train, num_eval, seed)
    factors = [k for k, s in enumerate(lat_sizes) if s > 1]
    assert got == score
    assert set(helpers) == {"factors", "classes", "coef", "intercept", "solver_iterations", "train_confusion",
                            "eval_confusion"}
    assert helpers["factors"].tolist() == factors and helpers["factors"].dtype == torch.int64
    assert helpers["classes"].tolist() == [factors[c] for c in classes] and helpers["classes"].dtype == torch.int64
    assert np.array_equal(helpers["coef"].numpy(), W) and np.array_equal(helpers["intercept"].numpy(), b)
    assert np.array_equal(helpers["train_confusion"].numpy(), train_conf)
    assert np.array_equal(helpers["eval_confusion"].numpy(), eval_conf)
    assert helpers["solver_iterations"].dtype == torch.int32 and helpers["solver_iterations"].shape == ()
    assert helpers["solver_iterations"] >= 0
    return got, helpers


def test_host_path_equals_a_restatement(host_kernels):
    """Five scored factors and a size-1 one; dims aligned with factors, a noise dim and a constant dim."""
    lat_sizes = [4, 1, 2, 6, 3, 5]
    n = int(np.prod(lat_sizes))
    values = np.stack(np.unravel_index(np.arange(n), lat_sizes), 1).astype(np.float64)
    rng = np.random.default_rng(0)
    mu = np.c_[values[:, [0, 2, 3]] / 4 + 0.3 * rng.standard_normal((n, 3)), rng.standard_normal(n), np.full(n, 0.5)]
    score, helpers = _check_against_restatement(torch.from_numpy(mu).float(), lat_sizes, 8, 500, 300, 5)
    assert helpers["coef"].shape == (5, 5) and abs(float(helpers["intercept"].sum())) < 1e-12


def test_two_classes_fit_one_binary_model(host_kernels):
    lat_sizes = [3, 4]
    mu = torch.randn(12, 3, generator=torch.Generator().manual_seed(2))
    score, helpers = _check_against_restatement(mu, lat_sizes, 5, 200, 100, 1)
    assert helpers["coef"].shape == (1, 3) and helpers["classes"].tolist() == [0, 1]


def test_one_class_in_training_predicts_that_class(host_kernels):
    """A single training point: one class, no fit, every point predicted as that factor."""
    lat_sizes = [3, 1, 4, 5]
    mu = torch.randn(60, 3, generator=torch.Generator().manual_seed(4))
    score, helpers = _check_against_restatement(mu, lat_sizes, 6, 1, 90, 11)
    assert helpers["coef"].shape == (0, 3) and helpers["intercept"].shape == (0,) and len(helpers["classes"]) == 1
    k = int(np.searchsorted([0, 2, 3], int(helpers["classes"][0])))
    assert score["train_accuracy"] == 1.0
    assert helpers["eval_confusion"][:, k].sum() == 90                        # every point predicted as k
    assert score["eval_accuracy"] == helpers["eval_confusion"][k, k].item() / 90


def test_evaluation_labels_unseen_in_training_are_never_right(host_kernels):
    lat_sizes = [2, 3, 4, 5, 6]
    mu = torch.randn(720, 4, generator=torch.Generator().manual_seed(6))
    seed = next(s for s in range(100) if len(np.unique(_hand_draws(lat_sizes, s, 3, 50, 4)[0][0])) < 5)
    score, helpers = _check_against_restatement(mu, lat_sizes, 4, 3, 50, seed)
    unseen = sorted(set(range(5)) - set(np.searchsorted([0, 1, 2, 3, 4], helpers["classes"].numpy())))
    assert unseen and helpers["eval_confusion"][:, unseen].sum() == 0


def test_failed_fit_warns(monkeypatch, host_kernels):
    fit = host_kernels.fit

    def failing(*a):
        coef, pred, _ = fit(*a)
        return coef, pred, torch.tensor([-1], dtype=torch.int32)
    monkeypatch.setattr(evaluate, "logistic_fit", failing)
    with pytest.warns(RuntimeWarning, match="did not converge"):
        _, helpers = evaluate.beta_vae_score(torch.randn(12, 3), [3, 4], num_train=50, num_eval=20)
    assert helpers["solver_iterations"] == -1


# ---- the objective is LogisticRegression's ------------------------------------------------------------------------
@pytest.mark.parametrize("nc", [2, 3, 5])
def test_reference_fit_equals_sklearn_newton_cholesky(nc):
    """The fp64 minimiser equals LogisticRegression(C=1, solver="newton-cholesky", tol=1e-12) on beta-VAE-like
    features, near zero and offset far from it; the multinomial intercepts are centred as sklearn centres them."""
    linear_model = pytest.importorskip("sklearn.linear_model")
    rng = np.random.default_rng(nc)
    n, D = 3000, 6
    y = rng.integers(0, nc, n)
    x = 0.5 * np.abs(rng.standard_normal((n, D)))
    x[np.arange(n), y % D] += 0.4
    for xx in (x, x + 50.0):
        W, b, steps = R.fit(xx, y, nc)
        assert steps >= 0
        clf = linear_model.LogisticRegression(C=1.0, solver="newton-cholesky", tol=1e-12, max_iter=1000).fit(xx, y)
        assert W.shape == clf.coef_.shape and b.shape == clf.intercept_.shape
        scale = max(np.abs(clf.coef_).max(), np.abs(clf.intercept_).max())
        assert np.abs(W - clf.coef_).max() <= 1e-6 * scale and np.abs(b - clf.intercept_).max() <= 1e-6 * scale
        if nc > 2:
            assert abs(b.sum()) <= 1e-12 * scale and abs(clf.intercept_.sum()) <= 1e-9 * scale
        pred = R.predict(W, b, nc, xx)[0]
        assert (clf.classes_[pred] == clf.predict(xx)).mean() > 0.999
