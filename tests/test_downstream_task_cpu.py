"""The downstream-task score without a GPU: the fp64 restatement of tests/downstream_reference.py against sklearn's
LogisticRegressionCV (the fit, the choice of C, the fold class rules) and against disentanglement_lib's
downstream_task.py steps at sklearn's defaults; the draw order and the keys of `downstream_task` with the restatement
standing in for the kernels; and every refusal before any GPU work."""
import warnings

import numpy as np
import pytest
import torch

import downstream_reference as R
from disvae import evaluate
from score_stubs import _evaluator, _Grid, no_gpu  # noqa: F401

sklearn_lm = pytest.importorskip("sklearn.linear_model")
sklearn_ms = pytest.importorskip("sklearn.model_selection")


def _sklearn_cv(x, y, **kw):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return sklearn_lm.LogisticRegressionCV(Cs=10, cv=sklearn_ms.KFold(n_splits=5), **kw).fit(x, y)


def _data(nc, n, D, seed, shift=3.0, sep=0.8):
    rng = np.random.default_rng(seed)
    y = rng.integers(0, nc, n)
    x = rng.normal(size=(n, D)) + sep * y[:, None] * rng.normal(size=D)[None] + shift
    return x, y


# ---- the restatement against sklearn ------------------------------------------------------------------------------
@pytest.mark.parametrize("nc, n, D, seed", [(2, 150, 3, 1), (2, 400, 1, 2), (3, 200, 4, 3), (5, 300, 6, 4),
                                            (8, 500, 10, 5)])
def test_restatement_equals_sklearn_where_every_fold_has_every_class(nc, n, D, seed):
    """LogisticRegressionCV(Cs=10, cv=KFold(5), solver="newton-cholesky", tol=1e-12): the same C_, coefficients within
    1e-6, the same predictions and the same fold scores."""
    x, y = _data(nc, n, D, seed)
    for s0, s1 in R.fold_bounds(n):
        assert len(np.unique(np.r_[y[:s0], y[s1:]])) == nc
    ref = R.logistic_cv(x, y, nc, x)
    m = _sklearn_cv(x, y, solver="newton-cholesky", tol=1e-12, max_iter=1000)
    assert m.C_[0] == R.CS[ref["chosen"]]
    sb = m.intercept_ - (m.intercept_.mean() if nc > 2 else 0.0)
    scale = max(np.abs(ref["W"]).max(), np.abs(ref["b"]).max(), 1.0)
    assert np.abs(m.coef_ - ref["W"]).max() <= 1e-6 * scale and np.abs(sb - ref["b"]).max() <= 1e-6 * scale
    assert np.array_equal(m.predict(x), ref["pred"][:n])
    assert np.array_equal(m.scores_[m.classes_[-1]], ref["fold_acc"])
    assert (ref["fold_steps"] >= 0).all() and ref["steps"] >= 0


def test_fold_bounds_are_kfold():
    for n in (5, 6, 9, 10, 11, 12, 13, 14, 99, 1000):
        want = [(t[0], t[-1] + 1) for _, t in sklearn_ms.KFold(n_splits=5).split(np.zeros(n))]
        assert R.fold_bounds(n) == want


def _fold_case(nc, only_in_fold0, n=60, D=3, seed=6):
    """nc classes, class `only_in_fold0` on fold 0's rows only: fold 0's fit lacks it."""
    x, y = _data(nc - 1, n, D, seed, sep=1.5)
    s0, s1 = R.fold_bounds(n)[0]
    y[s0:s0 + 4] = only_in_fold0
    x[s0:s0 + 4] += 1.5
    return x, y


@pytest.mark.parametrize("nc", [3, 4])
def test_fold_class_rules_against_sklearn_scores(nc):
    """Fold 0's training part lacks the last class.  For nc = 3 its fit is the two-present-class multinomial (the
    binary fit at 2C), for nc = 4 a three-class multinomial; both are the limit of sklearn's fit over every class,
    whose missing-class intercept runs to -inf.  sklearn (lbfgs, its default, stops on that diverging direction at its
    tolerance) scores every fold and C the same as the restatement."""
    x, y = _fold_case(nc, nc - 1)
    ref = R.logistic_cv(x, y, nc, x)
    W, b, _, present, multi = R.fold_fit(x, y, nc, 0, 1.0)
    assert multi and present.tolist() == list(range(nc - 1)) and W.shape[0] == nc - 1
    if nc == 3:
        wb, bb, _ = R.fit(x[R.fold_bounds(len(x))[0][1]:], y[R.fold_bounds(len(x))[0][1]:], 2, False, 2.0)
        assert np.allclose(W[1] - W[0], wb[0]) and np.allclose(b[1] - b[0], bb[0])
    m = _sklearn_cv(x, y, tol=1e-10, max_iter=10000)
    differ = int((m.scores_[m.classes_[-1]] != ref["fold_acc"]).sum())
    print("fold class rule, %d classes: %d of %d fold scores differ from sklearn's" % (nc, differ,
                                                                                     ref["fold_acc"].size))
    assert differ == 0


def test_two_present_classes_differ_from_the_binary_fit_at_c():
    """The two-class multinomial at C is the binary fit at 2C, not at C."""
    x, y = _data(2, 80, 2, 7, sep=0.3)
    W, b, _ = R.fit(x, y, 2, True, 0.01)
    w1, b1, _ = R.fit(x, y, 2, False, 0.01)
    w2, b2, _ = R.fit(x, y, 2, False, 0.02)
    assert np.allclose(W[1] - W[0], w2[0], rtol=1e-9) and not np.allclose(W[1] - W[0], w1[0], rtol=1e-3)


# ---- against disentanglement_lib's steps at sklearn's defaults ----------------------------------------------------
def _compute_loss(x_train, y_train, x_test, y_test, predictor_fn):
    """downstream_task.py's _compute_loss, line by line (x [D, n], y [K, n])."""
    num_factors = y_train.shape[0]
    train_loss, test_loss = [], []
    for i in range(num_factors):
        model = predictor_fn()
        model.fit(x_train, y_train[i, :])
        train_loss.append(np.mean(model.predict(x_train) == y_train[i, :]))
        test_loss.append(np.mean(model.predict(x_test) == y_test[i, :]))
    return train_loss, test_loss


def test_agrees_with_disentanglement_lib_at_sklearn_defaults():
    """dSprites-shaped factors (3, 6, 40, 32, 32), 10 latents, sizes 10, 100, 1000 with 1000 test rows.  The library
    fits LogisticRegressionCV with lbfgs at its defaults (tol 1e-4, 100 iterations) on the raw values; the restatement
    is the exact fit; lbfgs stops short of it at the large Cs on unstandardised values, so fold scores, the chosen C and
    some predictions differ.  The library labels rows by their values, the restatement by sap_labels' classes (the
    same accuracies).  The count of differing accuracy cells and the largest difference are reported."""
    lat = [3, 6, 40, 32, 32]
    rng = np.random.default_rng(8)
    n_items = int(np.prod(lat))
    differ, cells, largest = 0, 0, 0.0
    for size in (10, 100, 1000):
        tr, te = rng.integers(0, n_items, size), rng.integers(0, n_items, 1000)
        v_tr, v_te = np.stack(np.unravel_index(tr, lat)), np.stack(np.unravel_index(te, lat))
        M = rng.normal(size=(5, 10))
        code = lambda v: (v.T / np.array(lat)) @ M + 0.05 * rng.normal(size=(v.shape[1], 10))  # noqa: E731
        x_tr, x_te = code(v_tr).astype(np.float32), code(v_te).astype(np.float32)
        factors, cls_tr, cls_te, ncl = R.labels(lat, tr, te)
        ours = np.stack([R.logistic_cv(x_tr, cls_tr[k], int(ncl[k]), x_te)["pred"] for k in range(5)])
        a_tr, a_te = R.accuracies(ours, cls_tr, cls_te)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            try:
                lib_tr, lib_te = _compute_loss(x_tr, v_tr, x_te, v_te, lambda: sklearn_lm.LogisticRegressionCV(
                    Cs=10, cv=sklearn_ms.KFold(n_splits=5)))
            except ValueError:                       # a factor seen with one value: sklearn refuses, we predict it
                continue
        gap = np.abs(np.r_[lib_tr, lib_te] - np.r_[a_tr, a_te])
        differ += int((gap > 0).sum())
        cells += gap.size
        largest = max(largest, float(gap.max()))
        print("size %d: %d of %d cells differ, by at most %.4f; mean test accuracy %.4f (library) and %.4f"
              % (size, int((gap > 0).sum()), gap.size, gap.max(), np.mean(lib_te), np.mean(a_te)))
        assert np.mean(a_te) >= np.mean(lib_te) - 0.02      # the exact fit predicts no worse than lbfgs's stop
    print("downstream task against disentanglement_lib at sklearn's defaults: %d of %d accuracy cells differ, by at "
          "most %.4f" % (differ, cells, largest))
    assert cells > 0


# ---- downstream_task with the restatement standing in for the kernels ---------------------------------------------
@pytest.fixture
def host_fits(monkeypatch):
    calls = []

    def logistic(mu, train_rows, test_rows, train_cls, n_classes, class_stride, Cs=R.CS, folds=False):
        calls.append(("lr", train_rows.clone(), test_rows.clone()))
        x = mu.double().numpy()
        K, n, S, D = len(n_classes), len(train_rows), class_stride, mu.shape[1]
        fold_acc, chosen = np.zeros((K, 5, len(Cs))), np.zeros(K, np.int32)
        coef, pred = np.full((K, S, D + 1), np.nan), np.zeros((K, n + len(test_rows)), np.int32)
        iters = np.zeros((K, 5 * len(Cs) + 1), np.int32)
        for k in range(K):
            f = R.logistic_cv(x[train_rows.numpy()], train_cls[k].numpy(), int(n_classes[k]), x[test_rows.numpy()],
                              Cs)
            fold_acc[k], chosen[k], pred[k] = f["fold_acc"], f["chosen"], f["pred"]
            coef[k, :len(f["b"])] = np.c_[f["W"], f["b"]]
            iters[k, :-1], iters[k, -1] = f["fold_steps"].ravel(), f["steps"]
        return tuple(torch.from_numpy(a) for a in (fold_acc, chosen, coef, pred, iters)) + (None, None)

    def trees(mu, train_rows, test_rows, train_cls, n_classes, counts):
        calls.append(("bt", train_rows.clone(), test_rows.clone()))
        x = mu.numpy()
        pred = np.stack([R.boosted_trees(x[train_rows.numpy()], train_cls[k].numpy(), int(n_classes[k]),
                                         x[test_rows.numpy()]) for k in range(len(n_classes))])
        return None, torch.from_numpy(pred).int(), None

    monkeypatch.setattr(evaluate, "downstream_logistic_cv", logistic)
    monkeypatch.setattr(evaluate, "dci_fit", trees)
    monkeypatch.setattr(evaluate.N, "require_cuda_f32", lambda *t: None)
    return calls


@pytest.mark.parametrize("predictor", ["logistic_regression", "boosted_trees"])
def test_draw_order_and_keys(host_fits, predictor):
    """For each size in order, the training rows and then that size's test rows from one generator seeded with
    `seed`; the classes are sap_labels'; the keys and values are downstream_task.py's."""
    lat = [3, 1, 4, 5]
    n = int(np.prod(lat))
    g = torch.Generator().manual_seed(9)
    v = torch.from_numpy(np.stack(np.unravel_index(np.arange(n), lat), 1)).float()
    mu = torch.cat([v / torch.tensor(lat).float(), torch.randn(n, 2, generator=g)], 1) + 0.1 * torch.randn(n, 6,
                                                                                                       generator=g)
    cpu = torch.get_rng_state()
    score, helpers = evaluate.downstream_task(mu, lat, predictor=predictor, num_train=(10, 30), num_test=17, seed=4)
    assert torch.equal(cpu, torch.get_rng_state())
    gen = torch.Generator().manual_seed(4)
    want = {}
    for call, size in zip(host_fits, (10, 30)):
        tr, te = torch.randint(n, (size,), generator=gen), torch.randint(n, (17,), generator=gen)
        assert call[0] == ("lr" if predictor == "logistic_regression" else "bt")
        assert torch.equal(call[1], tr) and torch.equal(call[2], te)
        factors, cls_tr, cls_te, ncl = R.labels(lat, tr.numpy(), te.numpy())
        x = mu.double().numpy()
        if predictor == "logistic_regression":
            pred = np.stack([R.logistic_cv(x[tr.numpy()], cls_tr[k], int(ncl[k]), x[te.numpy()])["pred"]
                             for k in range(len(factors))])
        else:
            pred = np.stack([R.boosted_trees(mu.numpy()[tr.numpy()], cls_tr[k], int(ncl[k]), mu.numpy()[te.numpy()])
                             for k in range(len(factors))])
        a_tr, a_te = R.accuracies(pred, cls_tr, cls_te)
        want.update(R.score_keys(size, a_tr, a_te))
        assert np.array_equal(helpers[size]["train_accuracy"].numpy(), a_tr)
        assert helpers[size]["classes"].shape == (3, 5)
    assert len(host_fits) == 2
    assert list(score) == list(want) and all(score[k] == want[k] for k in want)
    assert list(score)[:4] == ["10:mean_train_accuracy", "10:mean_test_accuracy", "10:min_train_accuracy",
                               "10:min_test_accuracy"]
    assert "30:test_accuracy_factor_2" in score and "30:test_accuracy_factor_3" not in score
    assert helpers["factors"].tolist() == [0, 2, 3]
    if predictor == "logistic_regression":
        h = helpers[30]
        assert h["fold_accuracy"].shape == (3, 5, 10) and h["solver_iterations"].shape == (3, 51)
        assert h["coef"].shape == (3, 5, 6) and h["intercept"].shape == (3, 5)
        assert np.array_equal(h["Cs"].numpy(), np.logspace(-4, 4, 10))


# ---- refusals ------------------------------------------------------------------------------------------------------
REFUSALS = [
    (_Grid([4, 5], factors=False), 10, {}, "has no lat_sizes / lat_names"),
    (_Grid([4, 5], n=21), 10, {}, "has 21 items, not the 20 of the full grid"),
    (_Grid([1, 1, 1]), 10, {}, r"every factor of \[1, 1, 1\] has one value"),
    (_Grid([4, 257]), 10, {}, "more than the kernel's limit of 256 values"),
    (_Grid([4, 5]), 10, {"predictor": "svm"}, "predictor must be one of"),
    (_Grid([4, 5]), 0, {}, r"latent_dim must be in \[1, 128\] for the logistic_regression predictor, got 0"),
    (_Grid([4, 5]), 129, {}, r"latent_dim must be in \[1, 128\] for the logistic_regression predictor, got 129"),
    (_Grid([4, 5]), 1025, {"predictor": "boosted_trees"}, r"latent_dim must be in \[1, 1024\]"),
    (_Grid([4, 5]), 10, {"num_train": ()}, "at least one training size"),
    (_Grid([4, 5]), 10, {"num_train": (10, 4)}, r"every num_train must be in \[5, 32768\].*got 4"),
    (_Grid([4, 5]), 10, {"num_train": 32769}, r"every num_train must be in \[5, 32768\].*got 32769"),
    (_Grid([4, 5]), 10, {"num_test": 0}, "num_test must be at least 1, got 0"),
]


@pytest.mark.parametrize("case", range(len(REFUSALS)))
def test_refusals_before_gpu_work(tmp_path, no_gpu, case):
    ds, latent_dim, settings, msg = REFUSALS[case]
    loader = torch.utils.data.DataLoader(ds, batch_size=10)
    with pytest.raises(ValueError, match=msg):
        _evaluator(tmp_path, latent_dim).compute_downstream_task(loader, **settings)
    with pytest.raises(ValueError, match=msg):
        evaluate.check_downstream_task(ds, latent_dim, **settings)
    if hasattr(ds, "lat_sizes"):
        with pytest.raises(ValueError, match=msg):
            evaluate.downstream_task(torch.zeros(len(ds), latent_dim), ds.lat_sizes, **settings)
    assert not list(tmp_path.iterdir())


def test_the_grid_is_numpys():
    assert evaluate.DOWNSTREAM_CS.dtype == np.float64
    assert np.array_equal(evaluate.DOWNSTREAM_CS, np.logspace(-4, 4, 10))
