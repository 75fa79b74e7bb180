"""The SAP score on the host (no GPU, no kernel): every refusal happens before any GPU work, the documented draw order
reproduces the rows and their labels, the host path of `sap_score` (with `sap_score_matrix` replaced by the fp64
numpy stand-in of tests/sap_reference.py) equals a line-by-line restatement of the definition, and the stand-in's fits
equal sklearn's LinearSVC(C=0.01, class_weight="balanced"), which pins the objective to disentanglement_lib's
classifier."""
import numpy as np
import pytest
import torch

import sap_reference as R
from disvae import evaluate
from score_stubs import _evaluator, _Grid, no_gpu  # noqa: F401


# (dataset, latent_dim, settings, message) of every refusal
REFUSALS = [
    (_Grid([4, 5], factors=False), 10, {}, "no lat_sizes / lat_names"),
    (_Grid([4, 5], n=21), 10, {}, "has 21 items, not the 20 of the full grid"),
    (_Grid([1, 1, 1]), 10, {}, "every factor of .* has one value"),
    (_Grid([2, 257]), 10, {}, "more than the kernel's limit of 256 values"),
    (_Grid([4, 5]), 1, {}, "latent_dim must be at least 2 .*, got 1"),
    (_Grid([4, 5]), 1025, {}, "latent_dim 1025 is above the kernel's limit of 1024"),
    (_Grid([4, 5]), 10, {"num_train": 1}, "num_train must be at least 2, got 1"),
    (_Grid([4, 5]), 10, {"num_train": 32769}, "num_train 32769 is above the kernel's limit of 32768"),
    (_Grid([4, 5]), 10, {"num_test": 0}, "num_test must be at least 1, got 0"),
    (_Grid([4, 5]), 10, {"C": 0.0}, "C must be finite and positive, got 0.0"),
    (_Grid([4, 5]), 10, {"C": -1.0}, "C must be finite and positive, got -1.0"),
    (_Grid([4, 5]), 10, {"C": float("nan")}, "C must be finite and positive, got nan"),
    (_Grid([4, 5]), 10, {"C": float("inf")}, "C must be finite and positive, got inf"),
]


@pytest.mark.parametrize("case", range(len(REFUSALS)))
def test_evaluator_refusals_before_gpu_work(tmp_path, no_gpu, case):
    ds, latent_dim, settings, msg = REFUSALS[case]
    loader = torch.utils.data.DataLoader(ds, batch_size=10)
    with pytest.raises(ValueError, match=msg):
        _evaluator(tmp_path, latent_dim).compute_sap_score(loader, **settings)
    if not settings:
        for is_metrics in (False, True):
            for is_factor_score in (False, True):
                with pytest.raises(ValueError, match=msg):
                    _evaluator(tmp_path, latent_dim)(loader, is_metrics=is_metrics, is_factor_score=is_factor_score,
                                                     is_sap_score=True)
    if hasattr(ds, "lat_sizes"):
        with pytest.raises(ValueError, match=msg):
            evaluate.sap_score(torch.zeros(len(ds), latent_dim), ds.lat_sizes, **settings)
    assert not list(tmp_path.iterdir())


# ---- the host path with an fp64 stand-in for the kernel -----------------------------------------------------------
class _Fp64Kernel:
    """Stands in for `sap_score_matrix` on the host: records its inputs, computes with tests/sap_reference.py."""

    def __init__(self):
        self.calls = []

    def __call__(self, mu, train_rows, test_rows, train_cls, test_cls, n_classes, counts, C, coef=None, iters=None):
        args = [t.clone() for t in (train_rows, test_rows, train_cls, test_cls, n_classes, counts)]
        self.calls.append(args + [C])
        score, c, steps, _ = R.score_matrix(mu.numpy(), *(t.numpy() for t in args), C)
        assert (steps >= 0).all()
        if coef is not None:
            coef.copy_(torch.from_numpy(c))
        if iters is not None:
            iters.copy_(torch.from_numpy(steps))
        return torch.from_numpy(score)


@pytest.fixture
def host_kernel(monkeypatch):
    k = _Fp64Kernel()
    monkeypatch.setattr(evaluate, "sap_score_matrix", k)
    monkeypatch.setattr(evaluate.N, "require_cuda_f32", lambda *t: None)
    return k


def _hand_draws(n, seed, num_train, num_test):
    """The draw order of INTEGRATION.md, restated."""
    g = torch.Generator().manual_seed(seed)
    return torch.randint(n, (num_train,), generator=g), torch.randint(n, (num_test,), generator=g)


def test_documented_draw_order_reproduces_the_rows_and_labels(host_kernel):
    lat_sizes, seed = [3, 1, 40, 2, 5], 31
    n = int(np.prod(lat_sizes))
    mu = torch.randn(n, 4, generator=torch.Generator().manual_seed(1))
    evaluate.sap_score(mu, lat_sizes, num_train=60, num_test=200, seed=seed)
    tr, te = _hand_draws(n, seed, 60, 200)
    train_rows, test_rows, train_cls, test_cls, n_classes, counts, C = host_kernel.calls[0]
    assert len(host_kernel.calls) == 1 and C == 0.01
    assert torch.equal(train_rows, tr) and torch.equal(test_rows, te)
    vt, ve = np.unravel_index(tr.numpy(), lat_sizes), np.unravel_index(te.numpy(), lat_sizes)
    assert counts.shape == (4, 40) and train_cls.dtype == test_cls.dtype == torch.int32
    for j, k in enumerate([0, 2, 3, 4]):                                        # the factors of more than one value
        classes = np.unique(vt[k])
        assert n_classes[j] == len(classes)
        assert np.array_equal(classes[train_cls[j].numpy()], vt[k])
        seen = np.isin(ve[k], classes)
        assert np.array_equal(classes[test_cls[j].numpy()[seen]], ve[k][seen])
        assert (test_cls[j].numpy()[~seen] == -1).all()
        assert np.array_equal(counts[j, :len(classes)].numpy(), [(vt[k] == v).sum() for v in classes])
        assert (counts[j, len(classes):] == 0).all()
    assert (~np.isin(ve[2], vt[2])).any()                 # 40 values over 60 rows: some test values are unseen


def _restated(mu, lat_sizes, num_train, num_test, C, seed):
    """Steps 1-4 of the definition, line by line: (score [D, K'] fp32, SAP, {(d, k): (classes, lines)})."""
    n, D = mu.shape
    tr, te = _hand_draws(n, seed, num_train, num_test)
    v_train = np.stack(np.unravel_index(tr.numpy(), lat_sizes), 1)
    v_test = np.stack(np.unravel_index(te.numpy(), lat_sizes), 1)
    x = mu.double().numpy()
    factors = [k for k, s in enumerate(lat_sizes) if s > 1]
    score = np.zeros((D, len(factors)), np.float32)
    fits = {}
    for d in range(D):
        for j, k in enumerate(factors):
            classes = np.unique(v_train[:, k])
            y = np.searchsorted(classes, v_train[:, k])
            if len(classes) == 1:
                lines = np.zeros((0, 2))
                pred = np.full(num_test, classes[0])
            else:
                s, c, pos = R.problems(y, len(classes), C, num_train)
                lines, steps = R.solve(np.tile(x[tr.numpy(), d], (len(pos), 1)), s, c)
                assert (steps >= 0).all()
                v = R.decisions(lines, x[te.numpy(), d])
                idx = (v[:, 0] > 0).astype(int) if len(classes) == 2 else np.argmax(v, axis=1)
                pred = classes[idx]
            fits[d, j] = (classes, lines)
            score[d, j] = np.float32(np.mean(pred == v_test[:, k]))
    top = np.sort(score.astype(np.float64), axis=0)
    return score, float(np.mean(top[-1] - top[-2])), fits


def _check_against_restatement(mu, lat_sizes, num_train, num_test, C, seed):
    got, helpers = evaluate.sap_score(mu, lat_sizes, num_train=num_train, num_test=num_test, C=C, seed=seed)
    score, want, fits = _restated(mu, lat_sizes, num_train, num_test, C, seed)
    assert np.array_equal(helpers["score_matrix"].numpy(), score)
    assert got == {"SAP": want}
    assert helpers["factors"].tolist() == [k for k, s in enumerate(lat_sizes) if s > 1]
    for (d, j), (classes, lines) in fits.items():
        assert np.array_equal(helpers["classes"][j, :len(classes)].numpy(), classes)
        assert (helpers["classes"][j, len(classes):] == -1).all()
        npb = len(lines)
        assert np.array_equal(helpers["coef"][d, j, :npb].numpy(), lines)
        assert np.isnan(helpers["coef"][d, j, npb:].numpy()).all()
        assert (helpers["solver_iterations"][d, j, :npb] >= 0).all()
    return helpers


def test_host_path_equals_a_restatement(host_kernel):
    """Multi-class, binary and size-1 factors; dims aligned with factors, a noise dim and a constant dim."""
    lat_sizes = [4, 1, 2, 6]
    n = int(np.prod(lat_sizes))
    values = np.stack(np.unravel_index(np.arange(n), lat_sizes), 1).astype(np.float64)
    rng = np.random.default_rng(0)
    mu = np.stack([values[:, 3] + 0.3 * rng.standard_normal(n), values[:, 2] + 0.2 * rng.standard_normal(n),
                   rng.standard_normal(n), np.full(n, 0.5), 100 + 0.01 * values[:, 0]], 1)
    helpers = _check_against_restatement(torch.from_numpy(mu).float(), lat_sizes, 500, 300, 0.01, 5)
    score = helpers["score_matrix"]
    assert score[0, 2] > 0.5 and score[1, 1] > 0.95                           # the aligned dims predict their factors


def test_one_class_factor_predicts_that_class(host_kernel):
    """A factor that shows one value among the training rows is not fitted: every test row is predicted as that
    value."""
    lat_sizes, num_train = [2, 3], 2
    n = int(np.prod(lat_sizes))
    seed = next(s for s in range(100) if len(set(np.unravel_index(_hand_draws(n, s, num_train, 50)[0].numpy(),
                                                                   lat_sizes)[0])) == 1)
    mu = torch.randn(n, 3, generator=torch.Generator().manual_seed(2))
    helpers = _check_against_restatement(mu, lat_sizes, num_train, 50, 0.01, seed)
    assert (helpers["classes"][0, 1:] == -1).all() and np.isnan(helpers["coef"][:, 0].numpy()).all()


# ---- the objective is LinearSVC's ---------------------------------------------------------------------------------
@pytest.mark.parametrize("nc", [2, 3, 7])
def test_stand_in_fits_equal_sklearn_linear_svc(nc):
    """The fp64 minimiser equals LinearSVC(C=0.01, class_weight="balanced", tol=1e-7) on unbalanced one-vs-rest and
    binary problems: the positives of a one-vs-rest problem carry their class weight, the negatives plain C."""
    svm = pytest.importorskip("sklearn.svm")
    rng = np.random.default_rng(nc)
    n = 3000
    p = np.r_[0.5, np.full(nc - 1, 0.5 / (nc - 1))]
    y = rng.choice(nc, size=n, p=p)
    for x in (0.8 * y + rng.standard_normal(n), 3.0 + 0.2 * rng.standard_normal(n)):
        x = x.astype(np.float32).astype(np.float64)
        s, c, pos = R.problems(y, nc, 0.01, n)
        z, steps = R.solve(np.tile(x, (len(pos), 1)), s, c)
        assert (steps >= 0).all()
        clf = svm.LinearSVC(C=0.01, class_weight="balanced", tol=1e-7, max_iter=200000).fit(x[:, None], y)
        want = np.c_[clf.coef_[:, 0], clf.intercept_]
        assert np.allclose(z, want, rtol=1e-6, atol=1e-8 * np.abs(want).max()), (z, want)
