"""The unsupervised scores without a GPU: every refusal of `check_unsupervised_scores`, the wrappers, the Evaluator, the
resident path and the sweep's switches before any GPU work; the draw order and the seed rule; the fp64 restatement of
tests/unsupervised_reference.py against disentanglement_lib's recalled formulas (np.cov, slogdet and scipy's sqrtm to
1e-12 relative, sklearn's mutual_info_score on np.digitize bins to 1e-12); the host combination
`unsupervised_from_fit` against the restatement; and the three deviations on a constant latent, duplicated latents and
all-constant codes."""
import types
import warnings

import numpy as np
import pytest
import scipy.linalg
import torch
from sklearn.metrics import mutual_info_score

import unsupervised_reference as R
from disvae import evaluate as E


# ---- refusals -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("args, match", [
    (dict(latent_dim=1), "latent_dim must be in"),
    (dict(latent_dim=129), "latent_dim must be in"),
    (dict(latent_dim=10, num_train=1), "num_train must be in"),
    (dict(latent_dim=10, num_train=32769), "num_train must be in"),
])
def test_check_refusals(args, match):
    with pytest.raises(ValueError, match=match):
        E.check_unsupervised_scores(**args)


def test_check_accepts_the_limits():
    E.check_unsupervised_scores(2, 2)
    E.check_unsupervised_scores(128, 32768)


def test_wrappers_refuse_before_any_gpu_work():
    mu = torch.zeros(20, 1)
    with pytest.raises(ValueError, match="latent_dim must be in"):
        E.unsupervised_scores(mu, mu)
    with pytest.raises(ValueError, match="num_train must be in"):
        E.unsupervised_scores(torch.zeros(20, 3), torch.zeros(20, 3), num_train=1)
    with pytest.raises(RuntimeError, match="CUDA"):
        E.unsupervised_fit(torch.zeros(20, 3), torch.zeros(20, 3), torch.zeros(4, dtype=torch.int64), torch.zeros(4, 3))
    model = types.SimpleNamespace(latent_dim=10, img_size=(1, 32, 32))
    with pytest.raises(ValueError, match="expected a disvae.data.DeviceLoader"):
        E.resident_unsupervised_scores(model, torch.utils.data.DataLoader([]))
    with pytest.raises(ValueError, match="latent_dim must be in"):
        E.resident_unsupervised_scores(types.SimpleNamespace(latent_dim=1, img_size=(1, 32, 32)),
                                       object.__new__(__import__("disvae.data", fromlist=["x"]).DeviceLoader))


def test_evaluator_refuses_before_any_gpu_work():
    ev = object.__new__(E.Evaluator)
    ev.model = types.SimpleNamespace(latent_dim=10)
    for bad in (None, object(), torch.utils.data.DataLoader([])):
        with pytest.raises(ValueError, match="non-empty dataset"):
            ev.compute_unsupervised_scores(bad)
    with pytest.raises(ValueError, match="num_train must be in"):
        ev.compute_unsupervised_scores(None, num_train=40000)
    ev.model = types.SimpleNamespace(latent_dim=1)
    with pytest.raises(ValueError, match="latent_dim must be in"):
        ev.compute_unsupervised_scores(torch.utils.data.DataLoader([1]))


def test_sweep_refuses_a_bad_unsupervised_every_before_any_gpu_work():
    from disvae.sweep import Sweep
    sweep = object.__new__(Sweep)
    sweep.members = []
    for bad in (-1, 1.5, True, "2"):
        with pytest.raises(ValueError, match="unsupervised_every must be a non-negative integer"):
            Sweep([], [], unsupervised_every=bad)
        sweep.unsupervised_every = bad                         # the attribute, changed between calls
        with pytest.raises(ValueError, match="unsupervised_every must be a non-negative integer"):
            sweep(None)
    sweep.unsupervised_every = 1
    sweep.members = [types.SimpleNamespace(model=types.SimpleNamespace(latent_dim=1), _resume=None)]
    with pytest.raises(ValueError, match="latent_dim must be in"):
        sweep(None)
    sweep.loader = None
    with pytest.raises(ValueError, match="no loader yet"):
        sweep.unsupervised_scores()


# ---- the draws and the seed rule ------------------------------------------------------------------------------------
def test_draw_order():
    """Rows from torch.randint first, then eps from torch.randn, on one generator seeded with the seed (mod 2^64)."""
    state = torch.get_rng_state()
    rows, eps = E.unsupervised_draws(737, 500, 7, seed=-3, device="cpu")
    assert torch.equal(torch.get_rng_state(), state), "a global generator moved"
    g = torch.Generator().manual_seed((-3) & 0xFFFFFFFFFFFFFFFF)
    assert torch.equal(rows, torch.randint(737, (500,), generator=g))
    assert torch.equal(eps, torch.randn(500, 7, generator=g))
    assert rows.dtype == torch.int64 and eps.dtype == torch.float32


def test_sweep_seed_rule():
    """Member k's seed after epoch e is evaluation_seed(its noise key, e): the metrics' rule, not UDR's."""
    from disvae.sweep import Sweep
    sweep = object.__new__(Sweep)
    sweep.device = torch.device("cpu")
    member = types.SimpleNamespace(model=types.SimpleNamespace(_noise_state=lambda dev: (1234567, 0)))
    assert sweep._unsupervised_seed(member, 4) == E.evaluation_seed(1234567, 4)
    assert sweep._unsupervised_seed(member, 4) != sweep._unsupervised_seed(member, 5)


def test_file_names():
    assert E.unsupervised_filenames() == ("unsupervised_scores.log", "unsupervised_scores_helpers.pth")
    assert E.unsupervised_filenames(0) == ("unsupervised_scores-0.log", "unsupervised_scores_helpers-0.pth")


# ---- the restatement against disentanglement_lib's formulas --------------------------------------------------------
def _codes(n, D, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, D)) @ (np.eye(D) + 0.6 / np.sqrt(D) * rng.standard_normal((D, D)))
    return (x * rng.uniform(0.5, 2.0, D)).astype(np.float32)


def _dlib_scores(x):
    """unsupervised_metrics.py's lines, on mus = x.T."""
    mus = np.asarray(x, np.float64).T
    cov = np.cov(mus)
    tc = 0.5 * (np.sum(np.log(np.diag(cov))) - np.linalg.slogdet(cov)[1])
    sqrtm = scipy.linalg.sqrtm(cov * np.expand_dims(np.diag(cov), axis=1))
    w = 2 * np.trace(cov) - 2 * np.trace(sqrtm)
    return tc, np.real(w), np.real(w) / np.trace(cov)


@pytest.mark.parametrize("n, D, seed", [(10000, 10, 0), (500, 3, 1), (2000, 2, 2), (3000, 32, 3)])
def test_gaussian_scores_match_the_recalled_formulas(n, D, seed):
    x = _codes(n, D, seed)
    C = R.cov(x)
    assert np.abs(C - np.cov(np.asarray(x, np.float64).T)).max() <= 1e-15 * np.abs(C).max()
    got = R.scores_from(C, *R.eigenvalues(C), np.zeros((D, D)))
    tc, w, wn = _dlib_scores(x)
    assert abs(got["gaussian_total_correlation"] - tc) <= 1e-12 * abs(tc) + 1e-14
    assert abs(got["gaussian_wasserstein_correlation"] - w) <= 1e-12 * np.trace(C)
    assert abs(got["gaussian_wasserstein_correlation_norm"] - wn) <= 1e-12


@pytest.mark.parametrize("n, D, seed", [(2000, 4, 0), (300, 3, 1)])
def test_mutual_info_matches_sklearn_on_digitized_bins(n, D, seed):
    x = _codes(n, D, seed)
    x[:, -1] = np.round(x[:, -1])                              # ties
    mus = x.T
    digit = np.stack([np.digitize(m, np.histogram(m, 20)[1][:-1]) for m in mus])
    assert np.array_equal(digit, R.bins(x))
    want = np.array([[mutual_info_score(digit[j], digit[i]) for j in range(D)] for i in range(D)])
    got = R.mutual_info_matrix(x)
    assert np.abs(got - want).max() <= 1e-12
    np.fill_diagonal(want, 0)
    assert abs(R.mutual_info_score(got) - want.sum() / (D * D - D)) <= 1e-12


# ---- the three deviations -------------------------------------------------------------------------------------------
def test_a_constant_latent_adds_nothing_to_the_total_correlation():
    x = _codes(3000, 5, 4)
    x[:, 2] = 1.25
    C = R.cov(x)
    with np.errstate(divide="ignore", invalid="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        assert np.isnan(_dlib_scores(x)[0])                    # numpy's answer
    keep = [0, 1, 3, 4]
    want = R.total_correlation(np.linalg.eigvalsh(R.correlation(C[np.ix_(keep, keep)])))
    tc = R.total_correlation(R.eigenvalues(C)[0])
    assert np.isfinite(tc) and abs(tc - want) <= 1e-12 * abs(want)
    m = R.mutual_info_matrix(x)
    assert (m[2] == 0).all() and (m[:, 2] == 0).all()


def test_duplicated_latents_have_infinite_total_correlation():
    x = _codes(3000, 4, 5)
    x[:, 3] = x[:, 1]
    assert R.total_correlation(R.eigenvalues(R.cov(x))[0]) == np.inf


def test_all_constant_codes():
    x = np.full((100, 3), 0.5, np.float32)
    C = R.cov(x)
    s = R.scores_from(C, *R.eigenvalues(C), R.mutual_info_matrix(x))
    assert s == {"gaussian_total_correlation": 0.0, "gaussian_wasserstein_correlation": 0.0,
                 "gaussian_wasserstein_correlation_norm": 0.0, "mutual_info_score": 0.0}


# ---- the package's host combination -------------------------------------------------------------------------------
def _combine(xs):
    """unsupervised_from_fit on what the kernel would return for the two codes xs, and the restatement's scores."""
    D = xs[0].shape[1]
    cov = np.stack([R.cov(x) for x in xs])
    eig = np.stack([np.stack(R.eigenvalues(c)) for c in cov])
    mi = np.stack([R.mutual_info_matrix(x) for x in xs])
    got = E.unsupervised_from_fit(torch.from_numpy(cov), torch.from_numpy(eig), torch.from_numpy(mi))
    want = [R.scores_from(cov[r], eig[r, 0], eig[r, 1], mi[r]) for r in range(2)]
    assert list(got) == ["mean", "sampled"] and D >= 2
    return got, want


def test_host_combination_matches_the_restatement():
    got, want = _combine([_codes(2000, 6, 6), _codes(2000, 6, 7)])
    for r, name in enumerate(("mean", "sampled")):
        assert set(got[name]) == set(R.KEYS)
        for k in R.KEYS:
            assert abs(got[name][k] - want[r][k]) <= 1e-12 * max(1.0, abs(want[r][k])), (name, k)


def test_host_combination_deviations():
    dup = _codes(500, 4, 8)
    dup[:, 3] = dup[:, 0]
    with pytest.warns(RuntimeWarning, match="linearly dependent"):
        got, _ = _combine([dup, np.full((500, 4), 2.0, np.float32)])
    assert got["mean"]["gaussian_total_correlation"] == float("inf")
    assert got["sampled"] == {"gaussian_total_correlation": 0.0, "gaussian_wasserstein_correlation": 0.0,
                              "gaussian_wasserstein_correlation_norm": 0.0, "mutual_info_score": 0.0}
