"""UDR without a GPU: every refusal of `check_udr`, `udr_fit`, `udr_score`, `udr` and the sweep's UDR switches before any
GPU work; the fp64 restatement of tests/udr_reference.py against sklearn's Lasso (to 1e-9, on fixtures with a unique
minimiser) and scipy's spearmanr (to 1e-12, tied values included); the pair score against a line-by-line numpy form of
disentanglement_lib's relative_strength_disentanglement; the medians of `udr_from_pairs`; and the seed rule."""
import types
import warnings

import numpy as np
import pytest
import torch

import udr_reference as R
from disvae import evaluate as E


# ---- refusals -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("args, match", [
    (dict(num_models=1, latent_dims=[10]), "at least 2 models"),
    (dict(num_models=2, latent_dims=[10, 8]), "different latent_dim"),
    (dict(num_models=2, latent_dims=[10, 10], img_sizes=[(1, 64, 64), (3, 64, 64)]), "different image shapes"),
    (dict(num_models=2, latent_dims=[0, 0]), "latent_dim must be in"),
    (dict(num_models=2, latent_dims=[129, 129]), "latent_dim must be in"),
    (dict(num_models=33, latent_dims=[128] * 33), "above the kernel's limit of 4096"),
    (dict(num_models=2, latent_dims=[10, 10], num_points=1), "num_points must be in"),
    (dict(num_models=2, latent_dims=[10, 10], num_points=16385), "num_points must be in"),
    (dict(num_models=2, latent_dims=[10, 10], correlation="pearson"), "correlation must be one of"),
    (dict(num_models=3, latent_dims=[10] * 3, groups=[[0, 1]]), "not a partition"),
    (dict(num_models=3, latent_dims=[10] * 3, groups=[[0, 1], [1, 2]]), "not a partition"),
    (dict(num_models=3, latent_dims=[10] * 3, groups=[[0, 1, 2, 3]]), "not a partition"),
    (dict(num_models=3, latent_dims=[10] * 3, groups=[[0, 1], [2]]), "fewer than 2 models"),
])
def test_check_udr_refusals(args, match):
    with pytest.raises(ValueError, match=match):
        E.check_udr(**args)


def test_check_udr_accepts_the_limits_and_returns_the_groups():
    assert E.check_udr(2, [10, 10]) == [[0, 1]]
    assert E.check_udr(32, [128] * 32, num_points=16384, correlation="spearman") == [list(range(32))]
    assert E.check_udr(4096, [1] * 4096, num_points=2) == [list(range(4096))]
    assert E.check_udr(4, [3] * 4, groups=[(3, 0), [2, 1]]) == [[3, 0], [2, 1]]


def test_wrappers_refuse_before_any_gpu_work():
    mu = torch.zeros(2, 10, 3)
    with pytest.raises(ValueError, match="udr_fit: mu must be a contiguous CUDA"):
        E.udr_fit(mu, mu)
    with pytest.raises(ValueError, match="at least 2 models"):
        E.udr_score(torch.zeros(1, 10, 3), torch.zeros(1, 10, 3))
    with pytest.raises(ValueError, match="correlation must be one of"):
        E.udr_score(mu, mu, correlation="kendall")
    model = types.SimpleNamespace(latent_dim=10, img_size=(1, 32, 32))
    with pytest.raises(ValueError, match="expected a disvae.data.DeviceLoader"):
        E.udr([model, model], torch.utils.data.DataLoader([]))


def test_sweep_refuses_a_bad_udr_every_before_any_gpu_work():
    from disvae.sweep import Sweep
    sweep = object.__new__(Sweep)
    sweep.members = []
    for bad in (-1, 1.5, True, "2"):
        with pytest.raises(ValueError, match="udr_every must be a non-negative integer"):
            Sweep([], [], udr_every=bad)
        sweep.udr_every = bad                                  # the attribute, changed between calls
        with pytest.raises(ValueError, match="udr_every must be a non-negative integer"):
            sweep(None)
    sweep.loader = None
    with pytest.raises(ValueError, match="no loader yet"):
        sweep.udr()


# ---- the restatement against sklearn and scipy ---------------------------------------------------------------------
def _codes(n, D, seed, informative=None):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, D)) @ (np.eye(D) + 0.3 * rng.standard_normal((D, D)))
    x = x.astype(np.float32)
    inf = np.ones(D, bool) if informative is None else np.asarray(informative, bool)
    return x, inf


@pytest.mark.parametrize("n, Di, Dj, seed", [(1000, 10, 10, 0), (200, 5, 7, 1), (50, 3, 1, 2), (1000, 1, 4, 3)])
def test_lasso_matches_sklearn(n, Di, Dj, seed):
    from sklearn.linear_model import Lasso
    xi, _ = _codes(n, Di, seed)
    xj, _ = _codes(n, Dj, seed + 100)
    xj[:, 0] = xj[:, 0] + 2.0 * xi[:, 0]                      # a target the inputs explain
    mi = np.ones(Di, bool)
    mj = np.ones(Dj, bool)
    if Di > 2:
        mi[1] = False                                          # a non-informative input column: all zeros
    if Dj > 2:
        mj[-1] = False                                         # a non-informative target: y = 0
    Zi, Zj = R.features(xi, mi, "lasso"), R.features(xj, mj, "lasso")
    got, sweeps = R.similarity(Zi, Zj, "lasso")
    assert (sweeps >= 0).all()
    want = np.abs(Lasso(alpha=0.1, tol=1e-12, max_iter=10 ** 6).fit(Zi, Zj).coef_.reshape(Dj, Di)).T
    assert np.abs(got - want).max() <= 1e-9, np.abs(got - want).max()
    assert got[~mi].max(initial=0) == 0 and got[:, ~mj].max(initial=0) == 0


@pytest.mark.parametrize("ties", [False, True])
def test_spearman_matches_scipy(ties):
    from scipy.stats import spearmanr
    rng = np.random.default_rng(7)
    xi = rng.standard_normal((300, 4)).astype(np.float32)
    xj = (xi[:, ::-1] + 0.5 * rng.standard_normal((300, 4))).astype(np.float32)
    if ties:
        xi = np.round(xi * 2) / 2                              # a handful of values: long runs of ties
        xj[:, 1] = np.round(xj[:, 1])
        xj[:40, 2] = xj[0, 2]
        xj[::2, 3] = -0.0
        xj[1::4, 3] = 0.0
    got, _ = R.similarity(R.features(xi, np.ones(4, bool), "spearman"), R.features(xj, np.ones(4, bool), "spearman"),
                          "spearman")
    rho = spearmanr(xi, xj).correlation[:4, 4:]
    assert np.abs(got - np.abs(rho)).max() <= 1e-12


def test_spearman_of_a_constant_column_is_zero():
    xi, _ = _codes(100, 2, 4)
    xj, _ = _codes(100, 2, 5)
    xj[:, 1] = 0.25
    got, _ = R.similarity(R.features(xi, [1, 1], "spearman"), R.features(xj, [1, 1], "spearman"), "spearman")
    assert (got[:, 1] == 0).all() and (got[:, 0] > 0).all()


def test_rank_of_ties_is_scipys_average_rank():
    from scipy.stats import rankdata
    x = np.array([[3.0], [1.0], [3.0], [2.0], [1.0], [3.0], [-0.0], [0.0]], np.float32)
    assert np.array_equal(R.average_ranks(x)[:, 0], rankdata(x[:, 0]))


# ---- the pair score ---------------------------------------------------------------------------------------------
def _relative_strength_disentanglement(corr_matrix):
    """disentanglement_lib's udr.py, line by line."""
    score_x = np.nanmean(np.nan_to_num(np.power(np.ndarray.max(corr_matrix, axis=0), 2) /
                                       np.sum(corr_matrix, axis=0), 0))
    score_y = np.nanmean(np.nan_to_num(np.power(np.ndarray.max(corr_matrix, axis=1), 2) /
                                       np.sum(corr_matrix, axis=1), 0))
    return (score_x + score_y) / 2


@pytest.mark.parametrize("case", ["dense", "zero_column", "zero_row", "zero_matrix", "one_by_one"])
def test_pair_score_is_relative_strength_disentanglement(case):
    rng = np.random.default_rng(11)
    R_ = np.abs(rng.standard_normal((6, 6)))
    mi = np.array([1, 1, 0, 1, 1, 1], bool)
    mj = np.array([1, 0, 1, 1, 1, 1], bool)
    if case == "zero_column":
        R_[:, 3] = 0
    elif case == "zero_row":
        R_[4] = 0
    elif case == "zero_matrix":
        R_[:] = 0
    elif case == "one_by_one":
        mi, mj = np.eye(6, dtype=bool)[2], np.eye(6, dtype=bool)[5]
    with np.errstate(invalid="ignore", divide="ignore"):
        want = _relative_strength_disentanglement(R_[mi][:, mj])
    assert abs(R.pair_score(R_, mi, mj) - want) <= 1e-15


def test_pair_score_of_an_empty_filter_is_zero():
    R_ = np.ones((3, 3))
    none, some = np.zeros(3, bool), np.ones(3, bool)
    assert R.pair_score(R_, none, some) == 0.0 and R.pair_score(R_, some, none) == 0.0
    for mi, mj in ((none, some), (some, none)):                 # the library's form has no value there
        with warnings.catch_warnings(), pytest.raises(ValueError, match="zero-size array"):
            warnings.simplefilter("ignore")
            _relative_strength_disentanglement(R_[mi][:, mj])


# ---- medians ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K, groups", [(2, None), (3, None), (4, None), (5, None), (6, [[0, 2, 4], [1, 3, 5]]),
                                       (7, [[6, 0], [1, 2, 3, 4, 5]]), (8, [[0, 1, 2, 3], [4, 5, 6, 7]])])
def test_model_scores_are_medians_over_the_group(K, groups):
    rng = np.random.default_rng(K)
    pair = rng.random((K, K))
    np.fill_diagonal(pair, np.nan)
    groups_ = E.check_udr(K, [10] * K, groups=groups)
    got = E.udr_from_pairs(torch.from_numpy(pair), groups_)
    want = R.model_scores(pair, groups_)
    assert np.array_equal(np.array(got), want)
    for g in groups_:                                          # k as the target: column k, the others' rows
        for k in g:
            assert got[k] == np.median(np.delete(pair[g][:, g][:, g.index(k)], g.index(k)))


# ---- seeds ------------------------------------------------------------------------------------------------------
def test_points_come_from_their_own_generator():
    loader = types.SimpleNamespace(device=torch.device("cpu"), n=737)
    state = torch.get_rng_state()
    rows = E.udr_points(loader, 1000, 5)
    assert torch.equal(torch.get_rng_state(), state)
    g = torch.Generator().manual_seed(5)
    assert torch.equal(rows, torch.randint(737, (1000,), generator=g))


def test_sweep_udr_seed_is_the_loader_seed_and_the_latest_epoch(monkeypatch):
    from disvae import sweep as S
    seen = []
    monkeypatch.setattr(S, "write_udr", lambda models, loader, dirs, seed, **kw: seen.append(seed))
    monkeypatch.setattr(S.torch.cuda, "device", lambda d: __import__("contextlib").nullcontext())
    member = lambda seed: types.SimpleNamespace(  # noqa: E731
        model=types.SimpleNamespace(latent_dim=10, img_size=(1, 32, 32)), save_dir=".", logger=None, _next_epoch=3,
        seed=seed)
    for members in ([member(1), member(2)], [member(7), member(1), member(3)]):
        sweep = object.__new__(S.Sweep)
        sweep.members, sweep.device = members, None
        sweep.loader = types.SimpleNamespace(seed=1234)
        sweep.udr()
        sweep.udr(seed=9)
    assert seen == [E.evaluation_seed(1234, 2), 9] * 2
