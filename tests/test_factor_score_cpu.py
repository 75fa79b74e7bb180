"""The FactorVAE score on the host (no GPU, no kernel): every refusal happens before any GPU work, the vote rows are
grid indices whose voted factor is constant within a vote, the documented draw order reproduces them, and the
classifier and accuracies match a numpy restatement, ties included.  The host path of `factor_vae_score` runs here
with `group_variance` replaced by an fp64 numpy stand-in."""
import numpy as np
import pytest
import torch

from disvae import _native, evaluate
from score_stubs import _evaluator, _Grid, no_gpu  # noqa: F401


# (dataset, latent_dim, settings, message) of every refusal
REFUSALS = [
    (_Grid([4, 5], factors=False), 10, {}, "no lat_sizes / lat_names"),
    (_Grid([4, 5], n=21), 10, {}, "has 21 items, not the 20 of the full grid"),
    (_Grid([1, 1, 1]), 10, {}, "every factor of .* has one value"),
    (_Grid([4, 5]), 10, {"batch_size": 1}, "batch_size must be at least 2, got 1"),
    (_Grid([4, 5]), 10, {"num_train": 0}, "num_train must be at least 1, got 0"),
    (_Grid([4, 5]), 10, {"num_eval": 0}, "num_eval must be at least 1, got 0"),
    (_Grid([4, 5]), 10, {"num_variance_estimate": 1}, "num_variance_estimate must be at least 2, got 1"),
    (_Grid([4, 5]), 1025, {}, "latent_dim 1025 is above the kernel's limit of 1024"),
]


@pytest.mark.parametrize("case", range(len(REFUSALS)))
def test_evaluator_refusals_before_gpu_work(tmp_path, no_gpu, case):
    ds, latent_dim, settings, msg = REFUSALS[case]
    loader = torch.utils.data.DataLoader(ds, batch_size=10)
    with pytest.raises(ValueError, match=msg):
        _evaluator(tmp_path, latent_dim).compute_factor_vae_score(loader, **settings)
    if not settings:
        for is_metrics in (False, True):
            with pytest.raises(ValueError, match=msg):
                _evaluator(tmp_path, latent_dim)(loader, is_metrics=is_metrics, is_factor_score=True)
    if hasattr(ds, "lat_sizes"):
        with pytest.raises(ValueError, match=msg):
            evaluate.factor_vae_score(torch.zeros(len(ds), latent_dim), ds.lat_sizes, **settings)
    assert not list(tmp_path.iterdir())


# ---- vote rows and the draw order ---------------------------------------------------------------------------------
@pytest.mark.parametrize("lat_sizes", [[1, 3, 6, 40, 32, 32], [7], [2, 1], [5, 1, 4, 1]])
def test_vote_rows_are_grid_indices_with_the_voted_factor_constant(lat_sizes):
    num, bs = 3000, 16
    factor, rows = evaluate.factor_vote_rows(lat_sizes, num, bs, torch.Generator().manual_seed(5))
    assert factor.shape == (num,) and rows.shape == (num, bs) and rows.dtype == torch.int64
    assert rows.min() >= 0 and rows.max() < np.prod(lat_sizes)
    values = np.stack(np.unravel_index(rows.numpy(), lat_sizes), axis=-1)        # [num, bs, K]
    assert np.array_equal(np.ravel_multi_index(tuple(np.moveaxis(values, -1, 0)), lat_sizes), rows.numpy())
    f = factor.numpy()
    assert set(f.tolist()) == {k for k, s in enumerate(lat_sizes) if s > 1}       # every varying factor, no size-1 one
    voted = values[np.arange(num), :, f]                                          # [num, bs]
    assert (voted == voted[:, :1]).all()
    # the other factors do vary within a vote (over many votes, a factor of size > 1 takes more than one value)
    for k, s in enumerate(lat_sizes):
        if s > 1 and (f != k).any():
            other = values[f != k, :, k]
            assert (other != other[:, :1]).any(), k


def _hand_draws(n, lat_sizes, seed, nve, num_train, num_eval, bs):
    """The draw order of INTEGRATION.md, restated call by call."""
    g = torch.Generator().manual_seed(seed)
    var_rows = torch.randint(n, (nve,), generator=g)
    strides = np.cumprod([1] + list(lat_sizes[::-1]))[:-1][::-1]
    varying = [k for k, s in enumerate(lat_sizes) if s > 1]
    out = [var_rows]
    for num in (num_train, num_eval):
        f = torch.tensor(varying)[torch.randint(len(varying), (num,), generator=g)]
        rows = torch.zeros(num, bs, dtype=torch.int64)
        for k, s in enumerate(lat_sizes):
            v = torch.randint(s, (num, bs), generator=g)
            v[f == k] = v[f == k][:, :1]
            rows += v * int(strides[k])
        out += [f, rows]
    return out


class _Fp64Kernel:
    """Stands in for `group_variance` on the host: records the rows, computes in fp64 numpy."""

    def __init__(self):
        self.calls = []

    def __call__(self, mu, rows, global_var=None, var_out=None, argmin_out=None):
        self.calls.append(rows.clone())
        x = mu.double().numpy()[rows.numpy()]                                     # [V, L, D]
        var = x.var(axis=1, ddof=1)
        if var_out is not None:
            var_out.copy_(torch.from_numpy(var))
        if argmin_out is not None:
            gv = global_var.double().numpy()
            ratio = np.where(gv >= evaluate.FACTOR_SCORE_MIN_VAR, var / gv, np.inf)
            argmin_out.copy_(torch.from_numpy(ratio.argmin(axis=1)))


@pytest.fixture
def host_kernel(monkeypatch):
    k = _Fp64Kernel()
    monkeypatch.setattr(evaluate, "group_variance", k)
    monkeypatch.setattr(_native, "require_cuda_f32", lambda *t: None)
    return k


def test_documented_draw_order_reproduces_the_rows(host_kernel):
    lat_sizes, seed, settings = [3, 1, 4, 5], 77, dict(batch_size=8, num_train=300, num_eval=200,
                                                         num_variance_estimate=500)
    n = int(np.prod(lat_sizes))
    mu = torch.randn(n, 6, generator=torch.Generator().manual_seed(1))
    score, helpers = evaluate.factor_vae_score(mu, lat_sizes, seed=seed, **settings)
    var_rows, tf, tr, ef, er = _hand_draws(n, lat_sizes, seed, 500, 300, 200, 8)
    assert len(host_kernel.calls) == 2
    assert torch.equal(host_kernel.calls[0], var_rows.view(1, -1))
    assert torch.equal(host_kernel.calls[1], torch.cat([tr, er]))
    assert helpers["train_votes"].sum(1).tolist() == torch.bincount(tf, minlength=4).tolist()
    assert helpers["eval_votes"].sum(1).tolist() == torch.bincount(ef, minlength=4).tolist()
    assert helpers["train_votes"][1].sum() == 0 and score["num_active_dims"] == 6
    assert helpers["active_dims"].dtype == torch.bool and helpers["classifier"].shape == (6,)


def test_no_active_dim_draws_no_votes(host_kernel):
    mu = 0.1 * torch.randn(60, 4, generator=torch.Generator().manual_seed(2))     # variance 0.01 < 0.05
    score, helpers = evaluate.factor_vae_score(mu, [3, 4, 5], seed=3)
    assert score == {"train_accuracy": 0.0, "eval_accuracy": 0.0, "num_active_dims": 0}
    assert len(host_kernel.calls) == 1 and not helpers["active_dims"].any()
    assert helpers["train_votes"].shape == helpers["eval_votes"].shape == (3, 4)
    assert helpers["train_votes"].sum() == helpers["eval_votes"].sum() == 0


def test_host_path_equals_an_fp64_restatement(host_kernel):
    """The whole host path (draws, vote counting, classifier, accuracies) against numpy on the same draws."""
    lat_sizes, seed = [4, 3, 5], 123
    n = int(np.prod(lat_sizes))
    g = torch.Generator().manual_seed(9)
    values = np.stack(np.unravel_index(np.arange(n), lat_sizes), axis=-1).astype(np.float64)
    mu = torch.from_numpy(np.concatenate([values[:, [1, 0]], 0.01 * np.random.default_rng(0).standard_normal((n, 1)),
                                          values[:, [2]]], axis=1)).float()
    mu += 0.3 * torch.randn(n, 4, generator=g) * torch.tensor([1.0, 1.0, 0.0, 1.0])  # dim 2 stays inactive
    score, helpers = evaluate.factor_vae_score(mu, lat_sizes, batch_size=6, num_train=400, num_eval=300,
                                               num_variance_estimate=100, seed=seed)
    var_rows, tf, tr, ef, er = _hand_draws(n, lat_sizes, seed, 100, 400, 300, 6)
    x = mu.double().numpy()
    gv = x[var_rows.numpy()].var(axis=0, ddof=1)
    active = gv >= 0.05
    assert np.array_equal(helpers["active_dims"].numpy(), active) and score["num_active_dims"] == active.sum() == 3

    def votes(f, rows):
        ratio = np.where(active, x[rows.numpy()].var(axis=1, ddof=1) / gv, np.inf)
        table = np.zeros((3, 4), dtype=np.int64)
        np.add.at(table, (f.numpy(), ratio.argmin(axis=1)), 1)
        return table
    train, ev = votes(tf, tr), votes(ef, er)
    assert np.array_equal(helpers["train_votes"].numpy(), train) and np.array_equal(helpers["eval_votes"].numpy(), ev)
    cls = train.argmax(axis=0)
    assert np.array_equal(helpers["classifier"].numpy(), cls)
    assert score["train_accuracy"] == train[cls, np.arange(4)].sum() / 400
    assert score["eval_accuracy"] == ev[cls, np.arange(4)].sum() / 300
    assert score["train_accuracy"] > 0.9


# ---- classifier and accuracies ------------------------------------------------------------------------------------
def _np_accuracies(train, ev):
    cls = np.argmax(train, axis=0)                                                # the first maximum: lowest k
    cols = np.arange(train.shape[1])
    return cls, train[cls, cols].sum() / train.sum(), ev[cls, cols].sum() / ev.sum()


@pytest.mark.parametrize("seed", range(6))
def test_classifier_and_accuracies_against_numpy(seed):
    rng = np.random.default_rng(seed)
    K, D = rng.integers(1, 7), rng.integers(1, 12)
    train = rng.integers(0, 4, size=(K, D))                                       # small counts: many ties
    ev = rng.integers(0, 4, size=(K, D))
    train[0, 0] = ev[0, 0] = 1                                                    # at least one vote each
    cls, acc_t, acc_e = evaluate.factor_vote_accuracies(torch.from_numpy(train), torch.from_numpy(ev))
    want = _np_accuracies(train, ev)
    assert np.array_equal(cls.numpy(), want[0]) and acc_t == want[1] and acc_e == want[2]


def test_classifier_ties_go_to_the_lowest_factor():
    train = torch.tensor([[2, 0, 5, 0], [2, 3, 5, 0], [1, 3, 5, 0]])
    ev = torch.tensor([[1, 1, 1, 1], [1, 1, 1, 1], [1, 1, 1, 1]])
    cls, acc_t, acc_e = evaluate.factor_vote_accuracies(train, ev)
    assert cls.tolist() == [0, 1, 0, 0]
    assert acc_t == (2 + 3 + 5 + 0) / 26 and acc_e == 4 / 12
