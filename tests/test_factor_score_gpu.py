"""The FactorVAE score on the GPU: `dv_group_variance` (csrc/dv_factor_score.cu) against fp64 numpy on the same rows,
in the interleaved q_zCx layout and a contiguous one; bit-identical repeats and refusals that launch nothing; known
answers of `factor_vae_score`; the Evaluator's score files over a DataLoader and over resident data, against an fp64
restatement of the score, and beside MIG / AAM.  The score in training, in sweeps and across a resume is tested
with the others in test_scores_gpu.py.
"""
import json
import logging
import os

import numpy as np
import pytest
import torch

from score_kernels import DEV, DV_ERR_BAD_ARG, DV_ERR_BAD_SHAPE, _layout, grid_values

pytestmark = pytest.mark.gpu
AMBIGUOUS = 1e-5                          # two ratios closer than this (relatively) may be ordered either way in fp32


def _variances(mu, rows):
    from disvae.evaluate import group_variance
    out = torch.full((rows.size(0), mu.size(1)), float("nan"), device=DEV)
    group_variance(mu, rows, var_out=out)
    return out


def _votes(mu, rows, gv):
    from disvae.evaluate import group_variance
    out = torch.full((rows.size(0),), -7, dtype=torch.int32, device=DEV)
    group_variance(mu, rows, global_var=gv, argmin_out=out)
    return out


def _fp64_var(x64, rows):
    return x64[rows].var(axis=1, ddof=1)


def _check_votes(got, var64, gv32, excluded=None):
    """Every vote whose two smallest fp64 ratios are more than AMBIGUOUS apart is the fp64 argmin; the others pick one
    of the near-tied dims.  Returns the share of ambiguous votes."""
    gv = gv32.astype(np.float64)
    active = gv32 >= np.float32(0.05)
    ratio = np.where(active, var64 / np.where(gv > 0, gv, 1.0), np.inf)
    if excluded is not None:
        ratio[:, excluded] = np.inf
    got = got.cpu().numpy()
    assert active[got].all(), "an inactive dim was voted for"
    best = ratio.min(axis=1, keepdims=True)
    near = ratio <= best * (1 + AMBIGUOUS) + 1e-300
    assert near[np.arange(len(got)), got].all()
    unique = near.sum(axis=1) == 1
    assert np.array_equal(got[unique], ratio.argmin(axis=1)[unique])
    return 1 - unique.mean()


# (N, D, V, L): D in {1, 10, 64, 1024}, L in {2, 64, 10000}, V in {1, 15000}
SHAPES = [(5000, 1, 15000, 2), (5000, 1, 1, 10000), (20000, 10, 15000, 64), (20000, 10, 1, 10000),
          (3000, 64, 15000, 64), (20000, 64, 1, 10000), (20000, 1024, 1, 10000), (2000, 1024, 15000, 2),
          (2000, 1024, 300, 64)]
REGIMES = ["normal", "far", "constant", "duplicate", "inactive"]


def _regime(n, d, regime, g):
    """(mu [n, d] on the device, columns that copy an earlier one) of one input regime."""
    x = torch.randn(n, d, generator=g, dtype=torch.float64)
    excluded = None
    if regime == "far":                                     # means near 100 with a spread of 0.01: every dim inactive
        x = 100 + 0.01 * x
    elif regime == "constant":
        x[:, ::3] = 3.25
    elif regime == "duplicate" and d > 1:
        x[:, 1::2] = x[:, :1]                               # every odd column is a copy of column 0: 0 must win
        excluded = np.arange(1, d, 2)
    elif regime == "inactive":                              # even columns: global variance 0.01, constant along runs
        x[:, ::2] = 0.2 * (torch.arange(n, dtype=torch.float64) >= n // 2).unsqueeze(1)
    return x.float().to(DEV), excluded


def _rows(n, v, l, regime, g):
    """Random rows; for "inactive", runs of consecutive items, where the inactive columns have the smallest ratio."""
    if regime == "inactive":
        return ((torch.randint(n, (v, 1), generator=g) + torch.arange(l)) % n).to(DEV)
    return torch.randint(n, (v, l), generator=g).to(DEV)


@pytest.mark.parametrize("layout", ["q_zCx", "contig"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "N%d-D%d-V%d-L%d" % s)
def test_kernel_against_fp64(shape, layout):
    n, d, v, l = shape
    g = torch.Generator().manual_seed(n + d + v + l)
    ambiguous = []
    for regime in REGIMES:
        x, excluded = _regime(n, d, regime, g)
        mu = _layout(x, layout)
        x64 = x.double().cpu().numpy()
        rows = _rows(n, v, l, regime, g)
        got = _variances(mu, rows).double().cpu().numpy()
        want = _fp64_var(x64, rows.cpu().numpy())
        err = np.abs(got - want)
        assert np.all(err <= 1e-5 * np.abs(want)), (regime, np.max(err / np.maximum(np.abs(want), 1e-300)))
        if regime == "constant":
            assert (got[:, ::3] == 0).all()
        gv = _variances(mu, torch.randint(n, (1, 10000), generator=g).to(DEV))[0]
        gv32 = gv.cpu().numpy()
        votes = _votes(mu, rows, gv)
        if not (gv32 >= np.float32(0.05)).any():
            assert regime in ("far", "constant", "inactive") and (votes == -1).all(), regime
            continue
        ambiguous.append(_check_votes(votes, want, gv32, excluded))
    assert max(ambiguous) < 0.01, ambiguous


def test_far_from_zero_keeps_its_precision():
    """Means near 100 with a spread of 0.01: the variance of a group keeps fp64's value to 1e-5, where a plain fp32
    sum of squares would keep none of it."""
    g = torch.Generator().manual_seed(4)
    x = (100 + 0.01 * torch.randn(8192, 16, generator=g, dtype=torch.float64)).float()
    rows = torch.randint(8192, (2000, 64), generator=g)
    got = _variances(_layout(x.to(DEV), "q_zCx"), rows.to(DEV)).double().cpu().numpy()
    want = _fp64_var(x.double().numpy(), rows.numpy())
    assert np.all(np.abs(got - want) <= 1e-5 * want)


def test_repeats_are_bit_identical():
    g = torch.Generator().manual_seed(8)
    mu = _layout(torch.randn(20000, 10, generator=g).to(DEV), "q_zCx")
    rows = torch.randint(20000, (15000, 64), generator=g).to(DEV)
    grows = torch.randint(20000, (1, 10000), generator=g).to(DEV)
    runs = []
    for _ in range(3):
        gv = _variances(mu, grows)[0]
        runs.append((gv, _variances(mu, rows), _votes(mu, rows, gv)))
    for r in runs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(r, runs[0]))


def test_refusals_launch_nothing():
    from disvae import _native
    L = _native.lib()
    mu = torch.randn(100, 8, device=DEV)
    rows = torch.zeros(4, 8, dtype=torch.int64, device=DEV)
    gv = torch.ones(8, device=DEV)
    var = torch.full((4, 8), 7.0, device=DEV)
    arg = torch.full((4,), 7, dtype=torch.int32, device=DEV)
    S = torch.cuda.current_stream().cuda_stream

    def args(mu=mu.data_ptr(), ld=1, rs=8, N=100, D=8, rows=rows.data_ptr(), V=4, Lr=8, gv=gv.data_ptr(),
             var=var.data_ptr(), arg=arg.data_ptr()):
        return (mu, ld, rs, N, D, rows, V, Lr, gv, 0.05, var, arg, S)

    def refused(rc_want, **kw):
        torch.cuda.synchronize()
        before = L.dv_launch_count()
        rc = L.dv_group_variance(*args(**kw))
        torch.cuda.synchronize()
        assert rc == rc_want and L.dv_launch_count() == before, (kw, rc)

    for shape in (dict(Lr=1), dict(Lr=0), dict(V=0), dict(N=0), dict(D=0), dict(D=1025), dict(ld=0), dict(ld=-1),
                  dict(rs=0), dict(rs=-8)):
        refused(DV_ERR_BAD_SHAPE, **shape)
    for bad in (dict(mu=None), dict(rows=None), dict(var=None, arg=None), dict(gv=None), dict(mu=mu.data_ptr() + 2),
                dict(rows=rows.data_ptr() + 4), dict(gv=gv.data_ptr() + 1), dict(var=var.data_ptr() + 2),
                dict(arg=arg.data_ptr() + 2)):
        refused(DV_ERR_BAD_ARG, **bad)
    assert (var == 7).all() and (arg == 7).all()
    before = L.dv_launch_count()
    assert L.dv_group_variance(*args(gv=None, arg=None)) == 0 and L.dv_launch_count() == before + 1


# ---- known answers ------------------------------------------------------------------------------------------------
LAT = [3, 4, 5, 6]


def _aligned_mu(lat_sizes, g):
    """Dim k = factor k's value scaled to variance > 0.05, a last dim of variance 0.0004, small noise on the rest."""
    v = grid_values(lat_sizes).double()
    mu = torch.cat([v / v.std(0) * 0.5, 0.02 * torch.randn(v.size(0), 1, generator=g, dtype=torch.float64)], 1)
    return mu.float().to(DEV)


def test_aligned_representation_scores_one():
    from disvae.evaluate import factor_vae_score
    mu = _aligned_mu(LAT, torch.Generator().manual_seed(1))
    for layout in ("q_zCx", "contig"):
        score, helpers = factor_vae_score(_layout(mu, layout), LAT, seed=5)
        assert score == {"train_accuracy": 1.0, "eval_accuracy": 1.0, "num_active_dims": len(LAT)}, layout
        assert helpers["classifier"][:len(LAT)].tolist() == list(range(len(LAT)))
        assert helpers["active_dims"].tolist() == [True] * len(LAT) + [False]
        assert helpers["train_votes"].sum() == 10000 and helpers["eval_votes"].sum() == 5000


def test_all_dims_inactive_scores_zero():
    from disvae.evaluate import factor_vae_score
    mu = 0.1 * torch.randn(int(np.prod(LAT)), 7, device=DEV)
    score, helpers = factor_vae_score(mu, LAT, seed=2)
    assert score == {"train_accuracy": 0.0, "eval_accuracy": 0.0, "num_active_dims": 0}
    assert helpers["train_votes"].sum() == 0 and helpers["eval_votes"].sum() == 0


def test_noise_scores_well_below_one():
    from disvae.evaluate import factor_vae_score
    score, _ = factor_vae_score(torch.randn(int(np.prod(LAT)), 6, device=DEV), LAT, seed=3)
    assert score["num_active_dims"] == 6 and score["eval_accuracy"] < 0.5, score


class _Images(torch.utils.data.Dataset):
    """Images whose first row holds the item's factor values (the encoder stub reads them)."""
    lat_names = tuple("f%d" % k for k in range(len(LAT)))
    lat_sizes = np.array(LAT)

    def __init__(self):
        v = grid_values(LAT).float()
        self.imgs = torch.zeros(v.size(0), 1, 32, 32)
        self.imgs[:, 0, 0, :len(LAT)] = v

    def __len__(self):
        return self.imgs.size(0)

    def __getitem__(self, i):
        return self.imgs[i], 0


class _StubModel(torch.nn.Module):
    latent_dim = len(LAT) + 1

    def __init__(self, scale):
        super().__init__()
        self.scale = scale

    def encoder(self, x):
        v = x[:, 0, 0, :len(LAT)]
        mean = torch.cat([v * self.scale, torch.zeros_like(v[:, :1])], 1)
        return mean, torch.zeros_like(mean)

    def reparameterize(self, mean, logvar):
        return mean


def test_evaluator_with_an_encoder_stub(tmp_path):
    import disvae
    from synthetic_factors import loader
    for scale, want in ((1.0, (1.0, 1.0, len(LAT))), (0.01, (0.0, 0.0, 0))):
        ev = disvae.Evaluator(_StubModel(scale), None, device=DEV, logger=logging.getLogger("factor-score"),
                              save_dir=str(tmp_path), is_progress_bar=False)
        s = ev.compute_factor_vae_score(loader(_Images(), 100), num_train=500, num_eval=300, seed=4)
        assert (s["train_accuracy"], s["eval_accuracy"], s["num_active_dims"]) == want, (scale, s)


# ---- the Evaluator on a Burgess model ----------------------------------------------------------------------------
from test_eval_resident_gpu import (K, _assert_same_eval_files, _checkpoint_model, _dataset, _evaluator,  # noqa: E402
                                    _loader, _loss, _n_samples)

SCORE_FILES = [("factor_vae_score.log",) * 2, ("factor_vae_score_helpers.pth",) * 2]


def _restated_score(mu, lat_sizes, seed, batch_size=64, num_train=10000, num_eval=5000, nve=10000):
    """The score in fp64 numpy on the documented draws, the kernel's choice taken only among near-tied dims."""
    from disvae.evaluate import factor_vote_rows
    n, d = mu.shape
    gen = torch.Generator(device=DEV)
    gen.manual_seed(seed)
    var_rows = torch.randint(n, (nve,), generator=gen, device=DEV)
    x64 = mu.double().cpu().numpy()
    gv64 = x64[var_rows.cpu().numpy()].var(axis=0, ddof=1)
    gv32 = _variances(mu, var_rows.view(1, -1))[0]
    assert np.all(np.abs(gv32.double().cpu().numpy() - gv64) <= 1e-5 * gv64)
    tf, tr = factor_vote_rows(lat_sizes, num_train, batch_size, gen)
    ef, er = factor_vote_rows(lat_sizes, num_eval, batch_size, gen)
    rows = torch.cat([tr, er])
    votes = _votes(mu, rows, gv32)
    ambiguous = _check_votes(votes, _fp64_var(x64, rows.cpu().numpy()), gv32.cpu().numpy())
    f = torch.cat([tf, ef]).cpu().numpy()
    dims = votes.cpu().numpy()
    tables = []
    for sl in (slice(0, num_train), slice(num_train, None)):
        t = np.zeros((len(lat_sizes), d), dtype=np.int64)
        np.add.at(t, (f[sl], dims[sl]), 1)
        tables.append(t)
    cls = tables[0].argmax(axis=0)
    acc = [t[cls, np.arange(d)].sum() / t.sum() for t in tables]
    return {"train_accuracy": acc[0], "eval_accuracy": acc[1],
            "num_active_dims": int((gv32.cpu().numpy() >= np.float32(0.05)).sum())}, tables, ambiguous


def test_evaluator_score_files(tmp_path):
    from synthetic_factors import loader
    ds = _dataset()
    model = _checkpoint_model()
    with _n_samples(512):
        for name, data, kw in (("host", loader(ds, 1000), dict(is_factor_score=True)),
                               ("dev", _loader(ds).in_order(1000), dict(is_factor_score=True)),
                               ("plain", loader(ds, 1000), {})):
            torch.manual_seed(7)
            _evaluator(model, _loss("btcvae", K ** 4), tmp_path / name)(data, is_metrics=True, is_losses=True,
                                                                           factor_score_seed=21, **kw)
    _assert_same_eval_files(tmp_path / "dev", tmp_path / "host", SCORE_FILES, "dev vs host")
    names = [(f, f) for f in ("metrics.log", "metric_helpers.pth", "test_losses.log")]
    _assert_same_eval_files(tmp_path / "host", tmp_path / "plain", names, "with vs without the score")
    assert not os.path.exists(tmp_path / "plain" / "factor_vae_score.log")
    score = json.load(open(tmp_path / "host" / "factor_vae_score.log"))
    helpers = torch.load(tmp_path / "host" / "factor_vae_score_helpers.pth", weights_only=False)
    assert set(helpers) == {"global_variances", "active_dims", "train_votes", "eval_votes", "classifier"}
    ev = _evaluator(model, None, tmp_path / "enc")
    model.eval()
    mean = ev._compute_q_zCx(loader(ds, 1000))[1][0]
    want, tables, ambiguous = _restated_score(mean, [int(s) for s in ds.lat_sizes], 21)
    assert ambiguous < 0.01
    assert score == want, (score, want)
    assert np.array_equal(helpers["train_votes"].numpy(), tables[0])
    assert np.array_equal(helpers["eval_votes"].numpy(), tables[1])
    alone = ev.compute_factor_vae_score(loader(ds, 1000), seed=21)
    assert alone == score
