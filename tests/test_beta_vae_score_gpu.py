"""The beta-VAE score on the GPU: `dv_pair_abs_diff_mean` bit for bit against in-order fp64 sums, in the interleaved
q_zCx layout and a contiguous one; `dv_logistic_fit` against the fp64 dense Newton solve of
tests/beta_vae_reference.py at the shapes a user meets and at the limits; bit-identical repeats and refusals that
launch nothing; known answers of `beta_vae_score`; the Evaluator's score files over a DataLoader and over resident
data, beside MIG / AAM, the FactorVAE score and SAP.  The score in training, in sweeps and across a resume is tested
with the others in test_scores_gpu.py.
"""
import json
import os

import numpy as np
import pytest
import torch

import beta_vae_reference as R

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
DV_ERR_BAD_SHAPE, DV_ERR_BAD_ARG, DV_ERR_WORKSPACE = -1, -2, -3
COEF_RTOL = 1e-7          # |(W, b) - fp64 (W, b)|_inf against the fp64 solution's |(W, b)|_inf
KKT_TOL = 1e-8            # |gradient of the fp64 objective at the GPU's (W, b)|_inf against its largest part
MARGIN = 1e-7             # rows whose top two decisions are closer than this (relatively) may go either way
DSPRITES = [1, 3, 6, 40, 32, 32]


def _layout(x, layout):
    """`x` [N, D] as the kernel reads it: a contiguous copy, or the mean half of an interleaved [N, D, 2] buffer."""
    if layout == "contig":
        return x.contiguous()
    q = torch.full(x.shape + (2,), float("nan"), device=x.device)
    q[..., 0] = x
    return q.unbind(-1)[0]


def _values(lat_sizes):
    n = int(np.prod(lat_sizes))
    return torch.from_numpy(np.stack(np.unravel_index(np.arange(n), lat_sizes), 1)).double()


def _points(lat_sizes, num_train, num_eval, L, seed):
    from disvae.evaluate import beta_vae_points
    gen = torch.Generator(device=DEV)
    gen.manual_seed(seed)
    return beta_vae_points(lat_sizes, num_train, L, gen), beta_vae_points(lat_sizes, num_eval, L, gen)


# ---- features -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["q_zCx", "contig"])
def test_features_are_in_order_fp64_sums(layout):
    from disvae.evaluate import pair_abs_diff_mean
    g = torch.Generator().manual_seed(1)
    n = int(np.prod(DSPRITES))
    mu = torch.randn(n, 10, generator=g)
    mu[:, 3] = 100 + 0.01 * mu[:, 3]                   # far from zero
    mu[:, 4] = 1e-30 * mu[:, 4]                       # tiny
    (_, ta, tb), (_, ea, eb) = _points(DSPRITES, 10000, 5000, 64, 2)
    a, b = torch.cat([ta, ea]), torch.cat([tb, eb])
    x = pair_abs_diff_mean(_layout(mu.to(DEV), layout), a, b)
    want = R.features(mu.numpy(), a.cpu().numpy(), b.cpu().numpy())
    assert x.dtype == torch.float64 and x.shape == (15000, 10)
    assert np.array_equal(x.cpu().numpy(), want)
    for L in (1, 3):                                  # other lengths, odd ones included
        x = pair_abs_diff_mean(_layout(mu.to(DEV), layout), a[:100, :L].contiguous(), b[:100, :L].contiguous())
        assert np.array_equal(x.cpu().numpy(), R.features(mu.numpy(), a[:100, :L].cpu(), b[:100, :L].cpu()))


# ---- the fit ------------------------------------------------------------------------------------------------------
def _fit(x, y, nc, K, num_train):
    from disvae.evaluate import logistic_fit
    xd = torch.from_numpy(np.ascontiguousarray(x, np.float64)).to(DEV)
    labels = torch.from_numpy(np.asarray(y[:num_train], np.int32)).to(DEV)
    coef, pred, iters = logistic_fit(xd, labels, torch.tensor([nc], dtype=torch.int32, device=DEV), K, num_train)
    return coef.cpu().numpy(), pred.cpu().numpy(), int(iters)


def _check_fit(x, y, nc, K=None, num_train=None):
    """The GPU fit of the first num_train rows of x against the fp64 solve: (W, b), the KKT residual at the GPU's
    (W, b), convergence, the NaN rows, and the predictions of every row up to those within MARGIN of a tie.  Returns
    (W, b, iters) of the GPU."""
    K = nc if K is None else K
    num_train = len(x) if num_train is None else num_train
    coef, pred, iters = _fit(x, y, nc, K, num_train)
    rows = nc if nc > 2 else nc - 1
    assert iters >= 0, "the fit did not converge"
    assert np.isnan(coef[rows:]).all() and not np.isnan(coef[:rows]).any()
    W, b = coef[:rows, :-1], coef[:rows, -1]
    xt, yt = x[:num_train], np.asarray(y[:num_train])
    wW, wb, steps = R.fit(xt, yt, nc)
    assert steps >= 0
    if rows:
        ref = max(np.abs(wW).max(), np.abs(wb).max(), 1e-300)
        err = max(np.abs(W - wW).max(), np.abs(b - wb).max())
        assert err <= COEF_RTOL * ref, err / ref
        _, gr, sc = R.objective(xt, yt, nc, W, b)
        assert np.abs(gr).max() <= KKT_TOL * sc.max(), np.abs(gr).max() / sc.max()
        if nc > 2:
            assert abs(b.sum()) <= 1e-12 * ref
    want, gap = R.predict(wW, wb, nc, x)
    scale = 1 + (np.abs(R.decisions(wW, wb, x)).max(1) if rows else 0)
    loose = gap <= MARGIN * scale
    assert np.array_equal(pred[~loose], want[~loose]), np.flatnonzero(pred[~loose] != want[~loose])[:10]
    return W, b, iters


def _dsprites_features(seed):
    """Features of the dSprites grid's score points (10,000 + 5,000, L = 64) for a 10-dim code whose first five dims
    follow the scored factors."""
    from disvae.evaluate import pair_abs_diff_mean
    g = torch.Generator().manual_seed(seed)
    v = _values(DSPRITES)
    noise = torch.randn(v.size(0), 10, generator=g, dtype=torch.float64)
    mu = noise.clone()
    mu[:, :5] = v[:, 1:] / torch.tensor(DSPRITES[1:]) + 0.2 * noise[:, :5]
    (tl, ta, tb), (el, ea, eb) = _points(DSPRITES, 10000, 5000, 64, seed)
    x = pair_abs_diff_mean(mu.float().to(DEV), torch.cat([ta, ea]), torch.cat([tb, eb])).cpu().numpy()
    return x, torch.cat([tl, el]).cpu().numpy()


def test_fit_dsprites_shape():
    x, y = _dsprites_features(3)
    assert len(np.unique(y[:10000])) == 5
    _check_fit(x, y, 5, num_train=10000)


def test_fit_two_classes():
    rng = np.random.default_rng(4)
    y = rng.integers(0, 2, 6000)
    x = 0.5 * np.abs(rng.standard_normal((6000, 10)))
    x[:, 0] += 0.3 * y
    _check_fit(x, y, 2, K=5, num_train=4000)


def test_fit_one_class():
    rng = np.random.default_rng(5)
    x = rng.standard_normal((300, 10))
    coef, pred, iters = _fit(x, np.zeros(300, np.int64), 1, 5, 200)
    assert iters == 0 and np.isnan(coef).all() and (pred == 0).all()


@pytest.mark.parametrize("nc", [2, 3, 5])
def test_fit_all_zero_features_closed_form(nc):
    """W = 0 and b = the centred log class frequencies (log(n_1 / n_0) for two classes)."""
    rng = np.random.default_rng(nc)
    y = rng.choice(nc, size=3000, p=np.arange(1, nc + 1) / (nc * (nc + 1) / 2))
    W, b, _ = _check_fit(np.zeros((3000, 10)), y, nc)
    logn = np.log(np.bincount(y, minlength=nc).astype(np.float64))
    want = logn - logn.mean() if nc > 2 else np.array([logn[1] - logn[0]])
    assert (W == 0).all() and np.allclose(b, want, rtol=1e-9, atol=1e-12)


def test_fit_features_far_from_zero():
    rng = np.random.default_rng(6)
    y = rng.integers(0, 4, 8000)
    x = 100 + 0.01 * np.abs(rng.standard_normal((8000, 10)))
    x[np.arange(8000), y] += 0.005
    _check_fit(x, y, 4, num_train=6000)


def test_fit_near_separable_aligned_code():
    x, y = _dsprites_features(7)
    x[:, :5] *= 20.0                                          # large margins: weights far from the origin
    _check_fit(x, y, 5, num_train=10000)


def test_fit_at_the_limits():
    from disvae.evaluate import BETA_VAE_MAX_DIM, BETA_VAE_MAX_FACTORS
    rng = np.random.default_rng(8)
    D, K = BETA_VAE_MAX_DIM, BETA_VAE_MAX_FACTORS
    y = rng.integers(0, K, 1500)
    x = 0.5 * np.abs(rng.standard_normal((1500, D)))
    x[np.arange(1500), y * (D // K)] += 0.2
    _check_fit(x, y, K, num_train=1000)


def test_repeats_are_bit_identical():
    from disvae.evaluate import beta_vae_score
    mu = _layout(torch.randn(int(np.prod(DSPRITES)), 10, device=DEV), "q_zCx")
    runs = [beta_vae_score(mu, DSPRITES, seed=3) for _ in range(3)]
    for score, helpers in runs[1:]:
        assert score == runs[0][0]
        for key, value in helpers.items():
            assert torch.equal(torch.as_tensor(value), torch.as_tensor(runs[0][1][key])), key


def test_refusals_launch_nothing():
    from disvae import _native
    L = _native.lib()
    S = torch.cuda.current_stream().cuda_stream
    mu = torch.randn(100, 8, device=DEV)
    rows = torch.zeros(16, 4, dtype=torch.int64, device=DEV)
    x = torch.full((16, 8), 7.0, dtype=torch.float64, device=DEV)

    def pair(mu=mu.data_ptr(), ld=1, rs=8, N=100, D=8, a=rows.data_ptr(), b=rows.data_ptr(), V=16, Lp=4,
             x=x.data_ptr()):
        return L.dv_pair_abs_diff_mean(mu, ld, rs, N, D, a, b, V, Lp, x, S)

    labels = torch.zeros(12, dtype=torch.int32, device=DEV)
    ncl = torch.tensor([1, 0], dtype=torch.int32, device=DEV)
    coef = torch.full((4, 9), 7.0, dtype=torch.float64, device=DEV)
    pred = torch.full((16,), 7, dtype=torch.int32, device=DEV)
    iters = torch.full((2,), 7, dtype=torch.int32, device=DEV)
    nbytes = L.dv_logistic_fit_workspace_bytes(12, 8, 4)
    ws = torch.empty(nbytes // 8 + 1, dtype=torch.float64, device=DEV)

    def fit(x=x.data_ptr(), D=8, ntr=12, nev=4, y=labels.data_ptr(), nc=ncl.data_ptr(), K=4, coef=coef.data_ptr(),
            pred=pred.data_ptr(), it=iters.data_ptr(), ws=ws.data_ptr(), wsb=nbytes):
        return L.dv_logistic_fit(x, D, ntr, nev, y, nc, K, coef, pred, it, ws, wsb, S)

    def refused(fn, rc_want, **kw):
        torch.cuda.synchronize()
        before = L.dv_launch_count()
        rc = fn(**kw)
        torch.cuda.synchronize()
        assert rc == rc_want and L.dv_launch_count() == before, (fn.__name__, kw, rc)

    for shape in (dict(N=0), dict(D=0), dict(V=0), dict(Lp=0), dict(V=2 ** 30, D=8), dict(ld=0), dict(ld=-1),
                  dict(rs=0), dict(rs=-8)):
        refused(pair, DV_ERR_BAD_SHAPE, **shape)
    for bad in (dict(mu=None), dict(a=None), dict(b=None), dict(x=None), dict(mu=mu.data_ptr() + 2),
                dict(a=rows.data_ptr() + 4), dict(b=rows.data_ptr() + 4), dict(x=x.data_ptr() + 4)):
        refused(pair, DV_ERR_BAD_ARG, **bad)
    assert (x == 7).all()
    for shape in (dict(ntr=0), dict(nev=-1), dict(D=0), dict(D=129), dict(K=0), dict(K=33),
                  dict(ntr=2 ** 30, nev=2 ** 30)):
        refused(fit, DV_ERR_BAD_SHAPE, **shape)
    assert L.dv_logistic_fit_workspace_bytes(12, 129, 4) == 0 and L.dv_logistic_fit_workspace_bytes(12, 8, 33) == 0
    for bad in (dict(x=None), dict(y=None), dict(nc=None), dict(coef=None), dict(pred=None), dict(it=None),
                dict(x=x.data_ptr() + 4), dict(y=labels.data_ptr() + 2), dict(nc=ncl.data_ptr() + 2),
                dict(coef=coef.data_ptr() + 4), dict(pred=pred.data_ptr() + 2), dict(it=iters.data_ptr() + 2),
                dict(ws=ws.data_ptr() + 4)):
        refused(fit, DV_ERR_BAD_ARG, **bad)
    for bad in (dict(ws=None), dict(wsb=nbytes - 8)):
        refused(fit, DV_ERR_WORKSPACE, **bad)
    assert (coef == 7).all() and (pred == 7).all() and (iters == 7).all()
    before = L.dv_launch_count()
    x.zero_()
    assert fit() == 0 and L.dv_launch_count() == before + 1
    torch.cuda.synchronize()
    assert (pred == 0).all() and int(iters[0]) == 0 and int(iters[1]) == 7 and torch.isnan(coef).all()   # one class


# ---- known answers ------------------------------------------------------------------------------------------------
def test_constant_code_scores_the_majority_class_share():
    from disvae.evaluate import beta_vae_score
    lat = [3, 4, 5, 2]
    score, helpers = beta_vae_score(torch.full((120, 6), 0.25, device=DEV), lat, num_train=500, num_eval=300, seed=2)
    (tl, _, _), (el, _, _) = _points(lat, 500, 300, 64, 2)
    counts = torch.bincount(tl.cpu(), minlength=4)
    top = int(torch.argmax(counts))                                    # lowest on a tie, as the argmax of b
    assert score == {"train_accuracy": int(counts[top]) / 500, "eval_accuracy": int((el.cpu() == top).sum()) / 300}
    assert (helpers["coef"] == 0).all() and helpers["train_confusion"][:, top].sum() == 500


@pytest.mark.parametrize("layout", ["q_zCx", "contig"])
def test_aligned_code_scores_one(layout):
    from disvae.evaluate import beta_vae_score
    v = _values(DSPRITES)
    g = torch.Generator().manual_seed(9)
    mu = torch.cat([v[:, 1:] / (torch.tensor(DSPRITES[1:]) - 1), torch.randn(v.size(0), 2, generator=g,
                                                                            dtype=torch.float64)], 1)
    score, helpers = beta_vae_score(_layout(mu.float().to(DEV), layout), DSPRITES, seed=4)
    assert score == {"train_accuracy": 1.0, "eval_accuracy": 1.0}, score
    assert helpers["classes"].tolist() == [1, 2, 3, 4, 5] and helpers["solver_iterations"] >= 0


# ---- the Evaluator on a Burgess model ----------------------------------------------------------------------------
from test_eval_resident_gpu import (K, _assert_same_eval_files, _checkpoint_model, _dataset, _evaluator,  # noqa: E402
                                    _loader, _loss, _n_samples)

SCORE_FILES = [("beta_vae_score.log",) * 2, ("beta_vae_score_helpers.pth",) * 2]
OTHER_FILES = [(f, f) for f in ("factor_vae_score.log", "factor_vae_score_helpers.pth", "sap_score.log",
                                "sap_score_helpers.pth")]


def test_evaluator_score_files(tmp_path, monkeypatch):
    import disvae
    from synthetic_factors import loader
    ds = _dataset()
    model = _checkpoint_model()
    passes = []
    encode = disvae.Evaluator._compute_q_zCx

    def counted(self, dl):
        passes.append(dl)
        return encode(self, dl)
    monkeypatch.setattr(disvae.Evaluator, "_compute_q_zCx", counted)
    with _n_samples(512):
        for name, data, kw in (("host", loader(ds, 1000), dict(is_beta_vae_score=True)),
                               ("dev", _loader(ds).in_order(1000), dict(is_beta_vae_score=True)),
                               ("plain", loader(ds, 1000), {})):
            torch.manual_seed(7)
            passes.clear()
            _evaluator(model, _loss("btcvae", K ** 4), tmp_path / name)(
                data, is_metrics=True, is_losses=True, is_factor_score=True, factor_score_seed=21, is_sap_score=True,
                sap_score_seed=21, beta_vae_score_seed=21, **kw)
            assert len(passes) == 1, name                      # one encoding for MIG / AAM and every score
    _assert_same_eval_files(tmp_path / "dev", tmp_path / "host", SCORE_FILES, "dev vs host", nan_equal=True)
    names = [(f, f) for f in ("metrics.log", "metric_helpers.pth", "test_losses.log")] + OTHER_FILES
    _assert_same_eval_files(tmp_path / "host", tmp_path / "plain", names, "with vs without the score", nan_equal=True)
    assert not os.path.exists(tmp_path / "plain" / "beta_vae_score.log")
    score = json.load(open(tmp_path / "host" / "beta_vae_score.log"))
    helpers = torch.load(tmp_path / "host" / "beta_vae_score_helpers.pth", weights_only=False)
    assert set(helpers) == {"factors", "classes", "coef", "intercept", "solver_iterations", "train_confusion",
                            "eval_confusion"}
    # the fp64 restatement: documented draws, in-order features, the dense solve, its predictions
    ev = _evaluator(model, None, tmp_path / "enc")
    model.eval()
    mean = ev._compute_q_zCx(loader(ds, 1000))[1][0]
    lat = [int(s) for s in ds.lat_sizes]
    (tl, ta, tb), (el, ea, eb) = _points(lat, 10000, 5000, 64, 21)
    x = R.features(mean.cpu().numpy(), torch.cat([ta, ea]).cpu().numpy(), torch.cat([tb, eb]).cpu().numpy())
    truth = torch.cat([tl, el]).cpu().numpy()
    classes = np.unique(truth[:10000])
    W, b, _ = _check_fit(x, np.searchsorted(classes, truth), len(classes), K=len(lat), num_train=10000)
    assert np.array_equal(helpers["coef"].numpy(), W) and np.array_equal(helpers["intercept"].numpy(), b)
    pred, gap = R.predict(*R.fit(x[:10000], np.searchsorted(classes, truth[:10000]), len(classes))[:2],
                          len(classes), x)
    right = classes[pred] == truth
    loose = int((gap <= MARGIN * (1 + np.abs(x).sum(1).max())).sum())
    assert abs(score["train_accuracy"] - right[:10000].mean()) <= loose / 10000 + 1e-12
    assert abs(score["eval_accuracy"] - right[10000:].mean()) <= loose / 5000 + 1e-12
    assert ev.compute_beta_vae_score(loader(ds, 1000), seed=21) == score
