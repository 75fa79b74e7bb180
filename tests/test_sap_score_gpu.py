"""The SAP score on the GPU: `dv_sap_score_matrix` (csrc/dv_sap.cu) against the fp64 numpy solve of
tests/sap_reference.py on the same rows and labels, in the interleaved q_zCx layout and a contiguous one; bit-identical
repeats and refusals that launch nothing; known answers of `sap_score`; the Evaluator's score files over a DataLoader
and over resident data, beside MIG / AAM and the FactorVAE score.  The score in training, in sweeps and across a
resume is tested with the others in test_scores_gpu.py.
"""
import json
import os

import numpy as np
import pytest
import torch

import sap_reference as R

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
DV_ERR_BAD_SHAPE, DV_ERR_BAD_ARG = -1, -2
COEF_RTOL = 1e-7          # |(w, b) - fp64 (w, b)|_inf against the fp64 solution's |(w, b)|_inf
KKT_TOL = 1e-8            # |gradient of the fp64 objective at the GPU's (w, b)|_inf against its scale
MARGIN = 1e-7             # test rows whose top two decisions are closer than this (relatively) may go either way


def _layout(x, layout):
    """`x` [N, D] as the kernel reads it: a contiguous copy, or the mean half of an interleaved [N, D, 2] buffer."""
    if layout == "contig":
        return x.contiguous()
    q = torch.full(x.shape + (2,), float("nan"), device=x.device)
    q[..., 0] = x
    return q.unbind(-1)[0]


def _run_kernel(mu, lat_sizes, train_rows, test_rows, C=0.01):
    from disvae.evaluate import sap_labels, sap_score_matrix
    factors, train_cls, test_cls, n_classes, counts, _ = sap_labels(lat_sizes, train_rows, test_rows)
    D, (K, S) = mu.size(1), counts.shape
    coef = torch.full((D, K, S, 2), 7.0, dtype=torch.float64, device=DEV)
    iters = torch.full((D, K, S), -7, dtype=torch.int32, device=DEV)
    score = sap_score_matrix(mu, train_rows, test_rows, train_cls, test_cls, n_classes, counts, C, coef, iters)
    inputs = [t.cpu().numpy() for t in (train_rows, test_rows, train_cls, test_cls, n_classes, counts)]
    return score.cpu().numpy(), coef.cpu().numpy(), iters.cpu().numpy(), inputs


def _check_against_fp64(x, lat_sizes, train_rows, test_rows, C=0.01):
    """The kernel in both layouts against the fp64 solve: (w, b), the KKT residual at the GPU's (w, b), convergence,
    and the score cells up to the test rows within MARGIN of a tie.  Returns (fp64 score matrix, the kernel's)."""
    x32 = x.cpu().numpy()
    want = None
    for layout in ("q_zCx", "contig"):
        score, coef, iters, inputs = _run_kernel(_layout(x, layout), lat_sizes, train_rows, test_rows, C)
        if want is None:
            want = R.score_matrix(x32, *inputs, C)
        w_score, w_coef, w_steps, gap = want
        _, _, train_cls, test_cls, n_classes, _ = inputs
        assert (w_steps[~np.isnan(w_coef[..., 0])] >= 0).all()
        fitted = ~np.isnan(w_coef[..., 0])
        assert np.array_equal(fitted, ~np.isnan(coef[..., 0])), layout
        assert (iters[fitted] >= 0).all(), (layout, "a fit did not converge")
        assert (iters[~fitted] == 0).all() and np.isnan(coef[~fitted]).all()
        err = np.abs(coef - w_coef).max(-1)[fitted]
        ref = np.maximum(np.abs(w_coef).max(-1)[fitted], 1e-300)
        assert (err <= COEF_RTOL * ref).all(), (layout, (err / ref).max())
        n_train = len(train_rows)
        x_train = x32[inputs[0]].astype(np.float64)
        for k in range(len(n_classes)):
            s, c, pos = R.problems(train_cls[k].astype(np.int64), int(n_classes[k]), C, n_train)
            if not pos:
                continue
            D = x_train.shape[1]
            g, scale = R.gradient(coef[:, k, :len(pos)].reshape(-1, 2), np.repeat(x_train.T, len(pos), axis=0),
                                  np.tile(s, (D, 1)), np.tile(c, (D, 1)))
            assert (np.abs(g).max(1) <= KKT_TOL * scale).all(), (layout, k, (np.abs(g).max(1) / scale).max())
        x_test = x32[inputs[1]].astype(np.float64)
        for d in range(x32.shape[1]):
            for k in range(len(n_classes)):
                lines = w_coef[d, k][fitted[d, k]]
                scale = 1 + (np.abs(R.decisions(lines, x_test[:, d])).max() if len(lines) else 0)
                loose = int((gap[d, k] <= MARGIN * scale).sum())
                assert abs(float(score[d, k]) - float(w_score[d, k])) <= loose / len(test_rows) + 1e-7, \
                    (layout, d, k, score[d, k], w_score[d, k], loose)
    return w_score, score


def _rows(n, num, g):
    return torch.randint(n, (num,), generator=g).to(DEV)


def _values(lat_sizes):
    n = int(np.prod(lat_sizes))
    return torch.from_numpy(np.stack(np.unravel_index(np.arange(n), lat_sizes), 1)).double()


def test_kernel_dsprites_shape():
    lat = [1, 3, 6, 40, 32, 32]
    g = torch.Generator().manual_seed(1)
    v = _values(lat)
    n = v.size(0)
    noise = torch.randn(n, 10, generator=g, dtype=torch.float64)
    x = noise.clone()
    x[:, :5] = v[:, 1:] / torch.tensor(lat[1:]) + 0.2 * noise[:, :5]       # dims 0-4 follow the factors
    _check_against_fp64(x.float().to(DEV), lat, _rows(n, 10000, g), _rows(n, 5000, g))


def test_kernel_binary_factors():
    lat = [2, 2, 2, 3]
    g = torch.Generator().manual_seed(2)
    v = _values(lat)
    x = torch.cat([2 * v[:, :3] - 1 + 0.7 * torch.randn(v.size(0), 3, generator=g, dtype=torch.float64),
                   torch.randn(v.size(0), 3, generator=g, dtype=torch.float64)], 1)
    _check_against_fp64(x.float().to(DEV), lat, _rows(v.size(0), 4000, g), _rows(v.size(0), 2000, g))


def test_kernel_factor_with_one_class_in_training():
    """Factor 0 takes one value over every training row: no fit, every test row predicted as that value."""
    lat = [2, 50]
    g = torch.Generator().manual_seed(3)
    n = 100
    x = torch.randn(n, 4, generator=g).to(DEV)
    train = 50 + _rows(50, 3000, g)                                            # factor 0 = 1 on every training row
    test = _rows(n, 2000, g)
    score = _check_against_fp64(x, lat, train, test)[1]
    share = float((test >= 50).double().mean())
    assert np.allclose(score[:, 0], np.float32(share))


def test_kernel_constant_and_near_constant_columns():
    lat = [4, 6]
    g = torch.Generator().manual_seed(4)
    v = _values(lat)
    n = v.size(0)
    x = torch.stack([torch.full((n,), 0.5, dtype=torch.float64),
                     0.5 + 1e-6 * torch.randn(n, generator=g, dtype=torch.float64),
                     torch.zeros(n, dtype=torch.float64),
                     v[:, 1] + 0.3 * torch.randn(n, generator=g, dtype=torch.float64)], 1)
    _check_against_fp64(x.float().to(DEV), lat, _rows(n, 5000, g), _rows(n, 3000, g))


def test_kernel_column_far_from_zero():
    """Means near 100 with a spread of 0.01, the spread carrying the factors."""
    lat = [5, 3]
    g = torch.Generator().manual_seed(5)
    v = _values(lat)
    n = v.size(0)
    spread = torch.cat([v / torch.tensor([5.0, 3.0]) + 0.3 * torch.randn(n, 2, generator=g, dtype=torch.float64),
                        torch.randn(n, 1, generator=g, dtype=torch.float64)], 1)
    x = 100 + 0.01 * spread
    _check_against_fp64(x.float().to(DEV), lat, _rows(n, 6000, g), _rows(n, 3000, g))


def test_kernel_dim_limit():
    lat = [2, 3]
    g = torch.Generator().manual_seed(6)
    n = 6
    x = torch.randn(n, 1024, generator=g).to(DEV)
    _check_against_fp64(x, lat, _rows(n, 2000, g), _rows(n, 1000, g))


def test_kernel_class_limit():
    lat = [256]
    g = torch.Generator().manual_seed(7)
    v = _values(lat)
    x = torch.cat([v / 256 + 0.05 * torch.randn(256, 1, generator=g, dtype=torch.float64),
                   torch.randn(256, 2, generator=g, dtype=torch.float64)], 1)
    train = _rows(256, 10000, g)
    assert len(torch.unique(train)) == 256
    _check_against_fp64(x.float().to(DEV), lat, train, _rows(256, 2000, g))


def test_repeats_are_bit_identical():
    from disvae.evaluate import sap_score
    lat = [1, 3, 6, 40, 32, 32]
    mu = _layout(torch.randn(int(np.prod(lat)), 10, device=DEV), "q_zCx")
    runs = [sap_score(mu, lat, seed=3) for _ in range(3)]
    for score, helpers in runs[1:]:
        assert score == runs[0][0]
        for key in ("score_matrix", "coef", "solver_iterations"):
            assert torch.equal(helpers[key].nan_to_num(0), runs[0][1][key].nan_to_num(0)), key


def test_refusals_launch_nothing():
    from disvae import _native
    L = _native.lib()
    mu = torch.randn(100, 8, device=DEV)
    rows = torch.zeros(16, dtype=torch.int64, device=DEV)
    cls = torch.zeros(2, 16, dtype=torch.int32, device=DEV)
    ncl = torch.ones(2, dtype=torch.int32, device=DEV)
    cnt = torch.full((2, 4), 16, dtype=torch.int32, device=DEV)
    score = torch.full((8, 2), 7.0, device=DEV)
    coef = torch.full((8, 2, 4, 2), 7.0, dtype=torch.float64, device=DEV)
    iters = torch.full((8, 2, 4), 7, dtype=torch.int32, device=DEV)
    S = torch.cuda.current_stream().cuda_stream

    def args(mu=mu.data_ptr(), ld=1, rs=8, N=100, D=8, tr=rows.data_ptr(), ntr=16, te=rows.data_ptr(), nte=16,
             trc=cls.data_ptr(), tec=cls.data_ptr(), ncl=ncl.data_ptr(), cnt=cnt.data_ptr(), K=2, cs=4, C=0.01,
             score=score.data_ptr(), coef=coef.data_ptr(), iters=iters.data_ptr()):
        return (mu, ld, rs, N, D, tr, ntr, te, nte, trc, tec, ncl, cnt, K, cs, C, score, coef, iters, S)

    def refused(rc_want, **kw):
        torch.cuda.synchronize()
        before = L.dv_launch_count()
        rc = L.dv_sap_score_matrix(*args(**kw))
        torch.cuda.synchronize()
        assert rc == rc_want and L.dv_launch_count() == before, (kw, rc)

    for shape in (dict(N=0), dict(D=0), dict(D=1025), dict(ntr=0), dict(ntr=32769), dict(nte=0), dict(K=0),
                  dict(cs=0), dict(cs=257), dict(ld=0), dict(ld=-1), dict(rs=0), dict(rs=-8)):
        refused(DV_ERR_BAD_SHAPE, **shape)
    for bad in (dict(mu=None), dict(tr=None), dict(te=None), dict(trc=None), dict(tec=None), dict(ncl=None),
                dict(cnt=None), dict(score=None), dict(C=0.0), dict(C=-1.0), dict(C=float("nan")),
                dict(C=float("inf")), dict(mu=mu.data_ptr() + 2), dict(tr=rows.data_ptr() + 4),
                dict(te=rows.data_ptr() + 4), dict(trc=cls.data_ptr() + 2), dict(tec=cls.data_ptr() + 2),
                dict(ncl=ncl.data_ptr() + 2), dict(cnt=cnt.data_ptr() + 2), dict(score=score.data_ptr() + 2),
                dict(coef=coef.data_ptr() + 4), dict(iters=iters.data_ptr() + 2)):
        refused(DV_ERR_BAD_ARG, **bad)
    assert (score == 7).all() and (coef == 7).all() and (iters == 7).all()
    before = L.dv_launch_count()
    assert L.dv_sap_score_matrix(*args(coef=None, iters=None)) == 0 and L.dv_launch_count() == before + 1
    torch.cuda.synchronize()
    assert (score == 1).all()                      # one class everywhere: every row predicted right


# ---- known answers ------------------------------------------------------------------------------------------------
def test_constant_representation_scores_zero():
    from disvae.evaluate import sap_score
    lat = [3, 4, 5]
    score, helpers = sap_score(torch.full((60, 6), 0.25, device=DEV), lat, seed=2)
    assert score == {"SAP": 0.0}
    m = helpers["score_matrix"]
    assert (m == m[:1]).all()


def test_aligned_binary_factors_score_one():
    from disvae.evaluate import sap_score
    lat = [2, 2, 2]
    g = torch.Generator().manual_seed(9)
    v = _values(lat)
    x = torch.cat([2 * v - 1, torch.randn(v.size(0), 1, generator=g, dtype=torch.float64)], 1).float().to(DEV)
    for layout in ("q_zCx", "contig"):
        score, helpers = sap_score(_layout(x, layout), lat, seed=4)
        m = helpers["score_matrix"].numpy()
        assert (m[[0, 1, 2], [0, 1, 2]] == 1).all(), m
        gen = torch.Generator(device=DEV)
        gen.manual_seed(4)
        train, test = torch.randint(8, (10000,), generator=gen, device=DEV), torch.randint(8, (5000,), generator=gen,
                                                                                         device=DEV)
        want, got = _check_against_fp64(x, lat, train, test)
        assert np.array_equal(m, got) and score == {"SAP": R.sap(got)}
        assert abs(score["SAP"] - R.sap(want)) <= np.abs(got - want).max() + 1e-12


# ---- the Evaluator on a Burgess model ----------------------------------------------------------------------------
from test_eval_resident_gpu import (K, _assert_same_eval_files, _checkpoint_model, _dataset, _evaluator,  # noqa: E402
                                    _loader, _loss, _n_samples)

SCORE_FILES = [("sap_score.log",) * 2, ("sap_score_helpers.pth",) * 2]
FACTOR_FILES = [("factor_vae_score.log",) * 2, ("factor_vae_score_helpers.pth",) * 2]


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
        for name, data, kw in (("host", loader(ds, 1000), dict(is_sap_score=True)),
                               ("dev", _loader(ds).in_order(1000), dict(is_sap_score=True)),
                               ("plain", loader(ds, 1000), {})):
            torch.manual_seed(7)
            passes.clear()
            _evaluator(model, _loss("btcvae", K ** 4), tmp_path / name)(data, is_metrics=True, is_losses=True,
                                                                           is_factor_score=True, factor_score_seed=21,
                                                                           sap_score_seed=21, **kw)
            assert len(passes) == 1, name                      # one encoding for MIG / AAM and both scores
    _assert_same_eval_files(tmp_path / "dev", tmp_path / "host", SCORE_FILES, "dev vs host", nan_equal=True)
    names = [(f, f) for f in ("metrics.log", "metric_helpers.pth", "test_losses.log")] + FACTOR_FILES
    _assert_same_eval_files(tmp_path / "host", tmp_path / "plain", names, "with vs without the score", nan_equal=True)
    assert not os.path.exists(tmp_path / "plain" / "sap_score.log")
    score = json.load(open(tmp_path / "host" / "sap_score.log"))
    helpers = torch.load(tmp_path / "host" / "sap_score_helpers.pth", weights_only=False)
    assert set(helpers) == {"score_matrix", "factors", "classes", "coef", "solver_iterations"}
    ev = _evaluator(model, None, tmp_path / "enc")
    model.eval()
    mean = ev._compute_q_zCx(loader(ds, 1000))[1][0]
    gen = torch.Generator(device=DEV)
    gen.manual_seed(21)
    n = len(ds)
    train, test = torch.randint(n, (10000,), generator=gen, device=DEV), torch.randint(n, (5000,), generator=gen,
                                                                                     device=DEV)
    _, got = _check_against_fp64(mean.contiguous(), [int(s) for s in ds.lat_sizes], train, test)
    assert np.array_equal(helpers["score_matrix"].numpy(), got) and score == {"SAP": R.sap(got)}
    assert ev.compute_sap_score(loader(ds, 1000), seed=21) == score
