"""The DCI score on the GPU: `dv_dci_fit` (csrc/dv_dci.cu) through the raw C ABI against the fp64 numpy restatement of
tests/dci_reference.py on the same rows and labels -- the same tree structure (latent and threshold bits of every
node), the same predictions, leaf values and importances within 1e-12 -- on guarded buffers, in four layouts of mu,
with bit-identical repeats; refusals that launch nothing; a full-size dSprites-shaped fit; and `dci_score` /
`Evaluator.compute_dci_score`: repeats, host and resident loaders, isolation from the other scores and the global
generators, and a known answer.
"""
import logging

import numpy as np
import pytest
import torch

import dci_reference as R
from score_kernels import (DEV, DV_ERR_BAD_ARG, DV_ERR_BAD_SHAPE, DV_ERR_WORKSPACE, LAYOUTS, Buf, _call, _Code, _code,
                           _Factors, _graph_replays, _lib, _rows, grid_values, place_mu)

pytestmark = pytest.mark.gpu
VALUE_RTOL = 1e-12        # leaf values, against max(1, |fp64 value|)
IMPORTANCE_TOL = 1e-12    # importances sum to 1


class DciCase:
    """One fit through the raw ABI, every operand in a guarded buffer."""

    def __init__(self, x, lat_sizes, train_rows, test_rows, stages, layout="contiguous"):
        from disvae.evaluate import sap_labels
        self.x, self.stages = x, stages
        self.tr, self.te = train_rows.to(DEV), test_rows.to(DEV)
        self.factors, train_cls, _, n_classes, counts, _ = sap_labels(lat_sizes, self.tr, self.te)
        self.mu, self.ld, self.rs = place_mu(x, layout)
        self.K, self.S = counts.shape
        self.n, self.m, self.D = len(train_rows), len(test_rows), x.shape[1]
        self.inputs = [Buf(t.numel(), t.dtype, t) for t in (self.tr, self.te, train_cls, n_classes, counts)]
        self.train_cls, self.n_classes = train_cls.cpu().numpy(), n_classes.cpu().numpy()
        L, _ = _lib()
        self.ws_bytes = L.dv_dci_workspace_bytes(self.D, self.n, self.m, self.K, self.S)
        assert self.ws_bytes > 0
        T = self.K * self.S * stages * R.NODES
        self.outs = [Buf(self.D * self.K, torch.float64), Buf(self.K * (self.n + self.m), torch.int32),
                     Buf(T, torch.int32), Buf(T, torch.float64), Buf(T, torch.float64)]
        self.ws = Buf((self.ws_bytes + 7) // 8, torch.float64, float("nan"))

    def args(self, **kw):
        tr, te, cls, ncl, cnt = (b.ptr for b in self.inputs)
        imp, pred, tf, tt, tv = (b.ptr for b in self.outs)
        a = dict(mu=self.mu.ptr, ld=self.ld, rs=self.rs, N=self.x.shape[0], D=self.D, tr=tr, ntr=self.n, te=te,
                 nte=self.m, cls=cls, ncl=ncl, cnt=cnt, K=self.K, S=self.S, stages=self.stages, imp=imp, pred=pred,
                 tf=tf, tt=tt, tv=tv, ws=self.ws.ptr, wsb=self.ws_bytes)
        a.update(kw)
        return tuple(a.values()) + (_lib()[1],)

    def run(self):
        """Two runs (the second on the first's workspace): bit-identical, inside their buffers -> numpy outputs."""
        got = []
        for _ in range(2):
            for b in self.outs:
                b.body.view(torch.uint8).fill_(0xA5)
            _call(4 + 2 * self.stages, "dv_dci_fit", *self.args())
            got.append([b.body.clone() for b in self.outs])
            assert all(b.intact() for b in self.outs + [self.ws] + self.inputs), "a write past a buffer"
            assert self.mu.intact()
        for a, b in zip(*got):
            assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), "a repeat differs"
        imp, pred, tf, tt, tv = (t.cpu().numpy() for t in got[0])
        shape = (self.K, self.S, self.stages, R.NODES)
        return (imp.reshape(self.D, self.K), pred.reshape(self.K, -1), tf.reshape(shape), tt.reshape(shape),
                tv.reshape(shape))

    def check(self, got=None, factors=None, stages=None):
        """The kernel's outputs against the restatement (on factors `factors`, the first `stages` stages)."""
        imp, pred, tf, tt, tv = self.run() if got is None else got
        stages = self.stages if stages is None else stages
        ks = range(self.K) if factors is None else factors
        x = self.x.cpu().numpy()
        tr, te = self.tr.cpu().numpy(), self.te.cpu().numpy()
        for k in ks:
            nc = int(self.n_classes[k])
            f = R.fit(x[tr], self.train_cls[k], nc, x[te], stages)
            cols = nc if nc > 2 else max(nc - 1, 0)
            assert (tf[k, cols:] == R.ABSENT).all() and np.isnan(tt[k, cols:]).all() and np.isnan(tv[k, cols:]).all()
            feat, thr, val = tf[k, :cols, :stages], tt[k, :cols, :stages], tv[k, :cols, :stages]
            bad = np.argwhere(feat != f["feature"])
            assert not len(bad), ("tree structure", k, bad[:3], feat[tuple(bad[0][:2])], f["feature"][tuple(bad[0][:2])])
            assert np.array_equal(np.isnan(thr), np.isnan(f["threshold"]))
            assert np.array_equal(thr[~np.isnan(thr)], f["threshold"][~np.isnan(thr)]), ("thresholds", k)
            assert np.array_equal(np.isnan(val), np.isnan(f["value"]))
            err = np.abs(val - f["value"])[~np.isnan(val)] / np.maximum(1, np.abs(f["value"][~np.isnan(val)]))
            assert err.size == 0 or err.max() <= VALUE_RTOL, ("leaf values", k, err.max())
            if stages == self.stages:
                assert np.array_equal(pred[k], np.concatenate([f["pred_train"], f["pred_test"]])), ("pred", k)
                assert np.abs(imp[:, k] - f["importance"]).max() <= IMPORTANCE_TOL, ("importance", k)
        return imp, pred, tf, tt, tv


# ---- kernel against the restatement -------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", LAYOUTS)
def test_class_counts_1_2_3_40_every_layout(layout):
    """Factor 0 shows one value in training (no trees), factor 1 two, factor 2 three, factor 3 forty; the four layouts
    of mu give the same bits."""
    lat = [2, 2, 3, 40]
    x = _code(lat, 10, 1)
    n = x.size(0)
    tr = _rows(n, 3000, 2, where=torch.arange(n // 2, n))          # factor 0 = 1 on every training row
    case = DciCase(x, lat, tr, _rows(n, 1000, 3), stages=4, layout=layout)
    assert case.n_classes.tolist() == [1, 2, 3, 40]
    got = case.check()
    assert (got[0][:, 0] == 0).all() and (got[1][0] == 0).all()
    if layout != "contiguous":
        base = DciCase(x, lat, tr, _rows(n, 1000, 3), stages=4).run()
        for a, b in zip(got, base):
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), layout


def test_256_classes():
    lat = [256, 2]
    x = _code(lat, 4, 4)
    case = DciCase(x, lat, _rows(512, 6000, 5), _rows(512, 500, 6), stages=2)
    assert case.n_classes.tolist() == [256, 2]
    case.check()


@pytest.mark.parametrize("D, n, m, stages", [(2, 800, 300, 10), (1024, 300, 100, 2), (5, 2, 50, 5), (3, 32768, 1000, 2),
                                             (10, 5000, 2000, 0)])
def test_dims_rows_and_stages(D, n, m, stages):
    lat = [4, 5]
    x = _code(lat, D, D + n)
    case = DciCase(x, lat, _rows(20, n, 7), _rows(20, m, 8), stages=stages)
    imp, pred, *_ = case.check()
    if stages == 0:
        assert (imp == 0).all()


def test_repeated_near_equal_constant_and_duplicated_latents():
    """Latent 0 on a grid of 0.25 (repeated values), latent 1 the same plus steps of 6e-8 (gaps at or below 1e-7,
    never a candidate) and of 2e-7, latent 2 constant, latent 3 a copy of latent 5 (the lowest latent wins the tie),
    latent 4 noise."""
    lat = [6, 5, 4]
    v = grid_values(lat).float()
    n = v.size(0)
    g = torch.Generator().manual_seed(9)
    base = torch.round((v[:, 0] / 2 + 0.5 * torch.randn(n, generator=g)) * 4) / 4
    steps = torch.randint(0, 3, (n,), generator=g).float()
    x5 = v[:, 1] + 0.4 * torch.randn(n, generator=g)
    x = torch.stack([base, (base.double() + torch.where(steps == 2, 2e-7, 6e-8 * steps).double()).float(),
                     torch.full((n,), 0.375), x5, torch.randn(n, generator=g), x5], 1)
    case = DciCase(x, lat, _rows(n, 4000, 10), _rows(n, 1000, 11), stages=5)
    imp, pred, tf, tt, tv = case.check()
    assert (tf != 5).all() and (tf == 3).any()                 # the copy never wins over the original
    assert (tf != 2).all()                                     # a constant latent has no candidate
    assert (imp[2] == 0).all() and (imp[5] == 0).all()


def test_equal_residuals_make_leaves():
    """A binary factor that latent 0 separates: after the root split every row of a child has the same residual,
    so the children are leaves by the impurity rule, above depth 3 and with many rows."""
    lat = [2, 3]
    v = grid_values(lat).float()
    x = torch.stack([v[:, 0] * 2 - 1, torch.randn(6, generator=torch.Generator().manual_seed(12))], 1)
    case = DciCase(x, lat, _rows(6, 3000, 13), _rows(6, 500, 14), stages=3)
    imp, pred, tf, tt, tv = case.check()
    assert (tf[0, 0, 0, :3] == [0, R.LEAF, R.LEAF]).all()
    assert imp[0, 0] == 1.0 and np.array_equal(pred[0, :case.n], case.train_cls[0])


def test_workspace_and_refusals_launch_nothing():
    lat = [3, 4]
    x = _code(lat, 4, 15)
    case = DciCase(x, lat, _rows(12, 100, 16), _rows(12, 50, 17), stages=2)
    L, _ = _lib()
    for b in case.outs:
        b.body.view(torch.uint8).fill_(0x11)

    def refused(want, **kw):
        torch.cuda.synchronize()
        before = L.dv_launch_count()
        rc = L.dv_dci_fit(*case.args(**kw))
        torch.cuda.synchronize()
        assert rc == want and L.dv_launch_count() == before, (kw, rc)

    for shape in (dict(N=0), dict(D=0), dict(D=1025), dict(ntr=0), dict(ntr=32769), dict(nte=0), dict(K=0),
                  dict(S=0), dict(S=257), dict(stages=-1), dict(ld=0), dict(ld=-1), dict(rs=0), dict(rs=-4),
                  dict(K=2, S=256, stages=2 ** 31 // (2 * 256 * 15) + 1)):
        refused(DV_ERR_BAD_SHAPE, **shape)
    for bad in (dict(mu=None), dict(tr=None), dict(te=None), dict(cls=None), dict(ncl=None), dict(cnt=None),
                dict(imp=None), dict(pred=None), dict(mu=case.mu.ptr + 2), dict(tr=case.inputs[0].ptr + 4),
                dict(te=case.inputs[1].ptr + 4), dict(cls=case.inputs[2].ptr + 2), dict(ncl=case.inputs[3].ptr + 2),
                dict(cnt=case.inputs[4].ptr + 2), dict(imp=case.outs[0].ptr + 4), dict(pred=case.outs[1].ptr + 2),
                dict(tf=case.outs[2].ptr + 2), dict(tt=case.outs[3].ptr + 4), dict(tv=case.outs[4].ptr + 4),
                dict(ws=case.ws.ptr + 4)):
        refused(DV_ERR_BAD_ARG, **bad)
    refused(DV_ERR_WORKSPACE, ws=None)
    refused(DV_ERR_WORKSPACE, wsb=case.ws_bytes - 1)
    for b in case.outs:
        assert (b.body.view(torch.uint8) == 0x11).all() and b.intact()
    for q in (dict(D=0), dict(D=1025), dict(ntr=0), dict(ntr=32769), dict(nte=0), dict(K=0), dict(S=257)):
        a = dict(D=4, ntr=100, nte=50, K=2, S=4)
        a.update(q)
        assert L.dv_dci_workspace_bytes(a["D"], a["ntr"], a["nte"], a["K"], a["S"]) == 0, q
    before = L.dv_launch_count()
    assert L.dv_dci_fit(*case.args(tf=None, tt=None, tv=None)) == 0 and L.dv_launch_count() == before + 8
    torch.cuda.synchronize()
    assert (case.outs[2].body.view(torch.uint8) == 0x11).all()     # no tree asked for, none written


def test_graph_replay_equals_eager():
    lat = [3, 6]
    case = DciCase(_code(lat, 5, 18), lat, _rows(18, 2000, 19), _rows(18, 300, 20), stages=3)
    case.run()
    L, _ = _lib()
    _graph_replays(lambda: L.dv_dci_fit(*case.args()), case.outs, "dv_dci_fit")


def test_full_size_dsprites_shape():
    """dSprites' factor grid (1, 3, 6, 40, 32, 32; 737,280 rows), 10 latents, 10,000 / 5,000 rows, 100 stages, all
    five scored factors in one fit.  The factors of 3 and 6 values are checked against the restatement at all 100
    stages; the 40- and 32-value factors (104 columns) on their first 3 stages, which a fit of 3 stages restates."""
    from disvae import evaluate
    lat = [1, 3, 6, 40, 32, 32]
    x = _code(lat[1:], 10, 21, noise=0.2)
    case = DciCase(x, lat, _rows(x.size(0), 10000, 22), _rows(x.size(0), 5000, 23), stages=100)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    got = case.run()
    start.record()
    _lib()[0].dv_dci_fit(*case.args())
    end.record()
    torch.cuda.synchronize()
    print("full-size dv_dci_fit: %.1f ms" % start.elapsed_time(end))
    case.check(got, factors=[0, 1])
    case.check(got, factors=[2, 3, 4], stages=3)
    score, helpers = evaluate.dci_score(x.to(DEV), lat, seed=24)
    assert 0 < score["disentanglement"] <= 1 and 0 < score["completeness"] <= 1


# ---- dci_score and the Evaluator ----------------------------------------------------------------------------------
from test_eval_resident_gpu import _assert_same_eval_files, _checkpoint_model, _dataset, _evaluator, _loader  # noqa
from test_eval_resident_gpu import _loss, _n_samples, K as GRID_K  # noqa: E402


def test_repeats_and_loaders_agree():
    import disvae
    from synthetic_factors import loader
    ds = _dataset()
    model = _checkpoint_model()
    ev = disvae.Evaluator(model, None, device=DEV, logger=logging.getLogger("dci"), save_dir="unused",
                          is_progress_bar=False)
    host = ev.compute_dci_score(loader(ds, 1000), seed=5)
    dev = ev.compute_dci_score(_loader(ds).in_order(1000), seed=5)
    assert host == dev
    from disvae.evaluate import dci_score
    mean = ev._compute_q_zCx(loader(ds, 1000))[1][0]
    runs = [dci_score(mean, [int(s) for s in ds.lat_sizes], seed=5) for _ in range(2)]
    assert runs[0][0] == runs[1][0] == host
    for key in runs[0][1]:
        assert torch.equal(runs[0][1][key], runs[1][1][key]), key
    assert set(runs[0][1]) == {"importance_matrix", "factors", "classes", "train_accuracy", "test_accuracy"}
    assert runs[0][1]["importance_matrix"].shape == (10, 4)


def test_isolation_from_rng_and_other_scores(tmp_path):
    from synthetic_factors import loader
    ds = _dataset()
    model = _checkpoint_model()
    files = [(f, f) for f in ("metrics.log", "metric_helpers.pth", "factor_vae_score.log",
                              "factor_vae_score_helpers.pth", "sap_score.log", "sap_score_helpers.pth",
                              "beta_vae_score.log", "beta_vae_score_helpers.pth")]
    with _n_samples(512):
        for name in ("a", "b"):
            ev = _evaluator(model, _loss("btcvae", GRID_K ** 4), tmp_path / name)
            if name == "b":                                     # a DCI score between the two evaluations
                from disvae.evaluate import dci_score
                mean = ev._compute_q_zCx(loader(ds, 1000))[1][0]
                cpu, cuda = torch.get_rng_state(), torch.cuda.get_rng_state()
                dci_score(mean, [int(s) for s in ds.lat_sizes], seed=3)
                assert torch.equal(cpu, torch.get_rng_state()) and torch.equal(cuda, torch.cuda.get_rng_state())
                ev.compute_dci_score(loader(ds, 1000), seed=3)
            torch.manual_seed(7)
            ev(loader(ds, 1000), is_metrics=True, is_losses=False, is_factor_score=True, is_sap_score=True,
               is_beta_vae_score=True)
    _assert_same_eval_files(tmp_path / "a", tmp_path / "b", files, "with vs without a DCI score", nan_equal=True)


def test_known_answer_aligned_and_rotated_codes(tmp_path):
    import disvae
    lat = [5, 6, 4, 5]
    ds = _Factors(lat, 0.01, 25)
    dl = torch.utils.data.DataLoader(ds, batch_size=200, shuffle=False)
    theta = torch.tensor(np.pi / 4)
    rot = torch.eye(4)
    rot[:2, :2] = torch.tensor([[torch.cos(theta), -torch.sin(theta)], [torch.sin(theta), torch.cos(theta)]])
    rot[2:, 2:] = rot[:2, :2]
    scores = {}
    for name, M in (("aligned", torch.eye(4)), ("rotated", rot)):
        ev = disvae.Evaluator(_Code(M), None, device=DEV, logger=logging.getLogger("dci"), save_dir=str(tmp_path),
                              is_progress_bar=False)
        scores[name] = ev.compute_dci_score(dl, num_train=2000, num_test=1000, seed=1)
    a, r = scores["aligned"], scores["rotated"]
    assert a["disentanglement"] > 0.9 and a["completeness"] > 0.9, a
    assert a["informativeness_test"] > 0.9, a
    assert r["disentanglement"] < a["disentanglement"] - 0.3 and r["completeness"] < a["completeness"] - 0.3, (a, r)
