"""Modularity and explicitness on the GPU: `dv_discrete_mutual_info` and `dv_explicitness_fit` (csrc/dv_modularity.cu)
through the raw C ABI against the fp64 numpy restatement of tests/modularity_reference.py on the same rows and labels,
on guarded buffers, in four layouts of mu, with bit-identical repeats:
- the histogram edges (so the bins and the contingency counts) bit for bit, the mutual information within 1e-12;
- the standardisation within 1e-12 (fp64 sums of up to 32,768 rows in another order), every fit to the restatement's minimiser (coefficients within 1e-7 of their scale
  and the KKT residual within 1e-8 of its scale, as tests/test_score_paths_gpu.py holds dv_logistic_fit), the
  probabilities within 1e-12 of the kernel's own coefficients, and every AUC exactly equal to the pair count over the
  kernel's own probabilities;
- refusals that launch nothing, a captured graph that replays to the eager bits, a full-size dSprites-shaped score;
and `modularity_explicitness` / `Evaluator.compute_modularity_explicitness`: host and resident loaders, isolation from
the other scores and the global generators, and a known ordering.
"""
import logging

import numpy as np
import pytest
import torch

import beta_vae_reference as BR
import modularity_reference as R
from score_kernels import (DEV, DV_ERR_BAD_ARG, DV_ERR_BAD_SHAPE, DV_ERR_WORKSPACE, LAYOUTS, Buf, _call, _Code, _code,
                           _Factors, _graph_replays, _lib, _rows, grid_values, place_mu)

pytestmark = pytest.mark.gpu
MI_TOL = 1e-12
STD_RTOL = 1e-12         # the kernel's fixed-order fp64 sums against numpy's pairwise ones
COEF_RTOL, KKT_TOL = 1e-7, 1e-8
PROBA_TOL = 1e-12


class ModCase:
    """One call of each entry point through the raw ABI, every operand in a guarded buffer."""

    def __init__(self, x, lat_sizes, train_rows, test_rows, layout="contiguous"):
        from disvae.evaluate import sap_labels
        self.x = x
        self.tr, self.te = train_rows.to(DEV), test_rows.to(DEV)
        self.factors, train_cls, test_cls, n_classes, counts, _ = sap_labels(lat_sizes, self.tr, self.te)
        self.mu, self.ld, self.rs = place_mu(x, layout)
        self.K, self.S = counts.shape
        self.n, self.m, self.D = len(train_rows), len(test_rows), x.shape[1]
        self.inputs = [Buf(t.numel(), t.dtype, t) for t in (self.tr, self.te, train_cls, test_cls, n_classes)]
        self.train_cls, self.test_cls = train_cls.cpu().numpy(), test_cls.cpu().numpy()
        self.n_classes = n_classes.cpu().numpy()
        L, _ = _lib()
        self.ws_bytes = L.dv_explicitness_workspace_bytes(self.D, self.n, self.m, self.K, self.S)
        assert self.ws_bytes > 0
        K, S, D, rows = self.K, self.S, self.D, self.n + self.m
        self.mi_outs = [Buf(D * K, torch.float64), Buf(D * 21, torch.float32)]
        self.outs = [Buf(K * S * (D + 1), torch.float64), Buf(2 * K * S, torch.float64), Buf(K, torch.int32),
                     Buf(D, torch.float64), Buf(D, torch.float64), Buf(K * S * rows, torch.float64)]
        self.ws = Buf((self.ws_bytes + 7) // 8, torch.float64, float("nan"))

    def mi_args(self, **kw):
        tr, _, cls, _, ncl = (b.ptr for b in self.inputs)
        a = dict(mu=self.mu.ptr, ld=self.ld, rs=self.rs, N=self.x.shape[0], D=self.D, tr=tr, ntr=self.n, cls=cls,
                 ncl=ncl, K=self.K, S=self.S, mi=self.mi_outs[0].ptr, edges=self.mi_outs[1].ptr)
        a.update(kw)
        return tuple(a.values()) + (_lib()[1],)

    def fit_args(self, **kw):
        tr, te, cls, tcls, ncl = (b.ptr for b in self.inputs)
        coef, auc, it, mean, std, proba = (b.ptr for b in self.outs)
        a = dict(mu=self.mu.ptr, ld=self.ld, rs=self.rs, N=self.x.shape[0], D=self.D, tr=tr, ntr=self.n, te=te,
                 nte=self.m, cls=cls, tcls=tcls, ncl=ncl, K=self.K, S=self.S, coef=coef, auc=auc, it=it, mean=mean,
                 std=std, proba=proba, ws=self.ws.ptr, wsb=self.ws_bytes)
        a.update(kw)
        return tuple(a.values()) + (_lib()[1],)

    def _twice(self, launches, name, args, outs):
        got = []
        for _ in range(2):
            for b in outs:
                b.body.view(torch.uint8).fill_(0xA5)
            _call(launches, name, *args)
            got.append([b.body.clone() for b in outs])
            assert all(b.intact() for b in outs + [self.ws] + self.inputs), "a write past a buffer"
            assert self.mu.intact()
        for a, b in zip(*got):
            assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), name + ": a repeat differs"
        return [t.cpu().numpy() for t in got[0]]

    def run(self):
        mi, edges = self._twice(1, "dv_discrete_mutual_info", self.mi_args(), self.mi_outs)
        fit = self._twice(3, "dv_explicitness_fit", self.fit_args(), self.outs)
        K, S, D, rows = self.K, self.S, self.D, self.n + self.m
        coef, auc, it, mean, std, proba = fit
        return (mi.reshape(D, K), edges.reshape(D, 21), coef.reshape(K, S, D + 1), auc.reshape(2, K, S), it, mean,
                std, proba.reshape(K, S, rows))

    def check(self, got=None, factors=None):
        """The kernels' outputs against the restatement (fits of the factors `factors`, all by default)."""
        mi, edges, coef, auc, it, mean, std, proba = self.run() if got is None else got
        x = self.x.cpu().numpy().astype(np.float32)
        tr, te = self.tr.cpu().numpy(), self.te.cpu().numpy()
        want_mi, want_edges = R.mutual_information(x[tr], self.train_cls)
        assert np.array_equal(edges, want_edges), "edges"
        assert np.abs(mi - want_mi).max() <= MI_TOL, ("mutual information", np.abs(mi - want_mi).max())
        ft, fe, wmean, wstd = R.standardise(x[tr], x[te])
        assert np.abs(mean - wmean).max() <= STD_RTOL * max(1.0, np.abs(wmean).max())
        assert np.abs(std - wstd).max() <= STD_RTOL * max(1.0, np.abs(wstd).max())
        feats = np.r_[ft, fe]
        for k in range(self.K) if factors is None else factors:
            nc = int(self.n_classes[k])
            cols = R.columns(nc)
            assert np.isnan(proba[k, cols:]).all() and np.isnan(auc[:, k, cols:]).all()
            if nc < 2:
                assert it[k] == 0 and np.isnan(coef[k]).all()
                continue
            rows = nc if nc > 2 else 1
            assert np.isnan(coef[k, rows:]).all() and not np.isnan(coef[k, :rows]).any()
            assert it[k] >= 0, ("did not converge", k)
            W, b = coef[k, :rows, :-1], coef[k, :rows, -1]
            wW, wb, _ = BR.fit(ft, self.train_cls[k], nc)
            ref = max(np.abs(wW).max(), np.abs(wb).max(), 1e-300)
            err = max(np.abs(W - wW).max(), np.abs(b - wb).max())
            _, gr, sc = BR.objective(ft, self.train_cls[k], nc, W, b)
            assert err <= COEF_RTOL * ref and np.abs(gr).max() <= KKT_TOL * sc.max(), ("fit", k, err / ref)
            p = R.probabilities(W, b, nc, feats)
            assert np.abs(proba[k, :cols].T - p).max() <= PROBA_TOL, ("probabilities", k)
            for c in range(cols):
                for s, (lab, sl) in enumerate(((self.train_cls[k], slice(0, self.n)),
                                               (self.test_cls[k], slice(self.n, None)))):
                    want = R.auc(proba[k, c, sl], lab, c)
                    assert (np.isnan(want) and np.isnan(auc[s, k, c])) or auc[s, k, c] == want, ("auc", k, c, s)
        return mi, edges, coef, auc, it, mean, std, proba


# ---- kernels against the restatement -------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", LAYOUTS)
def test_class_counts_1_2_3_40_every_layout(layout):
    """Factor 0 shows one value in training (no fit), factor 1 two, factor 2 three, factor 3 forty; the four layouts
    of mu give the same bits."""
    lat = [2, 2, 3, 40]
    x = _code(lat, 10, 1)
    n = x.size(0)
    tr = _rows(n, 3000, 2, where=torch.arange(n // 2, n))          # factor 0 = 1 on every training row
    case = ModCase(x, lat, tr, _rows(n, 1000, 3), layout=layout)
    assert case.n_classes.tolist() == [1, 2, 3, 40]
    got = case.check()
    assert (got[0][:, 0] == 0).all()                               # no mutual information with a one-class factor
    if layout != "contiguous":
        base = ModCase(x, lat, tr, _rows(n, 1000, 3)).run()
        for a, b in zip(got, base):
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), layout


def test_256_classes():
    lat = [256, 2]
    x = _code(lat, 2, 4)
    case = ModCase(x, lat, _rows(512, 6000, 5), _rows(512, 500, 6))
    assert case.n_classes.tolist() == [256, 2]
    case.check()


@pytest.mark.parametrize("D, n, m", [(1, 800, 300), (2, 2, 50), (10, 19, 40), (10, 20, 40), (10, 21, 40),
                                     (10, 10000, 5000), (3, 32768, 1000), (128, 1500, 300)])
def test_dims_and_rows(D, n, m):
    lat = [4, 5]
    x = _code(lat, D, D + n)
    case = ModCase(x, lat, _rows(20, n, 7), _rows(20, m, 8))
    case.check()


def test_one_training_row():
    lat = [4, 5]
    case = ModCase(_code(lat, 3, 9), lat, _rows(20, 1, 10), _rows(20, 30, 11))
    mi, edges, coef, auc, it, *_ = case.check()
    assert (mi == 0).all() and np.isnan(auc).all() and (it == 0).all()
    assert (np.diff(edges, axis=1) > 0).all()                    # one value: lo - 0.5 .. hi + 0.5


def test_constant_duplicated_edge_valued_and_refused_latents():
    """Latent 0 constant (std 1, one bin), latent 1 a copy of latent 4, latent 2 on the edges of its own histogram,
    latent 3 a range of a few ulps (numpy refuses it; the same edges bin it), latent 4 informative."""
    lat = [6, 5, 4]
    v = grid_values(lat).float()
    n = v.size(0)
    g = torch.Generator().manual_seed(12)
    x4 = v[:, 1] + 0.4 * torch.randn(n, generator=g)
    e = torch.from_numpy(R.edges(np.array([-1.0, 3.0], np.float32)))
    on_edges = e[torch.randint(0, 21, (n,), generator=g)]
    on_edges[:2] = torch.tensor([-1.0, 3.0])                       # the extremes are present: the edges are e
    ulps = (1.0 + torch.randint(0, 4, (n,), generator=g).double() * 2.0 ** -23).float()
    x = torch.stack([torch.full((n,), 0.375), x4, on_edges, ulps, x4], 1)
    tr = torch.cat([torch.tensor([int(torch.argmin(x[:, 2])), int(torch.argmax(x[:, 2]))]), _rows(n, 3998, 13)])
    case = ModCase(x, lat, tr, _rows(n, 1000, 14))
    mi, edges, coef, auc, it, mean, std, proba = case.check()
    assert std[0] == 1.0 and (mi[0] == 0).all()
    assert np.array_equal(mi[1], mi[4])
    assert np.array_equal(edges[2], e.numpy())
    assert (np.diff(edges[3]) <= 0).any()


def test_tied_probabilities_and_unseen_test_values():
    """One latent on a coarse grid, so rows share their probabilities (ties across positives and negatives, in
    column 0 of a binary factor as well); no training row has value 5 of the 6-value factor, which test rows have."""
    lat = [2, 6, 3]
    v = grid_values(lat).float()
    x = torch.round(v[:, :1] + 0.7 * torch.randn(v.size(0), 1, generator=torch.Generator().manual_seed(15)))
    case = ModCase(x, lat, _rows(v.size(0), 40, 16, where=torch.nonzero(v[:, 1] < 5)[:, 0]),
                   _rows(v.size(0), 2000, 17))
    assert case.n_classes.tolist() == [2, 5, 3]
    got = case.check()
    proba = got[-1]
    assert len(np.unique(proba[0, 0])) < 20
    assert (case.test_cls == -1).any()


def test_workspace_and_refusals_launch_nothing():
    lat = [3, 4]
    case = ModCase(_code(lat, 4, 18), lat, _rows(12, 100, 19), _rows(12, 50, 20))
    L, _ = _lib()
    for b in case.outs + case.mi_outs:
        b.body.view(torch.uint8).fill_(0x11)

    def refused(fn, args, want):
        torch.cuda.synchronize()
        before = L.dv_launch_count()
        rc = getattr(L, fn)(*args)
        torch.cuda.synchronize()
        assert rc == want and L.dv_launch_count() == before, (fn, rc)

    for shape in (dict(N=0), dict(D=0), dict(D=1025), dict(ntr=0), dict(ntr=32769), dict(K=0), dict(S=0),
                  dict(S=257), dict(ld=0), dict(rs=-1)):
        refused("dv_discrete_mutual_info", case.mi_args(**shape), DV_ERR_BAD_SHAPE)
    tr, te, cls, tcls, ncl = (b.ptr for b in case.inputs)
    for bad in (dict(mu=None), dict(tr=None), dict(cls=None), dict(ncl=None), dict(mi=None), dict(mu=case.mu.ptr + 2),
                dict(tr=tr + 4), dict(cls=cls + 2), dict(ncl=ncl + 2), dict(mi=case.mi_outs[0].ptr + 4),
                dict(edges=case.mi_outs[1].ptr + 2)):
        refused("dv_discrete_mutual_info", case.mi_args(**bad), DV_ERR_BAD_ARG)
    for shape in (dict(N=0), dict(D=0), dict(D=129), dict(ntr=0), dict(ntr=32769), dict(nte=0), dict(K=0),
                  dict(S=0), dict(S=257), dict(ld=0), dict(ld=-1), dict(rs=0)):
        refused("dv_explicitness_fit", case.fit_args(**shape), DV_ERR_BAD_SHAPE)
    o = [b.ptr for b in case.outs]
    for bad in (dict(mu=None), dict(tr=None), dict(te=None), dict(cls=None), dict(tcls=None), dict(ncl=None),
                dict(coef=None), dict(auc=None), dict(it=None), dict(mean=None), dict(std=None),
                dict(mu=case.mu.ptr + 2), dict(tr=tr + 4), dict(te=te + 4), dict(cls=cls + 2), dict(tcls=tcls + 2),
                dict(ncl=ncl + 2), dict(coef=o[0] + 4), dict(auc=o[1] + 4), dict(it=o[2] + 2), dict(mean=o[3] + 4),
                dict(std=o[4] + 4), dict(proba=o[5] + 4), dict(ws=case.ws.ptr + 4)):
        refused("dv_explicitness_fit", case.fit_args(**bad), DV_ERR_BAD_ARG)
    refused("dv_explicitness_fit", case.fit_args(ws=None), DV_ERR_WORKSPACE)
    refused("dv_explicitness_fit", case.fit_args(wsb=case.ws_bytes - 1), DV_ERR_WORKSPACE)
    for b in case.outs + case.mi_outs:
        assert (b.body.view(torch.uint8) == 0x11).all() and b.intact()
    for q in (dict(D=0), dict(D=129), dict(ntr=0), dict(ntr=32769), dict(nte=0), dict(K=0), dict(S=257)):
        a = dict(D=4, ntr=100, nte=50, K=2, S=4)
        a.update(q)
        assert L.dv_explicitness_workspace_bytes(a["D"], a["ntr"], a["nte"], a["K"], a["S"]) == 0, q
    before = L.dv_launch_count()
    assert L.dv_explicitness_fit(*case.fit_args(proba=None)) == 0 and L.dv_launch_count() == before + 3
    assert L.dv_discrete_mutual_info(*case.mi_args(edges=None)) == 0 and L.dv_launch_count() == before + 4
    torch.cuda.synchronize()
    assert (case.outs[5].body.view(torch.uint8) == 0x11).all()     # no probabilities asked for, none written
    assert (case.mi_outs[1].body.view(torch.uint8) == 0x11).all()


def test_graph_replay_equals_eager():
    lat = [3, 6]
    case = ModCase(_code(lat, 5, 21), lat, _rows(18, 2000, 22), _rows(18, 300, 23))
    case.run()
    L, _ = _lib()
    _graph_replays(lambda: L.dv_discrete_mutual_info(*case.mi_args()), case.mi_outs, "dv_discrete_mutual_info")
    _graph_replays(lambda: L.dv_explicitness_fit(*case.fit_args()), case.outs, "dv_explicitness_fit")


def test_full_size_dsprites_shape():
    """dSprites' factor grid (1, 3, 6, 40, 32, 32; 737,280 rows), 10 latents, 10,000 / 5,000 rows: every factor against
    the restatement, and the whole score through `modularity_explicitness`."""
    from disvae import evaluate
    lat = [1, 3, 6, 40, 32, 32]
    x = _code(lat[1:], 10, 24, noise=0.2)
    case = ModCase(x, lat, _rows(x.size(0), 10000, 25), _rows(x.size(0), 5000, 26))
    got = case.run()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    _lib()[0].dv_explicitness_fit(*case.fit_args())
    end.record()
    torch.cuda.synchronize()
    print("full-size dv_explicitness_fit: %.1f ms, Newton steps %s" % (start.elapsed_time(end), got[4].tolist()))
    case.check(got)
    score, helpers = evaluate.modularity_explicitness(x.to(DEV), lat, seed=27)
    assert 0 < score["modularity_score"] <= 1
    assert 0.5 < score["explicitness_score_test"] <= 1 and 0.5 < score["explicitness_score_train"] <= 1
    assert helpers["mutual_information"].shape == (10, 5) and (helpers["solver_iterations"] >= 0).all()


# ---- modularity_explicitness and the Evaluator ---------------------------------------------------------------------
from test_eval_resident_gpu import _assert_same_eval_files, _checkpoint_model, _dataset, _evaluator, _loader  # noqa
from test_eval_resident_gpu import _loss, _n_samples, K as GRID_K  # noqa: E402


def test_repeats_and_loaders_agree():
    import disvae
    from synthetic_factors import loader
    ds = _dataset()
    model = _checkpoint_model()
    ev = disvae.Evaluator(model, None, device=DEV, logger=logging.getLogger("mod"), save_dir="unused",
                          is_progress_bar=False)
    host = ev.compute_modularity_explicitness(loader(ds, 1000), seed=5)
    dev = ev.compute_modularity_explicitness(_loader(ds).in_order(1000), seed=5)
    assert host == dev
    from disvae.evaluate import modularity_explicitness
    mean = ev._compute_q_zCx(loader(ds, 1000))[1][0]
    runs = [modularity_explicitness(mean, [int(s) for s in ds.lat_sizes], seed=5) for _ in range(2)]
    assert runs[0][0] == runs[1][0] == host
    for key in runs[0][1]:
        a, b = runs[0][1][key], runs[1][1][key]
        assert torch.equal(a.nan_to_num(7.0), b.nan_to_num(7.0)) if a.is_floating_point() else torch.equal(a, b), key
    assert runs[0][1]["mutual_information"].shape == (10, 4)
    assert set(host) == {"modularity_score", "explicitness_score_train", "explicitness_score_test"}


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
            if name == "b":                                     # a modularity score between the two evaluations
                from disvae.evaluate import modularity_explicitness
                mean = ev._compute_q_zCx(loader(ds, 1000))[1][0]
                cpu, cuda = torch.get_rng_state(), torch.cuda.get_rng_state()
                modularity_explicitness(mean, [int(s) for s in ds.lat_sizes], seed=3)
                assert torch.equal(cpu, torch.get_rng_state()) and torch.equal(cuda, torch.cuda.get_rng_state())
                ev.compute_modularity_explicitness(loader(ds, 1000), seed=3)
            torch.manual_seed(7)
            ev(loader(ds, 1000), is_metrics=True, is_losses=False, is_factor_score=True, is_sap_score=True,
               is_beta_vae_score=True)
    _assert_same_eval_files(tmp_path / "a", tmp_path / "b", files, "with vs without a modularity score",
                            nan_equal=True)


def test_known_ordering_aligned_rotated_and_noise(tmp_path):
    """An axis-aligned code has higher modularity than the same code rotated by 45 degrees in pairs of latents; an
    informative code has higher explicitness than pure noise, whose AUCs sit near 0.5."""
    import disvae
    lat = [5, 6, 4, 5]
    ds = _Factors(lat, 0.01, 28)
    dl = torch.utils.data.DataLoader(ds, batch_size=200, shuffle=False)
    theta = torch.tensor(np.pi / 4)
    rot = torch.eye(4)
    rot[:2, :2] = torch.tensor([[torch.cos(theta), -torch.sin(theta)], [torch.sin(theta), torch.cos(theta)]])
    rot[2:, 2:] = rot[:2, :2]
    scores = {}
    for name, M in (("aligned", torch.eye(4)), ("rotated", rot), ("noise", torch.zeros(4, 4))):
        model = _Code(M)
        if name == "noise":                                        # means independent of the factors
            g = torch.Generator().manual_seed(29)
            noise = torch.randn(len(ds), 4, generator=g)
            ds_noise = _Factors(lat, 0.0, 28)
            ds_noise.imgs.view(len(ds), -1)[:, :4] = noise
            dl_use = torch.utils.data.DataLoader(ds_noise, batch_size=200, shuffle=False)
            model = _Code(torch.eye(4))
        else:
            dl_use = dl
        ev = disvae.Evaluator(model, None, device=DEV, logger=logging.getLogger("mod"), save_dir=str(tmp_path),
                              is_progress_bar=False)
        scores[name] = ev.compute_modularity_explicitness(dl_use, num_train=2000, num_test=1000, seed=1)
    a, r, z = scores["aligned"], scores["rotated"], scores["noise"]
    assert a["modularity_score"] > 0.9 and r["modularity_score"] < a["modularity_score"] - 0.2, (a, r)
    assert a["explicitness_score_test"] > 0.9, a
    assert abs(z["explicitness_score_test"] - 0.5) < 0.05 and z["explicitness_score_test"] < a["explicitness_score_test"]
