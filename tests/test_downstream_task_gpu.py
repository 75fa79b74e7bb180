"""The downstream-task score on the GPU: `dv_downstream_logistic_cv` (csrc/dv_downstream.cu) through the raw C ABI
against the fp64 numpy restatement of tests/downstream_reference.py on the same rows and labels, on guarded buffers,
in every layout of mu, with bit-identical repeats:
- every fold fit and every refit to the restatement's minimiser (the KKT residual within 1e-8 of its scale, and up
  to C = 100 the coefficients within 1e-7 of their scale, as tests/test_score_paths_gpu.py holds dv_logistic_fit;
  above it the raw-mean fits are too ill-conditioned for a coefficient bound), every prediction equal
  to the restatement's from the kernel's own coefficients wherever the deciding values are apart, every fold accuracy
  exactly the count over the kernel's own fold predictions, and the chosen C the restatement's;
- the paths: 10 rows against a 40-value factor, a fold with one class, a training set with one class, binary
  factors, a two-present-class multinomial fold, separable data at C = 1e4, D = 1 and 128, a 256-value factor;
- refusals that launch nothing, a captured graph that replays to the eager bits, and a refit at C = 1 bit-identical
  to dv_logistic_fit on the same rows (the shared solver's C and multinomial flag leave the existing fits alone);
and `downstream_task` / `Evaluator.compute_downstream_task`: both predictors, the boosted trees equal to `dci_fit`'s,
host and resident loaders, isolation from the other scores and the global generators.
"""
import ctypes
import logging

import numpy as np
import pytest
import torch

import downstream_reference as R
from score_kernels import (DEV, DV_ERR_BAD_ARG, DV_ERR_BAD_SHAPE, DV_ERR_WORKSPACE, LAYOUTS, Buf, _call, _code,
                           _graph_replays, _lib, _rows, _same, grid_values, place_mu)

pytestmark = pytest.mark.gpu
COEF_RTOL, KKT_TOL = 1e-7, 1e-8
COEF_MAX_C = 100.0       # the largest C whose fits are also held to COEF_RTOL
GAP_RTOL = 1e-9          # deciding values closer than this (relative) may round either way


class DsCase:
    """One call of dv_downstream_logistic_cv through the raw ABI, every operand in a guarded buffer."""

    def __init__(self, x, lat_sizes, train_rows, test_rows, Cs=R.CS, layout="contiguous"):
        from disvae.evaluate import sap_labels
        self.x = x
        self.tr, self.te = train_rows.to(DEV), test_rows.to(DEV)
        self.factors, train_cls, test_cls, n_classes, counts, _ = sap_labels(lat_sizes, self.tr, self.te)
        self.mu, self.ld, self.rs = place_mu(x, layout)
        self.K, self.S = counts.shape
        self.n, self.m, self.D = len(train_rows), len(test_rows), x.shape[1]
        self.Cs = np.ascontiguousarray(Cs, np.float64)
        self.nC = len(self.Cs)
        self.inputs = [Buf(t.numel(), t.dtype, t) for t in (self.tr, self.te, train_cls, n_classes)]
        self.train_cls, self.test_cls = train_cls.cpu().numpy(), test_cls.cpu().numpy()
        self.n_classes = n_classes.cpu().numpy()
        L, _ = _lib()
        self.ws_bytes = L.dv_downstream_workspace_bytes(self.D, self.n, self.K, self.S, self.nC)
        assert self.ws_bytes > 0
        K, S, D, n, m, nC = self.K, self.S, self.D, self.n, self.m, self.nC
        self.outs = [Buf(K * 5 * nC, torch.float64), Buf(K, torch.int32), Buf(K * S * (D + 1), torch.float64),
                     Buf(K * (n + m), torch.int32), Buf(K * (5 * nC + 1), torch.int32),
                     Buf(K * 5 * nC * S * (D + 1), torch.float64), Buf(K * nC * n, torch.int32)]
        self.ws = Buf((self.ws_bytes + 7) // 8, torch.float64, float("nan"))

    def args(self, **kw):
        tr, te, cls, ncl = (b.ptr for b in self.inputs)
        acc, chosen, coef, pred, it, fcoef, fpred = (b.ptr for b in self.outs)
        a = dict(mu=self.mu.ptr, ld=self.ld, rs=self.rs, N=self.x.shape[0], D=self.D, tr=tr, ntr=self.n, te=te,
                 nte=self.m, cls=cls, ncl=ncl, K=self.K, S=self.S, cs=self.Cs.ctypes.data, nC=self.nC, acc=acc,
                 chosen=chosen, coef=coef, pred=pred, it=it, fcoef=fcoef, fpred=fpred, ws=self.ws.ptr,
                 wsb=self.ws_bytes)
        a.update(kw)
        return tuple(a.values()) + (_lib()[1],)

    def run(self):
        got = []
        for _ in range(2):
            for b in self.outs:
                b.body.view(torch.uint8).fill_(0xA5)
            _call(2, "dv_downstream_logistic_cv", *self.args())
            got.append([b.body.clone() for b in self.outs])
            assert all(b.intact() for b in self.outs + [self.ws] + self.inputs), "a write past a buffer"
            assert self.mu.intact()
        for a, b in zip(*got):
            assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), "a repeat differs"
        K, S, D, n, m, nC = self.K, self.S, self.D, self.n, self.m, self.nC
        acc, chosen, coef, pred, it, fcoef, fpred = (t.cpu().numpy() for t in got[0])
        return dict(acc=acc.reshape(K, 5, nC), chosen=chosen, coef=coef.reshape(K, S, D + 1),
                    pred=pred.reshape(K, n + m), iters=it.reshape(K, 5 * nC + 1),
                    fold_coef=fcoef.reshape(K, 5, nC, S, D + 1), fold_pred=fpred.reshape(K, nC, n))

    def _check_fit(self, got, x, y, p, multi, C, rows, tag):
        """One fit's rows `got` [S, D + 1] (model rows at `rows`, NaN elsewhere) against the restatement ->
        (the kernel's W, b, the restatement's W, b)."""
        model = len(rows)
        others = np.ones(self.S, bool)
        others[rows] = False
        assert np.isnan(got[others]).all(), tag
        if model == 0:
            return np.zeros((0, self.D)), np.zeros(0), np.zeros((0, self.D)), np.zeros(0)
        W, b = got[rows, :-1], got[rows, -1]
        assert not np.isnan(W).any() and not np.isnan(b).any(), tag
        wW, wb, _ = R.fit(x, y, p, multi, C)
        ref = max(np.abs(wW).max(), np.abs(wb).max(), 1e-300)
        err = max(np.abs(W - wW).max(), np.abs(b - wb).max())
        gr, sc = R.kkt(x, y, multi, C, W, b)
        # Above COEF_MAX_C on raw, nearly separable means the minimiser is ill-conditioned (the loss's curvature
        # vanishes where p is near 0 or 1, and the intercepts are unpenalised): two points that both pass the stopping
        # rule can differ by more than 1e-7 of the coefficients.  There the KKT residual is the test.
        assert (C > COEF_MAX_C or err <= COEF_RTOL * ref) and np.abs(gr).max() <= KKT_TOL * sc.max(), (
            tag, err / ref, np.abs(gr).max() / sc.max())
        return W, b, wW, wb

    def _agree(self, got, W, b, multi, classes, x, tag):
        want, gap = R.predict(W, b, multi, classes, x)
        scale = 1.0 + (np.abs(np.c_[W, b]).max() * (1.0 + np.abs(x).max()) if len(b) else 0.0)
        clear = gap > GAP_RTOL * scale
        assert np.array_equal(got[clear], want[clear]), tag
        return want

    def check(self, got=None, factors=None):
        got = self.run() if got is None else got
        x64 = self.x.cpu().numpy().astype(np.float32).astype(np.float64)
        xt, xe = x64[self.tr.cpu().numpy()], x64[self.te.cpu().numpy()]
        n, nC = self.n, self.nC
        for k in range(self.K) if factors is None else factors:
            nc, cls = int(self.n_classes[k]), self.train_cls[k]
            multi = nc > 2
            ref_acc = np.zeros((5, nC))
            for f, (s0, s1) in enumerate(R.fold_bounds(n)):
                keep = np.r_[0:s0, s1:n]
                present = np.unique(cls[keep])
                place = np.full(max(nc, 1), -1)
                place[present] = np.arange(len(present))
                p = len(present)
                rows = [] if p < 2 else (list(present) if multi else [0])
                for c, C in enumerate(self.Cs):
                    tag = ("fold", k, f, c)
                    W, b, wW, wb = self._check_fit(got["fold_coef"][k, f, c], xt[keep], place[cls[keep]], p, multi,
                                                   C, rows, tag)
                    steps = got["iters"][k, f * nC + c]
                    assert steps >= 0 if rows else steps == 0, (tag, steps)
                    fp = got["fold_pred"][k, c, s0:s1]
                    self._agree(fp, W, b, multi, present, xt[s0:s1], tag)
                    assert got["acc"][k, f, c] == (fp == cls[s0:s1]).sum() / (s1 - s0), tag
                    ref_acc[f, c] = (R.predict(wW, wb, multi, present, xt[s0:s1])[0] == cls[s0:s1]).sum() / (s1 - s0)
            total, want = got["acc"][k, 0], ref_acc[0]
            for f in range(1, 5):
                total, want = total + got["acc"][k, f], want + ref_acc[f]
            assert got["chosen"][k] == int(np.argmax(total)) == int(np.argmax(want)), ("chosen", k)
            C = self.Cs[got["chosen"][k]]
            rows = [] if nc < 2 else (list(range(nc)) if multi else [0])
            W, b, _, _ = self._check_fit(got["coef"][k], xt, cls, nc, multi, C, rows, ("refit", k))
            steps = got["iters"][k, 5 * nC]
            assert steps >= 0 if rows else steps == 0, ("refit", k, steps)
            self._agree(got["pred"][k], W, b, multi, np.arange(max(nc, 1)), np.r_[xt, xe], ("pred", k))
        return got


# ---- the kernel against the restatement ------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", LAYOUTS)
def test_every_layout(layout):
    lat = [2, 3, 6]
    x = _code(lat, 4, 1)
    case = DsCase(x, lat, _rows(36, 200, 2), _rows(36, 100, 3), layout=layout)
    got = case.check()
    if layout != "contiguous":
        base = DsCase(x, lat, _rows(36, 200, 2), _rows(36, 100, 3)).run()
        for key in got:
            assert np.array_equal(got[key].view(np.uint8), base[key].view(np.uint8)), (layout, key)


def test_ten_rows_against_a_40_value_factor():
    """Two rows per fold: every fold misses most of the factor's values."""
    lat = [40, 3]
    case = DsCase(_code(lat, 10, 4), lat, _rows(120, 10, 5), _rows(120, 500, 6))
    assert case.n_classes[0] >= 8
    case.check()


def test_fold_and_training_set_with_one_class_and_two_present_multinomial():
    """lat (2, 2, 3): factor 0 shows one value in training (no fit anywhere); factor 1 shows value 1 only on fold 0's
    rows, so fold 0 fits one class and predicts it; factor 2 shows value 2 only on fold 0's rows, so fold 0's fit is
    the multinomial over two present classes (the binary fit at 2C)."""
    lat = [2, 2, 3]
    v = grid_values(lat)
    ones = torch.nonzero((v[:, 0] == 0) & (v[:, 1] == 1) & (v[:, 2] == 2))[:, 0]
    rest = torch.nonzero((v[:, 0] == 0) & (v[:, 1] == 0) & (v[:, 2] < 2))[:, 0]
    tr = torch.cat([ones.repeat(8), rest[_rows(len(rest), 32, 7)]])      # fold 0 = the first 8 of 40 rows
    x = _code(lat, 3, 8)
    case = DsCase(x, lat, tr, _rows(12, 50, 9))
    assert case.n_classes.tolist() == [1, 2, 3]
    got = case.check()
    assert (got["fold_pred"][1, :, :8] == 0).all() and (got["iters"][1, :10] == 0).all()
    assert np.isnan(got["fold_coef"][2, 0, :, 2]).all() and not np.isnan(got["fold_coef"][2, 0, :, :2]).any()
    assert (got["pred"][0] == 0).all() and np.isnan(got["coef"][0]).all()


def test_binary_factors():
    lat = [2, 2]
    case = DsCase(_code(lat, 5, 10, noise=0.6), lat, _rows(4, 333, 11), _rows(4, 100, 12))
    assert case.n_classes.tolist() == [2, 2]
    case.check()


def test_separable_data_at_large_c():
    """Separated classes: the fits at C = 1e4 grow large weights and stop on the gradient test."""
    lat = [2, 3]
    case = DsCase(_code(lat, 3, 13, noise=0.01), lat, _rows(6, 400, 14), _rows(6, 100, 15), Cs=[1e2, 1e4])
    got = case.check()
    print("separable, C = 1e4: Newton steps", got["iters"][:, 1::2].tolist())


@pytest.mark.parametrize("D", [1, 128])
def test_one_and_128_latents(D):
    lat = [3, 4]
    case = DsCase(_code(lat, D, 16 + D), lat, _rows(12, 300, 17), _rows(12, 100, 18), Cs=R.CS[::3])
    case.check()


def test_256_values():
    lat = [256, 2]
    case = DsCase(_code(lat, 2, 19), lat, _rows(512, 3000, 20), _rows(512, 300, 21), Cs=[1e-2, 1.0])
    assert case.n_classes.tolist() == [256, 2]
    case.check()


def test_refit_at_c_1_equals_dv_logistic_fit_bitwise():
    """The same rows through dv_logistic_fit (C = 1, multinomial above two classes): the refit's coefficients,
    predictions of the training rows and Newton steps are the same bits."""
    lat = [2, 5, 7]
    x = _code(lat, 6, 22)
    case = DsCase(x, lat, _rows(70, 900, 23), _rows(70, 50, 24), Cs=[1.0])
    got = case.run()
    L, stream = _lib()
    xt = x.to(DEV, torch.float32).double()[case.tr].contiguous()
    D, n = case.D, case.n
    for k in range(case.K):
        K = case.S
        labels = torch.from_numpy(case.train_cls[k]).to(DEV).contiguous()
        ncl = torch.tensor([int(case.n_classes[k])], dtype=torch.int32, device=DEV)
        coef = torch.empty(K, D + 1, dtype=torch.float64, device=DEV)
        pred = torch.empty(n, dtype=torch.int32, device=DEV)
        it = torch.empty(1, dtype=torch.int32, device=DEV)
        nbytes = L.dv_logistic_fit_workspace_bytes(n, D, K)
        ws = torch.empty(nbytes // 8 + 1, dtype=torch.float64, device=DEV)
        _call(1, "dv_logistic_fit", xt.data_ptr(), D, n, 0, labels.data_ptr(), ncl.data_ptr(), K, coef.data_ptr(),
              pred.data_ptr(), it.data_ptr(), ws.data_ptr(), ctypes.c_size_t(nbytes), stream)
        _same(torch.from_numpy(got["coef"][k]), coef.cpu(), "refit coef %d" % k)
        _same(torch.from_numpy(got["pred"][k, :n]), pred.cpu(), "refit pred %d" % k)
        assert int(it) == got["iters"][k, -1] >= 0


def test_workspace_and_refusals_launch_nothing():
    lat = [3, 4]
    case = DsCase(_code(lat, 4, 25), lat, _rows(12, 100, 26), _rows(12, 50, 27), Cs=[0.5, 2.0])
    L, _ = _lib()
    for b in case.outs:
        b.body.view(torch.uint8).fill_(0x11)

    def refused(args, want):
        torch.cuda.synchronize()
        before = L.dv_launch_count()
        rc = L.dv_downstream_logistic_cv(*args)
        torch.cuda.synchronize()
        assert rc == want and L.dv_launch_count() == before, (rc, want)

    for shape in (dict(N=0), dict(D=0), dict(D=129), dict(ntr=4), dict(ntr=32769), dict(nte=0), dict(K=0),
                  dict(S=0), dict(S=257), dict(nC=0), dict(nC=33), dict(ld=0), dict(rs=-1)):
        refused(case.args(**shape), DV_ERR_BAD_SHAPE)
    tr, te, cls, ncl = (b.ptr for b in case.inputs)
    o = [b.ptr for b in case.outs]
    bad_c = [np.array([0.5, v]) for v in (0.0, -1.0, np.inf, np.nan)]
    for bad in ([dict(mu=None), dict(tr=None), dict(te=None), dict(cls=None), dict(ncl=None), dict(cs=None),
                 dict(acc=None), dict(chosen=None), dict(coef=None), dict(pred=None), dict(it=None),
                 dict(mu=case.mu.ptr + 2), dict(tr=tr + 4), dict(te=te + 4), dict(cls=cls + 2), dict(ncl=ncl + 2),
                 dict(acc=o[0] + 4), dict(chosen=o[1] + 2), dict(coef=o[2] + 4), dict(pred=o[3] + 2),
                 dict(it=o[4] + 2), dict(fcoef=o[5] + 4), dict(fpred=o[6] + 2), dict(ws=case.ws.ptr + 4)] +
                [dict(cs=c.ctypes.data) for c in bad_c]):
        refused(case.args(**bad), DV_ERR_BAD_ARG)
    refused(case.args(ws=None), DV_ERR_WORKSPACE)
    refused(case.args(wsb=case.ws_bytes - 1), DV_ERR_WORKSPACE)
    for b in case.outs:
        assert (b.body.view(torch.uint8) == 0x11).all() and b.intact()
    for q in (dict(D=0), dict(D=129), dict(n=4), dict(n=32769), dict(K=0), dict(S=257), dict(nC=0), dict(nC=33)):
        a = dict(D=4, n=100, K=2, S=4, nC=2)
        a.update(q)
        assert L.dv_downstream_workspace_bytes(a["D"], a["n"], a["K"], a["S"], a["nC"]) == 0, q
    # the slots: one per fold fit up to 132, each for one fit of num_train rows
    one = L.dv_downstream_workspace_bytes(10, 10000, 1, 40, 1) // 5          # five fold fits, five slots
    assert L.dv_downstream_workspace_bytes(10, 10000, 5, 40, 10) == 132 * one
    assert L.dv_downstream_workspace_bytes(10, 10000, 50, 40, 10) == 132 * one
    assert L.dv_downstream_workspace_bytes(128, 32768, 8, 256, 10) <= (8 << 30)
    before = L.dv_launch_count()
    assert L.dv_downstream_logistic_cv(*case.args(fcoef=None, fpred=None)) == 0 and L.dv_launch_count() == before + 2
    torch.cuda.synchronize()
    assert (case.outs[5].body.view(torch.uint8) == 0x11).all() and (case.outs[6].body.view(torch.uint8) == 0x11).all()


def test_graph_replay_equals_eager():
    lat = [3, 6]
    case = DsCase(_code(lat, 5, 28), lat, _rows(18, 300, 29), _rows(18, 60, 30))
    case.run()
    L, _ = _lib()
    _graph_replays(lambda: L.dv_downstream_logistic_cv(*case.args()), case.outs, "dv_downstream_logistic_cv")


# ---- downstream_task and the Evaluator ----------------------------------------------------------------------------
from test_eval_resident_gpu import _assert_same_eval_files, _checkpoint_model, _dataset, _evaluator, _loader  # noqa
from test_eval_resident_gpu import _loss, _n_samples, K as GRID_K  # noqa: E402


def test_downstream_task_both_predictors():
    """The logistic score equals the kernel's predictions on each size's draws; the boosted trees' accuracies equal
    `dci_fit`'s on the same rows."""
    from disvae import evaluate
    lat = [3, 1, 6, 8]
    x = _code(lat, 5, 31).to(DEV)
    sizes = (10, 100, 400)
    scores = {p: evaluate.downstream_task(x, lat, predictor=p, num_train=sizes, num_test=300, seed=2)
              for p in evaluate.DOWNSTREAM_PREDICTORS}
    gen = torch.Generator(device=DEV)
    gen.manual_seed(2)
    for size in sizes:
        tr = torch.randint(x.shape[0], (size,), generator=gen, device=DEV)
        te = torch.randint(x.shape[0], (300,), generator=gen, device=DEV)
        factors, train_cls, test_cls, n_classes, counts, _ = evaluate.sap_labels(lat, tr, te)
        assert factors == [0, 2, 3]
        truth = torch.cat([train_cls, test_cls], 1)
        _, pred, _ = evaluate.dci_fit(x, tr, te, train_cls, n_classes, counts)
        lr = evaluate.downstream_logistic_cv(x, tr, te, train_cls, n_classes, counts.shape[1])
        for p, pr in (("boosted_trees", pred), ("logistic_regression", lr[3])):
            score, helpers = scores[p]
            right = (pr == truth).double()
            assert torch.equal(helpers[size]["train_accuracy"], right[:, :size].mean(1).cpu()), (p, size)
            assert torch.equal(helpers[size]["test_accuracy"], right[:, size:].mean(1).cpu()), (p, size)
            assert score["%d:min_test_accuracy" % size] == float(right[:, size:].mean(1).min())
        h = scores["logistic_regression"][1][size]
        assert torch.equal(h["chosen_C"], torch.from_numpy(R.CS)[lr[1].cpu().long()])
        assert (h["solver_iterations"] >= 0).all()
    assert len(scores["logistic_regression"][0]) == 3 * (4 + 2 * 3)


def test_full_size_dsprites_shape():
    """dSprites' factor grid (1, 3, 6, 40, 32, 32), 10 latents, 1,000 training rows against the restatement for the
    3- and 40-value factors, and the whole default score's time."""
    from disvae import evaluate
    lat = [1, 3, 6, 40, 32, 32]
    x = _code(lat[1:], 10, 32, noise=0.2)
    case = DsCase(x, lat, _rows(x.size(0), 1000, 33), _rows(x.size(0), 500, 34))
    case.check(factors=[0, 2])
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    score, helpers = evaluate.downstream_task(x.to(DEV), lat, seed=35)
    end.record()
    torch.cuda.synchronize()
    print("full-size downstream_task (logistic): %.1f ms; largest Newton steps %s" % (
        start.elapsed_time(end), [int(helpers[s]["solver_iterations"].max()) for s in (10, 100, 1000, 10000)]))
    assert score["10000:mean_test_accuracy"] > score["10:mean_test_accuracy"]
    assert all((helpers[s]["solver_iterations"] >= 0).all() for s in (10, 100, 1000, 10000))


def test_loaders_agree_and_isolation(tmp_path):
    import disvae
    from disvae.evaluate import downstream_task
    from synthetic_factors import loader
    ds = _dataset()
    model = _checkpoint_model()
    ev = disvae.Evaluator(model, None, device=DEV, logger=logging.getLogger("ds"), save_dir="unused",
                          is_progress_bar=False)
    host = ev.compute_downstream_task(loader(ds, 1000), num_train=(10, 200), num_test=100, seed=5)
    dev = ev.compute_downstream_task(_loader(ds).in_order(1000), num_train=(10, 200), num_test=100, seed=5)
    assert host == dev and "200:test_accuracy_factor_0" in host
    files = [(f, f) for f in ("metrics.log", "metric_helpers.pth", "factor_vae_score.log",
                              "factor_vae_score_helpers.pth", "sap_score.log", "sap_score_helpers.pth",
                              "beta_vae_score.log", "beta_vae_score_helpers.pth")]
    with _n_samples(512):
        for name in ("a", "b"):
            ev = _evaluator(model, _loss("btcvae", GRID_K ** 4), tmp_path / name)
            if name == "b":                                     # a downstream score between the two evaluations
                mean = ev._compute_q_zCx(loader(ds, 1000))[1][0]
                cpu, cuda = torch.get_rng_state(), torch.cuda.get_rng_state()
                downstream_task(mean, [int(s) for s in ds.lat_sizes], num_train=(50,), num_test=50, seed=3)
                downstream_task(mean, [int(s) for s in ds.lat_sizes], predictor="boosted_trees", num_train=(50,),
                                num_test=50, seed=3)
                assert torch.equal(cpu, torch.get_rng_state()) and torch.equal(cuda, torch.cuda.get_rng_state())
            torch.manual_seed(7)
            ev(loader(ds, 1000), is_metrics=True, is_losses=False, is_factor_score=True, is_sap_score=True,
               is_beta_vae_score=True)
    _assert_same_eval_files(tmp_path / "a", tmp_path / "b", files, "with vs without a downstream score",
                            nan_equal=True)
