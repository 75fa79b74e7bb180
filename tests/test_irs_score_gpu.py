"""IRS on the GPU: `dv_irs_fit` (csrc/dv_irs.cu) through the raw C ABI against the fp64 numpy restatement of
tests/irs_reference.py on the same rows and values, on guarded buffers, in four layouts of mu, with bit-identical
repeats:
- the edges and group counts (so the bins) exactly, the active flags exactly;
- the max deviations and group deviations within 1e-12 of the latent's scale (the group means are fp64 sums in another
  order), the IRS matrix within that error over the latent's max deviation;
- refusals that launch nothing, a captured graph that replays to the eager bits;
and `irs_score` / `Evaluator.compute_irs_score`: host and resident loaders, SAP's training rows, isolation from the
other scores and the global generators, exact scores of axis-aligned codes, and a known ordering at full dSprites size.
"""
import logging

import numpy as np
import pytest
import torch

import irs_reference as R
from score_kernels import (DEV, DV_ERR_BAD_ARG, DV_ERR_BAD_SHAPE, DV_ERR_WORKSPACE, LAYOUTS, Buf, _call, _Code,
                           _Factors, _graph_replays, _lib, place_mu)

pytestmark = pytest.mark.gpu
RTOL = 1e-12


class IrsCase:
    """One raw `dv_irs_fit` call, every operand in a guarded buffer."""

    def __init__(self, x, rows, values, dq=0.99, layout="contiguous"):
        self.x = x.float()
        self.rows = torch.as_tensor(rows, dtype=torch.int64)
        self.values = torch.as_tensor(np.asarray(values), dtype=torch.int32).reshape(-1, len(self.rows))
        self.dq = dq
        self.mu, self.ld, self.rs = place_mu(self.x, layout)
        self.n, self.D, self.K = len(self.rows), x.shape[1], self.values.shape[0]
        self.inputs = [Buf(self.n, torch.int64, self.rows.to(DEV)), Buf(self.K * self.n, torch.int32,
                                                                         self.values.to(DEV))]
        L, _ = _lib()
        self.ws_bytes = L.dv_irs_workspace_bytes(self.D, self.n, self.K)
        assert self.ws_bytes > 0
        D, K = self.D, self.K
        self.outs = [Buf(D, torch.float64), Buf(D, torch.int32), Buf(D * K, torch.float64),
                     Buf(K * 20 * D, torch.float64), Buf(K * 20, torch.int32), Buf(K * 21, torch.float64)]
        self.ws = Buf((self.ws_bytes + 7) // 8, torch.float64, float("nan"))

    def args(self, **kw):
        rows, values = (b.ptr for b in self.inputs)
        md, act, irs, gd, gc, e = (b.ptr for b in self.outs)
        a = dict(mu=self.mu.ptr, ld=self.ld, rs=self.rs, N=self.x.shape[0], D=self.D, rows=rows, n=self.n,
                 values=values, K=self.K, dq=float(self.dq), md=md, act=act, irs=irs, gd=gd, gc=gc, e=e,
                 ws=self.ws.ptr, wsb=self.ws_bytes)
        a.update(kw)
        return tuple(a.values()) + (_lib()[1],)

    def run(self):
        got = []
        for _ in range(2):
            for b in self.outs:
                b.body.view(torch.uint8).fill_(0xA5)
            _call(3, "dv_irs_fit", *self.args())
            got.append([b.body.clone() for b in self.outs])
            assert all(b.intact() for b in self.outs + [self.ws] + self.inputs), "a write past a buffer"
            assert self.mu.intact()
        for a, b in zip(*got):
            assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), "dv_irs_fit: a repeat differs"
        md, act, irs, gd, gc, e = (t.cpu().numpy() for t in got[0])
        D, K = self.D, self.K
        return dict(max_deviation=md, active=act, irs_matrix=irs.reshape(D, K), group_deviation=gd.reshape(K, 20, D),
                    group_count=gc.reshape(K, 20), edges=e.reshape(K, 21))

    def check(self):
        got = self.run()
        xs = self.x.numpy()[self.rows.numpy()]
        want = R.fit(xs, self.values.numpy(), self.dq)
        assert np.array_equal(got["edges"], want["edges"]), "edges"
        assert np.array_equal(got["group_count"], want["group_count"]), "group counts"
        assert np.array_equal(got["active"].astype(bool), want["active"]), "active"
        scale = np.abs(xs.astype(np.float64)).max(0)                # [D]
        tol = RTOL * scale
        assert (np.abs(got["max_deviation"] - want["max_deviation"]) <= tol).all(), "max deviation"
        gd, wgd = got["group_deviation"], want["group_deviation"]
        assert np.array_equal(np.isnan(gd), np.isnan(wgd)), "empty bins"
        ok = ~np.isnan(wgd)
        assert (np.abs(gd - wgd)[ok] <= np.broadcast_to(tol, gd.shape)[ok]).all(), (
            "group deviation", np.nanmax(np.abs(gd - wgd)))
        M, W = got["irs_matrix"], want["irs_matrix"]
        assert np.array_equal(np.isnan(M), np.isnan(W)), "inactive rows"
        act = want["active"]
        mtol = np.maximum(RTOL, 2 * tol[act] / want["max_deviation"][act])[:, None]
        assert (np.abs(M[act] - W[act]) <= mtol).all(), ("irs matrix", np.abs(M[act] - W[act]).max())
        return got, want


def _grid_case(lat, D, n, seed, layout="contiguous", noise=0.2, dq=0.99):
    """Codes of a grid: latent d follows scored factor d plus noise, further latents noise; n random rows."""
    g = torch.Generator().manual_seed(seed)
    N = int(np.prod(lat))
    v = torch.from_numpy(np.stack(np.unravel_index(np.arange(N), lat), 1)).float()
    x = torch.randn(N, D, generator=g)
    scored = [k for k, s in enumerate(lat) if s > 1]
    for d, k in enumerate(scored[:D]):
        x[:, d] = v[:, k] / lat[k] + noise * x[:, d]
    rows = torch.randint(N, (n,), generator=g)
    return IrsCase(x, rows, R.draw_values(lat, rows.numpy())[1], dq=dq, layout=layout)


@pytest.mark.parametrize("layout", LAYOUTS)
def test_every_layout(layout):
    case = _grid_case([3, 6, 40, 32, 32], 10, 10000, 1, layout=layout)
    got, _ = case.check()
    if layout != "contiguous":
        base = _grid_case([3, 6, 40, 32, 32], 10, 10000, 1).run()
        for k in base:
            assert np.array_equal(got[k].view(np.uint8), base[k].view(np.uint8)), (layout, k)


@pytest.mark.parametrize("D, n", [(1, 1), (1, 2), (2, 3), (10, 10000), (16, 32768), (1024, 2048)])
def test_dims_and_rows(D, n):
    _grid_case([4, 5, 3], D, n, D + n).check()


def test_factor_sizes_and_an_fp32_edge_range():
    """Factors of 2, 3, 20, 21, 40, 256 values, and values 0 .. 324, where fp32 edges would bin differently."""
    g = np.random.default_rng(3)
    n = 6000
    sizes = [2, 3, 20, 21, 40, 256, 325]
    values = np.stack([g.integers(0, s, n) for s in sizes])
    values[:, 0], values[:, 1] = 0, np.array(sizes) - 1              # every range is full
    x = torch.randn(n, 7, generator=torch.Generator().manual_seed(4))
    x[:, :7] += torch.from_numpy(values.T / np.array(sizes)).float()
    got, _ = IrsCase(x, torch.arange(n), values).check()
    assert (got["group_count"][:2] > 0).sum() == 5                    # 2 and 3 values: one bin each
    assert (got["group_count"][2:] > 0).all()


@pytest.mark.parametrize("dq", [0.5, 0.0, 1.0, 0.99, 0.3])
def test_group_sizes_where_t_is_0_and_one_half(dq):
    """One factor of values 0 .. 6 (a bin each) with groups of 1, 2, 3, 4, 5, 100 and 101 rows: at dq = 0.5 odd groups
    have t = 0 and even ones t = 1/2; duplicated values throughout."""
    sizes = [1, 2, 3, 4, 5, 100, 101]
    values = np.concatenate([np.full(m, v) for v, m in enumerate(sizes)])
    n = len(values)
    g = torch.Generator().manual_seed(5)
    x = torch.round(4 * torch.randn(n, 3, generator=g)) / 4           # many ties
    IrsCase(x, torch.arange(n), values[None], dq=dq).check()


def test_constant_signed_zero_duplicated_and_offset_latents():
    """Latent 0 constant, latent 1 +0.0 and -0.0 only (inactive), latent 2 a copy of latent 4, latent 3 at 1e4 plus
    noise of 1e-3, latent 4 informative; factors of 12 values, of 2,900 values (merged bins) and of one row against
    all the others (a one-row group)."""
    n = 3000
    g = torch.Generator().manual_seed(6)
    f = torch.randint(0, 12, (n,), generator=g)
    x4 = f.float() / 12 + 0.3 * torch.randn(n, generator=g)
    zeros = torch.where(torch.rand(n, generator=g) < 0.5, torch.tensor(0.0), torch.tensor(-0.0))
    x = torch.stack([torch.full((n,), 0.375), zeros, x4, 1e4 + 1e-3 * torch.randn(n, generator=g), x4], 1)
    wide = torch.randperm(n, generator=g) % 2900
    values = np.stack([f.numpy(), wide.numpy(), np.r_[np.zeros(n - 1, np.int64), 1]])
    got, want = IrsCase(x, torch.arange(n), values).check()
    assert got["active"].tolist() == [0, 0, 1, 1, 1]
    assert np.isnan(got["irs_matrix"][:2]).all()
    assert np.array_equal(got["irs_matrix"][2], got["irs_matrix"][4])
    assert got["group_count"][2].tolist() == [n - 1] + [0] * 18 + [1]   # a one-row group: deviation 0
    assert (got["group_deviation"][2, 19] == 0).all()


def test_all_constant_latents_score_zero():
    from disvae import evaluate
    lat = [4, 5]
    mu = torch.full((20, 3), 2.0, device=DEV)
    score, helpers = evaluate.irs_score(mu, lat, num_train=100)
    assert score == {"IRS": 0.0, "num_active_dims": 0}
    assert torch.isnan(helpers["irs_matrix"]).all() and (helpers["parents"] == -1).all()


def test_latents_equal_to_distinct_factors_score_exactly_one():
    from disvae import evaluate
    lat = [5, 1, 7, 20]
    v = torch.from_numpy(np.stack(np.unravel_index(np.arange(700), lat), 1)).float()
    mu = v[:, [3, 0, 2]].contiguous().to(DEV)
    score, helpers = evaluate.irs_score(mu, lat, num_train=5000, seed=2)
    assert score == {"IRS": 1.0, "num_active_dims": 3}
    assert helpers["parents"].tolist() == [2, 0, 1] and (helpers["disentanglement_scores"] == 1.0).all()


def test_workspace_and_refusals_launch_nothing():
    case = _grid_case([3, 4], 4, 100, 7)
    L, _ = _lib()
    for b in case.outs:
        b.body.view(torch.uint8).fill_(0x11)

    def refused(args, want):
        torch.cuda.synchronize()
        before = L.dv_launch_count()
        rc = L.dv_irs_fit(*args)
        torch.cuda.synchronize()
        assert rc == want and L.dv_launch_count() == before, rc

    for shape in (dict(N=0), dict(D=0), dict(D=1025), dict(n=0), dict(n=32769), dict(K=0), dict(ld=0), dict(rs=0),
                  dict(rs=-1), dict(dq=-0.01), dict(dq=1.01), dict(dq=float("nan")), dict(K=2 ** 30)):
        refused(case.args(**shape), DV_ERR_BAD_SHAPE)
    o = [b.ptr for b in case.outs]
    rows, values = (b.ptr for b in case.inputs)
    bad = [dict(mu=None), dict(rows=None), dict(values=None)] + [{k: None} for k in ("md", "act", "irs", "gd", "gc",
                                                                                     "e")]
    bad += [dict(mu=case.mu.ptr + 2), dict(rows=rows + 4), dict(values=values + 2), dict(md=o[0] + 4),
            dict(act=o[1] + 2), dict(irs=o[2] + 4), dict(gd=o[3] + 4), dict(gc=o[4] + 2), dict(e=o[5] + 4),
            dict(ws=case.ws.ptr + 4)]
    for b in bad:
        refused(case.args(**b), DV_ERR_BAD_ARG)
    refused(case.args(ws=None), DV_ERR_WORKSPACE)
    refused(case.args(wsb=case.ws_bytes - 1), DV_ERR_WORKSPACE)
    for b in case.outs:
        assert (b.body.view(torch.uint8) == 0x11).all() and b.intact()
    for q in ((0, 100, 2), (1025, 100, 2), (4, 0, 2), (4, 32769, 2), (4, 100, 0)):
        assert L.dv_irs_workspace_bytes(*q) == 0, q


def test_graph_replay_equals_eager():
    case = _grid_case([3, 6, 10], 5, 3000, 8)
    case.run()
    L, _ = _lib()
    _graph_replays(lambda: L.dv_irs_fit(*case.args()), case.outs, "dv_irs_fit")


# ---- irs_score and the Evaluator ---------------------------------------------------------------------------------
from test_eval_resident_gpu import _assert_same_eval_files, _checkpoint_model, _dataset, _evaluator, _loader  # noqa
from test_eval_resident_gpu import _loss, _n_samples, K as GRID_K  # noqa: E402


def test_rows_are_saps_training_rows(monkeypatch):
    from disvae import evaluate
    lat = [3, 1, 40, 5]
    mu = torch.randn(600, 4, device=DEV)
    seen = []
    fit = evaluate.irs_fit
    monkeypatch.setattr(evaluate, "irs_fit", lambda mu, rows, values, dq: seen.append(rows.clone()) or
                        fit(mu, rows, values, dq))
    evaluate.irs_score(mu, lat, num_train=777, seed=41)
    assert torch.equal(seen[0], evaluate._sap_draws(mu, lat, 777, 5, 41)[0])


def test_repeats_and_loaders_agree():
    import disvae
    from synthetic_factors import loader
    ds = _dataset()
    model = _checkpoint_model()
    ev = disvae.Evaluator(model, None, device=DEV, logger=logging.getLogger("irs"), save_dir="unused",
                          is_progress_bar=False)
    host = ev.compute_irs_score(loader(ds, 1000), seed=5)
    dev = ev.compute_irs_score(_loader(ds).in_order(1000), seed=5)
    assert host == dev and set(host) == {"IRS", "num_active_dims"}
    from disvae.evaluate import irs_score
    mean = ev._compute_q_zCx(loader(ds, 1000))[1][0]
    runs = [irs_score(mean, [int(s) for s in ds.lat_sizes], seed=5) for _ in range(2)]
    assert runs[0][0] == runs[1][0] == host
    for key in runs[0][1]:
        a, b = runs[0][1][key], runs[1][1][key]
        assert torch.equal(a.nan_to_num(7.0), b.nan_to_num(7.0)) if a.is_floating_point() else torch.equal(a, b), key


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
            if name == "b":                                     # an IRS score between the two evaluations
                from disvae.evaluate import irs_score
                mean = ev._compute_q_zCx(loader(ds, 1000))[1][0]
                cpu, cuda = torch.get_rng_state(), torch.cuda.get_rng_state()
                irs_score(mean, [int(s) for s in ds.lat_sizes], seed=3)
                assert torch.equal(cpu, torch.get_rng_state()) and torch.equal(cuda, torch.cuda.get_rng_state())
                ev.compute_irs_score(loader(ds, 1000), seed=3)
            torch.manual_seed(7)
            ev(loader(ds, 1000), is_metrics=True, is_losses=False, is_factor_score=True, is_sap_score=True,
               is_beta_vae_score=True)
    _assert_same_eval_files(tmp_path / "a", tmp_path / "b", files, "with vs without an IRS score", nan_equal=True)


class _Batches:
    """The dataset's images in index order, `batch_size` at a time (what DataLoader(shuffle=False) yields)."""

    def __init__(self, dataset, batch_size):
        self.dataset, self.batch_size = dataset, batch_size

    def __iter__(self):
        for a in range(0, len(self.dataset), self.batch_size):
            yield self.dataset.imgs[a:a + self.batch_size], 0


def test_full_size_dsprites_aligned_rotated_noise(tmp_path):
    """dSprites' factor grid (1, 3, 6, 40, 32, 32; 737,280 items), 10 latents, through `compute_irs_score`: codes
    aligned with the factors score above the same codes rotated by 45 degrees in pairs, and those above noise."""
    import disvae
    lat = [1, 3, 6, 40, 32, 32]
    ds = _Factors(lat, 0.01, 9)
    M = torch.zeros(6, 10)
    M[1:, :5] = torch.eye(5)
    c, s = np.cos(np.pi / 4), np.sin(np.pi / 4)
    rot = torch.eye(10)
    for a in (0, 2):
        rot[a:a + 2, a:a + 2] = torch.tensor([[c, -s], [s, c]])
    noise = _Factors(lat, 0.0, 9)
    noise.imgs.view(len(noise), -1)[:, :6] = torch.randn(len(noise), 6, generator=torch.Generator().manual_seed(10))
    scores = {}
    for name, code, data in (("aligned", M, ds), ("rotated", M @ rot, ds), ("noise", M, noise)):
        ev = disvae.Evaluator(_Code(code), None, device=DEV, logger=logging.getLogger("irs"), save_dir=str(tmp_path),
                              is_progress_bar=False)
        scores[name] = ev.compute_irs_score(_Batches(data, 10000), seed=1)
    a, r, z = scores["aligned"], scores["rotated"], scores["noise"]
    print("full-size IRS:", scores)
    assert a["num_active_dims"] == r["num_active_dims"] == z["num_active_dims"] == 5
    assert a["IRS"] > r["IRS"] > z["IRS"], scores
