"""The unsupervised scores on the GPU: `dv_unsupervised_fit` (csrc/dv_unsupervised.cu) through the raw C ABI on guarded
buffers, across the four layouts of mu and logvar, D in {2, 10, 128} and n in {2, 10000, 32768}, against the fp64 numpy
restatement of tests/unsupervised_reference.py, on independent, correlated and known-covariance codes, a constant
latent, duplicated latents, tied values and a latent whose range is a few ulps wide:
- `sampled` within expf's 2 ulp (times |eps|) plus the final rounding of the fp64 formula;
- `cov` within 1e-12 of max |C|; the eigenvalues within 1e-12 of the largest, against np.linalg.eigvalsh of R and S built
  from the kernel's own cov; TC and W within 1e-9 relative where eig_min(R) >= 1e-4;
- the mutual-information matrix within 1e-12 of the restatement (sklearn's mutual_info_score), the edges bit for bit;
- the launch count, refusals that launch nothing, intact guards, bit-identical repeats and a graph replay;
and the Evaluator and sweeps: `compute_unsupervised_scores` on an unlabelled dataset, `unsupervised_every` leaving
training, every other file and the global generators as they are, the epoch files against `Sweep.unsupervised_scores`, a
member against a one-member sweep of it, and a resumed sweep against the unbroken one."""
import logging
import os

import numpy as np
import pytest
import torch

import modularity_reference as MR
import unsupervised_reference as R
from score_kernels import (DEV, DV_ERR_BAD_ARG, DV_ERR_BAD_SHAPE, DV_ERR_WORKSPACE, LAYOUTS, Buf, _call,
                           _graph_replays, _lib, _same, layout_strides)

pytestmark = pytest.mark.gpu
LAUNCHES = 6


def _place(mu, lv, layout):
    """mu and logvar [N, D] at element (p, d) = p rs + d ld of guarded NaN-filled buffers -> (bufs, mu ptr, lv ptr,
    ld, rs); in the q_zCx layout both halves of one interleaved buffer."""
    N, D = mu.shape
    ld, rs = layout_strides(layout, N, D)
    idx = (torch.arange(N, device=DEV)[:, None] * rs + torch.arange(D, device=DEV)[None, :] * ld).reshape(-1)
    span = (N - 1) * rs + (D - 1) * ld + 1
    if layout == "q_zCx":
        buf = Buf(span + 1, torch.float32, float("nan"))
        buf.body[idx] = mu.to(DEV).reshape(-1)
        buf.body[idx + 1] = lv.to(DEV).reshape(-1)
        return [buf], buf.ptr, buf.ptr + 4, ld, rs
    bufs = []
    for x in (mu, lv):
        b = Buf(span, torch.float32, float("nan"))
        b.body[idx] = x.to(DEV).reshape(-1)
        bufs.append(b)
    return bufs, bufs[0].ptr, bufs[1].ptr, ld, rs


class UnsCase:
    """One dv_unsupervised_fit call through the raw ABI, every operand in a guarded buffer."""

    def __init__(self, mu, lv, rows, eps, layout="contiguous"):
        self.mu_h, self.lv_h, self.rows_h, self.eps_h = mu, lv, rows, eps
        self.N, self.D = mu.shape
        self.n = rows.numel()
        D, n = self.D, self.n
        self.bufs, self.mu_p, self.lv_p, self.ld, self.rs = _place(mu, lv, layout)
        self.inputs = self.bufs + [Buf(n, torch.int64, rows.to(DEV)), Buf(n * D, torch.float32, eps.to(DEV))]
        self.outs = [Buf(2 * D * D, torch.float64), Buf(4 * D, torch.float64), Buf(4, torch.int32),
                     Buf(2 * D * D, torch.float64), Buf(2 * D * 21, torch.float32), Buf(n * D, torch.float32)]
        L, _ = _lib()
        self.ws_bytes = L.dv_unsupervised_workspace_bytes(n, D)
        assert self.ws_bytes > 0
        self.ws = Buf((self.ws_bytes + 7) // 8, torch.float64, float("nan"))

    def args(self, **kw):
        o = self.outs
        a = dict(mu=self.mu_p, lv=self.lv_p, ld=self.ld, rs=self.rs, N=self.N, D=self.D, rows=self.inputs[-2].ptr,
                 n=self.n, eps=self.inputs[-1].ptr, cov=o[0].ptr, eig=o[1].ptr, sweeps=o[2].ptr, mi=o[3].ptr,
                 edges=o[4].ptr, sampled=o[5].ptr, ws=self.ws.ptr, wsb=self.ws_bytes)
        a.update(kw)
        return tuple(a.values()) + (_lib()[1],)

    def run(self):
        got = []
        for _ in range(2):
            for b in self.outs:
                b.body.view(torch.uint8).fill_(0xA5)
            _call(LAUNCHES, "dv_unsupervised_fit", *self.args())
            got.append([b.body.clone() for b in self.outs])
            assert all(b.intact() for b in self.outs + self.inputs + [self.ws]), "a write past a buffer"
        for a, b in zip(*got):
            _same(a, b, "dv_unsupervised_fit repeat")
        D, n = self.D, self.n
        cov, eig, sweeps, mi, edges, sampled = (t.cpu().numpy() for t in got[0])
        return (cov.reshape(2, D, D), eig.reshape(2, 2, D), sweeps.reshape(2, 2), mi.reshape(2, D, D),
                edges.reshape(2, D, 21), sampled.reshape(n, D))

    def check(self, mi_pairs=None, tc_checked=True):
        cov, eig, sweeps, mi, edges, sampled = self.run()
        rows = self.rows_h.numpy()
        mu, lv, eps = self.mu_h.numpy()[rows], self.lv_h.numpy()[rows], self.eps_h.numpy()
        # the sampled codes: fmaf(expf(lv / 2), eps, mu) against the fp64 formula, within expf's 2 ulp times |eps|
        # plus the one rounding of the sum
        want = R.sampled(mu, lv, eps)
        e = np.exp(lv.astype(np.float64) / 2).astype(np.float32)
        tol = (2 * np.spacing(e).astype(np.float64) * np.abs(eps.astype(np.float64))
               + 0.5 * np.spacing(np.abs(want).astype(np.float32)))
        err = np.abs(sampled - want)
        assert (err <= tol).all(), ("sampled", float((err / tol).max()))
        codes = [mu, sampled]
        lam_r_min = []
        for r in range(2):
            C = R.cov(codes[r])
            assert np.abs(cov[r] - C).max() <= 1e-12 * np.abs(C).max() + 1e-300, ("cov", r)
            assert np.array_equal(cov[r], cov[r].T)
            assert (sweeps[r] >= 0).all(), ("Jacobi cap", r, sweeps)
            for k, M in enumerate((R.correlation(cov[r]), R.s_matrix(cov[r]))):
                lam = np.linalg.eigvalsh(M)
                assert np.all(np.diff(eig[r, k]) >= 0), ("not ascending", r, k)
                assert np.abs(eig[r, k] - lam).max() <= 1e-12 * max(np.abs(lam).max(), 1e-300), ("eig", r, k)
            lam_r, lam_s = R.eigenvalues(C)
            lam_r_min.append(lam_r[0])
            if tc_checked and lam_r[0] >= 1e-4:
                from disvae.evaluate import unsupervised_from_fit
                got = unsupervised_from_fit(torch.from_numpy(cov), torch.from_numpy(eig), torch.from_numpy(mi))
                got = got[("mean", "sampled")[r]]
                want_s = R.scores_from(C, lam_r, lam_s, np.zeros((self.D, self.D)))
                for key in R.KEYS[:3]:
                    assert abs(got[key] - want_s[key]) <= 1e-9 * max(abs(want_s[key]), 1e-9 * np.trace(C)), (key, r)
            x = codes[r].astype(np.float32)
            E = np.stack([MR.edges(x[:, d]) for d in range(self.D)])
            _same(torch.from_numpy(edges[r]), torch.from_numpy(E), "edges")
            b = R.bins(x)
            pairs = mi_pairs if mi_pairs is not None else [(i, j) for i in range(self.D) for j in range(self.D)]
            for i, j in pairs:
                assert abs(mi[r, i, j] - MR.mutual_info(b[j], b[i])) <= 1e-12, ("mi", r, i, j)
        return cov, eig, sweeps, mi, lam_r_min


def _inputs(N, n, D, seed, kind="correlated"):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(N, D, generator=g, dtype=torch.float64)
    if kind == "correlated":
        z = z @ (torch.eye(D, dtype=torch.float64) + 0.6 / D ** 0.5 * torch.randn(D, D, generator=g, dtype=torch.float64))
    mu = (z * (0.5 + torch.rand(D, generator=g, dtype=torch.float64))).float()
    lv = (-2.0 + 0.5 * torch.randn(N, D, generator=g)).float()
    rows = torch.randint(N, (n,), generator=g)
    eps = torch.randn(n, D, generator=g)
    return mu, lv, rows, eps


def _sample_pairs(D, k, seed):
    if D * D <= 128:
        return None
    rng = np.random.default_rng(seed)
    return [(i, i) for i in range(0, D, 17)] + [tuple(rng.integers(D, size=2)) for _ in range(k)]


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("D, n", [(2, 2), (10, 10000), (128, 32768)])
def test_fit_matches_the_restatement(layout, D, n):
    mu, lv, rows, eps = _inputs(max(n, 64) + 7, n, D, seed=D + n)
    UnsCase(mu, lv, rows, eps, layout).check(mi_pairs=_sample_pairs(D, 48, D))


@pytest.mark.parametrize("D", [2, 10])
def test_independent_codes(D):
    mu, lv, rows, eps = _inputs(4000, 3000, D, seed=7, kind="independent")
    *_, lam_min = UnsCase(mu, lv, rows, eps).check()
    assert min(lam_min) > 0.8


def test_known_covariance():
    """Four points (+-1, 0), (0, +-1) and logvar far below fp32's range of exp: both representations have covariance
    2/3 I exactly, TC 0 and W 0."""
    mu = torch.tensor([[1.0, 0.0], [-1.0, 0.0], [0.0, 1.0], [0.0, -1.0]])
    lv = torch.full((4, 2), -300.0)
    case = UnsCase(mu, lv, torch.arange(4), torch.randn(4, 2, generator=torch.Generator().manual_seed(1)))
    cov, eig, sweeps, mi, _ = case.check()
    for r in range(2):
        assert np.abs(cov[r] - np.diag([2 / 3, 2 / 3])).max() <= 1e-16
        assert (eig[r, 0] == 1.0).all() and (sweeps[r] == 0).all()
    from disvae.evaluate import unsupervised_from_fit
    s = unsupervised_from_fit(*(torch.from_numpy(a) for a in (cov, eig, mi)))
    for rep in s.values():
        assert rep["gaussian_total_correlation"] == 0.0
        assert abs(rep["gaussian_wasserstein_correlation"]) <= 1e-15


def test_constant_duplicated_tied_and_narrow_latents():
    """Latent 1 constant (mean and sampled: logvar -300), latent 3 a copy of latent 0, latent 4 tied on a grid of 0.5,
    latent 5 three values one ulp apart (numpy refuses to bin it)."""
    mu, lv, rows, eps = _inputs(3000, 2500, 8, seed=11)
    mu[:, 1] = 1.5
    lv[:, 1] = -300.0
    mu[:, 3], lv[:, 3] = mu[:, 0], lv[:, 0]
    mu[:, 4] = torch.round(mu[:, 4] * 2) / 2
    one = np.float32(1.0)
    ulps = np.array([one, np.nextafter(one, np.float32(2)), np.nextafter(np.nextafter(one, np.float32(2)),
                                                                        np.float32(2))], np.float32)
    mu[:, 5] = torch.from_numpy(ulps[np.arange(3000) % 3])
    lv[:, 5] = -300.0
    case = UnsCase(mu, lv, rows, eps, "q_zCx")
    cov, eig, sweeps, mi, _ = case.check(tc_checked=False)
    assert (cov[:, 1, :] == 0).all() and (mi[:, 1, :] == 0).all() and (mi[:, :, 1] == 0).all()
    from disvae.evaluate import unsupervised_from_fit
    with pytest.warns(RuntimeWarning, match="linearly dependent"):
        s = unsupervised_from_fit(*(torch.from_numpy(a) for a in (cov, eig, mi)))
    assert s["mean"]["gaussian_total_correlation"] == float("inf")
    assert np.isfinite(s["sampled"]["gaussian_total_correlation"])   # eps differs between the copies


def test_refusals_launch_nothing():
    mu, lv, rows, eps = _inputs(100, 50, 4, seed=1)
    case = UnsCase(mu, lv, rows, eps)
    L, _ = _lib()
    torch.cuda.synchronize()
    before = L.dv_launch_count()
    for kw, code in [(dict(D=1), DV_ERR_BAD_SHAPE), (dict(D=129), DV_ERR_BAD_SHAPE), (dict(n=1), DV_ERR_BAD_SHAPE),
                     (dict(n=32769), DV_ERR_BAD_SHAPE), (dict(N=0), DV_ERR_BAD_SHAPE), (dict(ld=0), DV_ERR_BAD_SHAPE),
                     (dict(rs=0), DV_ERR_BAD_SHAPE), (dict(mu=None), DV_ERR_BAD_ARG), (dict(lv=None), DV_ERR_BAD_ARG),
                     (dict(rows=None), DV_ERR_BAD_ARG), (dict(eps=None), DV_ERR_BAD_ARG),
                     (dict(cov=None), DV_ERR_BAD_ARG), (dict(eig=None), DV_ERR_BAD_ARG),
                     (dict(sweeps=None), DV_ERR_BAD_ARG), (dict(mi=None), DV_ERR_BAD_ARG),
                     (dict(mu=case.mu_p + 2), DV_ERR_BAD_ARG), (dict(rows=case.inputs[-2].ptr + 4), DV_ERR_BAD_ARG),
                     (dict(cov=case.outs[0].ptr + 4), DV_ERR_BAD_ARG), (dict(sweeps=case.outs[2].ptr + 2), DV_ERR_BAD_ARG),
                     (dict(edges=case.outs[4].ptr + 2), DV_ERR_BAD_ARG), (dict(sampled=case.outs[5].ptr + 2), DV_ERR_BAD_ARG),
                     (dict(ws=case.ws.ptr + 4), DV_ERR_BAD_ARG), (dict(ws=None), DV_ERR_WORKSPACE),
                     (dict(wsb=case.ws_bytes - 1), DV_ERR_WORKSPACE)]:
        assert L.dv_unsupervised_fit(*case.args(**kw)) == code, kw
    assert L.dv_launch_count() == before
    assert L.dv_unsupervised_workspace_bytes(50, 1) == 0 and L.dv_unsupervised_workspace_bytes(32769, 4) == 0
    assert L.dv_unsupervised_workspace_bytes(1, 4) == 0 and L.dv_unsupervised_workspace_bytes(50, 129) == 0
    # edges and sampled are optional
    _call(LAUNCHES, "dv_unsupervised_fit", *case.args(edges=None, sampled=None))


def test_graph_replay_is_bit_identical():
    mu, lv, rows, eps = _inputs(5000, 4000, 16, seed=2)
    case = UnsCase(mu, lv, rows, eps, "padded")
    case.run()
    L, _ = _lib()
    _graph_replays(lambda: L.dv_unsupervised_fit(*case.args()), case.outs, "dv_unsupervised_fit")


# ---- the Python entry points ----------------------------------------------------------------------------------------
def test_unsupervised_scores_on_q_zCx_views():
    from disvae.evaluate import unsupervised_draws, unsupervised_scores
    mu, lv, _, _ = _inputs(3000, 2, 6, seed=3)
    q = torch.stack([mu, lv], -1).to(DEV)
    state = (torch.get_rng_state(), torch.cuda.get_rng_state(DEV))
    scores, h = unsupervised_scores(*q.unbind(-1), num_train=2000, seed=5)
    assert all(torch.equal(a, b) for a, b in zip(state, (torch.get_rng_state(), torch.cuda.get_rng_state(DEV))))
    rows, eps = unsupervised_draws(3000, 2000, 6, 5, DEV)
    assert torch.equal(h["rows"], rows.cpu())
    x = [mu[rows.cpu()].numpy(), None]
    cov = h["cov"].numpy()
    x[1] = (mu[rows.cpu()].double() + torch.exp(lv[rows.cpu()].double() / 2) * eps.cpu().double()).numpy()
    for r, name in enumerate(("mean", "sampled")):
        want = R.scores(x[r].astype(np.float32))
        for k in R.KEYS[:3]:
            assert abs(scores[name][k] - want[k]) <= 1e-6 * max(1.0, abs(want[k])), (name, k)
        assert abs(scores[name]["mutual_info_score"] - want["mutual_info_score"]) <= (1e-12 if r == 0 else 1e-2)
        assert np.abs(cov[r] - R.cov(x[r])).max() <= 1e-5 * np.abs(cov[r]).max()
    assert set(h) == {"rows", "cov", "eigenvalues", "constant", "mutual_information", "bin_edges", "solver_sweeps"}
    assert h["constant"].shape == (2, 6) and not h["constant"].any()
    assert (torch.diagonal(h["mutual_information"], dim1=1, dim2=2) == 0).all()


# ---- the Evaluator and sweeps ---------------------------------------------------------------------------------------
from test_udr_gpu import B, IMG, LOADER_SEED, SPECS, _labelled, _read, _same_helpers, _Unlabelled  # noqa: E402


def _sweep(tmp, specs, dataset, epochs, unsupervised_every=0, resume_from=None, **kw):
    import disvae
    from disvae.data import DeviceLoader
    from disvae.models.losses import get_loss_f
    from disvae.sweep import Sweep
    from disvae.utils.modelIO import load_training_state
    members = []
    for k, (kind, seed) in enumerate(specs):
        save_dir = str(tmp / ("m_%s_%d" % (kind, seed)))
        os.makedirs(save_dir, exist_ok=True)
        torch.manual_seed(seed)
        model = disvae.init_specific_model("Burgess", IMG, 10)
        loss_f = get_loss_f(kind, rec_dist="bernoulli", reg_anneal=100, betaH_B=4, betaB_initC=0, betaB_finC=25,
                            betaB_G=100, btcvae_A=-1, btcvae_B=6, btcvae_G=1, n_data=len(dataset), latent_dim=10,
                            device=DEV)
        tr = disvae.Trainer(model, torch.optim.Adam(model.parameters(), lr=5e-4), loss_f, device=DEV,
                            logger=logging.getLogger("uns-gpu"), save_dir=save_dir, is_progress_bar=False)
        if resume_from is not None:
            load_training_state(tr, os.path.join(str(resume_from / ("m_%s_%d" % (kind, seed))), "training-state-0.pt"))
        members.append(tr)
    sweep = Sweep(members, seeds=[s for _, s in specs], unsupervised_every=unsupervised_every)
    torch.manual_seed(0)
    sweep(DeviceLoader(dataset, B, seed=LOADER_SEED, device=DEV), epochs=epochs, checkpoint_every=1, **kw)
    return sweep


def _uns_files(d):
    return sorted(f for f in os.listdir(d) if f.startswith("unsupervised_scores"))


def _same_uns_files(a, b, names):
    for f in names:
        if f.endswith(".log"):
            assert _read(os.path.join(a, f)) == _read(os.path.join(b, f)), f
        else:
            _same_helpers(torch.load(os.path.join(a, f), weights_only=False),
                          torch.load(os.path.join(b, f), weights_only=False))


def test_unsupervised_every_leaves_training_and_every_file_as_they_are(tmp_path):
    from test_eval_resident_gpu import _n_samples
    with _n_samples(512):
        on = _sweep(tmp_path / "on", SPECS, _labelled(), 2, unsupervised_every=1, metrics_every=1, sap_score=True)
        rng_on = (torch.get_rng_state(), torch.cuda.get_rng_state(DEV))
        off = _sweep(tmp_path / "off", SPECS, _labelled(), 2, metrics_every=1, sap_score=True)
        rng_off = (torch.get_rng_state(), torch.cuda.get_rng_state(DEV))
    assert all(torch.equal(a, b) for a, b in zip(rng_on, rng_off)), "the scores moved a global generator"
    for a, b in zip(on.members, off.members):
        for (n, p), q in zip(a.model.named_parameters(), b.model.parameters()):
            assert torch.equal(p, q), n
        files = sorted(os.listdir(b.save_dir))
        assert sorted(f for f in os.listdir(a.save_dir) if not f.startswith("unsupervised")) == files
        for f in files:
            if f.endswith(".log"):
                assert _read(os.path.join(a.save_dir, f)) == _read(os.path.join(b.save_dir, f)), f
            elif f.endswith((".pt", ".pth")):
                x = torch.load(os.path.join(a.save_dir, f), weights_only=False)
                y = torch.load(os.path.join(b.save_dir, f), weights_only=False)
                if isinstance(x, dict) and all(torch.is_tensor(v) for v in x.values()):
                    _same_helpers(x, y)
        assert _uns_files(a.save_dir) == ["unsupervised_scores-0.log", "unsupervised_scores-1.log",
                                          "unsupervised_scores_helpers-0.pth", "unsupervised_scores_helpers-1.pth"]
    # the epoch-1 files are what Sweep.unsupervised_scores writes after epoch 1
    out = on.unsupervised_scores()
    for m, (scores, helpers) in zip(on.members, out):
        assert _read(os.path.join(m.save_dir, "unsupervised_scores.log")) == _read(
            os.path.join(m.save_dir, "unsupervised_scores-1.log"))
        got = torch.load(os.path.join(m.save_dir, "unsupervised_scores_helpers.pth"), weights_only=False)
        _same_helpers(got, torch.load(os.path.join(m.save_dir, "unsupervised_scores_helpers-1.pth"), weights_only=False))
        assert got["rows"].shape == (10000,) and (got["solver_sweeps"] >= 0).all()
        assert set(scores) == {"mean", "sampled"}
    assert all(not m.model.training for m in on.members)
    # member 1 alone writes the same files
    with _n_samples(512):
        lone = _sweep(tmp_path / "lone", SPECS[1:2], _labelled(), 2, unsupervised_every=1, metrics_every=1,
                      sap_score=True)
    names = ["unsupervised_scores-0.log", "unsupervised_scores-1.log", "unsupervised_scores_helpers-0.pth",
             "unsupervised_scores_helpers-1.pth"]
    _same_uns_files(on.members[1].save_dir, lone.members[0].save_dir, names)


def test_unsupervised_every_on_an_unlabelled_dataset_and_after_a_resume(tmp_path):
    specs = [("betaH", 1), ("btcvae", 2)]
    full = _sweep(tmp_path / "full", specs, _Unlabelled(), 2, unsupervised_every=1)
    _sweep(tmp_path / "first", specs, _Unlabelled(), 1, unsupervised_every=1, save_state=True)
    resumed = _sweep(tmp_path / "resumed", specs, _Unlabelled(), 1, unsupervised_every=1,
                     resume_from=tmp_path / "first")
    for a, b in zip(full.members, resumed.members):
        assert _uns_files(b.save_dir) == ["unsupervised_scores-1.log", "unsupervised_scores_helpers-1.pth"]
        _same_uns_files(a.save_dir, b.save_dir, _uns_files(b.save_dir))
        h = torch.load(os.path.join(a.save_dir, "unsupervised_scores_helpers-0.pth"), weights_only=False)
        assert h["cov"].shape == (2, 10, 10) and h["rows"].max() < 2048


def test_evaluator_on_an_unlabelled_dataset():
    import disvae
    from disvae.evaluate import unsupervised_scores
    torch.manual_seed(4)
    model = disvae.init_specific_model("Burgess", IMG, 10).to(DEV)
    ev = disvae.Evaluator(model, None, device=DEV, logger=logging.getLogger("uns-gpu"), save_dir="/nonexistent",
                          is_progress_bar=False)
    loader = torch.utils.data.DataLoader(_Unlabelled(), batch_size=512, shuffle=False)
    model.eval()
    got = ev.compute_unsupervised_scores(loader, num_train=3000, seed=9)
    mean, logvar = ev._compute_q_zCx(loader)[1]
    assert got == unsupervised_scores(mean, logvar, num_train=3000, seed=9)[0]
    assert set(got) == {"mean", "sampled"} and set(got["mean"]) == set(R.KEYS)
