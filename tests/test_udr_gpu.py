"""UDR on the GPU: `dv_udr_fit` (csrc/dv_udr.cu) through the raw C ABI on guarded buffers against the fp64 numpy
restatement of tests/udr_reference.py, in both modes, K in {2, 3, 8, the limit}, D in {1, 2, 10, 128} and n in {2, 1000,
16384}, with collapsed latents, fully collapsed models, constant informative latents, duplicated latents and tied
values:
- KL within 1e-12 of its scale and the informative masks equal;
- raw within 1e-9 where the Lasso minimiser is unique; everywhere, every target's l1 norm (sum over a of |w_a|, the same
  for every minimiser of a Lasso) within 1e-9;
- pair scores within 1e-9 (where the minimiser is unique);
- the launch count, refusals that launch nothing, bit-identical repeats and a captured graph that replays to the
  eager bits;
and `udr_score` on synthetic codes of known ordering, and `Sweep.udr` and `udr_every` on trained sweeps, over data with
and without known factors."""
import logging
import os

import numpy as np
import pytest
import torch

import udr_reference as R
from score_kernels import (DEV, DV_ERR_BAD_ARG, DV_ERR_BAD_SHAPE, DV_ERR_WORKSPACE, Buf, _call, _graph_replays, _lib,
                           _same)

pytestmark = pytest.mark.gpu
KL_RTOL = 1e-12
RAW_TOL = 1e-9
PAIR_TOL = 1e-9
MODES = {"lasso": 0, "spearman": 1}


def _models(K, n, D, seed, collapsed=(), dead_model=None, constant=(), duplicate=(), ties=False):
    """Codes [K, n, D] of K models over shared factors: model k's informative latents are a signed permutation of the
    factors mixed slightly plus noise.  `collapsed` latents (mu and logvar near 0: KL far below 0.01), a fully
    collapsed model `dead_model`, `constant` informative latents (mu = 1.5 on every point), latents in `duplicate`
    copying latent 0, and `ties` (values rounded to a grid of 0.25)."""
    g = torch.Generator().manual_seed(seed)
    F = torch.randn(n, D, generator=g, dtype=torch.float64)
    mu = torch.empty(K, n, D, dtype=torch.float64)
    lv = torch.empty(K, n, D, dtype=torch.float64)
    for k in range(K):
        perm = torch.randperm(D, generator=g)
        sign = torch.where(torch.rand(D, generator=g) < 0.5, -1.0, 1.0).double()
        mix = torch.eye(D, dtype=torch.float64)[perm] * sign + 0.2 * torch.randn(D, D, generator=g, dtype=torch.float64)
        mu[k] = F @ mix + 0.3 * torch.randn(n, D, generator=g, dtype=torch.float64)
        lv[k] = -2.0 + 0.1 * torch.randn(n, D, generator=g, dtype=torch.float64)
        dead = list(collapsed) + (list(range(D)) if k == dead_model else [])
        for d in dead:
            mu[k, :, d] = 1e-3 * torch.randn(n, generator=g, dtype=torch.float64)
            lv[k, :, d] = 1e-3 * torch.randn(n, generator=g, dtype=torch.float64)
        for d in constant:
            mu[k, :, d] = 1.5
        for d in duplicate:
            mu[k, :, d] = mu[k, :, 0]
            lv[k, :, d] = lv[k, :, 0]
    if ties:
        mu = torch.round(mu * 4) / 4
    return mu.float(), lv.float()


class UdrCase:
    """One dv_udr_fit call through the raw ABI, every operand in a guarded buffer."""

    def __init__(self, mu, lv, mode):
        self.mu_h, self.lv_h, self.mode = mu, lv, mode
        self.K, self.n, self.D = mu.shape
        K, D = self.K, self.D
        self.inputs = [Buf(mu.numel(), torch.float32, mu.to(DEV)), Buf(lv.numel(), torch.float32, lv.to(DEV))]
        self.outs = [Buf(K * K * D * D, torch.float64), Buf(K * K, torch.float64), Buf(K * D, torch.float64),
                     Buf(K * K, torch.int32)]
        L, _ = _lib()
        self.ws_bytes = L.dv_udr_workspace_bytes(K, self.n, D)
        assert self.ws_bytes > 0
        self.ws = Buf((self.ws_bytes + 7) // 8, torch.float64, float("nan"))

    def args(self, **kw):
        a = dict(mu=self.inputs[0].ptr, lv=self.inputs[1].ptr, K=self.K, n=self.n, D=self.D, mode=MODES[self.mode],
                 alpha=R.ALPHA, thr=R.KL_THRESHOLD, raw=self.outs[0].ptr, pair=self.outs[1].ptr, kl=self.outs[2].ptr,
                 it=self.outs[3].ptr, ws=self.ws.ptr, wsb=self.ws_bytes)
        a.update(kw)
        return tuple(a.values()) + (_lib()[1],)

    def run(self):
        got = []
        for _ in range(2):
            for b in self.outs:
                b.body.view(torch.uint8).fill_(0xA5)
            _call(3, "dv_udr_fit", *self.args())
            got.append([b.body.clone() for b in self.outs])
            assert all(b.intact() for b in self.outs + self.inputs + [self.ws]), "a write past a buffer"
        for a, b in zip(*got):
            _same(a, b, "dv_udr_fit repeat")
        K, D = self.K, self.D
        raw, pair, kl, it = (t.cpu().numpy() for t in got[0])
        return raw.reshape(K, K, D, D), pair.reshape(K, K), kl.reshape(K, D), it.reshape(K, K)

    def check(self, unique=True, pairs=None):
        """The kernel against the restatement on the ordered pairs `pairs` (all by default)."""
        raw, pair, kl, it = self.run()
        K, D = self.K, self.D
        mu, lv = self.mu_h.numpy(), self.lv_h.numpy()
        want_kl = np.stack([R.kl(mu[k], lv[k]) for k in range(K)])
        assert np.abs(kl - want_kl).max() <= KL_RTOL * max(1.0, np.abs(want_kl).max()), "kl"
        inf = want_kl > R.KL_THRESHOLD
        assert np.array_equal(kl > R.KL_THRESHOLD, inf), "informative"
        assert np.isnan(pair[np.arange(K), np.arange(K)]).all() and np.isnan(raw[np.arange(K), np.arange(K)]).all()
        assert (it[np.arange(K), np.arange(K)] == 0).all()
        Z = {}
        feats = lambda k: Z.setdefault(k, R.features(mu[k], inf[k], self.mode))   # noqa: E731
        for i, j in (pairs if pairs is not None else [(i, j) for i in range(K) for j in range(K) if i != j]):
            want, sweeps = R.similarity(feats(i), feats(j), self.mode)
            if self.mode == "lasso":
                assert it[i, j] >= 0 and (sweeps >= 0).all(), ("did not converge", i, j)
                l1 = np.abs(raw[i, j].sum(0) - want.sum(0)).max()
                assert l1 <= RAW_TOL, ("l1 norms", i, j, l1)
            else:
                assert it[i, j] == 0
            if unique:
                err = np.abs(raw[i, j] - want).max()
                assert err <= RAW_TOL, ("raw", i, j, err)
                assert abs(pair[i, j] - R.pair_score(want, inf[i], inf[j])) <= PAIR_TOL, ("pair", i, j)
            if not inf[i].any() or not inf[j].any():
                assert pair[i, j] == 0.0
        return raw, pair, kl, it


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("K, n, D", [(2, 1000, 1), (2, 1000, 2), (3, 1000, 10), (8, 1000, 10), (3, 16384, 10),
                                     (2, 1000, 128)])
def test_fit_matches_the_restatement(mode, K, n, D):
    mu, lv = _models(K, n, D, seed=K * 1000 + D, collapsed=[D - 1] if D > 2 else [])
    UdrCase(mu, lv, mode).check()


@pytest.mark.parametrize("mode", list(MODES))
def test_edge_latents(mode):
    """Collapsed latents, a fully collapsed model and constant informative latents (unique minimisers)."""
    mu, lv = _models(4, 1000, 10, seed=3, collapsed=[8], dead_model=2, constant=[5])
    raw, pair, kl, _ = UdrCase(mu, lv, mode).check()
    assert (pair[2, [0, 1, 3]] == 0).all() and (pair[[0, 1, 3], 2] == 0).all()
    assert (raw[0, 1][5] == 0).all() and (raw[0, 1][:, 5] == 0).all()       # a constant feature is 0
    assert (kl[:, 5] > R.KL_THRESHOLD).all()


@pytest.mark.parametrize("mode", list(MODES))
def test_duplicated_latents_and_ties(mode):
    mu, lv = _models(3, 1000, 10, seed=5, duplicate=[4])
    UdrCase(mu, lv, mode).check(unique=mode == "spearman")
    mu, lv = _models(3, 1000, 10, seed=6, ties=True)
    UdrCase(mu, lv, mode).check(unique=mode == "spearman")


@pytest.mark.parametrize("mode", list(MODES))
def test_two_points(mode):
    mu, lv = _models(3, 2, 10, seed=8)
    UdrCase(mu, lv, mode).check(unique=mode == "spearman")


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("K, D", [(32, 128), (4096, 1), (2048, 2), (409, 10)])
def test_column_limit(mode, K, D):
    """K D = the 4096-column limit (409 x 10 just below it), the pairs checked on a sample."""
    mu, lv = _models(K, 1000 if K * D <= 4096 // 4 or D >= 10 else 200, D, seed=K, collapsed=[0] if D == 128 else [])
    case = UdrCase(mu, lv, mode)
    rng = np.random.default_rng(K)
    pairs = [(0, 1), (1, 0), (K - 1, 0), (0, K - 1)] + [tuple(rng.choice(K, 2, replace=False)) for _ in range(4)]
    case.check(unique=D <= 10, pairs=pairs)


def test_refusals_launch_nothing():
    mu, lv = _models(3, 100, 4, seed=1)
    case = UdrCase(mu, lv, "lasso")
    L, _ = _lib()
    torch.cuda.synchronize()
    before = L.dv_launch_count()
    for kw, code in [(dict(K=1), DV_ERR_BAD_SHAPE), (dict(D=0), DV_ERR_BAD_SHAPE), (dict(D=129), DV_ERR_BAD_SHAPE),
                     (dict(K=33, D=128), DV_ERR_BAD_SHAPE), (dict(n=1), DV_ERR_BAD_SHAPE),
                     (dict(n=16385), DV_ERR_BAD_SHAPE), (dict(mu=None), DV_ERR_BAD_ARG),
                     (dict(lv=None), DV_ERR_BAD_ARG), (dict(raw=None), DV_ERR_BAD_ARG), (dict(pair=None), DV_ERR_BAD_ARG),
                     (dict(kl=None), DV_ERR_BAD_ARG), (dict(it=None), DV_ERR_BAD_ARG), (dict(mode=2), DV_ERR_BAD_ARG),
                     (dict(mode=-1), DV_ERR_BAD_ARG), (dict(alpha=0.0), DV_ERR_BAD_ARG),
                     (dict(alpha=float("nan")), DV_ERR_BAD_ARG), (dict(alpha=float("inf")), DV_ERR_BAD_ARG),
                     (dict(thr=-1.0), DV_ERR_BAD_ARG), (dict(thr=float("nan")), DV_ERR_BAD_ARG),
                     (dict(mu=case.inputs[0].ptr + 2), DV_ERR_BAD_ARG), (dict(raw=case.outs[0].ptr + 4), DV_ERR_BAD_ARG),
                     (dict(it=case.outs[3].ptr + 2), DV_ERR_BAD_ARG), (dict(ws=case.ws.ptr + 4), DV_ERR_BAD_ARG),
                     (dict(ws=None), DV_ERR_WORKSPACE), (dict(wsb=case.ws_bytes - 1), DV_ERR_WORKSPACE)]:
        assert L.dv_udr_fit(*case.args(**kw)) == code, kw
    assert L.dv_launch_count() == before
    assert L.dv_udr_workspace_bytes(1, 100, 4) == 0 and L.dv_udr_workspace_bytes(2, 16385, 4) == 0
    assert L.dv_udr_workspace_bytes(2, 100, 4) >= (8 * 100 + 64) * 8


@pytest.mark.parametrize("mode", list(MODES))
def test_graph_replay_is_bit_identical(mode):
    mu, lv = _models(5, 1000, 10, seed=2, collapsed=[3])
    case = UdrCase(mu, lv, mode)
    case.run()
    L, _ = _lib()
    _graph_replays(lambda: L.dv_udr_fit(*case.args()), case.outs, "dv_udr_fit " + mode)


# ---- udr_score on codes of known ordering --------------------------------------------------------------------
def _known(K, n, kind, seed):
    """Codes of 6 latents over 5 shared factors (uniform on [-1, 1]) plus noise, the 6th collapsed: `perm` models
    encode a signed permutation of the factors, `rot` models a random rotation of them."""
    g = torch.Generator().manual_seed(seed)
    F = torch.rand(n, 5, generator=g) * 2 - 1
    mu = torch.zeros(K, n, 6)
    lv = torch.zeros(K, n, 6)
    for k in range(K):
        if kind == "perm":
            M = torch.eye(5)[torch.randperm(5, generator=g)] * torch.where(torch.rand(5, generator=g) < 0.5, -1.0, 1.0)
        else:
            M = torch.linalg.qr(torch.randn(5, 5, generator=g))[0]
        mu[k, :, :5] = F @ M + 0.05 * torch.randn(n, 5, generator=g)
        lv[k, :, :5] = -3.0
        mu[k, :, 5] = 1e-3 * torch.randn(n, generator=g)
    return mu.to(DEV), lv.to(DEV)


@pytest.mark.parametrize("correlation", list(MODES))
def test_known_ordering(correlation):
    """A permuted, sign-flipped code scores near 1 (one strong coefficient or correlation per latent), a rotated one
    spreads each latent over several factors.  The test asks for a margin of 0.2 between the lowest permuted and the
    highest rotated model: well inside the expected gap (about 0.4 for random rotations of 5 factors), well outside
    the noise of 1000 points."""
    from disvae.evaluate import udr_score
    perm = udr_score(*_known(6, 1000, "perm", 1), correlation=correlation)[0]["model_scores"]
    rot = udr_score(*_known(6, 1000, "rot", 2), correlation=correlation)[0]["model_scores"]
    assert min(perm) > 0.8 and min(perm) - max(rot) >= 0.2, (perm, rot)


def test_udr_score_helpers_and_groups():
    from disvae.evaluate import udr_score
    mu, lv = _known(6, 500, "perm", 3)
    scores, h = udr_score(mu, lv, groups=[[0, 2, 4], [5, 3, 1]])
    ref = R.udr(mu.cpu().numpy(), lv.cpu().numpy(), "lasso", [[0, 2, 4], [5, 3, 1]])
    assert np.abs(np.array(scores["model_scores"]) - ref["model_scores"]).max() <= PAIR_TOL
    assert h["groups"] == [[0, 2, 4], [5, 3, 1]] and h["pairwise"].shape == (6, 6)
    assert h["raw_correlations"].shape == (6, 6, 6, 6) and h["solver_iterations"].dtype == torch.int32
    assert torch.equal(h["informative"], h["kl"] > R.KL_THRESHOLD) and not h["informative"][:, 5].any()


# ---- sweeps ------------------------------------------------------------------------------------------------------
IMG, B, LOADER_SEED = (1, 32, 32), 256, 99


class _Unlabelled(torch.utils.data.Dataset):
    """The first 2048 images of the factor rectangles, without lat_sizes / lat_names."""

    def __init__(self):
        from synthetic_factors import FactorRectangles
        self.imgs = torch.round(FactorRectangles(k=8, size=IMG[-1]).imgs[:2048] * 255) / 255

    def __len__(self):
        return len(self.imgs)

    def __getitem__(self, i):
        return self.imgs[i], 0


def _labelled():
    from synthetic_factors import FactorRectangles
    ds = FactorRectangles(k=8, size=IMG[-1])
    ds.imgs = torch.round(ds.imgs * 255) / 255
    return ds


def _sweep(tmp, specs, dataset, udr_every=0, **kw):
    import disvae
    from disvae.data import DeviceLoader
    from disvae.models.losses import get_loss_f
    from disvae.sweep import Sweep
    members = []
    for k, (kind, seed) in enumerate(specs):
        save_dir = str(tmp / ("m%d_%s_%d" % (k, kind, seed)))
        os.makedirs(save_dir, exist_ok=True)
        torch.manual_seed(seed)
        model = disvae.init_specific_model("Burgess", IMG, 10)
        loss_f = get_loss_f(kind, rec_dist="bernoulli", reg_anneal=100, betaH_B=4, betaB_initC=0, betaB_finC=25, betaB_G=100,
                            btcvae_A=-1, btcvae_B=6, btcvae_G=1, n_data=len(dataset), latent_dim=10, device=DEV)
        members.append(disvae.Trainer(model, torch.optim.Adam(model.parameters(), lr=5e-4), loss_f, device=DEV,
                                      logger=logging.getLogger("udr-gpu"), save_dir=save_dir, is_progress_bar=False))
    sweep = Sweep(members, seeds=[s for _, s in specs], udr_every=udr_every)
    torch.manual_seed(0)
    sweep(DeviceLoader(dataset, B, seed=LOADER_SEED, device=DEV), checkpoint_every=1, **kw)
    return sweep


def _read(path):
    with open(path, "rb") as f:
        return f.read()


def _same_helpers(a, b):
    assert a.keys() == b.keys()
    for k in a:
        if torch.is_tensor(a[k]):
            assert torch.equal(a[k].view(-1).view(torch.uint8) if a[k].is_floating_point() else a[k],
                               b[k].view(-1).view(torch.uint8) if b[k].is_floating_point() else b[k]), k
        else:
            assert a[k] == b[k], k


SPECS = [("betaH", 21), ("btcvae", 22), ("betaB", 23)]


def test_udr_every_leaves_training_and_every_file_as_they_are(tmp_path):
    from test_eval_resident_gpu import _n_samples       # the estimator's 10,000 samples lowered for 4096 items
    with _n_samples(512):
        on = _sweep(tmp_path / "on", SPECS, _labelled(), epochs=2, metrics_every=1, sap_score=True, udr_every=1)
        rng_on = (torch.get_rng_state(), torch.cuda.get_rng_state(DEV))
        off = _sweep(tmp_path / "off", SPECS, _labelled(), epochs=2, metrics_every=1, sap_score=True)
        rng_off = (torch.get_rng_state(), torch.cuda.get_rng_state(DEV))
    assert all(torch.equal(a, b) for a, b in zip(rng_on, rng_off)), "UDR moved a global generator"
    for a, b in zip(on.members, off.members):
        for (n, p), q in zip(a.model.named_parameters(), b.model.parameters()):
            assert torch.equal(p, q), n
        files = sorted(os.listdir(b.save_dir))
        assert sorted(f for f in os.listdir(a.save_dir) if not f.startswith("udr")) == files
        for f in files:
            if f.endswith(".log"):
                assert _read(os.path.join(a.save_dir, f)) == _read(os.path.join(b.save_dir, f)), f
            elif f.endswith((".pt", ".pth")):
                x = torch.load(os.path.join(a.save_dir, f), weights_only=False)
                y = torch.load(os.path.join(b.save_dir, f), weights_only=False)
                if isinstance(x, dict) and all(torch.is_tensor(v) for v in x.values()):
                    _same_helpers(x, y)
        assert {f for f in os.listdir(a.save_dir) if f.startswith("udr")} == {
            "udr-0.log", "udr-1.log", "udr_helpers-0.pth", "udr_helpers-1.pth"}
    # udr-1.log is what Sweep.udr writes after epoch 1
    scores, helpers = on.udr()
    for k, m in enumerate(on.members):
        assert _read(os.path.join(m.save_dir, "udr.log")) == _read(os.path.join(m.save_dir, "udr-1.log"))
        got = torch.load(os.path.join(m.save_dir, "udr_helpers.pth"), weights_only=False)
        _same_helpers(got, torch.load(os.path.join(m.save_dir, "udr_helpers-1.pth"), weights_only=False))
        assert got["member"] == k and got["rows"].shape == (1000,)
    # a reordered member list: the same points, the scores permuted
    from disvae.evaluate import udr
    rev, rev_helpers = udr([m.model for m in on.members[::-1]], on.loader, seed=helpers_seed(on))
    assert rev["model_scores"] == scores["model_scores"][::-1]
    assert torch.equal(rev_helpers["rows"], helpers["rows"])
    assert all(not m.model.training for m in on.members)


def helpers_seed(sweep):
    from disvae.evaluate import evaluation_seed
    return evaluation_seed(sweep.loader.seed, sweep.members[0]._next_epoch - 1)


def test_udr_every_on_a_dataset_without_known_factors(tmp_path):
    sweep = _sweep(tmp_path, [("betaH", 1), ("betaH", 2)], _Unlabelled(), epochs=1, udr_every=1)
    for m in sweep.members:
        assert os.path.exists(os.path.join(m.save_dir, "udr-0.log"))
        h = torch.load(os.path.join(m.save_dir, "udr_helpers-0.pth"), weights_only=False)
        assert h["pairwise"].shape == (2, 2) and (h["solver_iterations"] >= 0).all()
    with pytest.raises(ValueError, match="lat_sizes"):
        sweep(sweep.loader, epochs=1, metrics_every=1)
