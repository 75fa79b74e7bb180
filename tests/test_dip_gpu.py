"""DIP-VAE-I / DIP-VAE-II on the GPU: the covariance-penalty kernels against fp64 at training shapes and input edges,
whole-model gradients against the fp64 oracle on the same ReLU branch, and the loss on every path a loss runs on --
CUDA graph against eager (annealed, recording, uint8 batches), a sweep against lone runs, a resumed run against an
uninterrupted one, and the Evaluator's test_losses.log."""
import json
import logging
import os
from collections import OrderedDict, defaultdict

import pytest
import torch

from oracle import disvae_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
DV_ERR_BAD_SHAPE, DV_ERR_BAD_ARG = -1, -2
G_TERMS = (0.7, 1.3)                       # upstream gradient of (od, dd) in the kernel tests


def dip64(mu, logvar, dip_type):
    """(od, dd) of the issue's formulas in the dtype of the inputs (fp64 in the references), differentiable."""
    B = mu.shape[0]
    c = mu - mu.mean(0)
    C = c.t() @ c / B
    if dip_type == "II":
        C = C + torch.diag(logvar.exp().mean(0))
    d = torch.diagonal(C)
    return ((C - torch.diag(d)) ** 2).sum(), ((d - 1) ** 2).sum()


# ---- the kernels against fp64 ----------------------------------------------------------------------------------------
SHAPES = [(1, 10), (2, 10), (33, 7), (64, 10), (1000, 10), (1024, 10), (256, 64), (2048, 64), (1024, 1), (512, 1024)]
REGIMES = ["normal", "offset", "collapsed", "collinear", "wide_logvar"]


def _inputs(B, D, regime, seed):
    g = torch.Generator().manual_seed(seed)
    mu = torch.randn(B, D, generator=g)
    lv = 0.5 * torch.randn(B, D, generator=g)
    if regime == "offset":
        mu = 100 + 0.01 * torch.randn(B, D, generator=g)
    elif regime == "collapsed":
        mu[:, D // 2] = 3.25
    elif regime == "collinear":
        mu[:, 1:] = mu[:, :1] + 1e-3 * torch.randn(B, D - 1, generator=g)
    elif regime == "wide_logvar":
        lv = torch.rand(B, D, generator=g) * 30 - 20
    return mu, lv


def _run(mu, lv, dip_type, interleaved=True):
    """ops.DipFn on the encoder's interleaved [B, D, 2] layout (or contiguous mu / logvar) -> (terms, g_mu, g_logvar)."""
    from disvae import ops
    if interleaved:
        ml = torch.stack([mu, lv], dim=-1).to(DEV).requires_grad_(True)
        m, l = ml[..., 0], ml[..., 1]
    else:
        m, l = mu.to(DEV).requires_grad_(True), lv.to(DEV).requires_grad_(True)
    terms = ops.DipFn.apply(m, l, dip_type)
    terms.backward(torch.tensor(G_TERMS, device=DEV))
    if interleaved:
        return terms.detach(), ml.grad[..., 0].contiguous(), ml.grad[..., 1].contiguous()
    return terms.detach(), m.grad, l.grad if l.grad is not None else torch.zeros_like(l)


def _within(got, want, scale, tol, what):
    err = (got.detach().double().cpu() - want).abs().max().item()
    assert err <= tol * scale, "%s: |err| %.3e > %.1e x %.3e" % (what, err, tol, scale)


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("dip_type", ["I", "II"])
@pytest.mark.parametrize("B,D", SHAPES, ids=["%dx%d" % s for s in SHAPES])
def test_kernel_matches_fp64(B, D, dip_type, regime):
    if regime == "wide_logvar" and dip_type == "I":
        pytest.skip("DIP-VAE-I does not read logvar")
    if regime == "collinear" and D < 2:
        pytest.skip("one column")
    mu, lv = _inputs(B, D, regime, seed=B * 7919 + D + len(regime))
    m64, l64 = mu.double().requires_grad_(True), lv.double().requires_grad_(True)
    od, dd = dip64(m64, l64, dip_type)
    (G_TERMS[0] * od + G_TERMS[1] * dd).backward()
    g_lv64 = l64.grad if l64.grad is not None else torch.zeros_like(l64)      # DIP-VAE-I: no dependence on logvar
    terms, g_mu, g_lv = _run(mu, lv, dip_type)
    _within(terms[0], od.detach(), max(abs(od.item()), 1.0), 1e-5, "od")
    _within(terms[1], dd.detach(), max(abs(dd.item()), 1.0), 1e-5, "dd")
    _within(g_mu, m64.grad, m64.grad.abs().max().item(), 1e-5, "g_mu")
    _within(g_lv, g_lv64, g_lv64.abs().max().item(), 1e-5, "g_logvar")
    if dip_type == "I":
        assert not g_lv.any()
    if B == 1:
        assert not g_mu.any()                              # Cov_mu of one row is 0
    # bit-identical on a second call, and from contiguous inputs
    for again in (_run(mu, lv, dip_type), _run(mu, lv, dip_type, interleaved=False)):
        for a, b in zip(again, (terms, g_mu, g_lv)):
            assert torch.equal(a, b)


def test_refusals_launch_nothing():
    """Bad shapes, bad types and NULL or misaligned pointers come back as status codes with no launch."""
    from disvae import _native as N
    L, S = N.lib(), N.stream()
    buf = torch.zeros(1 << 16, device=DEV)
    a = buf.data_ptr()
    terms = torch.full((2,), 7.0, device=DEV)
    B, D = 8, 4

    def refused(rc_want, fn, *args):
        before = L.dv_launch_count()
        rc = getattr(L, fn)(*args)
        torch.cuda.synchronize()
        assert rc == rc_want and L.dv_launch_count() == before, (fn, args, rc)

    def fwd(mu=a, lv=a, B_=B, D_=D, t=1, out=terms.data_ptr(), ws=a):
        return (mu, lv, 2, 2 * D_, B_, D_, t, out, ws, S)

    def bwd(mu=a, lv=a, B_=B, D_=D, t=2, g=a, gm=a, gl=a, ws=a):
        return (mu, lv, 2, 2 * D_, B_, D_, t, g, gm, gl, ws, S)

    for shape in (dict(B_=0), dict(B_=-1), dict(D_=0), dict(D_=1025), dict(t=0), dict(t=3)):
        refused(DV_ERR_BAD_SHAPE, "dv_dip_fwd", *fwd(**shape))
        refused(DV_ERR_BAD_SHAPE, "dv_dip_bwd", *bwd(**shape))
    for bad in (dict(mu=None), dict(lv=None), dict(out=None), dict(ws=None), dict(mu=a + 2), dict(lv=a + 1),
                dict(out=terms.data_ptr() + 2), dict(ws=a + 4)):
        refused(DV_ERR_BAD_ARG, "dv_dip_fwd", *fwd(**bad))
    for bad in (dict(mu=None), dict(lv=None), dict(g=None), dict(ws=None), dict(g=a + 2), dict(gm=a + 2),
                dict(gl=a + 3), dict(ws=a + 8)):
        refused(DV_ERR_BAD_ARG, "dv_dip_bwd", *bwd(**bad))
    refused(0, "dv_dip_bwd", *bwd(gm=None, gl=None))           # nothing asked for: nothing launched
    assert torch.equal(terms, torch.full((2,), 7.0, device=DEV))
    for b, d in ((0, 10), (10, 0), (10, 1025)):
        assert L.dv_dip_workspace_bytes(b, d) == 0
    assert L.dv_dip_workspace_bytes(1, 1) > 0 and L.dv_dip_workspace_bytes(2048, 1024) % 16 == 0


# ---- whole-model gradients against the fp64 oracle on the same branch ---------------------------------------------
@pytest.mark.parametrize("dip_type", ["I", "II"])
@pytest.mark.parametrize("img,z,B", [((1, 64, 64), 10, 1024), ((3, 64, 64), 64, 256)], ids=["c2", "3x64x64-z64"])
def test_model_gradients_full_batch_same_branch(img, z, B, dip_type):
    import disvae
    from disvae import ops
    from disvae.models.losses import get_loss_f
    from oracle import same_branch as SB
    torch.manual_seed(1234)
    m = disvae.init_specific_model("Burgess", img, z).to(DEV)
    m.train()
    p32 = OrderedDict((k, v.detach().cpu().clone()) for k, v in m.state_dict().items())
    torch.manual_seed(B + z)
    x, eps = torch.rand(B, *img), torch.randn(B, z)
    lf = get_loss_f("dip" + dip_type, rec_dist="bernoulli", reg_anneal=0)
    xd = x.to(DEV)
    m.inject_noise([eps])
    ops.start_trace()
    recon, (mu, lv), _ = m(xd)
    trace = ops.stop_trace()
    loss = lf(xd, recon, (mu, lv), True, None)
    m.zero_grad()
    loss.backward()
    ours = {k: prm.grad for k, prm in m.named_parameters()}

    def run64(p, dp):
        ro, (mo, lo), _ = O.vae_forward(p, x.double(), eps.double())
        l, _ = O.loss_betaH(x.double(), ro, mo, lo, 1, "bernoulli", 1, 0)        # rec + kl
        od, dd = dip64(mo, lo, dip_type)
        l = l + lf.lambda_od * od + lf.lambda_d * dd
        l.backward()
        return l.item()
    ref = SB.same_branch_reference(trace, p32, run64)
    assert abs(loss.item() - ref["loss"]) <= 1e-4 * abs(ref["loss"]), (loss.item(), ref["loss"])
    assert ref["flip_max_rel"] <= 1e-3, "a ReLU flipped at |pre-activation| = %.2e of its layer's scale" % ref["flip_max_rel"]
    err, key = SB.grad_errors(ours, ref["grads"])
    print("dip%s B=%d z=%d: gradients vs fp64 on the same branch %.2e (worst %s, %d flipped units)"
          % (dip_type, B, z, err, key, ref["flips"]))
    assert err <= 3e-4, "grad %s: %.2e vs fp64 on the same branch" % (key, err)


# ---- every path a loss runs on ----------------------------------------------------------------------------------------
STEPS, EVERY = 20, 5


def _train(name, mode, tmp_path, u8=True):
    """One epoch of STEPS steps on 1x32x32 batches of 64, annealing over 7 steps, recording every 5th.
    mode: 'graph' | 'eager'.  u8: host uint8 batches (converted on the device), else the same batches as float / 255."""
    import disvae
    from disvae.models.losses import get_loss_f
    from test_anneal_graph_gpu import _state
    torch.manual_seed(1234)
    m = disvae.init_specific_model("Burgess", (1, 32, 32), 10)
    opt = torch.optim.Adam(m.parameters(), lr=5e-4)
    lf = get_loss_f(name, rec_dist="bernoulli", reg_anneal=7, dip_lambda_od=5)
    lf.record_loss_every = EVERY
    tr = disvae.Trainer(m, opt, lf, device=torch.device(DEV), logger=logging.getLogger("dip"), save_dir=str(tmp_path),
                        is_progress_bar=False)
    tr.use_cuda_graph = mode == "graph"
    m.train()
    g = torch.Generator().manual_seed(5)
    xs = [torch.randint(0, 256, (64, 1, 32, 32), generator=g, dtype=torch.uint8) for _ in range(STEPS)]
    if not u8:
        xs = [x.float() / 255 for x in xs]
    storer = defaultdict(list)
    tr._train_epoch([(x, None) for x in xs], storer, 0)
    torch.cuda.synchronize()
    return tr, storer, _state(tr)


@pytest.mark.parametrize("name", ["dipI", "dipII"])
def test_graph_equals_eager(name, tmp_path):
    tr_g, st_g, s_g = _train(name, "graph", tmp_path)
    tr_e, st_e, s_e = _train(name, "eager", tmp_path)
    _, st_f, s_f = _train(name, "eager", tmp_path, u8=False)
    assert len(tr_g._graphs) == 1 and not tr_e._graphs
    assert tr_g.loss_f.n_train_steps == STEPS and int(tr_g.loss_f._step_dev.item()) == STEPS
    for other in (s_e, s_f):
        assert s_g.keys() == other.keys()
        for k in s_g:
            assert torch.equal(s_g[k], other[k]), k
    keys = ["recon_loss", "kl_loss"] + ["kl_loss_%d" % i for i in range(10)] + ["dip_od_loss", "dip_d_loss", "loss"]
    assert list(st_g) == keys
    assert len(st_g["loss"]) == len(range(1, STEPS + 1, EVERY))
    assert list(st_g.items()) == list(st_e.items()) == list(st_f.items())


def test_sweep_equals_lone_runs(tmp_path):
    from test_sweep_gpu import EPOCHS, _assert_same, _lone, _sweep
    specs = [("dipI", 21), ("dipII", 22), ("btcvae", 23)]
    swept = _sweep(specs, tmp_path / "sweep")
    for (kind, seed), got in zip(specs, swept):
        want = _lone(kind, seed, str(tmp_path / ("lone_" + kind)))
        assert want["graphs"] == 1 and want["steps"] == EPOCHS * 64
        assert (kind.startswith("dip")) == ("dip_od_loss" in want["log"])
        _assert_same(got, want, kind)


def test_resumed_run_equals_uninterrupted(tmp_path):
    from test_resume_gpu import _split_and_resume
    _split_and_resume(tmp_path, dict(losses=["dipII"], img=32, loader="device", every=1))
    with open(tmp_path / "b" / "m0_dipII" / "train_losses.log") as f:
        assert {"dip_od_loss", "dip_d_loss"} <= {r.split(",")[1] for r in f.read().splitlines()[1:]}


@pytest.mark.parametrize("name", ["dipI", "dipII"])
def test_evaluator_losses(name, tmp_path):
    """test_losses.log of a DIP model: the documented keys, and values equal to fp64 on the model's own encoder outputs
    with the annealing at 1 (reg_anneal set, no training step taken)."""
    import disvae
    from disvae.evaluate import Evaluator
    from disvae.models.losses import get_loss_f
    torch.manual_seed(7)
    m = disvae.init_specific_model("Burgess", (1, 32, 32), 10).to(DEV)
    lf = get_loss_f(name, rec_dist="bernoulli", reg_anneal=1000, dip_lambda_od=2)
    x = torch.rand(128, 1, 32, 32)
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(x, torch.zeros(128)), batch_size=128)
    _, losses = Evaluator(m, lf, device=torch.device(DEV), logger=logging.getLogger("dip"), save_dir=str(tmp_path),
                          is_progress_bar=False)(loader, is_metrics=False, is_losses=True)
    keys = ["recon_loss", "kl_loss"] + ["kl_loss_%d" % i for i in range(10)] + ["dip_od_loss", "dip_d_loss", "loss"]
    assert list(losses) == keys
    with open(os.path.join(str(tmp_path), "test_losses.log")) as f:
        assert set(json.load(f)) == set(keys)
    m.eval()
    with torch.no_grad():
        recon, (mu, lv), _ = m(x.to(DEV))
    r64, mu64, lv64, x64 = recon.double().cpu(), mu.double().cpu(), lv.double().cpu(), x.double()
    rec = O.reconstruction_loss(x64, r64, "bernoulli").item()
    kl, kl_dims = O.kl_normal(mu64, lv64)
    od, dd = (t.item() for t in dip64(mu64, lv64, name[3:]))
    want = dict(recon_loss=rec, kl_loss=kl.item(), dip_od_loss=od, dip_d_loss=dd,
                loss=rec + kl.item() + lf.lambda_od * od + lf.lambda_d * dd)
    want.update(("kl_loss_%d" % i, v) for i, v in enumerate(kl_dims.tolist()))
    for k in keys:
        assert abs(losses[k] - want[k]) <= 1e-5 * max(abs(want[k]), 1.0), (k, losses[k], want[k])
