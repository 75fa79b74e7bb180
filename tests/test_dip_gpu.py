"""DIP-VAE-I / DIP-VAE-II on the GPU: whole-model gradients against the fp64 oracle on the same ReLU branch, and the
loss on every path a loss runs on -- CUDA graph against eager (annealed, recording, uint8 batches), a sweep against
lone runs, a resumed run against an uninterrupted one, and the Evaluator's test_losses.log.  The covariance-penalty
kernels themselves are tested path by path in test_dip_paths_gpu.py."""
import json
import logging
import os
from collections import OrderedDict, defaultdict

import pytest
import torch

from oracle import disvae_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


def dip64(mu, logvar, dip_type):
    """(od, dd) of the issue's formulas in the dtype of the inputs (fp64 in the references), differentiable."""
    B = mu.shape[0]
    c = mu - mu.mean(0)
    C = c.t() @ c / B
    if dip_type == "II":
        C = C + torch.diag(logvar.exp().mean(0))
    d = torch.diagonal(C)
    return ((C - torch.diag(d)) ** 2).sum(), ((d - 1) ** 2).sum()


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
