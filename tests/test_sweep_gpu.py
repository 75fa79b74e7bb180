"""disvae.sweep.Sweep on the GPU: every member of a sweep ends bit-identical to a lone Trainer run of its settings and
seed (parameters, Adam moments and step counters, train_losses.log, checkpoints), identical members stay identical
under concurrent replays, a sweep leaves no state behind that changes a later lone run, and the documented refusals
happen before any kernel launch.

Run as a script (`python tests/test_sweep_gpu.py KIND SEED OUT`) it trains one lone member in a fresh process and saves
its result to OUT.
"""
import logging
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda", 0)
IMG, B, EPOCHS, LOADER_SEED = (1, 32, 32), 64, 2, 99      # 4096 images: 64 steps per epoch, recording steps 1, 51, 101


def _dataset():
    """tests/synthetic_factors.FactorRectangles rounded to bytes (what ToTensor makes of 8-bit images)."""
    from synthetic_factors import FactorRectangles
    ds = FactorRectangles(k=8, size=IMG[-1])
    ds.imgs = torch.round(ds.imgs * 255) / 255
    return ds


def _loader():
    from disvae.data import DeviceLoader
    return DeviceLoader(_dataset(), B, seed=LOADER_SEED, device=DEV)


def _member(kind, seed, save_dir):
    """A Trainer as main.py builds one, after torch.manual_seed(seed)."""
    import disvae
    from disvae.models.losses import get_loss_f
    os.makedirs(save_dir, exist_ok=True)
    torch.manual_seed(seed)
    model = disvae.init_specific_model("Burgess", IMG, 10)
    opt = torch.optim.Adam(model.parameters(), lr=5e-4 if kind != "factor" else 1e-4)
    loss_f = get_loss_f(kind, rec_dist="bernoulli", reg_anneal=100, betaB_initC=0, betaB_finC=25, betaB_G=100,
                        btcvae_A=-1, btcvae_B=6, btcvae_G=1, n_data=4096, factor_G=6.4, latent_dim=10, lr_disc=1e-4,
                        device=DEV)
    return disvae.Trainer(model, opt, loss_f, device=DEV, logger=logging.getLogger("sweep-gpu"), save_dir=save_dir,
                          is_progress_bar=False)


def _result(tr, ckpts=EPOCHS):
    """Everything the contract covers, on the host: parameters, Adam moments and step counters (the discriminator's
    too), the train_losses.log text and every checkpoint's state dict."""
    out = {"graphs": len(tr._graphs), "steps": tr.loss_f.n_train_steps}
    nets = [("vae", tr.model, tr.optimizer)]
    if hasattr(tr.loss_f, "discriminator"):
        nets.append(("disc", tr.loss_f.discriminator, tr.loss_f.optimizer_d))
    for tag, net, opt in nets:
        for name, p in net.named_parameters():
            st = opt.state[p]
            out["%s.%s" % (tag, name)] = p.detach().cpu()
            for k in ("exp_avg", "exp_avg_sq", "step"):
                out["%s.%s.%s" % (tag, name, k)] = st[k].detach().cpu()
    with open(os.path.join(tr.save_dir, "train_losses.log")) as f:
        out["log"] = f.read()
    for e in range(ckpts):
        out["ckpt%d" % e] = torch.load(os.path.join(tr.save_dir, "model-%d.pt" % e), weights_only=True)
    return out


def _lone(kind, seed, save_dir):
    tr = _member(kind, seed, save_dir)
    torch.manual_seed(seed)
    tr(_loader(), epochs=EPOCHS, checkpoint_every=1)
    return _result(tr)


def _sweep(specs, tmp):
    from disvae.sweep import Sweep
    members = [_member(kind, seed, str(tmp / ("m%d_%s" % (k, kind)))) for k, (kind, seed) in enumerate(specs)]
    Sweep(members, seeds=[seed for _, seed in specs])(_loader(), epochs=EPOCHS, checkpoint_every=1)
    assert all(not m.model.training for m in members)
    return [_result(m) for m in members]


def _assert_same(got, want, what):
    assert got.keys() == want.keys(), what
    for k in want:
        a, b = got[k], want[k]
        if isinstance(b, dict):
            assert a.keys() == b.keys(), (what, k)
            for n in b:
                assert torch.equal(a[n], b[n]), (what, k, n)
        elif torch.is_tensor(b):
            assert torch.equal(a, b), (what, k)
        else:
            assert a == b, (what, k)


def test_mixed_sweep_equals_lone_runs(tmp_path):
    specs = [("btcvae", 11), ("betaB", 12), ("factor", 13)]
    swept = _sweep(specs, tmp_path / "sweep")
    for (kind, seed), got in zip(specs, swept):
        want = _lone(kind, seed, str(tmp_path / ("lone_" + kind)))
        assert want["graphs"] == 1 and want["steps"] == EPOCHS * 64
        assert want["log"].count("\n") > 2 * 3                 # header + rows of both epochs
        _assert_same(got, want, kind)


def test_identical_twins(tmp_path):
    a, b = _sweep([("btcvae", 7), ("btcvae", 7)], tmp_path / "sweep")
    _assert_same(a, b, "twins")
    _assert_same(a, _lone("btcvae", 7, str(tmp_path / "lone")), "twin vs lone")


def test_lone_trainer_after_sweep_equals_fresh_process(tmp_path):
    _sweep([("factor", 3), ("btcvae", 4)], tmp_path / "sweep")
    here = _lone("btcvae", 5, str(tmp_path / "here"))
    out = tmp_path / "fresh.pt"
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "btcvae", "5", str(tmp_path / "fresh"), str(out)],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    _assert_same(here, torch.load(out, weights_only=False), "after sweep vs fresh process")


def test_second_call_continues_like_a_lone_trainer_called_again(tmp_path):
    """One Sweep called twice (1 + 1 epochs) against lone Trainers called twice: the members' graphs keep their
    Philox counters, step counters and Adam state, and the loader continues its epochs."""
    from disvae.data import DeviceLoader
    from disvae.sweep import Sweep
    specs = [("btcvae", 21), ("factor", 22), ("betaB", 23)]
    members = [_member(kind, seed, str(tmp_path / ("m%d_%s" % (k, kind)))) for k, (kind, seed) in enumerate(specs)]
    sweep, loader = Sweep(members, seeds=[seed for _, seed in specs]), _loader()
    sweep(loader, epochs=1, checkpoint_every=1)
    sweep(loader, epochs=1, checkpoint_every=1)
    for m, (kind, seed) in zip(members, specs):
        lone = _member(kind, seed, str(tmp_path / ("lone_" + kind)))
        torch.manual_seed(seed)
        lone_loader = _loader()
        lone(lone_loader, epochs=1, checkpoint_every=1)
        lone(lone_loader, epochs=1, checkpoint_every=1)
        want = _result(lone, ckpts=1)
        assert want["graphs"] == 1 and want["steps"] == 2 * 64
        _assert_same(_result(m, ckpts=1), want, kind)
    # a torch DataLoader is converted once per Sweep: its epochs continue across calls too
    dl = torch.utils.data.DataLoader(_dataset(), batch_size=B, shuffle=True)
    one = _member("btcvae", 31, str(tmp_path / "dl_sweep"))
    sweep = Sweep([one], seeds=[31])
    torch.manual_seed(31)                                    # the converted loader's seed, as for the lone run below
    sweep(dl, epochs=1, checkpoint_every=1)
    sweep(dl, epochs=1, checkpoint_every=1)
    assert len(sweep._device_loaders) == 1 and isinstance(sweep._device_loaders[id(dl)][1], DeviceLoader)
    lone = _member("btcvae", 31, str(tmp_path / "dl_lone"))
    lone.device_data = True
    torch.manual_seed(31)
    lone(dl, epochs=1, checkpoint_every=1)
    lone(dl, epochs=1, checkpoint_every=1)
    _assert_same(_result(one, ckpts=1), _result(lone, ckpts=1), "DataLoader, two calls")


def _launches():
    from disvae import _native as N
    torch.cuda.synchronize()
    return N.lib().dv_launch_count()


def test_refusals_before_any_launch(tmp_path, monkeypatch):
    from disvae import sweep as S
    from disvae.data import DeviceLoader
    from synthetic_factors import FactorRectangles
    members = [_member("btcvae", 1, str(tmp_path / "a")), _member("betaB", 2, str(tmp_path / "b"))]
    ds64 = FactorRectangles(k=3, size=64)
    ds64.imgs = torch.round(ds64.imgs * 255) / 255
    big = DeviceLoader(ds64, 16, seed=1, device=DEV)
    n0 = _launches()
    sweep = S.Sweep(members, seeds=[1, 2])
    with pytest.raises(ValueError, match=r"the loader yields \(1, 64, 64\) images, the members take \(1, 32, 32\)"):
        sweep(big, epochs=1)
    with pytest.raises(ValueError, match=r"the loader yields \(1, 64, 64\) images"):
        sweep(torch.utils.data.DataLoader(ds64, batch_size=16), epochs=1)
    sgd = _member("btcvae", 3, str(tmp_path / "c"))
    sgd.optimizer = torch.optim.SGD(sgd.model.parameters(), lr=1e-3)
    with pytest.raises(ValueError, match="member 1's optimizer \\(SGD\\) is not a plain torch.optim.Adam"):
        S.Sweep([members[0], sgd], seeds=[1, 3])
    fac = _member("factor", 4, str(tmp_path / "d"))
    fac.loss_f.optimizer_d = torch.optim.Adam(fac.loss_f.discriminator.parameters(), lr=1e-4, amsgrad=True)
    with pytest.raises(ValueError, match="member 0's discriminator optimizer \\(Adam\\)"):
        S.Sweep([fac], seeds=[4])
    eager = _member("btcvae", 5, str(tmp_path / "e"))
    eager.use_cuda_graph = False
    with pytest.raises(ValueError, match="member 2 has use_cuda_graph=False"):
        S.Sweep(members + [eager], seeds=[1, 2, 5])
    trained = _member("btcvae", 6, str(tmp_path / "f"))
    trained.loss_f.n_train_steps = 5
    with pytest.raises(ValueError, match="member 1 has already taken training steps"):
        S.Sweep([members[0], trained], seeds=[1, 6])
    monkeypatch.setattr(S, "is_distributed", lambda: True)
    with pytest.raises(ValueError, match="torch.distributed is not supported"):
        S.Sweep(members, seeds=[1, 2])
    assert _launches() == n0
    assert all(m.loss_f.n_train_steps == 0 and not m._graphs for m in members)


if __name__ == "__main__":
    sys.path[:0] = [os.path.join(ROOT, "disentangling-vae_b200"), os.path.join(ROOT, "tests")]
    kind, seed, save_dir, out = sys.argv[1], int(sys.argv[2]), sys.argv[3], sys.argv[4]
    torch.save(_lone(kind, seed, save_dir), out)
