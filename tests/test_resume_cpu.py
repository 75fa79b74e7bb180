"""Training state on the host (no GPU, no kernel): the state-file round trip, every refusal of
`Trainer.load_training_state` and of the call that follows it, and train_losses.log rewritten from the saved rows and
then appended to."""
import logging
from collections import defaultdict

import pytest
import torch

import disvae
from disvae.models.losses import get_loss_f
from disvae.training import TRAINING_STATE_FORMAT, training_state_filename
from disvae.utils import modelIO

CPU = torch.device("cpu")


def _loss(name="btcvae", **over):
    kw = dict(rec_dist="bernoulli", reg_anneal=100, betaH_B=4, betaB_initC=0, betaB_finC=25, betaB_G=100, btcvae_A=1,
              btcvae_B=6, btcvae_G=1, n_data=1000, factor_G=6.4, latent_dim=10, lr_disc=1e-4, device=CPU)
    kw.update(over)
    return get_loss_f(name, **kw)


def _trainer(path, name="btcvae", img=(1, 32, 32), latent_dim=10, seed=0, **loss_over):
    path.mkdir(parents=True, exist_ok=True)
    torch.manual_seed(seed)
    model = disvae.init_specific_model("Burgess", img, latent_dim)
    loss_over.setdefault("latent_dim", latent_dim)
    return disvae.Trainer(model, torch.optim.Adam(model.parameters(), lr=5e-4), _loss(name, **loss_over), device=CPU,
                          logger=logging.getLogger("resume-cpu"), save_dir=str(path), is_progress_bar=False)


def _adam_steps(params, opt, n, seed):
    """`n` torch.optim.Adam steps on fixed random gradients: optimizer state without any of our kernels."""
    g = torch.Generator().manual_seed(seed)
    for _ in range(n):
        for p in params:
            p.grad = torch.randn(p.shape, generator=g)
        opt.step()


def _trained(path, name="btcvae", **kw):
    """A Trainer in the state 3 epochs of training leave behind, without running a step: Adam moments, step counters,
    Philox counters, log rows and a DataLoader's order state."""
    tr = _trainer(path, name, **kw)
    _adam_steps(list(tr.model.parameters()), tr.optimizer, 3, 1)
    tr.loss_f.n_train_steps = 321
    tr.model.seed_noise(0xFEDCBA9876543210, CPU)
    tr.model._rng_offset.fill_(4242)
    if name == "factor":
        lf = tr.loss_f
        _adam_steps(list(lf.discriminator.parameters()), lf.optimizer_d, 2, 2)
        lf.seed_permutations(2 ** 63 + 5, CPU)
        lf._perm_offset.fill_(777)
    for e in range(3):
        tr.losses_logger.log(e, {"loss": [1.0 + e, 2.0], "recon_loss": [0.5 * e]})
    tr._next_epoch = 3
    tr._data_loader = torch.utils.data.DataLoader(_Images(40), batch_size=16, shuffle=True)
    return tr


class _Images(torch.utils.data.Dataset):
    def __init__(self, n, img=(1, 32, 32)):
        self.n, self.img = n, img

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        return torch.zeros(self.img), 0


def _equal(a, b, where="state"):
    if torch.is_tensor(b):
        assert torch.is_tensor(a) and a.dtype == b.dtype and torch.equal(a, b), where
    elif isinstance(b, dict):
        assert isinstance(a, dict) and set(a) == set(b), where
        for k in b:
            _equal(a[k], b[k], "%s.%s" % (where, k))
    elif isinstance(b, (list, tuple)):
        assert type(a) is type(b) and len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            _equal(x, y, "%s[%d]" % (where, i))
    else:
        assert a == b, where


@pytest.mark.parametrize("name", ["VAE", "betaH", "betaB", "btcvae", "factor"])
def test_state_file_round_trip(tmp_path, name):
    src = _trained(tmp_path / "src", name)
    path = modelIO.save_training_state(src, str(tmp_path / "src"), training_state_filename(2))
    assert path.endswith("training-state-2.pt")
    saved = src.training_state()
    assert saved["format"] == TRAINING_STATE_FORMAT and saved["epoch"] == 3
    assert saved["world_size"] == 1 and saved["rank"] == 0
    assert saved["loader"]["kind"] == "host" and saved["loader"]["n"] == 40 and saved["loader"]["batch_size"] == 16
    rng = torch.get_rng_state()

    dst = _trainer(tmp_path / "dst", name, seed=99)                # other initial weights
    torch.manual_seed(12345)                                      # other CPU RNG state
    state = modelIO.load_training_state(dst, path)
    _equal(state, saved)
    assert torch.equal(torch.get_rng_state(), rng)                # a host loader's RandomSampler draws the same orders
    for (k, p), q in zip(src.model.state_dict().items(), dst.model.state_dict().values()):
        assert torch.equal(p, q), k
    assert dst.loss_f.n_train_steps == 321
    assert dst.model._rng_seed == 0xFEDCBA9876543210 and int(dst.model._rng_offset) == 4242
    if name == "factor":
        assert dst.loss_f._perm_seed == 2 ** 63 + 5 and int(dst.loss_f._perm_offset) == 777
        for p, q in zip(src.loss_f.discriminator.parameters(), dst.loss_f.discriminator.parameters()):
            assert torch.equal(p, q)
        _equal(dst.loss_f.optimizer_d.state_dict(), src.loss_f.optimizer_d.state_dict(), "optimizer_d")
    _equal(dst.optimizer.state_dict(), src.optimizer.state_dict(), "optimizer")
    assert dst._next_epoch == 3 and dst._resume[0] == 3
    _equal(dst.training_state(), saved)                           # loaded, not yet stepped: saves the same state

    # Adam continues from the loaded moments and counts: one more step on both agrees bit for bit
    _adam_steps(list(src.model.parameters()), src.optimizer, 1, 7)
    _adam_steps(list(dst.model.parameters()), dst.optimizer, 1, 7)
    for p, q in zip(src.model.parameters(), dst.model.parameters()):
        assert torch.equal(p, q)


def _refused(tmp_path, match, **kw):
    state = _trained(tmp_path / "src").training_state()
    dst = _trainer(tmp_path / "dst", **kw)
    before = {k: v.clone() for k, v in dst.model.state_dict().items()}
    with pytest.raises(ValueError, match=match):
        dst.load_training_state(state)
    assert all(torch.equal(v, before[k]) for k, v in dst.model.state_dict().items())      # nothing was applied
    assert dst.loss_f.n_train_steps == 0 and dst._resume is None and dst.model._rng_offset is None


def test_refuses_other_latent_dim(tmp_path):
    _refused(tmp_path, r"latent_dim is 10 in the saved state but 12 here", latent_dim=12)


def test_refuses_other_image_size(tmp_path):
    _refused(tmp_path, r"img_size is \[1, 32, 32\] in the saved state but \[1, 64, 64\] here", img=(1, 64, 64))


def test_refuses_other_loss_class(tmp_path):
    _refused(tmp_path, r"the loss class is 'BtcvaeLoss' in the saved state but 'BetaBLoss' here", name="betaB")


@pytest.mark.parametrize("over,match", [(dict(btcvae_B=5), r"loss hyper-parameter beta is 6 .* but 5 here"),
                                        (dict(reg_anneal=0), r"loss hyper-parameter steps_anneal is 100 .* but 0 here"),
                                        (dict(n_data=999), r"loss hyper-parameter n_data is 1000 .* but 999 here"),
                                        (dict(rec_dist="laplace"), r"loss hyper-parameter rec_dist is 'bernoulli'")])
def test_refuses_other_hyper_parameter(tmp_path, over, match):
    _refused(tmp_path, match, **over)


def test_refuses_other_world_size_and_rank(tmp_path):
    state = _trained(tmp_path / "src").training_state()
    for field, value, match in [("world_size", 2, "the world size is 2 in the saved state but 1 here"),
                                ("rank", 1, "the rank is 1 in the saved state but 0 here")]:
        bad = dict(state, **{field: value})
        dst = _trainer(tmp_path / ("dst_" + field))
        with pytest.raises(ValueError, match=match):
            dst.load_training_state(bad)
        assert dst._resume is None


@pytest.mark.parametrize("version", [0, 2, None])
def test_refuses_unknown_format(tmp_path, version):
    state = dict(_trained(tmp_path / "src").training_state(), format=version)
    with pytest.raises(ValueError, match="unknown training-state format"):
        _trainer(tmp_path / "dst").load_training_state(state)
    with pytest.raises(ValueError, match="unknown training-state format"):
        _trainer(tmp_path / "dst2").load_training_state([1, 2])


def test_refuses_a_trainer_that_stepped(tmp_path):
    state = _trained(tmp_path / "src").training_state()
    for what in ("n_train_steps", "graphs", "eligible", "fused"):
        dst = _trainer(tmp_path / ("dst_" + what))
        if what == "n_train_steps":
            dst.loss_f.n_train_steps = 1
        elif what == "graphs":
            dst._graphs[((4, 1, 32, 32), "torch.float32")] = object()
        elif what == "eligible":
            dst._eligible_steps = 1
        else:
            dst._fused = False                                    # the step decided on the optimizer path
        with pytest.raises(ValueError, match="already taken training steps"):
            dst.load_training_state(state)
    dst = _trainer(tmp_path / "twice")                            # loaded but not stepped: loading again is fine
    dst.load_training_state(state)
    dst.load_training_state(state)
    dst.loss_f.n_train_steps += 1                                 # ... stepped since: refused
    with pytest.raises(ValueError, match="already taken training steps"):
        dst.load_training_state(state)


@pytest.mark.parametrize("n,batch_size,shuffle,field",
                         [(41, 16, True, "n is 40"), (40, 8, True, "batch_size is 16"), (40, 16, False, "shuffle is True")])
def test_refuses_another_loader(tmp_path, n, batch_size, shuffle, field):
    state = _trained(tmp_path / "src").training_state()
    dst = _trainer(tmp_path / "dst")
    dst.load_training_state(state)
    other = torch.utils.data.DataLoader(_Images(n), batch_size=batch_size, shuffle=shuffle)
    with pytest.raises(ValueError, match="the loader's " + field):
        dst(other, epochs=1)                                      # refused before the first step
    assert dst.loss_f.n_train_steps == 321 and dst._resume is not None
    # a state saved over a DeviceLoader: checked against the DataLoader that DISVAE_DEVICE_DATA=1 would convert
    dev_state = dict(state, loader=dict(kind="device", seed=5, epoch=3, n=40, batch_size=16, shuffle=True,
                                        drop_last=False))
    dst = _trainer(tmp_path / "dst_dev")
    dst.load_training_state(dev_state)
    dst.device_data = True
    with pytest.raises(ValueError, match="the loader's " + field):
        dst(other, epochs=1)
    dst.device_data = False
    with pytest.raises(ValueError, match="read a device loader but this call passes a host one"):
        dst(torch.utils.data.DataLoader(_Images(40), batch_size=16, shuffle=True), epochs=1)


def test_refuses_factor_state_into_another_loss(tmp_path):
    state = _trained(tmp_path / "src", "factor").training_state()
    with pytest.raises(ValueError, match="the loss class is 'FactorKLoss'"):
        _trainer(tmp_path / "dst", "btcvae").load_training_state(state)


def test_losses_log_rewritten_then_appended(tmp_path):
    src = _trained(tmp_path / "src")
    src._end_epoch(3, {"loss": [7.0]}, 7.0, checkpoint_every=10)
    state = src.training_state()
    assert state["epoch"] == 4
    want = (tmp_path / "src" / "train_losses.log").read_text()
    assert want.startswith("Epoch,Loss,Value\n0,loss,1.5\n0,recon_loss,0.0\n") and want.endswith("3,loss,7.0\n")

    dst = _trainer(tmp_path / "fresh")                            # a fresh directory: the file holds only the header
    assert (tmp_path / "fresh" / "train_losses.log").read_text() == "Epoch,Loss,Value\n"
    dst.load_training_state(state)
    assert (tmp_path / "fresh" / "train_losses.log").read_text() == want
    storer = defaultdict(list)
    storer["loss"] += [2.0, 4.0]
    dst._end_epoch(4, storer, 3.0, checkpoint_every=10, save_state=True)
    assert (tmp_path / "fresh" / "train_losses.log").read_text() == want + "4,loss,3.0\n"
    assert not (tmp_path / "fresh" / "model-4.pt").exists()       # the checkpoint cadence is the caller's
    again = torch.load(str(tmp_path / "fresh" / "training-state-4.pt"), weights_only=True)
    assert again["epoch"] == 5 and again["log_rows"] == state["log_rows"] + ["4,loss,3.0"]
