"""Host stand-ins for the score tests that run without a GPU: a factor grid of blank images, a model stub, CPU
Evaluators and Trainers, a DeviceLoader and a Sweep as the host sees them, and `no_gpu`, which fails a test that
reaches GPU work."""
import logging

import numpy as np
import pytest
import torch

import disvae
from disvae import _native, data, ops, sweep
from disvae.data import DeviceLoader
from disvae.models.losses import get_loss_f

CPU = torch.device("cpu")


class _Grid(torch.utils.data.Dataset):
    """n blank 1x32x32 images over factors of `lat_sizes` (n defaults to their product)."""

    def __init__(self, lat_sizes, n=None, factors=True):
        self.n = int(np.prod(lat_sizes)) if n is None else n
        if factors:
            self.lat_sizes = np.array(lat_sizes)
            self.lat_names = tuple("f%d" % k for k in range(len(lat_sizes)))

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        return torch.zeros(1, 32, 32), 0


class _Stub(torch.nn.Module):
    def __init__(self, latent_dim=10):
        super().__init__()
        self.latent_dim = latent_dim


def _evaluator(tmp_path, latent_dim=10):
    return disvae.Evaluator(_Stub(latent_dim), None, device=CPU, logger=logging.getLogger("score-cpu"),
                            save_dir=str(tmp_path), is_progress_bar=False)


def _trainer(tmp_path, name="t"):
    torch.manual_seed(0)
    model = disvae.init_specific_model("Burgess", (1, 32, 32), 10)
    loss_f = get_loss_f("btcvae", rec_dist="bernoulli", reg_anneal=0, btcvae_A=1, btcvae_B=6, btcvae_G=1, n_data=1000,
                        latent_dim=10, device=CPU)
    save_dir = tmp_path / name
    save_dir.mkdir(exist_ok=True)
    return disvae.Trainer(model, torch.optim.Adam(model.parameters(), lr=5e-4), loss_f, device=CPU,
                          logger=logging.getLogger("score-cpu"), save_dir=str(save_dir), is_progress_bar=False)


def _device_loader(dataset, batch_size=64):
    """A DeviceLoader as the host sees it (no resident tensor: nothing here may reach the GPU)."""
    dl = DeviceLoader.__new__(DeviceLoader)
    dl.dataset, dl.n, dl.batch_size, dl.device, dl.data = dataset, len(dataset), batch_size, torch.device("cuda", 0), None
    dl.epoch, dl.seed = 3, 1234
    return dl


def _bare_sweep(members):
    """A Sweep past its constructor's checks, which need CUDA members."""
    sw = sweep.Sweep.__new__(sweep.Sweep)
    sw.members, sw.seeds, sw.loader, sw._device_loaders = members, [0] * len(members), None, {}
    sw.img_size, sw.device = (1, 32, 32), torch.device("cuda", 0)
    return sw


@pytest.fixture
def no_gpu(monkeypatch):
    """Every way into GPU work fails the test."""
    def reached(*a, **k):
        raise AssertionError("GPU work before the refusal")
    monkeypatch.setattr(_native, "call", reached)
    monkeypatch.setattr(_native, "require_cuda_f32", reached)
    monkeypatch.setattr(disvae.Evaluator, "_compute_q_zCx", reached)
    monkeypatch.setattr(ops, "gather_u8_to_f32", reached)
    monkeypatch.setattr(data, "device_loader_for", reached)
    monkeypatch.setattr(sweep, "device_loader_for", reached)
    monkeypatch.setattr(DeviceLoader, "__init__", reached)
    monkeypatch.setattr(disvae.Trainer, "_train_epoch", reached)
    monkeypatch.setattr(sweep.Sweep, "_run", reached)
    monkeypatch.setattr(torch.cuda, "synchronize", reached)
