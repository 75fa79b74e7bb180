"""Evaluation over resident data on the host (no GPU, no kernel): every refusal of `metrics_every` and of
`Sweep.evaluate` happens before any GPU work, `DeviceLoader.in_order` batches like a DataLoader without shuffling, and
the seed of an evaluation depends on the run's saved noise key and the epoch only."""
import json
import logging
import os

import numpy as np
import pytest
import torch

import disvae
from disvae import _native, data, evaluate, ops, sweep
from disvae.data import DeviceLoader, batch_windows
from disvae.models.losses import get_loss_f

CPU = torch.device("cpu")
MASK = 0xFFFFFFFFFFFFFFFF


class _Factors(torch.utils.data.Dataset):
    """n blank 1x32x32 images; with known factors unless `factors=False`."""

    def __init__(self, n, factors=True):
        self.n = n
        if factors:
            self.lat_sizes = np.array([n])
            self.lat_names = ("index",)

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        return torch.zeros(1, 32, 32), 0


def _trainer(tmp_path, name="t"):
    torch.manual_seed(0)
    model = disvae.init_specific_model("Burgess", (1, 32, 32), 10)
    loss_f = get_loss_f("btcvae", rec_dist="bernoulli", reg_anneal=0, btcvae_A=1, btcvae_B=6, btcvae_G=1, n_data=1000,
                        latent_dim=10, device=CPU)
    save_dir = tmp_path / name
    save_dir.mkdir(exist_ok=True)
    return disvae.Trainer(model, torch.optim.Adam(model.parameters(), lr=5e-4), loss_f, device=CPU,
                          logger=logging.getLogger("eval-resident-cpu"), save_dir=str(save_dir), is_progress_bar=False)


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
    monkeypatch.setattr(ops, "gather_u8_to_f32", reached)
    monkeypatch.setattr(data, "device_loader_for", reached)
    monkeypatch.setattr(sweep, "device_loader_for", reached)
    monkeypatch.setattr(DeviceLoader, "__init__", reached)
    monkeypatch.setattr(disvae.Trainer, "_train_epoch", reached)
    monkeypatch.setattr(sweep.Sweep, "_run", reached)
    monkeypatch.setattr(torch.cuda, "synchronize", reached)


def _refusals(n_ok=10000):
    """(loader, device_data, message) of every loader metrics_every refuses."""
    host = torch.utils.data.DataLoader(_Factors(n_ok), batch_size=64, shuffle=True)
    return [
        (host, False, "needs the dataset resident on the GPU"),
        (torch.utils.data.DataLoader(_Factors(n_ok, factors=False), batch_size=64), True, "no lat_sizes / lat_names"),
        (_device_loader(_Factors(n_ok, factors=False)), False, "no lat_sizes / lat_names"),
        (_device_loader(_Factors(n_ok - 1)), False, "has 9999 items, fewer than the 10000 samples"),
        (torch.utils.data.DataLoader(_Factors(n_ok - 1), batch_size=64), True, "fewer than the 10000 samples"),
        ([(torch.zeros(2, 1, 32, 32), 0)], True, "needs a disvae.data.DeviceLoader, got list"),
    ]


def test_trainer_refusals_before_gpu_work(tmp_path, no_gpu):
    tr = _trainer(tmp_path)
    for i, (loader, device_data, msg) in enumerate(_refusals()):
        tr.device_data = device_data
        with pytest.raises(ValueError, match=msg):
            tr(loader, epochs=1, metrics_every=1)
    dl = _device_loader(_Factors(10000))
    for bad in (-1, True, 1.5, "2"):
        with pytest.raises(ValueError, match="metrics_every must be a non-negative integer"):
            tr(dl, epochs=1, metrics_every=bad)
    with pytest.raises(ValueError, match="metrics_batch_size must be positive"):
        tr(dl, epochs=1, metrics_every=1, metrics_batch_size=0)
    assert tr.loss_f.n_train_steps == 0 and tr._data_loader is None and dl.epoch == 3


def test_trainer_refuses_metrics_under_distributed(tmp_path, no_gpu, monkeypatch):
    monkeypatch.setattr(evaluate, "is_distributed", lambda: True)
    tr = _trainer(tmp_path)
    with pytest.raises(ValueError, match="not supported under torch.distributed"):
        tr(_device_loader(_Factors(10000)), epochs=1, metrics_every=2)


def test_refused_call_keeps_a_loaded_state_pending(tmp_path, no_gpu):
    tr = _trainer(tmp_path)
    tr._resume = (2, None)
    with pytest.raises(ValueError, match="needs the dataset resident"):
        tr(torch.utils.data.DataLoader(_Factors(10000), batch_size=64), epochs=1, metrics_every=1)
    assert tr._resume == (2, None)


def test_sweep_refusals_before_gpu_work(tmp_path, no_gpu):
    sw = _bare_sweep([_trainer(tmp_path, "a"), _trainer(tmp_path, "b")])
    for loader, device_data, msg in _refusals():
        if device_data is False and isinstance(loader, torch.utils.data.DataLoader):
            continue                                  # a Sweep converts every DataLoader (tested below)
        with pytest.raises(ValueError, match=msg):
            sw(loader, epochs=1, metrics_every=1)
    with pytest.raises(ValueError, match="metrics_every must be a non-negative integer"):
        sw(_device_loader(_Factors(10000)), epochs=1, metrics_every=-2)
    with pytest.raises(ValueError, match="metrics_batch_size must be positive"):
        sw(_device_loader(_Factors(10000)), epochs=1, metrics_every=1, metrics_batch_size=-5)
    assert sw.loader is None and not sw._device_loaders


def test_sweep_evaluate_needs_a_loader(tmp_path, no_gpu):
    sw = _bare_sweep([_trainer(tmp_path, "a")])
    with pytest.raises(ValueError, match="the sweep has no loader yet"):
        sw.evaluate()
    with pytest.raises(ValueError, match="the sweep has no loader yet"):
        sw.evaluate(is_metrics=False)
    sw.loader = _device_loader(_Factors(9000))
    with pytest.raises(ValueError, match="fewer than the 10000 samples"):
        sw.evaluate()
    with pytest.raises(ValueError, match="batch_size must be positive"):
        sw.evaluate(is_metrics=False, batch_size=0)


@pytest.mark.parametrize("n,b", [(10000, 1000), (10000, 3000), (737280, 1000), (7, 7), (7, 100), (1, 1)])
def test_in_order_windows_and_len(n, b):
    dl = _device_loader(_Factors(n), batch_size=64)
    view = dl.in_order(b)
    assert len(view) == -(-n // b) and view.dataset is dl.dataset and view.batch_size == b
    starts = list(range(0, n, b))
    assert view.windows == [(s, min(b, n - s)) for s in starts] == batch_windows(n, b)
    assert sum(size for _, size in view.windows) == n
    assert len(view) == len(torch.utils.data.DataLoader(dl.dataset, batch_size=b, shuffle=False))
    assert dl.epoch == 3 and dl.seed == 1234 and dl.batch_size == 64


@pytest.mark.parametrize("b", [0, -1])
def test_in_order_refuses_nonpositive_batch(b):
    with pytest.raises(ValueError, match="in_order: batch_size must be positive"):
        _device_loader(_Factors(10)).in_order(b)


@pytest.mark.parametrize("key", [0, 5, 1234, 2 ** 63 + 17, MASK])
def test_evaluation_seed_is_a_function_of_key_and_epoch(key):
    seeds = [evaluate.evaluation_seed(key, e) for e in range(50)]
    assert seeds == [(key + 0x9E3779B97F4A7C15 * (e + 1)) & MASK for e in range(50)]
    assert len(set(seeds)) == 50 and all(0 <= s <= MASK for s in seeds)
    saved = torch.initial_seed()
    try:
        torch.manual_seed(99)
        torch.rand(3)
        assert [evaluate.evaluation_seed(key, e) for e in range(50)] == seeds
    finally:
        torch.manual_seed(saved)
    assert evaluate.evaluation_seed(key, 3) != evaluate.evaluation_seed((key + 1) & MASK, 3)


def test_epoch_metrics_take_the_saved_noise_key(tmp_path, monkeypatch):
    """write_epoch_metrics seeds from the model's noise key (what a training state saves) and the epoch, whatever the
    global generators hold, and writes metrics-{e}.log / metric_helpers-{e}.pth in the Evaluator's formats."""
    import contextlib
    seen = []

    @contextlib.contextmanager
    def rng(device, key, epoch):
        seen.append((key, epoch))
        yield

    class FakeEvaluator:
        def __init__(self, model, loss_f, device, logger, save_dir, is_progress_bar):
            self.save_dir = save_dir

        def __call__(self, loader, is_metrics, is_losses):
            assert is_metrics and not is_losses and loader.batch_size == 500
            with open(os.path.join(self.save_dir, evaluate.METRICS_FILENAME), "w") as f:
                json.dump({"MIG": 0.25, "AAM": 0.5}, f)
            torch.save({"mig": torch.tensor(0.25)}, os.path.join(self.save_dir, evaluate.METRIC_HELPERS_FILE))

    monkeypatch.setattr(evaluate, "evaluation_rng", rng)
    monkeypatch.setattr(evaluate, "Evaluator", FakeEvaluator)
    tr = _trainer(tmp_path)
    tr.model.seed_noise(0xFEDCBA9876543210, CPU)
    dl = _device_loader(_Factors(10000))
    dl.device = CPU
    for e, seed in ((4, 1), (4, 2), (7, 3)):
        torch.manual_seed(seed)
        evaluate.write_epoch_metrics(tr.model, dl, e, 500, tr.save_dir, tr.logger)
    assert seen == [(0xFEDCBA9876543210, 4)] * 2 + [(0xFEDCBA9876543210, 7)]
    assert tr.training_state()["noise"]["key"] == 0xFEDCBA9876543210
    files = sorted(os.listdir(tr.save_dir))
    assert files == ["metric_helpers-4.pth", "metric_helpers-7.pth", "metrics-4.log", "metrics-7.log",
                     "train_losses.log"]
    assert evaluate.epoch_metrics_filenames(7) == ("metrics-7.log", "metric_helpers-7.pth")
    with open(os.path.join(tr.save_dir, "metrics-7.log")) as f:
        assert json.load(f) == {"MIG": 0.25, "AAM": 0.5}
