"""Device-resident training data: the epoch permutation dv_index_permutation, the batch gather dv_gather_u8_to_f32,
disvae.data.DeviceLoader, the Trainer over it (bit-identical to a host loader yielding the same batches), the
DISVAE_DEVICE_DATA opt-in under the reference's unmodified main.py, and two-rank data parallelism."""
import json
import logging
import os
import socket
import subprocess
import sys
from collections import defaultdict

import numpy as np
import pytest
import torch

from ddp_device_data_worker import KDataset, digest
from ddp_device_data_worker import N as DDP_N, SHAPE as DDP_SHAPE
from test_factor_global_gpu import host_perms

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
SEED = 0x0123456789ABCDEF


def _offset(v):
    return torch.tensor([v], dtype=torch.int64, device=DEV)


# ---- dv_index_permutation --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 3, 4095, 4096, 4097, 12289, 202599, 737280])
def test_index_permutation_matches_host_philox_sort(n):
    from disvae import ops
    off = _offset(77)
    perm = ops.index_permutation(n, SEED, off)
    assert off.item() == 77 + n
    assert perm.dtype == torch.int64 and perm.shape == (n,)
    assert torch.equal(perm.sort().values.cpu(), torch.arange(n))
    assert torch.equal(perm.cpu(), host_perms(n, 1, SEED, 77)[0])


@pytest.mark.parametrize("n", [3, 4096, 12289, 202599])
def test_index_permutation_graph_replays_equal_eager_epochs(n):
    from disvae import ops
    off_e = _offset(5)
    eager = [ops.index_permutation(n, SEED, off_e).clone() for _ in range(3)]
    off_g = _offset(5)
    out = torch.empty(n, dtype=torch.int64, device=DEV)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.index_permutation(n, SEED, off_g, out=out)
    assert off_g.item() == 5                                              # capture ran nothing
    for e in eager:
        g.replay()
        assert torch.equal(out, e)
    assert off_g.item() == off_e.item() == 5 + 3 * n


def test_index_permutation_refusals():
    from disvae import _native as N
    L, st = N.lib(), N.stream()
    out, off = torch.empty(8192, dtype=torch.int64, device=DEV), _offset(0)
    ws = torch.empty(L.dv_index_permutation_workspace_bytes(8192), dtype=torch.uint8, device=DEV)
    assert L.dv_index_permutation_workspace_bytes(4096) == 0 and ws.numel() == 8192 * 8
    assert L.dv_index_permutation(0, 1, off.data_ptr(), out.data_ptr(), ws.data_ptr(), st) == -1
    assert L.dv_index_permutation(16, 1, None, out.data_ptr(), None, st) == -2
    assert L.dv_index_permutation(16, 1, off.data_ptr(), None, None, st) == -2
    assert L.dv_index_permutation(16, 1, off.data_ptr(), out.data_ptr() + 4, None, st) == -2
    assert L.dv_index_permutation(8192, 1, off.data_ptr(), out.data_ptr(), None, st) == -2
    assert L.dv_index_permutation(8192, 1, off.data_ptr(), out.data_ptr(), ws.data_ptr() + 4, st) == -2
    torch.cuda.synchronize()
    assert off.item() == 0                                                # nothing was launched


# ---- dv_gather_u8_to_f32 ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("chw", [(1, 32, 32), (1, 64, 64), (3, 64, 64)])
@pytest.mark.parametrize("nrows", [1, 7, 64, 1024])
def test_gather_u8_to_f32_is_indexing_then_totensor(chw, nrows):
    from disvae import ops
    g = torch.Generator().manual_seed(nrows)
    src = torch.randint(0, 256, (300,) + chw, dtype=torch.uint8, generator=g).to(DEV)
    src[0] = 255
    src[1] = 0
    idx = torch.randint(0, 300, (nrows,), generator=g)
    idx[-1] = idx[0]                                                      # a repeat in every case
    idx = idx.to(DEV)
    out = ops.gather_u8_to_f32(src, idx)
    assert out.shape == (nrows,) + chw and out.dtype == torch.float32
    # ToTensor divides on the host; torch's CUDA division by a scalar multiplies by its reciprocal (not bit-equal)
    assert torch.equal(out.cpu(), src[idx].cpu().float().div(255))
    assert torch.equal(out, ops.u8_to_f32(src[idx]))


def test_gather_u8_to_f32_refusals():
    from disvae import _native as N
    L, st = N.lib(), N.stream()
    src = torch.zeros(4, 64, dtype=torch.uint8, device=DEV)
    idx = torch.zeros(2, dtype=torch.int64, device=DEV)
    dst = torch.full((2, 64), -1.0, device=DEV)
    s, i, d = src.data_ptr(), idx.data_ptr(), dst.data_ptr()
    for nrows, row_bytes in [(0, 64), (2, 0), (2, 8), (2, 24), (2, 63)]:
        assert L.dv_gather_u8_to_f32(s, i, nrows, row_bytes, d, st) == -1, (nrows, row_bytes)
    for args in [(None, i, d), (s, None, d), (s, i, None), (s + 1, i, d), (s, i + 4, d), (s, i, d + 4)]:
        assert L.dv_gather_u8_to_f32(args[0], args[1], 2, 64, args[2], st) == -2, args
    torch.cuda.synchronize()
    assert (dst == -1).all()                                              # nothing was launched


# ---- DeviceLoader ----------------------------------------------------------------------------------------------------
def _orders(dl, epochs):
    return [torch.cat([idx for _, idx in dl]).cpu() for _ in range(epochs)]


@pytest.mark.parametrize("n,b,chw", [(1000, 64, (1, 32, 32)), (300, 32, (3, 64, 64)), (5000, 4096, (1, 64, 64))])
@pytest.mark.parametrize("shuffle", [True, False])
def test_device_loader_batches_are_the_datasets_items(n, b, chw, shuffle):
    from disvae.data import DeviceLoader
    ds = KDataset(n, chw, seed=n)
    for drop_last in (False, True):
        dl = DeviceLoader(ds, b, shuffle=shuffle, drop_last=drop_last, seed=11)
        assert dl.dataset is ds
        assert len(dl) == len(torch.utils.data.DataLoader(ds, batch_size=b, drop_last=drop_last))
        orders = []
        for epoch in range(2):
            seen, steps = [], 0
            for x, idx in dl:
                assert x.is_cuda and idx.is_cuda and x.dtype == torch.float32 and idx.dtype == torch.int64
                assert torch.equal(x, torch.stack([ds[int(i)][0] for i in idx.cpu()]).to(DEV))
                seen.append(idx.cpu())
                steps += 1
            assert steps == len(dl)
            order = torch.cat(seen)
            if drop_last:
                assert order.numel() == n // b * b and order.unique().numel() == order.numel()
            else:
                assert torch.equal(order.sort().values, torch.arange(n))   # every index once
            orders.append(order)
        if shuffle:
            assert not torch.equal(orders[0], orders[1])
            full = host_perms(n, 1, 11, n)[0]                             # epoch 1: offset 1 * n
            assert torch.equal(orders[1], full[:orders[1].numel()])
        else:
            assert torch.equal(orders[0], torch.arange(orders[0].numel())) and torch.equal(orders[0], orders[1])


def test_device_loader_seeds():
    from disvae.data import DeviceLoader
    ds = KDataset(777, (1, 32, 32), seed=3)
    a, b, c = (DeviceLoader(ds, 100, seed=s) for s in (5, 5, 6))
    oa, ob, oc = _orders(a, 2), _orders(b, 2), _orders(c, 2)
    assert all(torch.equal(x, y) for x, y in zip(oa, ob))
    assert not torch.equal(oa[0], oc[0])
    torch.manual_seed(4321)
    assert DeviceLoader(ds, 100).seed == torch.initial_seed() == 4321


class _Normalised(KDataset):
    def __getitem__(self, i):
        x, y = super().__getitem__(i)
        return (x - 0.5) / 0.5, y


def test_device_loader_refuses_non_byte_images():
    from disvae.data import DeviceLoader
    ds = _Normalised(2000, (1, 32, 32), seed=1)
    with pytest.raises(RuntimeError, match="item 0 "):
        DeviceLoader(ds, 64)
    ds = KDataset(2000, (1, 32, 32), seed=1)
    ds.imgs = ds.imgs.astype(np.float32)
    ds.imgs[1500, 0, 3, 4] += 0.25                                        # 0.25/255 off a byte value
    with pytest.raises(RuntimeError, match="item 1500 "):
        DeviceLoader(ds, 64)


def test_device_loader_memory_check(monkeypatch):
    from disvae.data import DeviceLoader
    ds = KDataset(100, (3, 64, 64), seed=1)
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (100 * 3 * 64 * 64 - 1, 80 << 30))
    with pytest.raises(RuntimeError, match="%d bytes .* only %d bytes" % (100 * 3 * 64 * 64, 100 * 3 * 64 * 64 - 1)):
        DeviceLoader(ds, 10)
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (100 * 3 * 64 * 64, 80 << 30))
    assert len(DeviceLoader(ds, 10)) == 10


# ---- Trainer over a DeviceLoader == Trainer over host batches in the same order ----------------------------------------
def _train(loss, chw, n_data, loader, graph, tmp):
    import disvae
    from disvae.models.losses import get_loss_f
    torch.manual_seed(1234)
    m = disvae.init_specific_model("Burgess", chw, 10).to(DEV)
    opt = torch.optim.Adam(m.parameters(), lr=5e-4)
    lf = get_loss_f(loss, rec_dist="bernoulli", reg_anneal=0, btcvae_A=1, btcvae_B=6, btcvae_G=1, factor_G=6.4,
                    latent_dim=10, lr_disc=5e-5, n_data=n_data, device=torch.device(DEV))
    tmp.mkdir()
    tr = disvae.Trainer(m, opt, lf, device=torch.device(DEV), logger=logging.getLogger("dd"), save_dir=str(tmp),
                        is_progress_bar=False)
    tr.use_cuda_graph = graph
    m.train()
    losses, storers = [], []
    for epoch in range(2):
        st = defaultdict(list)
        losses.append(tr._train_epoch(loader, st, epoch))
        storers.append(dict(st))
    params = [p.detach().clone() for p in m.parameters()]
    if hasattr(lf, "discriminator"):
        params += [p.detach().clone() for p in lf.discriminator.parameters()]
    return losses, storers, params, tr


@pytest.mark.parametrize("loss,chw,b,n", [("btcvae", (1, 64, 64), 256, 256 * 7 + 100),
                                          ("factor", (3, 64, 64), 128, 128 * 7 + 64)])
@pytest.mark.parametrize("graph", [False, True])
def test_trainer_device_loader_equals_host_batches(loss, chw, b, n, graph, tmp_path):
    from disvae.data import DeviceLoader
    ds = KDataset(n, chw, seed=9)
    recorded = _orders(DeviceLoader(ds, b, seed=21), 2)
    host_epochs = [[(torch.stack([ds[int(i)][0] for i in order[s:s + b]]), order[s:s + b]) for s in range(0, n, b)]
                   for order in recorded]

    class HostLoader:                                                     # yields the recorded epochs, in order
        def __init__(self):
            self.epoch = 0

        def __iter__(self):
            self.epoch += 1
            return iter(host_epochs[self.epoch - 1])

        def __len__(self):
            return len(host_epochs[0])

    dev = _train(loss, chw, n, DeviceLoader(ds, b, seed=21), graph, tmp_path / "dev")
    host = _train(loss, chw, n, HostLoader(), graph, tmp_path / "host")
    if graph:
        assert dev[3]._graphs and len(dev[3]._graphs) == 2                # the full and the partial batch shape
        assert dev[3]._eligible_steps > 2 * len(host_epochs[0]) - 4
    assert dev[0] == host[0]
    assert dev[1] == host[1]
    assert len(dev[2]) == len(host[2])
    for a, c in zip(dev[2], host[2]):
        assert torch.equal(a, c)


# ---- DISVAE_DEVICE_DATA=1 under the reference's unmodified main.py ---------------------------------------------------
_DROPIN = r"""
import json, sys
sys.argv = ["run_reference_main.py"] + sys.argv[1:]
sys.path.insert(0, %(tests)r)
import run_reference_main as R
class ByteShapes(R.SyntheticShapes):          # the synthetic images rounded to bytes: what ToTensor makes of PNGs
    def __init__(self, img_size):
        super().__init__(img_size)
        self.imgs = (self.imgs * 255).round() / 255
R.SyntheticShapes = ByteShapes
from disvae import data
built = []
_init = data.DeviceLoader.__init__
def _counting_init(self, *a, **k):
    built.append(1)
    _init(self, *a, **k)
data.DeviceLoader.__init__ = _counting_init
R.main()
print(json.dumps({"device_loaders": len(built)}))
"""


def test_unmodified_main_with_device_data(tmp_path):
    if not os.path.isfile(os.path.join(ROOT, "oracle", "_ref", "main.py")):
        pytest.skip("oracle/_ref not installed (oracle/ship_reference.py needs a reference checkout)")
    env = dict(os.environ, DISVAE_DEVICE_DATA="1")
    r = subprocess.run([sys.executable, "-c", _DROPIN % dict(tests=os.path.join(ROOT, "tests")), "btcvae", str(tmp_path)],
                       capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + "\n" + r.stderr[-6000:]
    lines = r.stdout.strip().splitlines()
    assert json.loads(lines[-1]) == {"device_loaders": 1}                 # built once for the two epochs
    out = json.loads(lines[-2])
    assert {"model.pt", "specs.json", "train_losses.log", "test_losses.log", "model-0.pt"} <= set(out["files"])
    assert out["log_head"] == "Epoch,Loss,Value"
    assert {"recon_loss", "kl_loss", "loss", "kl_loss_0", "mi_loss", "tc_loss", "dw_kl_loss"} <= set(out["logged"])
    assert out["img_size"] == [1, 64, 64] and out["meta_loss"] == "btcvae"
    assert {"recon_loss", "kl_loss", "loss"} <= set(out["test_losses"])
    assert all(v == v and abs(v) < 1e9 for v in out["test_losses"].values())
    assert out["param_device"].startswith("cuda") and out["native_launches"] > 100


def test_trainer_wraps_a_dataloader_once_when_opted_in(tmp_path, monkeypatch):
    import disvae
    from disvae.data import DeviceLoader
    from disvae.models.losses import get_loss_f
    ds = KDataset(300, (1, 32, 32), seed=2)
    loader = torch.utils.data.DataLoader(ds, batch_size=64, shuffle=True, drop_last=True)
    m = disvae.init_specific_model("Burgess", (1, 32, 32), 10).to(DEV)
    lf = get_loss_f("VAE", rec_dist="bernoulli", reg_anneal=0)
    for flag, wrapped in (("0", False), ("1", True)):
        monkeypatch.setenv("DISVAE_DEVICE_DATA", flag)
        tr = disvae.Trainer(m, torch.optim.Adam(m.parameters(), lr=1e-4), lf, device=torch.device(DEV),
                            logger=logging.getLogger("dd"), save_dir=str(tmp_path), is_progress_bar=False)
        seen = []
        real_epoch = tr._train_epoch
        tr._train_epoch = lambda dl, storer, epoch: seen.append(dl) or real_epoch(dl, storer, epoch)
        tr(loader, epochs=1, checkpoint_every=100)
        tr(loader, epochs=1, checkpoint_every=100)
        if wrapped:
            assert isinstance(seen[0], DeviceLoader) and seen[0] is seen[1] and seen[0].dataset is ds
            assert seen[0].shuffle and seen[0].drop_last and seen[0].batch_size == 64 and len(seen[0]) == 4
        else:
            assert seen == [loader, loader]


# ---- two ranks -------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_two_rank_device_loader():
    from disvae.data import DeviceLoader
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "ddp_device_data_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    lines = [l for l in r.stdout.splitlines() if l.startswith("DDP_DEVICE_DATA ")]
    assert lines, r.stdout[-2000:] + "\n" + r.stderr[-6000:]
    rep = json.loads(lines[-1][len("DDP_DEVICE_DATA "):])
    assert rep["ok"] and r.returncode == 0, json.dumps(rep, indent=1)
    assert rep["world"] == 2
    single = DeviceLoader(KDataset(DDP_N, DDP_SHAPE, seed=5), 16)
    assert rep["digest"] == digest(single.data)
