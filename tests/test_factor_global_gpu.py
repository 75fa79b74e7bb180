"""Global-batch FactorVAE permutations (SURVEY.md 8e): the row-window permutation entry point dv_permute_dims_rows at
any batch size, FactorKLoss.global_batch under two-rank data parallelism, and the equal-rows check that guards its
gather.  Tests 1-6 need an H100 (pytest -m gpu); the equal-rows check runs on gloo without a GPU."""
import json
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
M32 = np.uint64(0xFFFFFFFF)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def philox_x(ctr, seed):
    """Word x of Philox4x32-10 (dv_common.cuh) at counters `ctr` (uint64 array) with the counter words (c_lo, c_hi,
    0x5eed, 0) and the key (seed_lo, seed_hi) that the permutation kernels use."""
    x, y = ctr & M32, ctr >> np.uint64(32)
    z, w = np.full_like(ctr, 0x5EED), np.zeros_like(ctr)
    k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64(seed >> 32)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * x, np.uint64(0xCD9E8D57) * z
        x, y, z, w = (p1 >> np.uint64(32)) ^ y ^ k0, p1 & M32, (p0 >> np.uint64(32)) ^ w ^ k1, p0 & M32
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & M32, (k1 + np.uint64(0xBB67AE85)) & M32
    return x


def host_perms(B, D, seed, offset):
    """[D, B] permutations: column d sorts the keys (x << 32) | b of counters offset + d*B + b ascending."""
    b = np.arange(B, dtype=np.uint64)
    out = np.empty((D, B), dtype=np.int64)
    for d in range(D):
        keys = (philox_x(np.uint64(offset + d * B) + b, seed) << np.uint64(32)) | b
        out[d] = (keys & M32)[np.argsort(keys)].astype(np.int64)
    return torch.from_numpy(out)


def apply_perms(z, perms):
    return torch.gather(z, 0, perms.t().to(z.device))


def _offset(v):
    return torch.tensor([v], dtype=torch.int64, device=DEV)


SEED = 0x0123456789ABCDEF


def _z(B, D):
    g = torch.Generator().manual_seed(B * 131 + D)
    return torch.randn(B, D, generator=g).to(DEV)


def _splits(B, k):
    """k windows covering [0, B), uneven when B % k != 0."""
    edges = [B * i // k for i in range(k + 1)]
    return [(a, b - a) for a, b in zip(edges[:-1], edges[1:]) if b > a]


# ---- 1: the B <= 4096 kernel -----------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("B,D", [(2, 1), (16, 10), (1000, 12), (4096, 10), (4096, 64)])
def test_full_window_is_dv_permute_dims(B, D):
    from disvae import ops
    z = _z(B, D)
    off_a, off_b = _offset(77), _offset(77)
    ref = ops.permute_dims(z, None, SEED, off_a)
    full = ops.permute_dims_rows(z, 0, B, None, SEED, off_b)
    assert torch.equal(full, ref)
    assert off_a.item() == off_b.item() == 77 + B * D
    for k in (2, 3, 8):
        parts = []
        for row0, n in _splits(B, k):
            off = _offset(77)
            parts.append(ops.permute_dims_rows(z, row0, n, None, SEED, off))
            assert off.item() == 77 + B * D
        assert torch.equal(torch.cat(parts), ref), k


# ---- 2: beyond 4096 rows ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("B,D", [(16, 10), (1000, 3), (4096, 10)])
def test_host_philox_restatement_matches_device(B, D):
    """The numpy restatement that referees the multi-CTA sort, checked where the single-CTA kernel is the referee."""
    from disvae import ops
    z = torch.arange(B, dtype=torch.float32, device=DEV).view(B, 1).expand(B, D).contiguous()
    dev = ops.permute_dims(z, None, SEED, _offset(5))
    assert torch.equal(dev.t().long().cpu(), host_perms(B, D, SEED, 5))


@pytest.mark.gpu
@pytest.mark.parametrize("B,D", [(4097, 10), (8192, 10), (50001, 3), (65536, 10)])
def test_beyond_4096_rows_matches_host_sort(B, D):
    from disvae import ops
    z = _z(B, D)
    off = _offset(123)
    full = ops.permute_dims_rows(z, 0, B, None, SEED, off)
    assert off.item() == 123 + B * D
    expect = apply_perms(z, host_perms(B, D, SEED, 123))
    assert torch.equal(full, expect)
    assert torch.equal(full.sort(0).values, z.sort(0).values)             # every column a permutation of its input
    off = _offset(123)
    assert torch.equal(ops.permute_dims(z, None, SEED, off), full) and off.item() == 123 + B * D
    for row0, n in _splits(B, 3) + [(B - 1, 1), (B // 8, B // 8)]:
        off = _offset(123)
        assert torch.equal(ops.permute_dims_rows(z, row0, n, None, SEED, off), full[row0:row0 + n]), (row0, n)
        assert off.item() == 123 + B * D


# ---- 3: given permutations -------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("B", [16, 5000])
def test_given_perms_windows_equal_indexing(B):
    from disvae import ops
    D = 7
    z = _z(B, D)
    g = torch.Generator().manual_seed(B)
    perms = torch.stack([torch.randperm(B, generator=g) for _ in range(D)])
    expect = apply_perms(z, perms)
    assert torch.equal(ops.permute_dims(z, perms), expect)
    for row0, n in [(0, B)] + _splits(B, 3) + [(B - 1, 1)]:
        assert torch.equal(ops.permute_dims_rows(z, row0, n, perms), expect[row0:row0 + n]), (row0, n)


# ---- 4: refusals -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_row_window_refusals():
    from disvae import _native as N
    L = N.lib()
    st = N.stream()
    for B in (100, 5000):
        D = 4
        z, out = torch.zeros(B, D, device=DEV), torch.zeros(B, D, device=DEV)
        off = _offset(0)
        ws = torch.empty(max(L.dv_permute_dims_workspace_bytes(B, D), 8), dtype=torch.uint8, device=DEV)
        assert L.dv_permute_dims_workspace_bytes(B, D) == (0 if B <= 4096 else 2 * B * D * 8)
        for row0, n in [(-1, 1), (0, 0), (0, B + 1), (B - 1, 2), (B, 1)]:
            assert L.dv_permute_dims_rows(z.data_ptr(), None, 1, off.data_ptr(), out.data_ptr(), B, D, row0, n,
                                          ws.data_ptr(), st) == -1, (B, row0, n)
        for b, d in [(0, D), (B, 0), (B, (1 << 31) // B + 1)]:
            assert L.dv_permute_dims_rows(z.data_ptr(), None, 1, off.data_ptr(), out.data_ptr(), b, d, 0, 1,
                                          ws.data_ptr(), st) == -1, (b, d)
        assert L.dv_permute_dims_rows(z.data_ptr(), None, 1, None, out.data_ptr(), B, D, 0, B, ws.data_ptr(), st) == -2
        assert L.dv_permute_dims_rows(None, None, 1, off.data_ptr(), out.data_ptr(), B, D, 0, B, ws.data_ptr(), st) == -2
        torch.cuda.synchronize()
        assert off.item() == 0                                            # nothing was launched
    B, D = 5000, 4
    z, out, off = torch.zeros(B, D, device=DEV), torch.zeros(B, D, device=DEV), _offset(0)
    assert L.dv_permute_dims_rows(z.data_ptr(), None, 1, off.data_ptr(), out.data_ptr(), B, D, 0, B, None, st) == -2
    assert L.dv_permute_dims(z.data_ptr(), None, 1, off.data_ptr(), out.data_ptr(), B, D, st) == -1   # its limit stays


# ---- 5: one process, FactorVAE above the old limit ------------------------------------------------------------------
@pytest.mark.gpu
def test_single_process_factor_step_above_4096_rows(tmp_path):
    import logging
    import disvae
    from disvae.models.losses import get_loss_f
    torch.manual_seed(1234)
    m = disvae.init_specific_model("Burgess", (1, 32, 32), 10).to(DEV)
    opt = torch.optim.Adam(m.parameters(), lr=5e-4)
    lf = get_loss_f("factor", rec_dist="bernoulli", reg_anneal=0, factor_G=6.4, latent_dim=10, lr_disc=1e-4,
                    device=torch.device(DEV))
    tr = disvae.Trainer(m, opt, lf, device=torch.device(DEV), logger=logging.getLogger("t"), save_dir=str(tmp_path),
                        is_progress_bar=False)
    m.train()
    g = torch.Generator().manual_seed(3)
    x = torch.rand(9216, 1, 32, 32, generator=g).to(DEV)                  # two halves of 4608 rows
    losses = [tr._step(x, None).item() for _ in range(5)]                # 2 eager warm-up steps, capture, replays
    assert len(tr._graphs) == 1, "graph path was not taken"
    assert lf._perm_offset.item() == 5 * 4608 * 10
    assert all(np.isfinite(losses)), losses
    for p in list(m.parameters()) + list(lf.discriminator.parameters()):
        assert torch.isfinite(p).all()


# ---- 6: two ranks ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_two_rank_global_factor_parity():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "ddp_factor_global_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    lines = [l for l in r.stdout.splitlines() if l.startswith("DDP_FACTOR_GLOBAL ")]
    assert lines, r.stdout[-2000:] + "\n" + r.stderr[-6000:]
    rep = json.loads(lines[-1][len("DDP_FACTOR_GLOBAL "):])
    assert rep["ok"] and r.returncode == 0, json.dumps(rep, indent=1)
    assert rep["world"] == 2


# ---- 7: the equal-rows check, gloo on the host -----------------------------------------------------------------------
def _equal_rows_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from disvae import parallel
    from disvae.models.losses import FactorKLoss
    res = {}
    try:
        parallel.check_equal_rows(8)
        res["equal"] = True
    except RuntimeError:
        res["equal"] = False
    gathers = []
    real_gather = parallel.all_gather_rows
    parallel.all_gather_rows = lambda t, group=None: gathers.append(t) or real_gather(t, group)
    lf = FactorKLoss(torch.device("cpu"), disc_kwargs=dict(latent_dim=3))
    try:
        lf._permute_global(torch.zeros(4 + rank, 3))                     # rank 0: 4 rows, rank 1: 5
        res["unequal"] = "no error"
    except RuntimeError as e:
        res["unequal"] = "rows" in str(e) and "4" in str(e) and "5" in str(e)
    res["gathers"] = len(gathers)
    q.put((rank, res))
    dist.destroy_process_group()


def test_equal_rows_check_world2_gloo():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_equal_rows_worker, args=(r, 2, port, q)) for r in range(2)]
    try:
        for p in procs:
            p.start()
        res = sorted(q.get(timeout=120) for _ in procs)
        for p in procs:
            p.join(30)
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
            p.join(10)
    assert res == [(r, dict(equal=True, unequal=True, gathers=0)) for r in range(2)]
