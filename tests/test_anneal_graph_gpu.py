"""Annealing and loss-recording training steps on the CUDA-graph path.

The coefficients of an annealed loss and the scalars of a recording step follow the loss's device step counter, so the
Trainer replays its captured graph for those steps too.  Everything a step computes must stay bit-identical to the eager
path: parameters, Adam moments, the FactorVAE discriminator and every value handed to the storer -- and the storer must
also equal what the host path (`_record` on every recording step) gives.
"""
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

from test_anneal_log_cpu import device_coef

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEPS, ANNEAL, EVERY = 40, 7, 5

LOSS_CASES = [("VAE", "bernoulli"), ("betaH", "bernoulli"), ("betaB", "bernoulli"), ("betaB", "laplace"),
              ("factor", "bernoulli"), ("btcvae", "bernoulli")]
GEOMETRIES = [((1, 32, 32), 64), ((1, 64, 64), 256)]


class _CountingLoader:
    """Device batches; notes (direct launches, graph-replayed launches) each time a batch is drawn."""

    def __init__(self, xs):
        self.xs, self.counts = xs, []

    def __len__(self):
        return len(self.xs)

    def __iter__(self):
        from disvae import _native as N
        for x in self.xs:
            self.counts.append((N.lib().dv_launch_count(), N.GRAPH_LAUNCHES))
            yield x, None


def _train(loss_name, rec_dist, img, B, mode, tmp_path):
    """One epoch of STEPS steps.  mode: 'graph' | 'eager' (device loss log) | 'host' (eager, `_record` on the host)."""
    import disvae
    from disvae.models.losses import get_loss_f
    torch.manual_seed(1234)
    m = disvae.init_specific_model("Burgess", img, 10)
    opt = torch.optim.Adam(m.parameters(), lr=5e-4)
    lf = get_loss_f(loss_name, rec_dist=rec_dist, reg_anneal=ANNEAL, betaH_B=4, betaB_initC=0, betaB_finC=25,
                    betaB_G=100, btcvae_A=1, btcvae_B=6, btcvae_G=1, n_data=737280, factor_G=6.4, latent_dim=10,
                    lr_disc=1e-4, device=torch.device(DEV))
    lf.record_loss_every = EVERY

    class HostLogTrainer(disvae.Trainer):
        def _step(self, data, storer):                  # no device loss log: the host path of every recording step
            return self._run_step(data, storer)
    cls = HostLogTrainer if mode == "host" else disvae.Trainer
    tr = cls(m, opt, lf, device=torch.device(DEV), logger=logging.getLogger("t"), save_dir=str(tmp_path),
             is_progress_bar=False)
    tr.use_cuda_graph = mode == "graph"
    m.train()
    g = torch.Generator().manual_seed(5)
    loader = _CountingLoader([torch.rand(B, *img, generator=g).to(DEV) for _ in range(STEPS)])
    storer = defaultdict(list)
    tr._train_epoch(loader, storer, 0)
    torch.cuda.synchronize()
    from disvae import _native as N
    return tr, storer, loader.counts + [(N.lib().dv_launch_count(), N.GRAPH_LAUNCHES)]


def _state(tr):
    """Every tensor a step writes: parameters and Adam moments (and the discriminator's)."""
    out = {}
    nets = [("vae", tr.model, tr.optimizer)]
    if hasattr(tr.loss_f, "discriminator"):
        nets.append(("disc", tr.loss_f.discriminator, tr.loss_f.optimizer_d))
    for tag, net, opt in nets:
        for k, p in net.named_parameters():
            out["%s.%s" % (tag, k)] = p.detach()
            st = opt.state[p]
            out["%s.%s.exp_avg" % (tag, k)] = st["exp_avg"]
            out["%s.%s.exp_avg_sq" % (tag, k)] = st["exp_avg_sq"]
    return out


@pytest.mark.parametrize("img,B", GEOMETRIES, ids=["1x32x32-b64", "1x64x64-b256"])
@pytest.mark.parametrize("loss_name,rec_dist", LOSS_CASES, ids=["-".join(c) for c in LOSS_CASES])
def test_annealed_recording_steps_replay_bit_identical(loss_name, rec_dist, img, B, tmp_path):
    tr_g, st_g, counts = _train(loss_name, rec_dist, img, B, "graph", tmp_path)
    tr_e, st_e, _ = _train(loss_name, rec_dist, img, B, "eager", tmp_path)
    tr_h, st_h, _ = _train(loss_name, rec_dist, img, B, "host", tmp_path)
    assert len(tr_g._graphs) == 1 and not tr_e._graphs and not tr_h._graphs
    for tr in (tr_g, tr_e, tr_h):
        assert tr.loss_f.n_train_steps == STEPS and int(tr.loss_f._step_dev.item()) == STEPS
    s_g, s_e = _state(tr_g), _state(tr_e)
    assert s_g.keys() == s_e.keys()
    for k in s_g:
        assert torch.equal(s_g[k], s_e[k]), k
    for k, v in _state(tr_h).items():
        assert torch.equal(v, s_e[k]), k
    # the storer: 8 recording steps (1, 6, .., 36), same keys in the same order, same values -- and as the host path
    assert len(st_g["loss"]) == len(range(1, STEPS + 1, EVERY)) == 8
    assert list(st_g.items()) == list(st_e.items())
    assert list(st_e.items()) == list(st_h.items())
    # every step after the two eager warm-up steps was a replay: the third step captured (its launches count once as
    # direct ones) and replayed; from the fourth on nothing launches directly and each step replays n_kernels
    n_kernels = next(iter(tr_g._graphs.values())).n_kernels
    assert n_kernels > 0
    # counts[k] is noted when batch k is drawn: the prefetcher draws one batch ahead, so after steps 0 .. k-2; the
    # last entry is noted after the epoch
    after3, final = counts[4], counts[-1]
    assert final[0] - after3[0] == 0, "direct launches after the graph was captured"
    assert final[1] - counts[0][1] == (STEPS - 2) * n_kernels
    assert final[1] - after3[1] == (STEPS - 3) * n_kernels


def test_graph_replays_follow_a_hand_set_step_counter(tmp_path):
    """n_train_steps set by hand between steps (as a resumed run or a parity check does) re-writes the device counter
    before the next replay: the coefficients and the recording rule follow the host value."""
    import disvae
    from disvae.models.losses import get_loss_f

    def run(use_graph):
        torch.manual_seed(1234)
        m = disvae.init_specific_model("Burgess", (1, 32, 32), 10)
        opt = torch.optim.Adam(m.parameters(), lr=5e-4)
        lf = get_loss_f("btcvae", rec_dist="bernoulli", reg_anneal=20, btcvae_A=1, btcvae_B=6, btcvae_G=1, n_data=6400)
        lf.record_loss_every = 4
        tr = disvae.Trainer(m, opt, lf, device=torch.device(DEV), logger=logging.getLogger("t"), save_dir=str(tmp_path),
                            is_progress_bar=False)
        tr.use_cuda_graph = use_graph
        m.train()
        g = torch.Generator().manual_seed(5)
        xs = [torch.rand(64, 1, 32, 32, generator=g).to(DEV) for _ in range(12)]
        storer = defaultdict(list)
        for i, x in enumerate(xs):
            if i == 6:
                lf.n_train_steps = 16
            tr._step(x, storer)
        tr._flush_loss_log()
        return tr, storer
    tr_g, st_g = run(True)
    tr_e, st_e = run(False)
    assert len(tr_g._graphs) == 1
    assert tr_g.loss_f.n_train_steps == 22 and int(tr_g.loss_f._step_dev.item()) == 22
    assert list(st_g.items()) == list(st_e.items()) and len(st_g["loss"]) == 4       # steps 1, 5, 17, 21
    for (k, a), (_, b) in zip(tr_g.model.state_dict().items(), tr_e.model.state_dict().items()):
        assert torch.equal(a, b), k


@pytest.mark.parametrize("base,steps_anneal", [(4, 10000), (10, 10000), (6.4, 10000), (1, 7)])
def test_device_coefficient_near_end_of_annealing(base, steps_anneal):
    """The scheduled combination's coefficient (its debug output) == the host formula == Python's value rounded by
    ctypes, and its loss and gradients are bit-identical to the host-coefficient kernel's."""
    from disvae import ops
    from disvae.models.losses import linear_annealing
    g = torch.Generator(device=DEV).manual_seed(3)
    a0 = torch.rand(12, device=DEV, generator=g) * 100
    b0 = torch.rand(3, device=DEV, generator=g) * 10
    for s in list(range(steps_anneal - 4, steps_anneal + 4)) + [1]:
        step = torch.full((1,), s - 1, dtype=torch.int64, device=DEV)
        a, b = a0.clone().requires_grad_(True), b0.clone().requires_grad_(True)
        loss, coefs = ops.LossCombineSchedFn.apply(a, b, [1.0], [1, 6, base], 1 << 3, (0, 1, steps_anneal), True, step, None)
        assert int(step.item()) == s                                          # advanced on the device
        want = device_coef(base, 0, 1, [s], steps_anneal)[0]
        host = np.float32(linear_annealing(0, 1, s, steps_anneal) * base)
        got = np.float32(coefs[3].item())
        assert got.view(np.uint32) == want.view(np.uint32) == host.view(np.uint32), (s, got, want, host)
        ar, br = a0.clone().requires_grad_(True), b0.clone().requires_grad_(True)
        ref = ops.LossCombineFn.apply(ar, br, [1.0], [1, 6, linear_annealing(0, 1, s, steps_anneal) * base])
        assert torch.equal(loss, ref), s
        ga, gb = torch.autograd.grad(loss * 3.0, [a, b])
        gar, gbr = torch.autograd.grad(ref * 3.0, [ar, br])
        assert torch.equal(ga, gar) and torch.equal(gb, gbr), s
    # outside training: the final coefficient, the counter untouched (not even read)
    loss, coefs = ops.LossCombineSchedFn.apply(a0, None, [1.0, base], None, 1 << 1, (0, 1, steps_anneal), False, None, None)
    assert np.float32(coefs[1].item()) == np.float32(1 * base)


@pytest.mark.parametrize("c_fin,steps_anneal", [(25, 100000), (50, 100000), (25, 7)])
def test_betab_kernel_matches_torch_expression(c_fin, steps_anneal):
    """rec + gamma * |kl - C| and its gradient: the fused kernels against the torch expression of the host path, bit for
    bit -- including kl == C (torch's abs backward gives 0 there) and both signs."""
    from disvae import ops
    from disvae.models.losses import linear_annealing
    for s in list(range(steps_anneal - 3, steps_anneal + 3)) + [1, 2]:
        C = linear_annealing(0, c_fin, s, steps_anneal)
        for kl in (np.float32(C), np.float32(C) + 1.5, np.float32(C) - 0.75, np.float32(3.3)):
            out0 = torch.tensor([123.456, float(kl), 0.5, 1.25, 7.0], device=DEV)
            out = out0.clone().requires_grad_(True)
            step = torch.full((1,), s - 1, dtype=torch.int64, device=DEV)
            loss, consts = ops.BetaBLossFn.apply(out, 100, (0, c_fin, steps_anneal), True, step, None)
            assert int(step.item()) == s
            assert np.float32(consts[0].item()) == device_coef(None, 0, c_fin, [s], steps_anneal)[0] == np.float32(C)
            ref_in = out0.clone().requires_grad_(True)
            ref = ref_in[0] + 100 * (ref_in[1] - C).abs()
            assert torch.equal(loss, ref), (s, kl)
            g, = torch.autograd.grad(loss, out)
            gr, = torch.autograd.grad(ref, ref_in)
            assert torch.equal(g, gr), (s, kl, g, gr)
    loss, consts = ops.BetaBLossFn.apply(out0, 100, (0, c_fin, steps_anneal), False, None, None)
    assert consts[0].item() == c_fin


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.parametrize("loss", ["btcvae", "factor"])
def test_two_rank_annealed_graph_equals_eager(loss):
    """Two ranks (NCCL on two GPUs, gloo over CUDA tensors on one): annealed, recording steps on the graph path are
    bit-identical to the eager path on each rank (parameters, moments, discriminator, storer)."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "ddp_anneal_worker.py"), "--loss", loss]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    lines = [l for l in r.stdout.splitlines() if l.startswith("DDP_ANNEAL ")]
    assert lines, r.stdout[-2000:] + "\n" + r.stderr[-6000:]
    rep = json.loads(lines[-1][len("DDP_ANNEAL "):])
    assert rep["ok"] and r.returncode == 0, json.dumps(rep, indent=1)
    assert rep["world"] == 2
