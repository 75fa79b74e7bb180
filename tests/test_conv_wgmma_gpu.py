"""The determinism of a whole c2 training step (whose 32-channel convolutions run on the wgmma kernels of
dv_conv_tc.cu) across Trainers of one fresh process and with the weight-gradient side stream on or off.  The kernels
themselves are checked against fp64 in test_conv_paths_gpu.py."""
import collections
import logging
import os
import subprocess
import sys
import tempfile

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda", 0)


def _c2_trainer(seed):
    """The benchmark's default job: beta-TCVAE, Burgess 1x64x64, z = 10, batch 1024."""
    import disvae
    from disvae.models.losses import get_loss_f
    torch.manual_seed(seed)
    model = disvae.init_specific_model("Burgess", (1, 64, 64), 10).to(DEV)
    opt = torch.optim.Adam(model.parameters(), lr=5e-4)
    loss_f = get_loss_f("btcvae", rec_dist="bernoulli", reg_anneal=0, btcvae_A=1, btcvae_B=6, btcvae_G=1,
                        n_data=737280, latent_dim=10, device=DEV)
    tr = disvae.Trainer(model, opt, loss_f, device=DEV, logger=logging.getLogger("wgmma-gpu"),
                        save_dir=tempfile.mkdtemp(prefix="dvwgmma"), is_progress_bar=False)
    model.train()
    return tr


def _params_after_each_step(batches, seed=5):
    """Two eager steps, the step that captures the graph, one replay: the parameters after each, on the host."""
    tr = _c2_trainer(seed)
    out = []
    for x in batches:
        tr._step(x, collections.defaultdict(list))
        torch.cuda.synchronize()
        out.append([p.detach().cpu() for p in tr.model.parameters()])
    assert len(tr._graphs) == 1
    return out


def _three_trainers():
    """In this process: a first c2 Trainer (the process's first steps: scratch growth, first allocations, the side
    stream's creation), a second one from the same seed, and a third with the weight-gradient side stream off."""
    g = torch.Generator().manual_seed(11)
    batches = [(torch.randint(0, 256, (1024, 1, 64, 64), generator=g).float() / 255).to(DEV) for _ in range(4)]
    first = _params_after_each_step(batches)
    second = _params_after_each_step(batches)
    os.environ["DISVAE_SIDE_STREAM"] = "0"
    no_side = _params_after_each_step(batches)
    return dict(first=first, second=second, no_side=no_side)


def test_c2_steps_identical_across_trainers_and_side_stream(tmp_path):
    """Run in a fresh process, so that its first Trainer really takes the process's first steps: its parameters after
    every step must equal those of a second Trainer built from the same seed, and with the side stream switched off."""
    out = tmp_path / "params.pt"
    env = dict(os.environ)
    env.pop("DISVAE_SIDE_STREAM", None)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), str(out)], capture_output=True, text=True,
                       timeout=900, env=env)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    res = torch.load(out, weights_only=False)
    for step in range(4):
        for a, b, c in zip(res["first"][step], res["second"][step], res["no_side"][step]):
            assert torch.equal(a, b), "step %d: second Trainer differs" % (step + 1)
            assert torch.equal(a, c), "step %d: side stream off differs" % (step + 1)


if __name__ == "__main__":
    sys.path[:0] = [os.path.join(ROOT, "disentangling-vae_b200"), os.path.join(ROOT, "tests")]
    torch.save(_three_trainers(), sys.argv[1])
