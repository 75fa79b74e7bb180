"""The 32-channel down and up convolutions (wgmma kernels of dv_conv_tc.cu) at the shapes of the training steps, with
every epilogue those steps use, against fp64; and the determinism of a whole c2 training step across Trainers of one
fresh process and with the weight-gradient side stream on or off."""
import collections
import logging
import os
import subprocess
import sys
import tempfile

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda", 0)
TOL = 4e-6          # of the output scale: fp32-grade (single-pass tf32 lands near 5e-4)


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def rel_err(a, b):
    a, b = a.double(), b.double()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def words(t):
    """[t > 0] of a [..., 32] tensor as one int32 word per pixel (bit c = channel c)."""
    bits = (t > 0).to(torch.int64) << torch.arange(32, device=t.device)
    w = bits.sum(-1)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


# batch per GPU of c2 (1x64x64), c3 (3x64x64) and c5 (3x64x64, z=64); the 32-channel layers of both networks run at
# lo 16, 8 and 4 on 64x64 images
SHAPES = [(B, H) for B in (1024, 512, 256) for H in (16, 8, 4)]


@pytest.mark.parametrize("B,H", SHAPES)
def test_conv_down_epilogues_vs_fp64(B, H):
    from disvae import ops
    torch.manual_seed(B + H)
    x = torch.randn(B, 32, 2 * H, 2 * H, device=DEV)
    w = torch.randn(32, 32, 4, 4, device=DEV) * 0.1
    b = torch.randn(32, device=DEV)
    wp = ops.conv_pack(w, 32)
    hi = nhwc(x)
    ref = nhwc(F.conv2d(x.double(), w.double(), None, stride=2, padding=1))            # [B, H, H, 32]

    # encoder forward: bias, ReLU, [out > 0] words for the backward pass
    lo, bits = ops.conv_down(hi, wp, b, None, B, H, H, 32, 0, ops.ACT_RELU, want_bits=True)
    want = torch.relu(ref + b.double())
    assert rel_err(lo, want) <= TOL
    assert torch.equal(bits, words(lo))
    lo2, bits2 = ops.conv_down(hi, wp, b, None, B, H, H, 32, 0, ops.ACT_RELU, want_bits=True)
    assert torch.equal(lo, lo2) and torch.equal(bits, bits2)

    # decoder backward: no activation, float mask with its words, channel sums of the result
    mask = torch.randn(B, H, H, 32, device=DEV)
    g, cs = ops.conv_down(hi, wp, None, mask, B, H, H, 32, 0, ops.ACT_NONE, want_colsum=True, mask_bits=words(mask))
    want = ref * (mask > 0)
    assert rel_err(g, want) <= TOL
    assert rel_err(cs, want.sum((0, 1, 2))) <= TOL
    # ... and the float mask alone (the decoder's first layer)
    g1 = ops.conv_down(hi, wp, None, mask, B, H, H, 32, 0, ops.ACT_NONE)
    assert torch.equal(g1, g)


@pytest.mark.parametrize("B,H", SHAPES)
def test_conv_up_epilogues_vs_fp64(B, H):
    from disvae import ops
    torch.manual_seed(B + H + 1)
    lo_nchw = torch.randn(B, 32, H, H, device=DEV)
    w = torch.randn(32, 32, 4, 4, device=DEV) * 0.1
    b = torch.randn(32, device=DEV)
    wp = ops.conv_pack(w, 32)
    lo = nhwc(lo_nchw)
    ref = nhwc(F.conv_transpose2d(lo_nchw.double(), w.double(), None, stride=2, padding=1))   # [B, 2H, 2H, 32]

    # decoder forward: bias, ReLU, [out > 0] words
    hi, bits = ops.conv_up(lo, wp, b, None, B, H, H, 32, 0, ops.ACT_RELU, want_bits=True)
    want = torch.relu(ref + b.double())
    assert rel_err(hi, want) <= TOL
    assert torch.equal(bits, words(hi))
    hi2, bits2 = ops.conv_up(lo, wp, b, None, B, H, H, 32, 0, ops.ACT_RELU, want_bits=True)
    assert torch.equal(hi, hi2) and torch.equal(bits, bits2)

    # encoder backward: no activation, float mask with its words, and the float mask alone
    mask = torch.randn(B, 2 * H, 2 * H, 32, device=DEV)
    g = ops.conv_up(lo, wp, None, mask, B, H, H, 32, 0, ops.ACT_NONE, mask_bits=words(mask))
    assert rel_err(g, ref * (mask > 0)) <= TOL
    assert torch.equal(ops.conv_up(lo, wp, None, mask, B, H, H, 32, 0, ops.ACT_NONE), g)


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
