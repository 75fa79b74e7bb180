"""Model / loss / training-step parity of the CUDA path against (a) golden fixtures produced by
the unmodified reference (tests/golden/make_golden.py) and (b) the oracle on the same seeded
inputs at larger sizes.  Tolerance: 1e-4 relative fp32 on losses and reconstructions
(BASELINE.json north_star).  Run on an H100: pytest -m gpu."""
import logging
import os
from collections import OrderedDict, defaultdict

import pytest
import torch

from oracle import disvae_oracle as O

pytestmark = pytest.mark.gpu

SEED = 1234
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RTOL = 1e-4
DEV = "cuda"


def rel_err(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def assert_close(a, b, tol=RTOL, what=""):
    assert tuple(a.shape) == tuple(b.shape), (what, a.shape, b.shape)
    e = rel_err(a, b)
    assert e <= tol, "%s: rel err %.3e > %.1e" % (what, e, tol)


def digest_close(t, dg, rtol, atol=0.0):
    """`atol`: extra absolute slack per element (and 4x that on the sums) -- see the Adam note below.
    Head/tail elements are held to rtol of the TENSOR's scale (its mean magnitude, or the sample's own max if
    larger): rounding differences are absolute at the tensor's scale, a sample of 8 elements can be 100x smaller."""
    t = t.detach().double().flatten().cpu()
    assert t.numel() == dg["n"]
    scale = dg["abssum"] / max(1, dg["n"])
    for ours, ref in ((t[:8].float(), dg["head"]), (t[-8:].float(), dg["tail"])):
        assert torch.allclose(ours, ref, rtol=rtol, atol=1e-7 + atol + rtol * max(scale, ref.abs().max().item()))
    tol = rtol * max(1.0, dg["abssum"]) + 4 * atol
    assert abs(t.sum().item() - dg["sum"]) <= tol
    assert abs(t.abs().sum().item() - dg["abssum"]) <= tol


def make_model(img_size, z, ckpt=None):
    import disvae
    torch.manual_seed(SEED)
    m = disvae.init_specific_model("Burgess", img_size, z)
    if ckpt is not None:
        m.load_state_dict(torch.load(os.path.join(GOLDEN, "ckpt", ckpt + ".pt")), strict=False)
    return m.to(DEV)


@pytest.mark.parametrize("name", ["c1_1x32x32", "c2_1x64x64", "c3_3x64x64", "c5_3x64x64_z64",
                                  "ckpt_btcvae_dsprites", "ckpt_VAE_mnist"])
def test_forward_backward_matches_reference_golden(golden, name):
    c = golden("forward.pt")[name]
    m = make_model(c["img_size"], c["latent_dim"], c["ckpt"])
    m.train()
    x = c["x"].to(DEV)
    recon, (mu, logvar), z = m(x, eps=c["eps"].to(DEV))
    assert recon.is_contiguous() and tuple(recon.shape) == tuple(c["recon"].shape)
    assert_close(mu.cpu(), c["mu"], what="mu")
    assert_close(logvar.cpu(), c["logvar"], what="logvar")
    assert_close(z.cpu(), c["z"], what="z")
    assert_close(recon.cpu(), c["recon"], what="recon")
    wr = torch.linspace(0.5, 1.5, recon.numel()).view_as(recon).to(DEV)
    probe = (recon * wr).sum() + (mu * 0.3).sum() - (logvar * 0.2).sum()
    assert abs(probe.item() - c["probe"]) <= RTOL * abs(c["probe"])
    m.zero_grad()
    probe.backward()
    for k, p in m.named_parameters():
        digest_close(p.grad, c["grad_digest"][k], rtol=RTOL)
        if k in c["grad_small"]:
            assert_close(p.grad.cpu(), c["grad_small"][k], what="grad " + k)
    # eval mode: latent sample == mean (vae.py:69-71), encoder/decoder callable on their own
    m.eval()
    with torch.no_grad():
        recon_e, (mu_e, _), z_e = m(x)
        assert torch.equal(z_e, mu_e)
        assert_close(m.decoder(mu_e).cpu(), recon_e.cpu(), tol=0)
        assert_close(m.sample_latent(x).cpu(), mu_e.cpu(), tol=0)


@pytest.mark.parametrize("img_size,z,B", [((3, 64, 64), 10, 37), ((1, 64, 64), 10, 64), ((1, 32, 32), 10, 130),
                                          ((3, 64, 64), 64, 16)])
def test_forward_backward_matches_oracle_larger_batches(img_size, z, B):
    m = make_model(img_size, z)
    m.train()
    p = O.make_leaf_params(OrderedDict((k, v.detach().cpu()) for k, v in m.state_dict().items()))
    torch.manual_seed(B)
    x = torch.rand(B, *img_size)
    eps = torch.randn(B, z)
    recon_o, (mu_o, lv_o), z_o = O.vae_forward(p, x, eps)
    loss_o, _ = O.loss_betaH(x, recon_o, mu_o, lv_o, 4, "bernoulli", 1, 0)
    loss_o.backward()
    from disvae import ops
    from disvae.models.losses import get_loss_f
    from oracle import same_branch as SB
    ops.start_trace()
    recon, (mu, lv), zz = m(x.to(DEV), eps=eps.to(DEV))
    trace = ops.stop_trace()
    lf = get_loss_f("betaH", rec_dist="bernoulli", reg_anneal=0, betaH_B=4)
    loss = lf(x.to(DEV), recon, (mu, lv), True, None)
    assert_close(recon.cpu(), recon_o.detach(), what="recon")
    assert abs(loss.item() - loss_o.item()) <= RTOL * abs(loss_o.item())
    m.zero_grad()
    loss.backward()
    # Gradients: two fp32 evaluation orders (MKL/oneDNN on CPU vs 3xTF32 tensor cores) may round a ReLU pre-activation
    # to opposite sides of zero, which switches a whole back-propagated path.  Referee = the fp64 oracle on the SAME
    # branch of the network as the CUDA path (oracle/same_branch.py), held to 1e-4; every flipped unit must be
    # numerically ambiguous.  Where no unit flipped, the plain fp32 oracle must agree to 1e-4 as well.
    def run64(pp, dd):
        r64, (m64, l64), _ = O.vae_forward(pp, x.double(), eps.double())
        l = O.loss_betaH(x.double(), r64, m64, l64, 4, "bernoulli", 1, 0)[0]
        l.backward()
        return l.item()
    ref = SB.same_branch_reference(trace, OrderedDict((k, v.detach().cpu()) for k, v in m.state_dict().items()), run64)
    assert ref["flip_max_rel"] <= 1e-3, ref
    ours = {k: prm.grad for k, prm in m.named_parameters()}
    err, key = SB.grad_errors(ours, ref["grads"])
    assert err <= RTOL, "grad %s: %.2e vs fp64 on the same branch (%d flipped units)" % (key, err, ref["flips"])
    if ref["flips"] == 0:
        e32, k32 = SB.grad_errors(ours, {k: v.grad for k, v in p.items()})
        assert e32 <= RTOL, (k32, e32)


@pytest.mark.parametrize("loss_name", ["VAE", "betaH", "betaB", "btcvae"])
@pytest.mark.parametrize("rec_dist", ["bernoulli", "laplace", "gaussian"])
@pytest.mark.parametrize("anneal,n_calls", [(0, 1), (100, 3)])
def test_losses_match_reference_golden(golden, loss_name, rec_dist, anneal, n_calls):
    from disvae.models.losses import get_loss_f
    G = golden("losses.pt")
    i = G["inputs"]
    g = G["%s_%s_a%d" % (loss_name, rec_dist, anneal)]
    kw = dict(rec_dist=rec_dist, reg_anneal=anneal, betaH_B=4, betaB_initC=0, betaB_finC=25, betaB_G=100, factor_G=6,
              latent_dim=10, lr_disc=5e-5, btcvae_A=1, btcvae_B=6, btcvae_G=1, device=torch.device(DEV), n_data=737280)
    lf = get_loss_f(loss_name, **kw)
    data = i["data"].to(DEV)
    for _ in range(n_calls):
        recon = i["recon"].to(DEV).requires_grad_(True)
        mu = i["mu"].to(DEV).requires_grad_(True)
        lv = i["logvar"].to(DEV).requires_grad_(True)
        z = mu + torch.exp(0.5 * lv) * i["eps"].to(DEV)
        storer = defaultdict(list)
        loss = lf(data, recon, (mu, lv), True, storer, latent_sample=z)
    assert lf.n_train_steps == g["n_train_steps"]
    assert abs(loss.item() - g["loss"]) <= RTOL * abs(g["loss"])
    gr = torch.autograd.grad(loss, [recon, mu, lv])
    digest_close(gr[0], g["g_recon"], rtol=RTOL)
    assert_close(gr[1].cpu(), g["g_mu"], what="g_mu")
    assert_close(gr[2].cpu(), g["g_logvar"], what="g_logvar")
    if n_calls == 1:        # step 1 records (losses.py:109): every logged key and value must match
        assert set(storer.keys()) == set(g["storer_train"].keys())
        for k, v in g["storer_train"].items():
            assert abs(storer[k][0] - v[0]) <= RTOL * max(1e-3, abs(v[0])), k
    else:
        assert len(storer) == 0
    st = defaultdict(list)
    with torch.no_grad():
        ze = i["mu"] + torch.exp(0.5 * i["logvar"]) * i["eps"]
        le = lf(data, i["recon"].to(DEV), (i["mu"].to(DEV), i["logvar"].to(DEV)), False, st, latent_sample=ze.to(DEV))
    assert abs(le.item() - g["loss_eval"]) <= RTOL * abs(g["loss_eval"])
    assert set(st.keys()) == set(g["storer_eval"].keys())
    for k, v in g["storer_eval"].items():
        assert abs(st[k][0] - v[0]) <= RTOL * max(1e-3, abs(v[0])), k


def _cpu_noise_stream(loss_name, b, z, n_steps):
    """The reference's CPU RNG consumption per iteration (training.py:153, losses.py:254,286,505)."""
    torch.manual_seed(SEED + 5)
    out = []
    for _ in range(n_steps):
        if loss_name == "factor":
            torch.randn(b, z)                                   # discarded full-batch forward (trap T6)
            e1, e2 = torch.randn(b // 2, z), torch.randn(b // 2, z)
            perms = torch.stack([torch.randperm(b // 2) for _ in range(z)])
            out.append((e1, e2, perms))
        else:
            out.append(torch.randn(b, z))
    return out


@pytest.mark.parametrize("loss_name", ["VAE", "betaH", "betaB", "btcvae", "factor"])
def test_train_steps_match_reference_golden(golden, loss_name, tmp_path):
    """3 optimisation steps through disvae.Trainer on the GPU == the reference Trainer on CPU."""
    import disvae
    from disvae.models.losses import get_loss_f
    g = golden("train_steps.pt")[loss_name]
    over = g["over"]
    m = make_model(g["img_size"], 10)
    opt = torch.optim.Adam(m.parameters(), lr=over["lr"])
    kw = dict(rec_dist="bernoulli", reg_anneal=0, betaH_B=4, betaB_initC=0, betaB_finC=25, betaB_G=100, factor_G=6,
              latent_dim=10, lr_disc=5e-5, btcvae_A=1, btcvae_B=6, btcvae_G=1, device=torch.device(DEV),
              n_data=g["n_data"])
    kw.update({k: v for k, v in over.items() if k != "lr"})
    lf = get_loss_f(loss_name, **kw)                 # factor: discriminator drawn here, after the model (same RNG order)
    trainer = disvae.Trainer(m, opt, lf, device=torch.device(DEV), logger=logging.getLogger("t"),
                             save_dir=str(tmp_path), is_progress_bar=False)
    m.train()
    torch.manual_seed(SEED + 4)
    xs = [torch.rand(g["batch"], *g["img_size"]) for _ in range(3)]
    noise = _cpu_noise_stream(loss_name, g["batch"], 10, 3)
    for i, x in enumerate(xs):
        storer = defaultdict(list)
        if loss_name == "factor":
            e1, e2, perms = noise[i]
            # the discarded forward of training.py:153 consumes one eps before the two halves
            m.inject_noise([torch.zeros(g["batch"], 10), e1, e2])
            lf._perm_queue = [perms]
        else:
            m.inject_noise([noise[i]])
        lv = trainer._train_iteration(x, storer)
        ref = g["steps"][i]
        assert abs(lv - ref["loss"]) <= RTOL * abs(ref["loss"]), (i, lv, ref["loss"])
        assert set(storer.keys()) == set(ref["storer"].keys()), i
        for k, v in ref["storer"].items():
            assert abs(storer[k][0] - v[0]) <= RTOL * max(1e-3, abs(v[0])), (i, k, storer[k][0], v[0])
    # Post-Adam parameters.  In its first steps Adam moves every parameter by ~ +-lr regardless of the
    # gradient's magnitude, so an entry whose gradient sign is numerically ambiguous (|g| ~ rounding noise,
    # e.g. biases of barely-active units) lands up to 2*lr apart per step in two correct fp32 implementations.
    # Losses and logged values above are held to 1e-4; parameters to 1e-4 of scale + 2.5*lr per element.
    for k, v in m.state_dict().items():
        digest_close(v, g["params"][k], rtol=RTOL, atol=2.5 * over["lr"])
    # Adam moments are NOT compared after 3 steps: from step 2 on the trajectory depends on which way Adam moved the
    # entries whose first gradient is numerically zero (+-lr whatever the magnitude: 2*lr/|w| ~ 0.5 % relative parameter
    # differences between two correct runs, several % on individual moment entries after three steps -- measured).  The
    # optimizer path is pinned after ONE step, where exp_avg = (1 - beta1) * grad exactly: next test.
    trainer._fused.flush_state()
    for k, prm in m.named_parameters():
        assert float(opt.state[prm]["step"]) == g["opt_state"][k]["step"] == 3.0
    if loss_name == "factor":
        for k, v in lf.discriminator.state_dict().items():
            digest_close(v, g["disc_params"][k], rtol=RTOL, atol=2.5 * over["lr_disc"])


@pytest.mark.parametrize("loss_name", ["VAE", "betaH", "betaB", "btcvae", "factor"])
def test_first_step_adam_moments_match_reference_golden(golden, loss_name, tmp_path):
    """After ONE Trainer step Adam's moments are exactly (1 - beta1) * grad and (1 - beta2) * grad^2: the gradient as the
    (fused) optimizer consumed it -- the check with teeth that the +-2.5 lr parameter bound cannot provide (VERDICT r1
    weak #4).  Against the reference Trainer's optimizer state after its first step; 1e-4 / 2e-4 of each tensor's scale."""
    import disvae
    from disvae.models.losses import get_loss_f
    g = golden("train_steps.pt")[loss_name]
    over = g["over"]
    m = make_model(g["img_size"], 10)
    opt = torch.optim.Adam(m.parameters(), lr=over["lr"])
    kw = dict(rec_dist="bernoulli", reg_anneal=0, betaH_B=4, betaB_initC=0, betaB_finC=25, betaB_G=100, factor_G=6,
              latent_dim=10, lr_disc=5e-5, btcvae_A=1, btcvae_B=6, btcvae_G=1, device=torch.device(DEV), n_data=g["n_data"])
    kw.update({k: v for k, v in over.items() if k != "lr"})
    lf = get_loss_f(loss_name, **kw)
    trainer = disvae.Trainer(m, opt, lf, device=torch.device(DEV), logger=logging.getLogger("t"), save_dir=str(tmp_path),
                             is_progress_bar=False)
    m.train()
    torch.manual_seed(SEED + 4)
    x = torch.rand(g["batch"], *g["img_size"])
    noise = _cpu_noise_stream(loss_name, g["batch"], 10, 1)[0]
    if loss_name == "factor":
        e1, e2, perms = noise
        m.inject_noise([torch.zeros(g["batch"], 10), e1, e2])
        lf._perm_queue = [perms]
    else:
        m.inject_noise([noise])
    from disvae import ops
    from oracle import same_branch as SB
    p32 = OrderedDict((k, v.detach().cpu().clone()) for k, v in m.state_dict().items())
    d32 = (OrderedDict((k, v.detach().cpu().clone()) for k, v in lf.discriminator.state_dict().items())
           if loss_name == "factor" else None)
    ops.start_trace()
    lv = trainer._train_iteration(x, None)
    trace = ops.stop_trace()
    assert abs(lv - g["steps"][0]["loss"]) <= RTOL * abs(g["steps"][0]["loss"])

    def moments_match_golden():
        try:
            for k, prm in m.named_parameters():
                st, ref = opt.state[prm], g["opt_state_step1"][k]
                digest_close(st["exp_avg"], ref["exp_avg"], rtol=RTOL)
                digest_close(st["exp_avg_sq"], ref["exp_avg_sq"], rtol=2 * RTOL)
            if loss_name == "factor":
                for k, prm in lf.discriminator.named_parameters():
                    st, ref = lf.optimizer_d.state[prm], g["disc_opt_state_step1"][k]
                    digest_close(st["exp_avg"], ref["exp_avg"], rtol=RTOL)
                    digest_close(st["exp_avg_sq"], ref["exp_avg_sq"], rtol=2 * RTOL)
            return True
        except AssertionError:
            return False

    if moments_match_golden():
        return
    # The reference run and this one may sit on different sides of a (Leaky)ReLU for a unit whose pre-activation is
    # numerically zero (oracle/same_branch.py).  Then -- and only then -- the referee is the fp64 oracle on THIS run's
    # branch: the trace must show at least one flipped, numerically ambiguous unit, and exp_avg = (1 - beta1) * grad must
    # match that oracle to 1e-4.
    if loss_name == "factor":
        # the Trainer's discarded full-batch forward (training.py:153) is the first encoder/decoder pass of the trace
        second_enc = [i for i, (n, _) in enumerate(trace) if n == "encoder.conv0"][1]
        trace = trace[second_enc:]
    cfg = dict(rec_dist="bernoulli", reg_anneal=kw["reg_anneal"], factor_G=kw["factor_G"])

    def run64(pp, dd):
        xx = x.double()
        if loss_name == "factor":
            l, _, _ = O.factor_step(pp, dd, O.make_adam(pp, 0.0), O.make_adam(dd, 0.0, betas=(0.5, 0.9)), xx, cfg, step=1,
                                    eps1=e1.double(), eps2=e2.double(), perms=perms)
            return l.item()
        ro, (mo, lo), zo = O.vae_forward(pp, xx, noise.double())
        if loss_name in ("VAE", "betaH"):
            l, _ = O.loss_betaH(xx, ro, mo, lo, 1 if loss_name == "VAE" else kw["betaH_B"], "bernoulli", 1, kw["reg_anneal"])
        elif loss_name == "betaB":
            l, _ = O.loss_betaB(xx, ro, mo, lo, kw["betaB_initC"], kw["betaB_finC"], kw["betaB_G"], "bernoulli", 1, kw["reg_anneal"])
        else:
            l, _ = O.loss_btcvae(xx, ro, mo, lo, zo, g["n_data"], kw["btcvae_A"], kw["btcvae_B"], kw["btcvae_G"], "bernoulli", 1,
                                 kw["reg_anneal"])
        l.backward()
        return l.item()
    ref = SB.same_branch_reference(trace, p32, run64, disc32=d32)
    assert ref["flips"] > 0 and ref["flip_max_rel"] <= 1e-3, ref
    ours = {k: opt.state[prm]["exp_avg"] / 0.1 for k, prm in m.named_parameters()}
    if loss_name == "factor":
        ours.update({"disc." + k: lf.optimizer_d.state[prm]["exp_avg"] / 0.5 for k, prm in lf.discriminator.named_parameters()})
    err, key = SB.grad_errors(ours, ref["grads"])
    assert err <= RTOL, "exp_avg/(1-beta1) of %s: %.2e vs fp64 on the same branch (%d flips)" % (key, err, ref["flips"])


def test_factor_step_matches_oracle_including_encoder_leak():
    """FactorVAE at a larger half-batch vs the oracle: covers the CE gradient that leaks into the
    encoder through the non-detached d_z (trap T5) and the discriminator update."""
    from disvae.models.losses import get_loss_f
    B, z, img = 64, 10, (3, 64, 64)
    m = make_model(img, z)
    m.train()
    lf = get_loss_f("factor", rec_dist="bernoulli", reg_anneal=0, factor_G=6.4, latent_dim=z, lr_disc=1e-4,
                    device=torch.device(DEV))
    p = O.make_leaf_params(OrderedDict((k, v.detach().cpu()) for k, v in m.state_dict().items()))
    dp = O.make_leaf_params(OrderedDict((k, v.detach().cpu()) for k, v in lf.discriminator.state_dict().items()))
    opt_o, optd_o = O.make_adam(p, 1e-4), O.make_adam(dp, 1e-4, betas=(0.5, 0.9))
    opt = torch.optim.Adam(m.parameters(), lr=1e-4)
    torch.manual_seed(77)
    x = torch.rand(B, *img)
    e1, e2 = torch.randn(B // 2, z), torch.randn(B // 2, z)
    perms = torch.stack([torch.randperm(B // 2) for _ in range(z)])
    cfg = dict(rec_dist="bernoulli", reg_anneal=0, factor_G=6.4)
    loss_o, logs, _ = O.factor_step(p, dp, opt_o, optd_o, x, cfg, step=1, eps1=e1, eps2=e2, perms=perms)
    storer = defaultdict(list)
    loss = lf.call_optimize(x.to(DEV), m, opt, storer, eps1=e1.to(DEV), eps2=e2.to(DEV), perms=perms)
    assert abs(loss.item() - loss_o.item()) <= RTOL * abs(loss_o.item())
    for k in ("recon_loss", "kl_loss", "tc_loss", "discrim_loss", "loss"):
        assert abs(storer[k][0] - logs[k].item()) <= RTOL * max(1e-3, abs(logs[k].item())), k
    for k, prm in m.named_parameters():
        assert_close(prm.grad.cpu(), p[k].grad, tol=3e-4, what="vae grad " + k)
    for k, prm in lf.discriminator.named_parameters():
        assert_close(prm.grad.cpu(), dp[k].grad, tol=3e-4, what="disc grad " + k)


def test_trainer_runs_epochs_logs_and_checkpoints(tmp_path):
    """disvae.Trainer end to end with device noise: loss goes down, log + checkpoints written."""
    import disvae
    from disvae.models.losses import get_loss_f
    from disvae.utils.modelIO import load_model
    torch.manual_seed(SEED)
    m = disvae.init_specific_model("Burgess", (1, 32, 32), 10)
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    lf = get_loss_f("btcvae", rec_dist="bernoulli", reg_anneal=0, btcvae_A=1, btcvae_B=6, btcvae_G=1, n_data=640)
    lf.record_loss_every = 5                      # record inside every epoch of this short run
    torch.manual_seed(3)
    base = (torch.rand(1, 1, 32, 32) > 0.5).float()
    batches = [((base.repeat(64, 1, 1, 1) * (torch.rand(64, 1, 32, 32) > 0.1).float()), torch.zeros(64)) for _ in range(10)]

    class Loader(list):
        dataset = list(range(640))
    trainer = disvae.Trainer(m, opt, lf, device=torch.device(DEV), logger=logging.getLogger("t"), save_dir=str(tmp_path),
                             is_progress_bar=False)
    first = trainer._train_iteration(batches[0][0], None)
    trainer(Loader(batches), epochs=3, checkpoint_every=2)
    last = trainer._step(batches[0][0], None).item()
    assert last < 0.8 * first, (first, last)
    assert not m.training                                                   # training.py:99
    log = open(os.path.join(str(tmp_path), "train_losses.log")).read().splitlines()
    assert log[0] == "Epoch,Loss,Value" and any(l.startswith("0,recon_loss,") for l in log)
    assert any(l.split(",")[1] == "kl_loss_9" for l in log) and any(l.split(",")[1] == "mi_loss" for l in log)
    assert os.path.exists(os.path.join(str(tmp_path), "model-0.pt")) and os.path.exists(os.path.join(str(tmp_path), "model-2.pt"))
    from disvae.utils.modelIO import save_model
    save_model(m, str(tmp_path), metadata=dict(img_size=[1, 32, 32], latent_dim=10, model_type="Burgess"))
    assert next(m.parameters()).is_cuda                                     # model stays on its device
    m2 = load_model(str(tmp_path))
    x = batches[0][0][:4].to(DEV)
    with torch.no_grad():
        assert torch.equal(m2(x)[0], m(x)[0])


def test_evaluator_losses():
    import disvae
    from disvae.models.losses import get_loss_f
    m = make_model((1, 32, 32), 10)
    lf = get_loss_f("factor", rec_dist="bernoulli", reg_anneal=0, factor_G=6, latent_dim=10, lr_disc=5e-5,
                    device=torch.device(DEV))

    class Loader(list):
        dataset = list(range(64))
    torch.manual_seed(0)
    m.eval()                      # Evaluator.__call__ does this before compute_losses (evaluate.py:75)
    ev = disvae.Evaluator(m, lf, device=torch.device(DEV), logger=logging.getLogger("t"), is_progress_bar=False)
    losses = ev.compute_losses(Loader([(torch.rand(16, 1, 32, 32), None)] * 4))
    assert {"recon_loss", "kl_loss", "loss", "tc_loss", "kl_loss_0"} <= set(losses)


@pytest.mark.parametrize("loss_name", ["btcvae", "betaB", "factor"])
def test_cuda_graph_step_equals_eager_step(loss_name, tmp_path):
    """The Trainer's captured whole-step graph (fwd + loss + bwd + fused Adam, device Philox noise) must walk the
    same trajectory as eager launches of the same kernels: identical seed -> identical parameters."""
    import disvae
    from disvae.models.losses import get_loss_f

    def run(use_graph):
        torch.manual_seed(SEED)
        m = disvae.init_specific_model("Burgess", (1, 32, 32), 10)
        opt = torch.optim.Adam(m.parameters(), lr=5e-4)
        lf = get_loss_f(loss_name, rec_dist="bernoulli", reg_anneal=0, betaB_initC=0, betaB_finC=25, betaB_G=100,
                        btcvae_A=1, btcvae_B=6, btcvae_G=1, n_data=6400, factor_G=6.4, latent_dim=10, lr_disc=1e-4,
                        device=torch.device(DEV))
        tr = disvae.Trainer(m, opt, lf, device=torch.device(DEV), logger=logging.getLogger("t"), save_dir=str(tmp_path),
                            is_progress_bar=False)
        tr.use_cuda_graph = use_graph
        m.train()
        g = torch.Generator().manual_seed(5)
        xs = [torch.rand(64, 1, 32, 32, generator=g).to(DEV) for _ in range(9)]
        losses = [tr._step(x, None).item() for x in xs]
        return m, losses, tr

    m_e, l_e, tr_e = run(False)
    m_g, l_g, tr_g = run(True)
    assert len(tr_g._graphs) == 1, "graph path was not taken"
    for a, b in zip(l_e, l_g):
        assert abs(a - b) <= 1e-6 * abs(a), (l_e, l_g)
    for (k, a), (_, b) in zip(m_e.state_dict().items(), m_g.state_dict().items()):
        assert torch.allclose(a, b, rtol=0, atol=1e-7), k
    if loss_name == "factor":       # FactorVAE: both backward passes and BOTH optimizer steps are inside the graph
        for (k, a), (_, b) in zip(tr_e.loss_f.discriminator.state_dict().items(), tr_g.loss_f.discriminator.state_dict().items()):
            assert torch.allclose(a, b, rtol=0, atol=1e-7), k
        assert tr_g.loss_f.n_train_steps == tr_e.loss_f.n_train_steps == 9


def test_train_epoch_mean_identical_in_graph_and_eager_mode(tmp_path):
    """_train_epoch's 'Average loss per image' over several epochs must not depend on whether steps replay the CUDA
    graph: the epoch accumulator once aliased the graph's static loss tensor (first step of epoch >= 2), which the
    next replay overwrote (ADVICE r1).  Same seed -> same device noise -> the two runs walk the same trajectory."""
    import disvae
    from disvae.models.losses import get_loss_f

    def run(use_graph):
        torch.manual_seed(SEED)
        m = disvae.init_specific_model("Burgess", (1, 32, 32), 10)
        opt = torch.optim.Adam(m.parameters(), lr=5e-4)
        lf = get_loss_f("btcvae", rec_dist="bernoulli", reg_anneal=0, btcvae_A=1, btcvae_B=6, btcvae_G=1, n_data=6400)
        tr = disvae.Trainer(m, opt, lf, device=torch.device(DEV), logger=logging.getLogger("t"), save_dir=str(tmp_path),
                            is_progress_bar=False)
        tr.use_cuda_graph = use_graph
        m.train()
        g = torch.Generator().manual_seed(5)
        loader = [(torch.rand(64, 1, 32, 32, generator=g), None) for _ in range(5)]
        means = [tr._train_epoch(loader, None, e) for e in range(3)]
        steps = float(opt.state[next(m.parameters())]["step"])
        return means, steps, tr

    means_e, steps_e, _ = run(False)
    means_g, steps_g, tr_g = run(True)
    assert len(tr_g._graphs) == 1, "graph path was not taken"
    for a, b in zip(means_e, means_g):
        assert abs(a - b) <= 1e-6 * abs(a), (means_e, means_g)
    assert means_g[0] > means_g[1] > means_g[2]
    assert steps_e == steps_g == 15.0                  # FusedAdam.flush_state at every epoch end (ADVICE r1)


def test_factor_discriminator_adam_step_count_at_epoch_end(tmp_path):
    """FactorVAE: at every epoch end optimizer_d.state[p]["step"] counts the discriminator's Adam steps, as torch's Adam
    would report them -- after eager steps and after graph replays alike (its FusedAdam's counter is flushed too)."""
    import disvae
    from disvae.models.losses import get_loss_f

    def run(use_graph):
        torch.manual_seed(SEED)
        m = disvae.init_specific_model("Burgess", (1, 32, 32), 10)
        opt = torch.optim.Adam(m.parameters(), lr=5e-4)
        lf = get_loss_f("factor", rec_dist="bernoulli", reg_anneal=0, factor_G=6.4, latent_dim=10, lr_disc=1e-4,
                        device=torch.device(DEV))
        tr = disvae.Trainer(m, opt, lf, device=torch.device(DEV), logger=logging.getLogger("t"), save_dir=str(tmp_path),
                            is_progress_bar=False)
        tr.use_cuda_graph = use_graph
        m.train()
        g = torch.Generator().manual_seed(5)
        loader = [(torch.rand(64, 1, 32, 32, generator=g), None) for _ in range(5)]
        counts = []
        for e in range(2):
            tr._train_epoch(loader, None, e)
            counts.append(({float(opt.state[p]["step"]) for p in m.parameters()},
                           {float(lf.optimizer_d.state[p]["step"]) for p in lf.discriminator.parameters()}))
        return counts, tr

    counts_e, _ = run(False)
    counts_g, tr_g = run(True)
    assert len(tr_g._graphs) == 1, "graph path was not taken"
    assert counts_e == counts_g == [({5.0}, {5.0}), ({10.0}, {10.0})]


def test_uint8_batches_train_like_float_batches(tmp_path):
    """SURVEY.md 8f-3: a uint8 host batch (bytes over PCIe, /255 on the device by dv_u8_to_f32 -- in graph mode straight
    into the captured input buffer) walks exactly the trajectory of the same batch converted by ToTensor on the host."""
    import disvae
    from disvae.models.losses import get_loss_f

    def run(as_u8):
        torch.manual_seed(SEED)
        m = disvae.init_specific_model("Burgess", (1, 32, 32), 10)
        opt = torch.optim.Adam(m.parameters(), lr=5e-4)
        lf = get_loss_f("betaH", rec_dist="bernoulli", reg_anneal=0, betaH_B=4)
        tr = disvae.Trainer(m, opt, lf, device=torch.device(DEV), logger=logging.getLogger("t"), save_dir=str(tmp_path),
                            is_progress_bar=False)
        m.train()
        g = torch.Generator().manual_seed(5)
        us = [torch.randint(0, 256, (64, 1, 32, 32), generator=g, dtype=torch.uint8) for _ in range(6)]
        loader = [((u.pin_memory() if as_u8 else u.float().div(255).pin_memory()), None) for u in us]
        means = [tr._train_epoch(loader, None, e) for e in range(2)]
        return means, m, tr

    mf, m_f, _ = run(False)
    mu8, m_u, tr_u = run(True)
    assert len(tr_u._graphs) == 1
    assert mf == mu8
    for (k, a), (_, b) in zip(m_f.state_dict().items(), m_u.state_dict().items()):
        assert torch.equal(a, b), k
