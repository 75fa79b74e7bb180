"""MIG / AAM from the resident dataset on the GPU: an Evaluator over `DeviceLoader.in_order(b)` writes the files an
Evaluator over `DataLoader(shuffle=False)` writes, bit for bit; `metrics_every` leaves training bit-identical and
writes each epoch's metrics as a standalone Evaluator under the documented seed does, in a lone Trainer, in a Sweep
and across a resume; `Sweep.evaluate` writes every member's files as its lone run does.

The factor datasets here are smaller than the estimator's 10,000 samples, so its default `n_samples` is lowered for
each test (as test_metrics_gpu.py's golden test does) to the size of the smallest factor slice.

Run as a script (`python tests/test_eval_resident_gpu.py PHASE SAVE_DIR OUT`) it trains the resume case's stopped
("first") or continued ("resume") run in a fresh process and saves its result to OUT.
"""
import contextlib
import json
import logging
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DEV = torch.device("cuda", 0)
IMG, B, K, EPOCHS, LOADER_SEED = (1, 32, 32), 64, 8, 3, 99    # 8**4 = 4096 images: 64 c1-sized steps per epoch


@contextlib.contextmanager
def _n_samples(n):
    """The estimator's default n_samples lowered to `n` (the golden test's device; no public option)."""
    import disvae
    fn = disvae.Evaluator._estimate_latent_entropies
    old = fn.__defaults__
    fn.__defaults__ = (n,)
    try:
        yield
    finally:
        fn.__defaults__ = old


def _dataset(k=K):
    """tests/synthetic_factors.FactorRectangles rounded to bytes (what ToTensor makes of 8-bit images)."""
    from synthetic_factors import FactorRectangles
    ds = FactorRectangles(k=k, size=IMG[-1])
    ds.imgs = torch.round(ds.imgs * 255) / 255
    return ds


def _loss(kind, n):
    from disvae.models.losses import get_loss_f
    return get_loss_f(kind, rec_dist="bernoulli", reg_anneal=100, betaB_initC=0, betaB_finC=25, betaB_G=100,
                      btcvae_A=-1, btcvae_B=6, btcvae_G=1, n_data=n, factor_G=6.4, latent_dim=10, lr_disc=1e-4,
                      device=DEV)


def _evaluator(model, loss_f, save_dir):
    import disvae
    os.makedirs(save_dir, exist_ok=True)
    return disvae.Evaluator(model, loss_f, device=DEV, logger=logging.getLogger("eval-resident"), save_dir=str(save_dir),
                            is_progress_bar=False)


def _checkpoint_model():
    import disvae
    torch.manual_seed(1234)
    m = disvae.init_specific_model("Burgess", IMG, 10)
    m.load_state_dict(torch.load(os.path.join(HERE, "golden", "ckpt", "VAE_mnist.pt")))
    return m.to(DEV)


def _member(kind, seed, save_dir):
    """A Trainer as main.py builds one, after torch.manual_seed(seed)."""
    import disvae
    os.makedirs(save_dir, exist_ok=True)
    torch.manual_seed(seed)
    model = disvae.init_specific_model("Burgess", IMG, 10)
    opt = torch.optim.Adam(model.parameters(), lr=5e-4 if kind != "factor" else 1e-4)
    return disvae.Trainer(model, opt, _loss(kind, K ** 4), device=DEV, logger=logging.getLogger("eval-resident"),
                          save_dir=str(save_dir), is_progress_bar=False)


def _loader(ds=None):
    from disvae.data import DeviceLoader
    return DeviceLoader(_dataset() if ds is None else ds, B, seed=LOADER_SEED, device=DEV)


def _read(path):
    with open(path, "rb") as f:
        return f.read()


def _assert_same_helpers(a, b, what, nan_equal=False):
    ha, hb = torch.load(a, weights_only=False), torch.load(b, weights_only=False)
    assert ha.keys() == hb.keys(), what
    for k in hb:
        x, y = ha[k], hb[k]
        if nan_equal and torch.is_floating_point(y):
            assert torch.equal(x.isnan(), y.isnan()), (what, k)
            x, y = x[~x.isnan()], y[~y.isnan()]
        assert torch.equal(x, y), (what, k)


def _assert_same_eval_files(dir_a, dir_b, names, what, nan_equal=False):
    """Logs byte for byte and helper tensors bit for bit; with `nan_equal`, NaN where the other file has NaN (the
    unused slots of SAP's "coef") and bit for bit elsewhere."""
    for fa, fb in names:
        pa, pb = os.path.join(dir_a, fa), os.path.join(dir_b, fb)
        if fa.endswith(".pth"):
            _assert_same_helpers(pa, pb, (what, fa, fb), nan_equal)
        else:
            assert _read(pa) == _read(pb), (what, fa, fb, _read(pa), _read(pb))


def _state(tr):
    """Parameters, Adam moments and step counters (the discriminator's too), train_losses.log and the checkpoints."""
    out = {"graphs": len(tr._graphs), "steps": tr.loss_f.n_train_steps}
    nets = [("vae", tr.model, tr.optimizer)]
    if hasattr(tr.loss_f, "discriminator"):
        nets.append(("disc", tr.loss_f.discriminator, tr.loss_f.optimizer_d))
    for tag, net, opt in nets:
        for name, p in net.named_parameters():
            out["%s.%s" % (tag, name)] = p.detach().cpu()
            for k in ("exp_avg", "exp_avg_sq", "step"):
                out["%s.%s.%s" % (tag, name, k)] = opt.state[p][k].detach().cpu()
    out["log"] = _read(os.path.join(tr.save_dir, "train_losses.log"))
    for f in sorted(os.listdir(tr.save_dir)):
        if f.startswith("model-"):
            out[f] = _read(os.path.join(tr.save_dir, f))
    return out


def _assert_same_state(got, want, what):
    assert got.keys() == want.keys(), what
    for k in want:
        if torch.is_tensor(want[k]):
            assert torch.equal(got[k], want[k]), (what, k)
        else:
            assert got[k] == want[k], (what, k)


def _standalone_epoch_metrics(kind, save_dir, epoch, noise_key, out_dir):
    """The documented reproduction of metrics-{epoch}.log: model-{epoch}.pt in a fresh model, an Evaluator over
    DataLoader(dataset, 1000, shuffle=False) inside evaluation_rng(device, noise key, epoch)."""
    import disvae
    from disvae.evaluate import evaluation_rng
    from synthetic_factors import loader
    m = disvae.init_specific_model("Burgess", IMG, 10)
    m.load_state_dict(torch.load(os.path.join(save_dir, "model-%d.pt" % epoch), weights_only=True))
    with evaluation_rng(DEV, noise_key, epoch):
        _evaluator(m.to(DEV), _loss(kind, K ** 4), out_dir)(loader(_dataset(), 1000), is_metrics=True, is_losses=False)


# ---- 1, 2: in_order against a DataLoader ------------------------------------------------------------------------
@pytest.mark.parametrize("b", [1000, 768])
def test_in_order_evaluator_equals_dataloader_evaluator(tmp_path, b):
    """N = 10,000: b = 1000 divides it, b = 768 leaves a last batch of 16."""
    from synthetic_factors import loader
    ds = _dataset(k=10)
    dl = _loader(ds)
    list(dl.epoch_indices())                                  # the parent has run an epoch: irrelevant to in_order
    view = dl.in_order(b)
    assert len(view) == len(loader(ds, b)) == -(-10000 // b) and view.dataset is ds
    model = _checkpoint_model()
    with _n_samples(1000):
        torch.manual_seed(7)
        _evaluator(model, _loss("btcvae", 10000), tmp_path / "dev")(view, is_metrics=True, is_losses=True)
        torch.manual_seed(7)
        _evaluator(model, _loss("btcvae", 10000), tmp_path / "host")(loader(ds, b), is_metrics=True, is_losses=True)
    assert dl.epoch == 1 and dl.seed == LOADER_SEED
    names = [(f, f) for f in ("metrics.log", "metric_helpers.pth", "test_losses.log")]
    _assert_same_eval_files(tmp_path / "dev", tmp_path / "host", names, "b=%d" % b)
    idx = torch.cat([i for _, i in view])
    assert torch.equal(idx.cpu(), torch.arange(10000))


def test_in_order_with_reference_draws_matches_golden(golden, tmp_path):
    """The golden metrics case (reference index draws injected) over resident data: the same files as over the
    DataLoader, and MIG / AAM within test_evaluator_metrics_match_reference_golden's bounds of the reference's (the
    dataset is rounded to bytes here, as a DeviceLoader stores it)."""
    from synthetic_factors import loader
    g = golden("metrics.pt")["full"]
    ds = _dataset(k=g["k"])
    model = _checkpoint_model()
    with _n_samples(g["n_samples"]):
        for name, data in (("dev", _loader(ds).in_order(1000)), ("host", loader(ds, 1000))):
            ev = _evaluator(model, None, tmp_path / name)
            ev._perm_queue = list(g["perms"])
            ev(data, is_metrics=True, is_losses=False)
            assert not ev._perm_queue
    _assert_same_eval_files(tmp_path / "dev", tmp_path / "host",
                            [("metrics.log", "metrics.log"), ("metric_helpers.pth", "metric_helpers.pth")], "golden")
    metrics = json.load(open(tmp_path / "dev" / "metrics.log"))
    assert abs(metrics["MIG"] - g["metrics"]["MIG"]) < 1e-4 and abs(metrics["AAM"] - g["metrics"]["AAM"]) < 1e-4, \
        (metrics, g["metrics"])


# ---- 3: metrics during training ----------------------------------------------------------------------------------
def test_metrics_every_leaves_training_unchanged(tmp_path):
    seed = 17
    runs = {}
    with _n_samples(512):
        for every in (0, 1):
            tr = _member("btcvae", seed, tmp_path / ("every%d" % every))
            torch.manual_seed(seed)
            tr(_loader(), epochs=EPOCHS, checkpoint_every=1, metrics_every=every)
            runs[every] = tr
    _assert_same_state(_state(runs[1]), _state(runs[0]), "metrics_every=1 vs 0")
    assert runs[1]._graphs.keys() == runs[0]._graphs.keys() and len(runs[1]._graphs) == 1
    assert not any(f.startswith("metric") for f in os.listdir(runs[0].save_dir))
    key = runs[1].training_state()["noise"]["key"]
    assert key == seed
    with _n_samples(512):
        for e in range(EPOCHS):
            out = tmp_path / ("standalone%d" % e)
            _standalone_epoch_metrics("btcvae", runs[1].save_dir, e, key, out)
            _assert_same_eval_files(runs[1].save_dir, out, [("metrics-%d.log" % e, "metrics.log"),
                                                            ("metric_helpers-%d.pth" % e, "metric_helpers.pth")], e)
    # the global generators are left as they were
    with _n_samples(512):
        tr = _member("btcvae", seed, tmp_path / "rng")
        torch.manual_seed(5)
        before = (torch.get_rng_state(), torch.cuda.get_rng_state(DEV))
        tr(_loader(), epochs=1, checkpoint_every=1, metrics_every=1)
        assert torch.equal(torch.get_rng_state(), before[0]) and torch.equal(torch.cuda.get_rng_state(DEV), before[1])


def test_metrics_every_k_cadence_and_host_loader(tmp_path):
    """k = 2 over 3 epochs writes epochs 0 and 2 (the last); a host DataLoader is converted under
    DISVAE_DEVICE_DATA=1."""
    tr = _member("betaB", 3, tmp_path / "k2")
    tr.device_data = True
    torch.manual_seed(3)
    with _n_samples(512):
        tr(torch.utils.data.DataLoader(_dataset(), batch_size=B, shuffle=True), epochs=EPOCHS, checkpoint_every=1,
           metrics_every=2)
    files = sorted(f for f in os.listdir(tr.save_dir) if f.startswith("metric"))
    assert files == ["metric_helpers-0.pth", "metric_helpers-2.pth", "metrics-0.log", "metrics-2.log"]
    assert len(tr._device_loaders) == 1 and not tr.model.training


# ---- 4: sweeps ---------------------------------------------------------------------------------------------------
SPECS = [("btcvae", 11), ("betaB", 12), ("factor", 13)]


def _lone_with_eval(kind, seed, save_dir):
    """A lone Trainer with metrics_every=1, then a standalone Evaluator of its last epoch under the documented seed
    over DataLoader(shuffle=False): what Sweep.evaluate() must reproduce."""
    from disvae.evaluate import evaluation_rng
    from synthetic_factors import loader
    tr = _member(kind, seed, save_dir)
    torch.manual_seed(seed)
    tr(_loader(), epochs=EPOCHS, checkpoint_every=1, metrics_every=1)
    with evaluation_rng(DEV, seed, EPOCHS - 1):
        _evaluator(tr.model, tr.loss_f, save_dir)(loader(_dataset(), 1000), is_metrics=True, is_losses=True)
    return tr


def test_sweep_metrics_and_evaluate_equal_lone_runs(tmp_path):
    from disvae.sweep import Sweep
    with _n_samples(512):
        members = [_member(kind, seed, tmp_path / ("m%d_%s" % (k, kind))) for k, (kind, seed) in enumerate(SPECS)]
        sweep = Sweep(members, seeds=[seed for _, seed in SPECS])
        sweep(_loader(), epochs=EPOCHS, checkpoint_every=1, metrics_every=1)
        sweep.evaluate()
        lones = [_lone_with_eval(kind, seed, tmp_path / ("lone_" + kind)) for kind, seed in SPECS]
    names = [("metrics-%d.log" % e,) * 2 for e in range(EPOCHS)] + [("metric_helpers-%d.pth" % e,) * 2
                                                                   for e in range(EPOCHS)]
    names += [(f, f) for f in ("metrics.log", "metric_helpers.pth", "test_losses.log")]
    for m, lone, (kind, _) in zip(members, lones, SPECS):
        _assert_same_state(_state(m), _state(lone), kind)
        _assert_same_eval_files(m.save_dir, lone.save_dir, names, kind)
        # evaluate() seeds as the metrics of the last epoch: the same MIG / AAM at the same batch size
        _assert_same_eval_files(m.save_dir, m.save_dir, [("metrics.log", "metrics-%d.log" % (EPOCHS - 1))], kind)


# ---- 5: resume ---------------------------------------------------------------------------------------------------
def _resume_run(phase, save_dir):
    """'full': EPOCHS epochs; 'first': 1 epoch; 'resume': load training-state-0.pt and train EPOCHS - 1 more.  All with
    save_state=True and metrics_every=1."""
    from disvae.utils.modelIO import load_training_state
    tr = _member("factor", 29, save_dir)
    if phase == "resume":
        load_training_state(tr, os.path.join(str(save_dir), "training-state-0.pt"))
    torch.manual_seed(29)
    epochs = {"full": EPOCHS, "first": 1, "resume": EPOCHS - 1}[phase]
    with _n_samples(512):
        tr(_loader(), epochs=epochs, checkpoint_every=1, save_state=True, metrics_every=1)
    torch.cuda.synchronize()
    return _state(tr)


def test_resumed_run_writes_the_same_later_metrics(tmp_path):
    full = _resume_run("full", tmp_path / "a")
    for phase in ("first", "resume"):
        r = subprocess.run([sys.executable, os.path.abspath(__file__), phase, str(tmp_path / "b"),
                            str(tmp_path / (phase + ".pt"))], capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, (phase, r.stdout[-2000:] + r.stderr[-4000:])
    got = torch.load(tmp_path / "resume.pt", weights_only=False)
    _assert_same_state(got, full, "resumed")
    names = [("metrics-%d.log" % e,) * 2 for e in range(EPOCHS)] + [("metric_helpers-%d.pth" % e,) * 2
                                                                   for e in range(EPOCHS)]
    _assert_same_eval_files(tmp_path / "b", tmp_path / "a", names, "resume")


if __name__ == "__main__":
    sys.path[:0] = [os.path.join(ROOT, "disentangling-vae_b200"), HERE]
    phase, save_dir, out = sys.argv[1], sys.argv[2], sys.argv[3]
    torch.cuda.set_device(DEV)
    torch.save(_resume_run(phase, save_dir), out)
