"""The plumbing every disentanglement score shares, on the host (no GPU, no kernel): for every entry of
`disvae.evaluate.SCORES`, a Trainer, a Trainer or Sweep under torch.distributed, and a Sweep refuse what the score
cannot be written for before any GPU work; the checks of several scores run in the documented order; the public
signatures that name each score and the file names stay as documented."""
import inspect
import re

import pytest
import torch

import disvae
from disvae import evaluate
from disvae.evaluate import SCORES
from score_stubs import _bare_sweep, _device_loader, _evaluator, _Grid, _trainer, no_gpu  # noqa: F401

IDS = [s.flag for s in SCORES]

# (dataset, latent_dim, message) of the training refusals every score shares; "{label}" is the score's label
SHARED_REFUSALS = [
    (_Grid([100, 100], n=10001), 10, "{label}: the dataset has 10001 items, not the 10000"),
    (_Grid([1] * 3, n=10000), 10, "{label}: the dataset has 10000 items, not the 1 of the full grid"),
    (_Grid([10000], factors=False), 10, "no lat_sizes / lat_names"),
]
# and those of one score
OWN_REFUSALS = {
    "factor_score": [],
    "sap_score": [(_Grid([2, 5000]), 10, "more than the kernel's limit of 256 values")],
    "beta_vae_score": [(_Grid([1, 10000]), 10, "has 1 factors of more than one value")],
}
# the smallest latent_dim above each score's kernel limit, and that limit
LATENT_LIMITS = {"factor_score": (1025, 1024), "sap_score": (1025, 1024), "beta_vae_score": (129, 128)}


def _match(score, msg):
    return re.escape(msg.format(label=score.label))


@pytest.mark.parametrize("score", SCORES, ids=IDS)
def test_trainer_refusals_before_gpu_work(tmp_path, no_gpu, score):
    tr = _trainer(tmp_path)
    good = _device_loader(_Grid([100, 100]))
    with pytest.raises(ValueError, match="%s=True needs metrics_every > 0" % score.flag):
        tr(good, epochs=1, **{score.flag: True})
    for ds, latent_dim, msg in SHARED_REFUSALS + OWN_REFUSALS[score.flag]:
        tr.model.latent_dim = latent_dim
        with pytest.raises(ValueError, match=_match(score, msg)):
            tr(_device_loader(ds), epochs=1, metrics_every=1, **{score.flag: True})
    assert tr.loss_f.n_train_steps == 0 and tr._data_loader is None and good.epoch == 3


@pytest.mark.parametrize("score", SCORES, ids=IDS)
def test_trainer_refuses_a_latent_dim_above_the_limit(tmp_path, no_gpu, score):
    tr = _trainer(tmp_path)
    tr.model.latent_dim, limit = LATENT_LIMITS[score.flag]
    msg = "{label}: latent_dim %d is above the kernel's limit of %d" % (tr.model.latent_dim, limit)
    with pytest.raises(ValueError, match=_match(score, msg)):
        tr(_device_loader(_Grid([100, 100])), epochs=1, metrics_every=1, **{score.flag: True})


@pytest.mark.parametrize("score", SCORES, ids=IDS)
def test_trainer_and_sweep_refuse_scores_under_distributed(tmp_path, no_gpu, monkeypatch, score):
    monkeypatch.setattr(evaluate, "is_distributed", lambda: True)
    tr = _trainer(tmp_path)
    with pytest.raises(ValueError, match="not supported under torch.distributed"):
        tr(_device_loader(_Grid([100, 100])), epochs=1, metrics_every=1, **{score.flag: True})
    with pytest.raises(ValueError, match="%s=True needs metrics_every > 0" % score.flag):
        tr(_device_loader(_Grid([100, 100])), epochs=1, **{score.flag: True})
    sw = _bare_sweep([_trainer(tmp_path, "a")])
    with pytest.raises(ValueError, match="not supported under torch.distributed"):
        sw(_device_loader(_Grid([100, 100])), epochs=1, metrics_every=1, **{score.flag: True})


@pytest.mark.parametrize("score", SCORES, ids=IDS)
def test_sweep_refusals_before_gpu_work(tmp_path, no_gpu, score):
    sw = _bare_sweep([_trainer(tmp_path, "a"), _trainer(tmp_path, "b")])
    with pytest.raises(ValueError, match="%s=True needs metrics_every > 0" % score.flag):
        sw(_device_loader(_Grid([100, 100])), epochs=1, **{score.flag: True})
    msg = _match(score, "{label}: the dataset has 10001 items, not the 10000")
    with pytest.raises(ValueError, match=msg):
        sw(_device_loader(_Grid([100, 100], n=10001)), epochs=1, metrics_every=1, **{score.flag: True})
    assert sw.loader is None and not sw._device_loaders
    sw.loader = _device_loader(_Grid([100, 100], n=10001))
    with pytest.raises(ValueError, match=msg):
        sw.evaluate(is_metrics=False, is_losses=False, **{"is_" + score.flag: True})


def test_checks_run_in_table_order(tmp_path, no_gpu):
    """With every score on, the first refusal in table order wins; a Sweep's training checks each member in turn for
    every score, and `Sweep.evaluate` each score in turn for every member."""
    every = {s.flag: True for s in SCORES}
    sap_first = "more than the kernel's limit of 256 values"                   # SAP refuses it, beta-VAE refuses 129
    tr = _trainer(tmp_path)
    tr.model.latent_dim = 129
    with pytest.raises(ValueError, match=sap_first):
        tr(_device_loader(_Grid([2, 5000])), epochs=1, metrics_every=1, **every)
    with pytest.raises(ValueError, match=sap_first):
        _evaluator(tmp_path, 129)(torch.utils.data.DataLoader(_Grid([2, 5000]), batch_size=10),
                                  **{"is_" + s.flag: True for s in SCORES})
    sw = _bare_sweep([_trainer(tmp_path, "a"), _trainer(tmp_path, "b")])
    sw.members[0].model.latent_dim = 129                                      # beta-VAE refuses member 0,
    sw.members[1].model.latent_dim = 1                                        # SAP member 1
    with pytest.raises(ValueError, match="beta-VAE score: latent_dim 129"):
        sw(_device_loader(_Grid([100, 100])), epochs=1, metrics_every=1, **every)
    sw.loader = _device_loader(_Grid([100, 100]))
    with pytest.raises(ValueError, match="SAP score: latent_dim must be at least 2"):
        sw.evaluate(is_metrics=False, is_losses=False, **{"is_" + s.flag: True for s in SCORES})


def test_public_signatures():
    """The keywords that name each score are public API (README, INTEGRATION.md)."""
    def sig(fn):
        return str(inspect.signature(fn))
    assert sig(disvae.Evaluator.__call__) == (
        "(self, data_loader, is_metrics=False, is_losses=True, is_factor_score=False, factor_score_seed=0, "
        "is_sap_score=False, sap_score_seed=0, is_beta_vae_score=False, beta_vae_score_seed=0)")
    assert sig(disvae.Evaluator.compute_factor_vae_score) == (
        "(self, dataloader, batch_size=64, num_train=10000, num_eval=5000, num_variance_estimate=10000, seed=0)")
    assert sig(disvae.Evaluator.compute_sap_score) == "(self, dataloader, num_train=10000, num_test=5000, C=0.01, seed=0)"
    assert sig(disvae.Evaluator.compute_beta_vae_score) == (
        "(self, dataloader, batch_size=64, num_train=10000, num_eval=5000, seed=0)")
    training = ("(self, data_loader, epochs=10, checkpoint_every=10, save_state=False, metrics_every=0, "
                "metrics_batch_size=1000, factor_score=False, sap_score=False, beta_vae_score=False)")
    assert sig(disvae.Trainer.__call__) == training
    from disvae.sweep import Sweep
    assert sig(Sweep.__call__) == training
    assert sig(Sweep.evaluate) == ("(self, is_metrics=True, is_losses=True, batch_size=1000, is_factor_score=False, "
                                   "is_sap_score=False, is_beta_vae_score=False)")


def test_score_file_names():
    assert [(s.flag, s.label) for s in SCORES] == [("factor_score", "FactorVAE score"), ("sap_score", "SAP score"),
                                                   ("beta_vae_score", "beta-VAE score")]
    assert [(s.filename, s.helpers_file) + evaluate.epoch_score_filenames(s, 7) for s in SCORES] == [
        ("factor_vae_score.log", "factor_vae_score_helpers.pth", "factor_vae_score-7.log",
         "factor_vae_score_helpers-7.pth"),
        ("sap_score.log", "sap_score_helpers.pth", "sap_score-7.log", "sap_score_helpers-7.pth"),
        ("beta_vae_score.log", "beta_vae_score_helpers.pth", "beta_vae_score-7.log", "beta_vae_score_helpers-7.pth")]
