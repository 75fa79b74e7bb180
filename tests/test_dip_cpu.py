"""DIP-VAE-I / DIP-VAE-II without a GPU: the factory's parsing and defaults, the refusals, the exported names, and the
loss's fields in a training state (and their checks on load)."""
import math

import pytest
import torch

from disvae.models import losses
from disvae.models.losses import DIP_LOSSES, LOSSES, DipVAELoss, get_loss_f
from disvae.training import loss_hparams
from test_resume_cpu import _trained, _trainer

ARGS = dict(rec_dist="bernoulli", reg_anneal=0)


def test_names():
    assert LOSSES == ["VAE", "betaH", "betaB", "factor", "btcvae"]      # main.py's -l choices, unchanged
    assert DIP_LOSSES == ["dipI", "dipII"] and losses.DIP_LOSSES is DIP_LOSSES
    assert not set(DIP_LOSSES) & set(LOSSES)


@pytest.mark.parametrize("name,dip_type,lambda_d", [("dipI", "I", 100.0), ("dipII", "II", 10.0)])
def test_factory_defaults(name, dip_type, lambda_d):
    lf = get_loss_f(name, **ARGS)
    assert type(lf) is DipVAELoss
    assert (lf.dip_type, lf.lambda_od, lf.lambda_d) == (dip_type, 10.0, lambda_d)
    assert (lf.rec_dist, lf.steps_anneal, lf.record_loss_every) == ("bernoulli", 0, 50)


@pytest.mark.parametrize("name,lambda_d", [("dipI", 20.0), ("dipII", 2.0)])
def test_factory_lambda_od_sets_the_default_lambda_d(name, lambda_d):
    lf = get_loss_f(name, dip_lambda_od=2, **ARGS)
    assert (lf.lambda_od, lf.lambda_d) == (2.0, lambda_d)
    assert isinstance(lf.lambda_od, float) and isinstance(lf.lambda_d, float)


@pytest.mark.parametrize("name", DIP_LOSSES)
def test_factory_explicit_values_and_extra_keys(name):
    # the whole argparse dictionary of main.py: keys of the other losses are ignored
    kw = dict(rec_dist="laplace", reg_anneal=500, betaH_B=4, betaB_initC=0, betaB_finC=25, betaB_G=100, factor_G=6.4,
              latent_dim=10, lr_disc=5e-5, btcvae_A=1, btcvae_B=6, btcvae_G=1, n_data=737280, device=torch.device("cpu"),
              dip_lambda_od=5, dip_lambda_d=0.5, unrelated="x")
    lf = get_loss_f(name, **kw)
    assert (lf.lambda_od, lf.lambda_d, lf.rec_dist, lf.steps_anneal) == (5.0, 0.5, "laplace", 500)


@pytest.mark.parametrize("bad", [-1.0, -1e-30, math.inf, -math.inf, math.nan, "10", True])
@pytest.mark.parametrize("which", ["lambda_od", "lambda_d"])
def test_refuses_bad_lambdas(which, bad):
    with pytest.raises(ValueError, match=which):
        DipVAELoss("I", **{"lambda_od": 10.0, "lambda_d": 1.0, which: bad})
    key = "dip_" + which
    with pytest.raises(ValueError, match=which):
        get_loss_f("dipII", **dict(ARGS, **{key: bad}))


def test_refuses_missing_lambda_od():
    with pytest.raises(ValueError, match="lambda_od"):
        DipVAELoss("II", lambda_od=None)


def test_zero_lambdas_allowed():
    lf = DipVAELoss("II", lambda_od=0, lambda_d=0)
    assert (lf.lambda_od, lf.lambda_d) == (0.0, 0.0)


@pytest.mark.parametrize("bad", ["III", "i", 1, None, "dipI"])
def test_refuses_unknown_type(bad):
    with pytest.raises(ValueError, match="DIP-VAE type"):
        DipVAELoss(bad)


def test_unknown_loss_name_still_refused():
    with pytest.raises(ValueError, match="Uknown loss"):
        get_loss_f("dipIII", **ARGS)


@pytest.mark.parametrize("name", DIP_LOSSES)
def test_training_state_fields(tmp_path, name):
    tr = _trained(tmp_path, name, reg_anneal=7, dip_lambda_od=2.5)
    st = tr.training_state()
    assert st["loss"]["cls"] == "DipVAELoss" and st["factor"] is None
    hp = st["loss"]["hparams"]
    assert hp == loss_hparams(tr.loss_f)
    assert hp == dict(dip_type=name[3:], lambda_od=2.5, lambda_d=25.0 if name == "dipI" else 2.5,
                      rec_dist="bernoulli", record_loss_every=50, steps_anneal=7)
    dst = _trainer(tmp_path / "dst", name, reg_anneal=7, dip_lambda_od=2.5)
    dst.load_training_state(st)
    assert dst.loss_f.n_train_steps == 321


@pytest.mark.parametrize("src,dst,match", [
    (dict(name="dipI"), dict(name="dipII"), "loss hyper-parameter dip_type"),
    (dict(name="dipII"), dict(name="dipI"), "loss hyper-parameter dip_type"),
    (dict(name="dipI"), dict(name="dipI", dip_lambda_od=20), "loss hyper-parameter lambda_d"),
    (dict(name="dipII"), dict(name="dipII", dip_lambda_d=3), "loss hyper-parameter lambda_d"),
    (dict(name="dipII", dip_lambda_d=10), dict(name="dipII", dip_lambda_od=5, dip_lambda_d=10),
     "loss hyper-parameter lambda_od"),
    (dict(name="dipI"), dict(name="btcvae"), "the loss class"),
    (dict(name="betaH"), dict(name="dipII"), "the loss class"),
])
def test_load_refuses_another_dip_setting(tmp_path, src, dst, match):
    state = _trained(tmp_path / "src", **src).training_state()
    tr = _trainer(tmp_path / "dst", **dst)
    with pytest.raises(ValueError, match=match):
        tr.load_training_state(state)
