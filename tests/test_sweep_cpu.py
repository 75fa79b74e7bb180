"""Host-side checks of disvae.sweep.Sweep (no GPU needed): the argument checks that run before any GPU work, and the
mapping from a member's seed to the Philox keys of its training draws."""
import logging

import pytest
import torch

import disvae
from disvae import sweep as S
from disvae.models.losses import get_loss_f

CPU = torch.device("cpu")
MASK = 0xFFFFFFFFFFFFFFFF


def _loss(name="btcvae"):
    return get_loss_f(name, rec_dist="bernoulli", reg_anneal=0, btcvae_A=1, btcvae_B=6, btcvae_G=1, n_data=1000,
                      factor_G=6.4, latent_dim=10, lr_disc=1e-4, device=CPU)


def _trainer(tmp_path, name, img=(1, 32, 32), device=CPU, graph=True):
    model = disvae.init_specific_model("Burgess", img, 10)
    tr = disvae.Trainer(model, torch.optim.Adam(model.parameters(), lr=5e-4), _loss(), device=device,
                        logger=logging.getLogger("sweep-cpu"), save_dir=str(tmp_path / name), is_progress_bar=False)
    tr.use_cuda_graph = graph
    return tr


@pytest.fixture
def dirs(tmp_path):
    for name in ("a", "b"):
        (tmp_path / name).mkdir()
    return tmp_path


def test_empty_and_seed_count(dirs):
    with pytest.raises(ValueError, match="no members"):
        S.Sweep([], [])
    with pytest.raises(ValueError, match="2 members but 1 seeds"):
        S.Sweep([_trainer(dirs, "a"), _trainer(dirs, "b")], [1])
    with pytest.raises(ValueError, match="seeds must be integers"):
        S.Sweep([_trainer(dirs, "a")], [1.5])


def test_members_must_be_trainers(dirs):
    with pytest.raises(ValueError, match="member 0 is a str"):
        S.Sweep(["results/a"], [1])


def test_graph_path_required(dirs):
    with pytest.raises(ValueError, match="member 1 has use_cuda_graph=False"):
        S.Sweep([_trainer(dirs, "a"), _trainer(dirs, "b", graph=False)], [1, 2])


def test_trained_members_refused(dirs):
    a, b = _trainer(dirs, "a"), _trainer(dirs, "b")
    b.loss_f.n_train_steps = 3
    with pytest.raises(ValueError, match="member 1 has already taken training steps"):
        S.Sweep([a, b], [1, 2])


def test_distributed_refused(dirs, monkeypatch):
    monkeypatch.setattr(S, "is_distributed", lambda: True)
    with pytest.raises(ValueError, match="torch.distributed is not supported"):
        S.Sweep([_trainer(dirs, "a")], [1])


def test_shared_objects_refused(dirs):
    a = _trainer(dirs, "a")
    b = disvae.Trainer(a.model, torch.optim.Adam(a.model.parameters()), _loss(), device=CPU,
                       logger=logging.getLogger("sweep-cpu"), save_dir=str(dirs / "b"), is_progress_bar=False)
    with pytest.raises(ValueError, match="members share a model object"):
        S.Sweep([a, b], [1, 2])
    with pytest.raises(ValueError, match="members share a model object"):
        S.Sweep([a, a], [1, 1])


def test_image_shape_must_match(dirs):
    with pytest.raises(ValueError, match=r"member 1 takes \(1, 64, 64\) images but member 0 takes \(1, 32, 32\)"):
        S.Sweep([_trainer(dirs, "a"), _trainer(dirs, "b", img=(1, 64, 64))], [1, 2])


def test_cuda_device_required(dirs):
    with pytest.raises(ValueError, match="member 0 is on cpu; a sweep runs on a CUDA device"):
        S.Sweep([_trainer(dirs, "a"), _trainer(dirs, "b")], [1, 2])


@pytest.mark.parametrize("seed", [0, 1, 1234, 0x9E3779B97F4A7C15, MASK, 2 ** 63 + 17])
def test_seed_to_philox_keys(seed):
    """philox_keys(seed) are the keys a lone single-process run fixes at its first step after torch.manual_seed(seed):
    the formulas of VAE._noise_state and FactorKLoss._perm_state with rank salt 0, and what they actually compute."""
    noise, perm = S.philox_keys(seed)
    assert noise == seed & MASK
    assert perm == (seed ^ 0x9E3779B97F4A7C15) & MASK
    saved = torch.initial_seed()
    try:
        torch.manual_seed(seed)
        model = disvae.init_specific_model("Burgess", (1, 32, 32), 10)
        loss = _loss("factor")
        assert model._noise_state(CPU)[0] == noise
        assert loss._perm_state(CPU)[0] == perm
    finally:
        torch.manual_seed(saved)
    model.seed_noise(noise, CPU)
    loss.seed_permutations(perm, CPU)
    assert model._rng_seed == noise and int(model._rng_offset) == 0
    assert loss._perm_seed == perm and int(loss._perm_offset) == 0
    assert model._noise_state(CPU)[0] == noise and loss._perm_state(CPU)[0] == perm    # kept by the first step
