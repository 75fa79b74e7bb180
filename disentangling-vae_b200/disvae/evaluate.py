"""Evaluator with the reference's API (disvae/evaluate.py:22-317).  Test losses run on the CUDA path; the MIG / AAM
disentanglement metrics run their one expensive piece -- the marginal-entropy estimator (evaluate.py:233-297), the
same pairwise Gaussian log-density pattern as the beta-TCVAE kernel -- in `dv_latent_entropy` instead of 1000
materialised [N, D, 10] tensors per call (SURVEY.md 8f-4).  Everything else (index bookkeeping, the two metric
formulas on a [n_factors, latent_dim] table) is host code that mirrors the reference line for line, quirks included.
"""
import contextlib
import inspect
import logging
import math
import os
import tempfile
import warnings
from collections import defaultdict
from functools import reduce
from timeit import default_timer
from typing import Callable, NamedTuple

import torch
from tqdm import tqdm

from disvae import _native as N
from disvae.parallel import is_distributed
from disvae.utils.modelIO import save_metadata

TEST_LOSSES_FILE = "test_losses.log"
METRICS_FILENAME = "metrics.log"
METRIC_HELPERS_FILE = "metric_helpers.pth"
FACTOR_SCORE_MIN_VAR = 0.05                # a dim whose global variance is below this is inactive (factor_vae.py)
FACTOR_SCORE_MAX_DIM = 1024                # dv_group_variance's limit
SAP_MAX_DIM = 1024                         # dv_sap_score_matrix's limits: latents,
SAP_MAX_TRAIN = 32768                      # training rows staged in shared memory,
SAP_MAX_CLASSES = 256                      # and values of a scored factor
BETA_VAE_MAX_DIM = 128                     # dv_logistic_fit's limits: latents,
BETA_VAE_MAX_FACTORS = 32                  # and scored factors (classes)
EVAL_SEED_STRIDE = 0x9E3779B97F4A7C15      # odd 64-bit constant: consecutive epochs get unrelated seeds


def epoch_metrics_filenames(epoch):
    """(`metrics-{epoch}.log`, `metric_helpers-{epoch}.pth`): the metrics written after training epoch `epoch`."""
    return "metrics-{}.log".format(epoch), "metric_helpers-{}.pth".format(epoch)


def epoch_score_filenames(score, epoch):
    """(`{stem}-{epoch}.log`, `{stem}_helpers-{epoch}.pth`): the files of `score` (an entry of SCORES) written after
    training epoch `epoch`."""
    return "{}-{}.log".format(score.stem, epoch), "{}_helpers-{}.pth".format(score.stem, epoch)


def evaluation_seed(noise_key, epoch):
    """Seed of the device generator for the evaluation of a run's model after epoch `epoch` (numbered from 0, as in
    `model-{epoch}.pt`): (noise_key + EVAL_SEED_STRIDE * (epoch + 1)) mod 2**64, where `noise_key` is the Philox key of
    the run's reparameterisation noise (`training_state()["noise"]["key"]`).  Nothing else enters it."""
    return (int(noise_key) + EVAL_SEED_STRIDE * (int(epoch) + 1)) & 0xFFFFFFFFFFFFFFFF


@contextlib.contextmanager
def evaluation_rng(device, noise_key, epoch):
    """Inside: `device`'s default CUDA generator is seeded with `evaluation_seed(noise_key, epoch)`, which the
    estimator's index draws (`torch.randperm`) read.  On exit the CPU generator and that CUDA generator are back in the
    state they had before."""
    device = torch.device(device)
    index = torch.cuda.current_device() if device.index is None else device.index
    with torch.random.fork_rng(devices=[index]):
        torch.cuda.default_generators[index].manual_seed(evaluation_seed(noise_key, epoch))
        yield


def check_resident_metrics(loader, metrics_batch_size, device_data):
    """ValueError unless MIG / AAM can be computed from `loader`'s resident data: a DeviceLoader (or a torch DataLoader
    that `device_data` converts to one) over a dataset with `lat_sizes` and `lat_names` and at least the estimator's
    n_samples items, in one process.  No GPU work."""
    from disvae.data import DeviceLoader
    if is_distributed():
        raise ValueError("metrics_every is not supported under torch.distributed; evaluate the saved checkpoints "
                         "with an Evaluator in one process instead")
    if isinstance(loader, torch.utils.data.DataLoader):
        if not device_data:
            raise ValueError("metrics_every needs the dataset resident on the GPU: pass a disvae.data.DeviceLoader or "
                             "set DISVAE_DEVICE_DATA=1 (evaluating through the host DataLoader every few epochs costs "
                             "more than the epochs themselves)")
    elif not isinstance(loader, DeviceLoader):
        raise ValueError("metrics_every needs a disvae.data.DeviceLoader, got %s" % type(loader).__name__)
    ds = loader.dataset
    if not (hasattr(ds, "lat_sizes") and hasattr(ds, "lat_names")):
        raise ValueError("metrics_every: the dataset %s has no lat_sizes / lat_names (known factors of variation), "
                         "which MIG and AAM need" % type(ds).__name__)
    n_samples = inspect.signature(Evaluator._estimate_latent_entropies).parameters["n_samples"].default
    if len(ds) < n_samples:
        raise ValueError("metrics_every: the dataset has %d items, fewer than the %d samples the entropy estimator "
                         "draws" % (len(ds), n_samples))
    if int(metrics_batch_size) < 1:
        raise ValueError("metrics_batch_size must be positive, got %d" % int(metrics_batch_size))


def select_scores(switches, prefix=""):
    """The entries of SCORES, in table order, whose switch `prefix + flag` is true in the mapping `switches` (a
    caller's keyword arguments: `factor_score=...` for a Trainer, `is_factor_score=...` for an Evaluator)."""
    return tuple(s for s in SCORES if switches[prefix + s.flag])


def score_evaluator_args(scores, seed):
    """The Evaluator keywords that write every score of `scores`, each drawn from a generator seeded with `seed`."""
    args = {}
    for s in scores:
        args.update({"is_" + s.flag: True, s.flag + "_seed": seed})
    return args


def check_epoch_scores(scores, metrics_every, loader, latent_dim):
    """ValueError unless every score of `scores` (entries of SCORES) can be written with the metrics of every
    `metrics_every` epochs (after `check_resident_metrics` has accepted `loader`).  No GPU work."""
    for s in scores:
        if not metrics_every:
            raise ValueError("%s=True needs metrics_every > 0: the score is written with the metrics of those epochs"
                             % s.flag)
        s.check(loader.dataset, latent_dim)


def write_epoch_metrics(model, loader, epoch, batch_size, save_dir, logger, scores=()):
    """MIG / AAM of `model` over `loader.in_order(batch_size)` (a DeviceLoader) into `save_dir` as
    `epoch_metrics_filenames(epoch)`, with the index draws seeded by `evaluation_rng(.., model's noise key, epoch)`.
    Every score of `scores` (entries of SCORES) is written from the same encodings as `epoch_score_filenames(score,
    epoch)`, each drawn from its own generator seeded with `evaluation_seed(model's noise key, epoch)`.  The model's
    train / eval mode is kept."""
    device = loader.device
    key = model._noise_state(device)[0]           # fixed at the first training step; this fixes it the same way
    moves = list(zip((METRICS_FILENAME, METRIC_HELPERS_FILE), epoch_metrics_filenames(epoch)))
    for s in scores:
        moves += zip((s.filename, s.helpers_file), epoch_score_filenames(s, epoch))
    with tempfile.TemporaryDirectory(dir=save_dir) as tmp, evaluation_rng(device, key, epoch):
        Evaluator(model, None, device=device, logger=logger, save_dir=tmp, is_progress_bar=False)(
            loader.in_order(batch_size), is_metrics=True, is_losses=False,
            **score_evaluator_args(scores, evaluation_seed(key, epoch)))
        for src, dst in moves:
            os.replace(os.path.join(tmp, src), os.path.join(save_dir, dst))


# ---- what every score needs of the dataset ------------------------------------------------------------------------
def _dataset_lat_sizes(label, dataset):
    """`dataset.lat_sizes`; ValueError prefixed with the score's `label` unless the dataset has known factors."""
    if not (hasattr(dataset, "lat_sizes") and hasattr(dataset, "lat_names")):
        raise ValueError("%s: the dataset %s has no lat_sizes / lat_names (known factors of variation)"
                         % (label, type(dataset).__name__))
    return dataset.lat_sizes


def _full_grid(label, lat_sizes, n):
    """`lat_sizes` as a list of ints; ValueError prefixed with the score's `label` unless `n` items are their full
    grid."""
    lat_sizes = [int(s) for s in lat_sizes]
    if n != reduce(lambda x, y: x * y, lat_sizes, 1):
        raise ValueError("%s: the dataset has %d items, not the %d of the full grid of its factors %s"
                         % (label, n, reduce(lambda x, y: x * y, lat_sizes, 1), lat_sizes))
    return lat_sizes


# ---- FactorVAE score (Kim & Mnih 2018, section 4; the conventions of disentanglement_lib's factor_vae.py) ----------
def check_factor_score(dataset, latent_dim, batch_size=64, num_train=10000, num_eval=5000,
                       num_variance_estimate=10000):
    """ValueError unless the FactorVAE score can be computed over `dataset` for a `latent_dim` model with these
    settings: the dataset has known factors (`lat_sizes`, `lat_names`), is their full grid, and has a factor of more
    than one value.  No GPU work.  Returns lat_sizes as a list of ints."""
    return _check_factor_grid(_dataset_lat_sizes("FactorVAE score", dataset), len(dataset), latent_dim, batch_size,
                              num_train, num_eval, num_variance_estimate)


def _check_factor_grid(lat_sizes, n, latent_dim, batch_size, num_train, num_eval, num_variance_estimate):
    lat_sizes = _full_grid("FactorVAE score", lat_sizes, n)
    if all(s == 1 for s in lat_sizes):
        raise ValueError("FactorVAE score: every factor of %s has one value; there is nothing to vote on" % lat_sizes)
    for name, value, least in (("batch_size", batch_size, 2), ("num_train", num_train, 1), ("num_eval", num_eval, 1),
                               ("num_variance_estimate", num_variance_estimate, 2)):
        if int(value) < least:
            raise ValueError("FactorVAE score: %s must be at least %d, got %d" % (name, least, int(value)))
    if int(latent_dim) > FACTOR_SCORE_MAX_DIM:
        raise ValueError("FactorVAE score: latent_dim %d is above the kernel's limit of %d"
                         % (int(latent_dim), FACTOR_SCORE_MAX_DIM))
    return lat_sizes


def factor_vote_rows(lat_sizes, num_votes, batch_size, generator):
    """(factor [num_votes], rows [num_votes, batch_size]) of `num_votes` votes, drawn from `generator` on its device:
    one randint for the factor of every vote (among the factors of more than one value), then one randint per factor k,
    k = 0 .. K-1 in order (size-1 factors included), for the [num_votes, batch_size] values of factor k.  Factor k of
    a vote on k takes row 0's value in every row.  Rows are the C-order grid indices, the last factor fastest; each
    value is below its factor's size, so every row is in [0, prod(lat_sizes))."""
    device = generator.device
    varying = torch.tensor([k for k, s in enumerate(lat_sizes) if s > 1], dtype=torch.int64, device=device)
    factor = varying[torch.randint(len(varying), (num_votes,), generator=generator, device=device)]
    rows = torch.zeros(num_votes, batch_size, dtype=torch.int64, device=device)
    stride = 1
    strides = []
    for s in reversed(lat_sizes):
        strides.insert(0, stride)
        stride *= s
    for k, s in enumerate(lat_sizes):
        values = torch.randint(s, (num_votes, batch_size), generator=generator, device=device)
        values = torch.where((factor == k).unsqueeze(1), values[:, :1], values)
        rows += values * strides[k]
    return factor, rows


def group_variance(mu, rows, global_var=None, var_out=None, argmin_out=None):
    """`dv_group_variance` on `mu` [N, D] (any strides, a view of q_zCx included) and int64 `rows` [V, L]: the
    unbiased variance of every group into `var_out` [V, D], and / or into int32 `argmin_out` [V] the dim minimising
    var / global_var over the dims with global_var >= FACTOR_SCORE_MIN_VAR."""
    N.require_cuda_f32(mu)
    n, d = mu.shape
    V, L = rows.shape
    if rows.dtype != torch.int64 or not rows.is_contiguous():
        raise ValueError("group_variance: rows must be a contiguous int64 tensor")
    for name, t, dtype, shape in (("var_out", var_out, torch.float32, (V, d)),
                                  ("argmin_out", argmin_out, torch.int32, (V,)),
                                  ("global_var", global_var, torch.float32, (d,))):
        if t is not None and (t.dtype != dtype or not t.is_contiguous() or not t.is_cuda or tuple(t.shape) != shape):
            raise ValueError("group_variance: %s must be a contiguous CUDA %s tensor of shape %s" % (name, dtype, shape))
    N.call("dv_group_variance", N.ptr(mu), mu.stride(1), mu.stride(0), n, d, N.ptr(rows), V, L, N.ptr(global_var),
           FACTOR_SCORE_MIN_VAR, N.ptr(var_out), N.ptr(argmin_out), N.stream())


def factor_vae_score(mu, lat_sizes, batch_size=64, num_train=10000, num_eval=5000, num_variance_estimate=10000,
                     seed=0):
    """FactorVAE score of the encoder means `mu` [N, D] (CUDA fp32, dataset index order) of the full factor grid
    `lat_sizes` -> ({"train_accuracy", "eval_accuracy", "num_active_dims"}, helpers).  The draws come from a device
    torch.Generator seeded with `seed`, in this order: the `num_variance_estimate` variance rows
    (`torch.randint(N, (num_variance_estimate,))`), then `factor_vote_rows` for the training votes, then for the
    evaluation votes; no vote is drawn when no dim is active.  The global generators are not touched."""
    lat_sizes = _check_factor_grid(lat_sizes, mu.shape[0], mu.shape[1], batch_size, num_train, num_eval,
                                   num_variance_estimate)
    N.require_cuda_f32(mu)
    n, D = mu.shape
    K = len(lat_sizes)
    gen = torch.Generator(device=mu.device)
    gen.manual_seed(int(seed))
    var_rows = torch.randint(n, (int(num_variance_estimate),), generator=gen, device=mu.device)
    global_var = torch.empty(1, D, dtype=torch.float32, device=mu.device)
    group_variance(mu, var_rows.view(1, -1), var_out=global_var)
    global_var = global_var[0]
    active = global_var >= FACTOR_SCORE_MIN_VAR
    num_active = int(active.sum())
    if num_active == 0:
        train_votes = torch.zeros(K, D, dtype=torch.int64)
        eval_votes = torch.zeros(K, D, dtype=torch.int64)
    else:
        train_factor, train_rows = factor_vote_rows(lat_sizes, int(num_train), int(batch_size), gen)
        eval_factor, eval_rows = factor_vote_rows(lat_sizes, int(num_eval), int(batch_size), gen)
        dims = torch.empty(int(num_train) + int(num_eval), dtype=torch.int32, device=mu.device)
        group_variance(mu, torch.cat([train_rows, eval_rows]), global_var=global_var, argmin_out=dims)
        cells = (torch.cat([train_factor, eval_factor]) * D + dims.long()).cpu()
        train_votes = torch.bincount(cells[:num_train], minlength=K * D).view(K, D)
        eval_votes = torch.bincount(cells[num_train:], minlength=K * D).view(K, D)
    classifier, train_accuracy, eval_accuracy = factor_vote_accuracies(train_votes, eval_votes)
    score = {"train_accuracy": train_accuracy, "eval_accuracy": eval_accuracy, "num_active_dims": num_active}
    helpers = {"global_variances": global_var.cpu(), "active_dims": active.cpu(), "train_votes": train_votes,
               "eval_votes": eval_votes, "classifier": classifier}
    return score, helpers


def factor_vote_accuracies(train_votes, eval_votes):
    """(classifier [D], train accuracy, eval accuracy) of vote tables [K, D]: classifier[d] = argmax_k
    train_votes[k, d], the lowest k on a tie; an accuracy is the share of a table's votes the classifier gets right."""
    classifier = torch.argmax(train_votes, dim=0)
    cols = torch.arange(train_votes.size(1))

    def accuracy(votes):
        total = int(votes.sum())
        return int(votes[classifier, cols].sum()) / total if total else 0.0
    return classifier, accuracy(train_votes), accuracy(eval_votes)


# ---- SAP score (Kumar et al. 2018, section 3; the discrete variant of disentanglement_lib's sap_score.py) -----------
def check_sap_score(dataset, latent_dim, num_train=10000, num_test=5000, C=0.01):
    """ValueError unless the SAP score can be computed over `dataset` for a `latent_dim` model with these settings: the
    dataset has known factors (`lat_sizes`, `lat_names`) and is their full grid.  No GPU work.  Returns lat_sizes as a
    list of ints."""
    return _check_sap_grid(_dataset_lat_sizes("SAP score", dataset), len(dataset), latent_dim, num_train, num_test, C)


def _check_sap_grid(lat_sizes, n, latent_dim, num_train, num_test, C):
    lat_sizes = _full_grid("SAP score", lat_sizes, n)
    if all(s == 1 for s in lat_sizes):
        raise ValueError("SAP score: every factor of %s has one value; there is nothing to predict" % lat_sizes)
    if max(lat_sizes) > SAP_MAX_CLASSES:
        raise ValueError("SAP score: a factor of %s has more than the kernel's limit of %d values"
                         % (lat_sizes, SAP_MAX_CLASSES))
    if int(latent_dim) < 2:
        raise ValueError("SAP score: latent_dim must be at least 2 (the score compares the two most predictive dims), "
                         "got %d" % int(latent_dim))
    if int(latent_dim) > SAP_MAX_DIM:
        raise ValueError("SAP score: latent_dim %d is above the kernel's limit of %d" % (int(latent_dim), SAP_MAX_DIM))
    if int(num_train) < 2:
        raise ValueError("SAP score: num_train must be at least 2, got %d" % int(num_train))
    if int(num_train) > SAP_MAX_TRAIN:
        raise ValueError("SAP score: num_train %d is above the kernel's limit of %d" % (int(num_train), SAP_MAX_TRAIN))
    if int(num_test) < 1:
        raise ValueError("SAP score: num_test must be at least 1, got %d" % int(num_test))
    if not (math.isfinite(float(C)) and float(C) > 0):
        raise ValueError("SAP score: C must be finite and positive, got %r" % (C,))
    return lat_sizes


def sap_labels(lat_sizes, train_rows, test_rows):
    """Class labels of the scored factors (those of more than one value, ascending) for grid rows `train_rows` /
    `test_rows` (C-order grid indices, the last factor fastest), all on the rows' device without a host sync ->
    (factors [K'] list, train_cls int32 [K', num_train], test_cls int32 [K', num_test], n_classes int32 [K'],
    counts int32 [K', S], present bool [K', S]) with S the largest size of a scored factor.  The classes of factor k are
    the values seen among the training rows, ascending; a row's class is its value's place among them, -1 for a test
    value no training row has; counts[k, c] is the training rows of class c and present[k, v] marks value v."""
    device = train_rows.device
    factors = [k for k, s in enumerate(lat_sizes) if s > 1]
    S = max(lat_sizes[k] for k in factors)
    strides = [reduce(lambda x, y: x * y, lat_sizes[k + 1:], 1) for k in range(len(lat_sizes))]
    values = torch.arange(S, device=device)
    train_cls, test_cls, counts, present = [], [], [], []
    for k in factors:
        vt = train_rows // strides[k] % lat_sizes[k]
        ve = test_rows // strides[k] % lat_sizes[k]
        cnt = (vt.unsqueeze(1) == values).sum(0)                  # [S]; values >= lat_sizes[k] count 0
        seen = cnt > 0
        place = torch.cumsum(seen, 0) - 1
        train_cls.append(place[vt])
        test_cls.append(torch.where(seen[ve], place[ve], -1))
        counts.append(torch.zeros(S + 1, dtype=cnt.dtype, device=device).scatter_(
            0, torch.where(seen, place, S), cnt)[:S])
        present.append(seen)
    present = torch.stack(present)
    return (factors, torch.stack(train_cls).int(), torch.stack(test_cls).int(), present.sum(1).int(),
            torch.stack(counts).int(), present)


def sap_score_matrix(mu, train_rows, test_rows, train_cls, test_cls, n_classes, counts, C, coef=None, iters=None):
    """`dv_sap_score_matrix` on `mu` [N, D] (any strides, a view of q_zCx included) -> the fp32 score [D, K'] of
    `sap_labels`' classes; optionally the fitted lines into fp64 `coef` [D, K', S, 2] and the Newton steps into int32
    `iters` [D, K', S]."""
    N.require_cuda_f32(mu)
    n, d = mu.shape
    K, S = counts.shape
    for name, t, dtype in (("train_rows", train_rows, torch.int64), ("test_rows", test_rows, torch.int64),
                           ("train_cls", train_cls, torch.int32), ("test_cls", test_cls, torch.int32),
                           ("n_classes", n_classes, torch.int32), ("counts", counts, torch.int32),
                           ("coef", coef, torch.float64), ("iters", iters, torch.int32)):
        if t is not None and (t.dtype != dtype or not t.is_contiguous() or not t.is_cuda):
            raise ValueError("sap_score_matrix: %s must be a contiguous CUDA %s tensor" % (name, dtype))
    score = torch.empty(d, K, dtype=torch.float32, device=mu.device)
    N.call("dv_sap_score_matrix", N.ptr(mu), mu.stride(1), mu.stride(0), n, d, N.ptr(train_rows), train_rows.numel(),
           N.ptr(test_rows), test_rows.numel(), N.ptr(train_cls), N.ptr(test_cls), N.ptr(n_classes), N.ptr(counts), K,
           S, float(C), N.ptr(score), N.ptr(coef), N.ptr(iters), N.stream())
    return score


def sap_from_matrix(score_matrix):
    """SAP of a score matrix [D, K'] (D >= 2): the mean over factors of the largest minus the second largest score of
    the factor's column, in fp64."""
    m = torch.sort(score_matrix.double().cpu(), dim=0, descending=True)[0]
    return float((m[0] - m[1]).mean())


def sap_score(mu, lat_sizes, num_train=10000, num_test=5000, C=0.01, seed=0):
    """SAP score of the encoder means `mu` [N, D] (CUDA fp32, dataset index order) of the full factor grid `lat_sizes`
    -> ({"SAP"}, helpers).  The draws come from a device torch.Generator seeded with `seed`: `torch.randint(N,
    (num_train,))` for the training rows, then `torch.randint(N, (num_test,))` for the test rows; the global generators
    are not touched.  For every latent and scored factor `dv_sap_score_matrix` fits LinearSVC(C,
    class_weight="balanced") exactly and scores it on the test rows; SAP is `sap_from_matrix` of that table.
    helpers: "score_matrix" fp32 [D, K'], "factors" (the scored factor indices, ascending), "classes" int64 [K', S]
    (each factor's training values, ascending, -1 beyond), "coef" fp64 [D, K', S, 2] (w, b of each problem: class c's
    one-vs-rest problem in slot c, the two-class problem in slot 0, NaN beyond) and "solver_iterations" int32
    [D, K', S] (Newton steps, -1 for a fit that did not converge, which also raises a RuntimeWarning)."""
    lat_sizes = _check_sap_grid(lat_sizes, mu.shape[0], mu.shape[1], num_train, num_test, C)
    N.require_cuda_f32(mu)
    n, D = mu.shape
    gen = torch.Generator(device=mu.device)
    gen.manual_seed(int(seed))
    train_rows = torch.randint(n, (int(num_train),), generator=gen, device=mu.device)
    test_rows = torch.randint(n, (int(num_test),), generator=gen, device=mu.device)
    factors, train_cls, test_cls, n_classes, counts, present = sap_labels(lat_sizes, train_rows, test_rows)
    K, S = counts.shape
    coef = torch.empty(D, K, S, 2, dtype=torch.float64, device=mu.device)
    iters = torch.empty(D, K, S, dtype=torch.int32, device=mu.device)
    matrix = sap_score_matrix(mu, train_rows, test_rows, train_cls, test_cls, n_classes, counts, C, coef, iters)
    matrix, coef, iters, present = matrix.cpu(), coef.cpu(), iters.cpu(), present.cpu()
    failed = int((iters < 0).sum())
    if failed:
        warnings.warn("SAP score: %d of the linear-SVM fits did not converge in the solver's step limit; see "
                      "helpers['solver_iterations'] (-1)" % failed, RuntimeWarning)
    values = torch.arange(S).expand(K, S)
    classes = torch.sort(torch.where(present, values, S), dim=1)[0]           # the values seen, ascending, then S
    helpers = {"score_matrix": matrix, "factors": torch.tensor(factors, dtype=torch.int64),
               "classes": torch.where(classes < S, classes, -1), "coef": coef, "solver_iterations": iters}
    return {"SAP": sap_from_matrix(matrix)}, helpers


# ---- beta-VAE score (Higgins et al. 2017, section 3; the conventions of disentanglement_lib's beta_vae.py) ---------
def check_beta_vae_score(dataset, latent_dim, batch_size=64, num_train=10000, num_eval=5000):
    """ValueError unless the beta-VAE score can be computed over `dataset` for a `latent_dim` model with these
    settings: the dataset has known factors (`lat_sizes`, `lat_names`), is their full grid and has between 2 and
    BETA_VAE_MAX_FACTORS factors of more than one value.  No GPU work.  Returns lat_sizes as a list of ints."""
    return _check_beta_vae_grid(_dataset_lat_sizes("beta-VAE score", dataset), len(dataset), latent_dim, batch_size,
                                num_train, num_eval)


def _check_beta_vae_grid(lat_sizes, n, latent_dim, batch_size, num_train, num_eval):
    lat_sizes = _full_grid("beta-VAE score", lat_sizes, n)
    scored = sum(s > 1 for s in lat_sizes)
    if scored < 2:
        raise ValueError("beta-VAE score: %s has %d factors of more than one value; the score needs at least 2 to "
                         "tell apart" % (lat_sizes, scored))
    if scored > BETA_VAE_MAX_FACTORS:
        raise ValueError("beta-VAE score: %s has %d factors of more than one value, above the kernel's limit of %d"
                         % (lat_sizes, scored, BETA_VAE_MAX_FACTORS))
    if int(latent_dim) > BETA_VAE_MAX_DIM:
        raise ValueError("beta-VAE score: latent_dim %d is above the kernel's limit of %d"
                         % (int(latent_dim), BETA_VAE_MAX_DIM))
    for name, value in (("batch_size", batch_size), ("num_train", num_train), ("num_eval", num_eval)):
        if int(value) < 1:
            raise ValueError("beta-VAE score: %s must be at least 1, got %d" % (name, int(value)))
    return lat_sizes


def beta_vae_points(lat_sizes, count, batch_size, generator):
    """(label [count], rows_a, rows_b [count, batch_size]) of `count` points drawn from `generator` on its device: one
    randint for the label of every point (its scored factor's place among the factors of more than one value), then
    for every factor k, k = 0 .. K-1 in order (size-1 factors included), one randint [count, batch_size] for its `a`
    values and one for its `b` values; factor k of a point on k takes the `a` values in `b` too.  Rows are the C-order
    grid indices, the last factor fastest."""
    device = generator.device
    varying = torch.tensor([k for k, s in enumerate(lat_sizes) if s > 1], dtype=torch.int64, device=device)
    label = torch.randint(len(varying), (count,), generator=generator, device=device)
    factor = varying[label]
    rows_a = torch.zeros(count, batch_size, dtype=torch.int64, device=device)
    rows_b = torch.zeros(count, batch_size, dtype=torch.int64, device=device)
    stride = reduce(lambda x, y: x * y, lat_sizes, 1)
    for k, s in enumerate(lat_sizes):
        stride //= s
        a = torch.randint(s, (count, batch_size), generator=generator, device=device)
        b = torch.randint(s, (count, batch_size), generator=generator, device=device)
        b = torch.where((factor == k).unsqueeze(1), a, b)
        rows_a += a * stride
        rows_b += b * stride
    return label, rows_a, rows_b


def pair_abs_diff_mean(mu, rows_a, rows_b):
    """`dv_pair_abs_diff_mean` on `mu` [N, D] (any strides, a view of q_zCx included) and int64 `rows_a`, `rows_b`
    [V, L] -> fp64 x [V, D], x[v, d] = mean over l of |mu[rows_a[v, l], d] - mu[rows_b[v, l], d]|, added in order."""
    N.require_cuda_f32(mu)
    n, d = mu.shape
    V, L = rows_a.shape
    for name, t in (("rows_a", rows_a), ("rows_b", rows_b)):
        if t.dtype != torch.int64 or not t.is_contiguous() or t.shape != (V, L):
            raise ValueError("pair_abs_diff_mean: %s must be a contiguous int64 tensor of shape %s" % (name, (V, L)))
    x = torch.empty(V, d, dtype=torch.float64, device=mu.device)
    N.call("dv_pair_abs_diff_mean", N.ptr(mu), mu.stride(1), mu.stride(0), n, d, N.ptr(rows_a), N.ptr(rows_b), V, L,
           N.ptr(x), N.stream())
    return x


def logistic_fit(x, labels, n_classes, K, num_train):
    """`dv_logistic_fit` on fp64 features `x` [V, D] (the first `num_train` rows train) with int32 class indices
    `labels` [num_train] and the class count in int32 `n_classes` [1] on the device -> (coef fp64 [K, D + 1], pred
    int32 [V], iters int32 [1]); see include/disvae_b200.h for the objective and the layout of coef."""
    V, D = x.shape
    for name, t, dtype in (("x", x, torch.float64), ("labels", labels, torch.int32),
                           ("n_classes", n_classes, torch.int32)):
        if t.dtype != dtype or not t.is_contiguous() or not t.is_cuda:
            raise ValueError("logistic_fit: %s must be a contiguous CUDA %s tensor" % (name, dtype))
    L = N.lib()
    nbytes = L.dv_logistic_fit_workspace_bytes(int(num_train), D, int(K))
    ws = torch.empty(max(nbytes, 8) // 8, dtype=torch.float64, device=x.device)
    coef = torch.empty(int(K), D + 1, dtype=torch.float64, device=x.device)
    pred = torch.empty(V, dtype=torch.int32, device=x.device)
    iters = torch.empty(1, dtype=torch.int32, device=x.device)
    N.call("dv_logistic_fit", N.ptr(x), D, int(num_train), V - int(num_train), N.ptr(labels), N.ptr(n_classes), int(K),
           N.ptr(coef), N.ptr(pred), N.ptr(iters), N.ptr(ws), nbytes, N.stream())
    return coef, pred, iters


def beta_vae_score(mu, lat_sizes, batch_size=64, num_train=10000, num_eval=5000, seed=0):
    """beta-VAE score of the encoder means `mu` [N, D] (CUDA fp32, dataset index order) of the full factor grid
    `lat_sizes` -> ({"train_accuracy", "eval_accuracy"}, helpers).  The draws come from a device torch.Generator seeded
    with `seed`: `beta_vae_points` for the `num_train` training points, then for the `num_eval` evaluation points; the
    global generators are not touched.  A point's feature is `pair_abs_diff_mean` of its rows, and `logistic_fit` fits
    LogisticRegression(C=1) exactly to the training points, over the scored factors seen among them.
    helpers: "factors" int64 [K'] (the scored factors, ascending), "classes" int64 (the factors seen in training,
    ascending), "coef" fp64 [rows, D] and "intercept" fp64 [rows] (rows = the classes for more than two, 1 for two
    with classes[1] the positive class, 0 for one), "solver_iterations" int32 scalar (Newton steps, -1 for a fit that
    did not converge, which also raises a RuntimeWarning), "train_confusion" and "eval_confusion" int64 [K', K'] (points by
    true x predicted scored factor)."""
    lat_sizes = _check_beta_vae_grid(lat_sizes, mu.shape[0], mu.shape[1], batch_size, num_train, num_eval)
    N.require_cuda_f32(mu)
    num_train, num_eval, batch_size = int(num_train), int(num_eval), int(batch_size)
    device = mu.device
    gen = torch.Generator(device=device)
    gen.manual_seed(int(seed))
    train_label, train_a, train_b = beta_vae_points(lat_sizes, num_train, batch_size, gen)
    eval_label, eval_a, eval_b = beta_vae_points(lat_sizes, num_eval, batch_size, gen)
    x = pair_abs_diff_mean(mu, torch.cat([train_a, eval_a]), torch.cat([train_b, eval_b]))
    factors = [k for k, s in enumerate(lat_sizes) if s > 1]
    K = len(factors)
    seen = torch.bincount(train_label, minlength=K) > 0
    place = torch.cumsum(seen, 0) - 1
    classes = torch.sort(torch.where(seen, torch.arange(K, device=device), K))[0]    # seen labels, ascending, then K
    n_classes = seen.sum().int().view(1)
    coef, pred, iters = logistic_fit(x, place[train_label].int(), n_classes, K, num_train)
    pred = classes[pred.long()]
    truth = torch.cat([train_label, eval_label])
    cells = truth * K + pred
    train_conf = torch.bincount(cells[:num_train], minlength=K * K).view(K, K)
    eval_conf = torch.bincount(cells[num_train:], minlength=K * K).view(K, K)
    nc, steps = int(n_classes), int(iters)
    train_conf, eval_conf, coef, classes = train_conf.cpu(), eval_conf.cpu(), coef.cpu(), classes.cpu()
    if steps < 0:
        warnings.warn("beta-VAE score: the logistic-regression fit did not converge in the solver's step limit; see "
                      "helpers['solver_iterations'] (-1)", RuntimeWarning)
    rows = nc if nc > 2 else nc - 1
    factors = torch.tensor(factors, dtype=torch.int64)
    helpers = {"factors": factors, "classes": factors[classes[:nc]], "coef": coef[:rows, :-1].clone(),
               "intercept": coef[:rows, -1].clone(), "solver_iterations": iters.cpu()[0], "train_confusion": train_conf,
               "eval_confusion": eval_conf}
    score = {"train_accuracy": int(train_conf.trace()) / num_train, "eval_accuracy": int(eval_conf.trace()) / num_eval}
    return score, helpers


# ---- the scores the Evaluator, training and sweeps write ----------------------------------------------------------
class Score(NamedTuple):
    """A disentanglement score the Evaluator writes beside MIG / AAM.  `flag` names its switches: the Evaluator's
    `is_{flag}` and `{flag}_seed`, and `{flag}` of training and sweeps.  Its files are `{stem}.log` and
    `{stem}_helpers.pth`, during training `epoch_score_filenames`.  `label` names it in the log.  `check(dataset,
    latent_dim)` refuses, before any GPU work, what `compute(mu, lat_sizes, seed=...)` cannot score at its default
    settings."""
    flag: str
    stem: str
    label: str
    check: Callable
    compute: Callable

    @property
    def filename(self):
        return self.stem + ".log"

    @property
    def helpers_file(self):
        return self.stem + "_helpers.pth"


SCORES = (
    Score("factor_score", "factor_vae_score", "FactorVAE score", check_factor_score, factor_vae_score),
    Score("sap_score", "sap_score", "SAP score", check_sap_score, sap_score),
    Score("beta_vae_score", "beta_vae_score", "beta-VAE score", check_beta_vae_score, beta_vae_score),
)


class Evaluator:
    def __init__(self, model, loss_f, device=torch.device("cpu"), logger=logging.getLogger(__name__),
                 save_dir="results", is_progress_bar=True):
        self.device = device
        self.loss_f = loss_f
        self.model = model.to(self.device)
        self.logger = logger
        self.save_dir = save_dir
        self.is_progress_bar = is_progress_bar
        self._perm_queue = []         # injected sample indices (parity tests), consumed FIFO by _estimate_latent_entropies
        self.logger.info("Testing Device: {}".format(self.device))

    def __call__(self, data_loader, is_metrics=False, is_losses=True, is_factor_score=False, factor_score_seed=0,
                 is_sap_score=False, sap_score_seed=0, is_beta_vae_score=False, beta_vae_score_seed=0):
        """evaluate.py:59-96.  Like the reference, the first returned value is always None (it assigns the metrics to
        a differently named variable, :77-79); the metrics are logged and written to metrics.log.
        For every entry of SCORES, `is_{flag}=True` also writes that score (`compute_factor_vae_score`,
        `compute_sap_score` or `compute_beta_vae_score` with its default settings and `seed={flag}_seed`) to
        `{stem}.log` and its tables to `{stem}_helpers.pth`: factor_vae_score, sap_score and beta_vae_score.  The
        checks of every score asked for run before any GPU work, and the dataset is encoded once for all of them."""
        args = locals()                           # the per-score keywords are is_{flag} and {flag}_seed
        scores = select_scores(args, "is_")
        start = default_timer()
        for s in scores:
            s.check(getattr(data_loader, "dataset", None), self.model.latent_dim)
        is_still_training = self.model.training
        self.model.eval()
        metric, losses = None, None
        encoded = None
        if is_metrics:
            self.logger.info('Computing metrics...')
            lat_sizes, lat_names = self._known_factors(data_loader)
            self.logger.info("Computing the empirical distribution q(z|x).")
            encoded = self._compute_q_zCx(data_loader)
            metrics = self._metrics_of(encoded, lat_sizes, lat_names)
            self.logger.info('Losses: {}'.format(metrics))
            save_metadata(metrics, self.save_dir, filename=METRICS_FILENAME)
        for s in scores:
            self.logger.info('Computing the {}...'.format(s.label))
            if encoded is None:
                encoded = self._compute_q_zCx(data_loader)
            score, helpers = s.compute(encoded[1][0], data_loader.dataset.lat_sizes, seed=args[s.flag + "_seed"])
            self.logger.info('{}: {}'.format(s.label, score))
            save_metadata(score, self.save_dir, filename=s.filename)
            torch.save(helpers, os.path.join(self.save_dir, s.helpers_file))
        if is_losses:
            self.logger.info('Computing losses...')
            losses = self.compute_losses(data_loader)
            self.logger.info('Losses: {}'.format(losses))
            save_metadata(losses, self.save_dir, filename=TEST_LOSSES_FILE)
        if is_still_training:
            self.model.train()
        self.logger.info('Finished evaluating after {:.1f} min.'.format((default_timer() - start) / 60))
        return metric, losses

    def compute_losses(self, dataloader):
        """evaluate.py:98-117, including its first-batch-only early return (trap T17)."""
        storer = defaultdict(list)
        for data, _ in tqdm(dataloader, leave=False, disable=not self.is_progress_bar):
            data = data.to(self.device)
            with torch.no_grad():
                try:
                    recon_batch, latent_dist, latent_sample = self.model(data)
                    _ = self.loss_f(data, recon_batch, latent_dist, self.model.training, storer,
                                    latent_sample=latent_sample)
                except ValueError:
                    _ = self.loss_f.call_optimize(data, self.model, None, storer)
            return {k: sum(v) / len(dataloader) for k, v in storer.items()}

    # ---- MIG / AAM (evaluate.py:119-317) ------------------------------------------------------------------
    def compute_metrics(self, dataloader):
        """evaluate.py:119-161"""
        lat_sizes, lat_names = self._known_factors(dataloader)
        self.logger.info("Computing the empirical distribution q(z|x).")
        return self._metrics_of(self._compute_q_zCx(dataloader), lat_sizes, lat_names)

    def compute_factor_vae_score(self, dataloader, batch_size=64, num_train=10000, num_eval=5000,
                                 num_variance_estimate=10000, seed=0):
        """FactorVAE score (Kim & Mnih 2018, section 4) of the model's encoder means over `dataloader` (the dataset in
        index order: DataLoader(shuffle=False) or DeviceLoader.in_order) -> {"train_accuracy", "eval_accuracy",
        "num_active_dims"}; see `factor_vae_score` for the definition and the order of the draws."""
        return self._score(check_factor_score, factor_vae_score, dataloader, seed, batch_size=batch_size,
                           num_train=num_train, num_eval=num_eval, num_variance_estimate=num_variance_estimate)

    def compute_sap_score(self, dataloader, num_train=10000, num_test=5000, C=0.01, seed=0):
        """SAP score (Kumar et al. 2018, section 3) of the model's encoder means over `dataloader` (the dataset in index
        order: DataLoader(shuffle=False) or DeviceLoader.in_order) -> {"SAP"}; see `sap_score` for the definition and
        the order of the draws."""
        return self._score(check_sap_score, sap_score, dataloader, seed, num_train=num_train, num_test=num_test, C=C)

    def compute_beta_vae_score(self, dataloader, batch_size=64, num_train=10000, num_eval=5000, seed=0):
        """beta-VAE score (Higgins et al. 2017, section 3) of the model's encoder means over `dataloader` (the dataset
        in index order: DataLoader(shuffle=False) or DeviceLoader.in_order) -> {"train_accuracy", "eval_accuracy"};
        see `beta_vae_score` for the definition and the order of the draws."""
        return self._score(check_beta_vae_score, beta_vae_score, dataloader, seed, batch_size=batch_size,
                           num_train=num_train, num_eval=num_eval)

    def _score(self, check, compute, dataloader, seed, **settings):
        """`compute(encoder means, lat_sizes, seed=seed, **settings)`'s score, after `check(dataset, latent_dim,
        **settings)` has accepted the dataset."""
        check(getattr(dataloader, "dataset", None), self.model.latent_dim, **settings)
        mean = self._compute_q_zCx(dataloader)[1][0]
        return compute(mean, dataloader.dataset.lat_sizes, seed=seed, **settings)[0]

    def _known_factors(self, dataloader):
        try:
            return dataloader.dataset.lat_sizes, dataloader.dataset.lat_names
        except AttributeError:
            raise ValueError("Dataset needs to have known true factors of variations to compute the metric. This does not "
                             "seem to be the case for {}".format(type(dataloader.__dict__["dataset"]).__name__))

    def _metrics_of(self, encoded, lat_sizes, lat_names):
        """MIG / AAM from `_compute_q_zCx`'s (samples, params)."""
        samples_zCx, params_zCx = encoded
        len_dataset, latent_dim = samples_zCx.shape

        self.logger.info("Estimating the marginal entropy.")
        H_z = self._estimate_latent_entropies(samples_zCx, params_zCx)            # H(z_j)

        samples_zCx = samples_zCx.view(*lat_sizes, latent_dim)                    # H(z_j | v_k)
        params_zCx = tuple(p.view(*lat_sizes, latent_dim) for p in params_zCx)
        H_zCv = self._estimate_H_zCv(samples_zCx, params_zCx, lat_sizes, lat_names)

        H_z = H_z.cpu()
        H_zCv = H_zCv.cpu()
        mut_info = - H_zCv + H_z                                                  # I[z_j; v_k] = H[z_j] - H[z_j | v_k]
        sorted_mut_info = torch.sort(mut_info, dim=1, descending=True)[0].clamp(min=0)

        metric_helpers = {'marginal_entropies': H_z, 'cond_entropies': H_zCv}
        mig = self._mutual_information_gap(sorted_mut_info, lat_sizes, storer=metric_helpers)
        aam = self._axis_aligned_metric(sorted_mut_info, storer=metric_helpers)
        metrics = {'MIG': mig.item(), 'AAM': aam.item()}
        torch.save(metric_helpers, os.path.join(self.save_dir, METRIC_HELPERS_FILE))
        return metrics

    def _mutual_information_gap(self, sorted_mut_info, lat_sizes, storer=None):
        """evaluate.py:163-185 (H(v_k) = log |V_k|: balanced factors)."""
        delta_mut_info = sorted_mut_info[:, 0] - sorted_mut_info[:, 1]
        H_v = torch.as_tensor(lat_sizes).float().log()
        mig_k = delta_mut_info / H_v
        mig = mig_k.mean()
        if storer is not None:
            storer["mig_k"] = mig_k
            storer["mig"] = mig
        return mig

    def _axis_aligned_metric(self, sorted_mut_info, storer=None):
        """evaluate.py:187-198"""
        numerator = (sorted_mut_info[:, 0] - sorted_mut_info[:, 1:].sum(dim=1)).clamp(min=0)
        aam_k = numerator / sorted_mut_info[:, 0]
        aam_k[torch.isnan(aam_k)] = 0
        aam = aam_k.mean()
        if storer is not None:
            storer["aam_k"] = aam_k
            storer["aam"] = aam
        return aam

    def _compute_q_zCx(self, dataloader):
        """evaluate.py:200-231: (mean, logvar) of every example through the encoder (CUDA path), one 'sample' per
        example -- in eval mode reparameterize returns the mean (vae.py:69-71)."""
        len_dataset = len(dataloader.dataset)
        latent_dim = self.model.latent_dim
        q_zCx = torch.zeros(len_dataset, latent_dim, 2, device=self.device)
        n = 0
        with torch.no_grad():
            for x, label in dataloader:
                batch_size = x.size(0)
                idcs = slice(n, n + batch_size)
                q_zCx[idcs, :, 0], q_zCx[idcs, :, 1] = self.model.encoder(x.to(self.device))
                n += batch_size
            params_zCX = q_zCx.unbind(-1)
            samples_zCx = self.model.reparameterize(*params_zCX)
        return samples_zCx, params_zCX

    def _estimate_latent_entropies(self, samples_zCx, params_zCX, n_samples=10000):
        """evaluate.py:233-297 -> H_z [latent_dim].

        Kept on purpose: the reference draws `n_samples` example indices and then RESHAPES (not transposes) the
        selected [n_samples, latent_dim] block to [latent_dim, n_samples] (:270) -- row j of that view is a contiguous
        run of the flattened block, so "the samples of dimension j" mix all dimensions.  The kernel receives exactly that
        view.  Like the reference this needs len_dataset >= n_samples."""
        len_dataset, latent_dim = samples_zCx.shape
        device = samples_zCx.device
        if self._perm_queue:
            samples_x = self._perm_queue.pop(0).to(device)[:n_samples]
        else:
            samples_x = torch.randperm(len_dataset, device=device)[:n_samples]
        zs = samples_zCx.index_select(0, samples_x).view(latent_dim, n_samples).contiguous()
        mean, log_var = params_zCX
        N.require_cuda_f32(zs, mean, log_var)
        if mean.stride() != log_var.stride():
            mean, log_var = mean.contiguous(), log_var.contiguous()
        L = N.lib()
        ws = torch.empty((L.dv_latent_entropy_workspace_bytes(len_dataset, latent_dim, n_samples) + 3) // 4,
                         dtype=torch.float32, device=device)
        H_z = torch.empty(latent_dim, dtype=torch.float32, device=device)
        N.call("dv_latent_entropy", N.ptr(zs), N.ptr(mean), N.ptr(log_var), mean.stride(1), mean.stride(0), len_dataset,
               latent_dim, n_samples, N.ptr(H_z), None, N.ptr(ws), N.stream())
        return H_z

    def _estimate_H_zCv(self, samples_zCx, params_zCx, lat_sizes, lat_names):
        """evaluate.py:299-317: H[z_j | v_k] = mean over the values of factor k of the entropy within that slice."""
        latent_dim = samples_zCx.size(-1)
        len_dataset = reduce((lambda x, y: x * y), lat_sizes)
        H_zCv = torch.zeros(len(lat_sizes), latent_dim, device=self.device)
        for i_fac_var, (lat_size, lat_name) in enumerate(zip(lat_sizes, lat_names)):
            idcs = [slice(None)] * len(lat_sizes)
            for i in range(lat_size):
                self.logger.info("Estimating conditional entropies for the {}th value of {}.".format(i, lat_name))
                idcs[i_fac_var] = i
                samples_zxCv = samples_zCx[tuple(idcs)].contiguous().view(len_dataset // lat_size, latent_dim)
                params_zxCv = tuple(p[tuple(idcs)].contiguous().view(len_dataset // lat_size, latent_dim)
                                    for p in params_zCx)
                H_zCv[i_fac_var] += self._estimate_latent_entropies(samples_zxCv, params_zxCv) / lat_size
        return H_zCv
