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

import numpy as np
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
DCI_MAX_DIM = 1024                         # dv_dci_fit's limits: latents,
DCI_MAX_TRAIN = 32768                      # training rows,
DCI_MAX_CLASSES = 256                      # and values of a scored factor
DCI_STAGES = 100                           # GradientBoostingClassifier()'s n_estimators
MODULARITY_MAX_DIM = 128                   # dv_explicitness_fit's limits: latents,
MODULARITY_MAX_TRAIN = 32768               # training rows,
MODULARITY_MAX_CLASSES = 256               # and values of a scored factor
MODULARITY_BINS = 20                       # disentanglement_lib's num_bins of the mutual information
DOWNSTREAM_PREDICTORS = ("logistic_regression", "boosted_trees")
DOWNSTREAM_MAX_DIM = 128                   # dv_downstream_logistic_cv's limits: latents,
DOWNSTREAM_MIN_TRAIN = 5                   # training rows of a size (every fold holds one),
DOWNSTREAM_MAX_TRAIN = 32768
DOWNSTREAM_MAX_CLASSES = 256               # and values of a scored factor
DOWNSTREAM_CS = np.logspace(-4, 4, 10)     # LogisticRegressionCV(Cs=10)'s grid, numpy's bits
DOWNSTREAM_FOLDS = 5                       # KFold(n_splits=5)
IRS_MAX_DIM = 1024                         # dv_irs_fit's limits: latents,
IRS_MAX_TRAIN = 32768                      # and drawn rows (one latent's sort in shared memory)
IRS_BINS = 20                              # disentanglement_lib's make_discretizer of the factors
UDR_MAX_DIM = 128                          # dv_udr_fit's limits: latents of a model,
UDR_MAX_COLUMNS = 4096                     # models x latents,
UDR_MAX_POINTS = 16384                     # and points
UDR_CORRELATIONS = {"lasso": 0, "spearman": 1}   # UDR_L and UDR_S: dv_udr_fit's modes
UDR_LASSO_ALPHA = 0.1                      # udr.py's Lasso(alpha=0.1)
UDR_KL_THRESHOLD = 0.01                    # a latent is informative when its mean KL is above this
UDR_ENCODE_BATCH = 1000                    # points per encoder call
UDR_FILENAME = "udr.log"
UDR_HELPERS_FILE = "udr_helpers.pth"
UNSUPERVISED_MAX_DIM = 128                 # dv_unsupervised_fit's limits: latents (the Jacobi matrix in shared memory),
UNSUPERVISED_MAX_POINTS = 32768            # and drawn points (dv_discrete_mutual_info's)
UNSUPERVISED_REPRESENTATIONS = ("mean", "sampled")
UNSUPERVISED_DBL_EPSILON = 2.0 ** -52
UNSUPERVISED_FILENAME = "unsupervised_scores.log"
UNSUPERVISED_HELPERS_FILE = "unsupervised_scores_helpers.pth"
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


# ---- what every wrapper of a score kernel checks and passes -------------------------------------------------------
def _mu_args(mu):
    """`mu` [N, D] (CUDA fp32, any strides, a view of q_zCx included) as the score kernels take it: (ptr, ld,
    row_stride, N, D), with latent d of row i at ptr[i * row_stride + d * ld]."""
    N.require_cuda_f32(mu)
    n, d = mu.shape
    return N.ptr(mu), mu.stride(1), mu.stride(0), n, d


def _require_operands(fn, optional=False, **operands):
    """ValueError `{fn}: {name} must be a contiguous CUDA {dtype} tensor[ of shape {shape}]` unless every operand
    name=(tensor, dtype[, shape]) is one; with `optional`, a None tensor passes."""
    for name, (t, dtype, *shape) in operands.items():
        if t is None and optional:
            continue
        if t.dtype != dtype or not t.is_contiguous() or not t.is_cuda or (shape and tuple(t.shape) != shape[0]):
            raise ValueError("%s: %s must be a contiguous CUDA %s tensor%s"
                             % (fn, name, dtype, " of shape %s" % (shape[0],) if shape else ""))


def _f64_workspace(nbytes, device):
    """A kernel workspace of at least `nbytes` bytes (8-byte aligned, never empty)."""
    return torch.empty(max(nbytes, 8) // 8, dtype=torch.float64, device=device)


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
    mu_args, d = _mu_args(mu), mu.shape[1]
    V, L = rows.shape
    if rows.dtype != torch.int64 or not rows.is_contiguous():
        raise ValueError("group_variance: rows must be a contiguous int64 tensor")
    _require_operands("group_variance", var_out=(var_out, torch.float32, (V, d)),
                      argmin_out=(argmin_out, torch.int32, (V,)), global_var=(global_var, torch.float32, (d,)),
                      optional=True)
    N.call("dv_group_variance", *mu_args, N.ptr(rows), V, L, N.ptr(global_var), FACTOR_SCORE_MIN_VAR, N.ptr(var_out),
           N.ptr(argmin_out), N.stream())


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


def _train_rows(mu, num_train, seed):
    """(generator, rows): a device torch.Generator seeded with `seed` and its first draw, `torch.randint(N,
    (num_train,))`, for `mu` [N, D] (CUDA fp32).  The global generators are not touched."""
    N.require_cuda_f32(mu)
    gen = torch.Generator(device=mu.device)
    gen.manual_seed(int(seed))
    return gen, torch.randint(mu.shape[0], (int(num_train),), generator=gen, device=mu.device)


def _sap_draws(mu, lat_sizes, num_train, num_test, seed):
    """The rows of the SAP, DCI, modularity and explicitness scores of `mu` [N, D] (CUDA fp32) -> (train_rows,
    test_rows) + `sap_labels`' tuple.  They come from a device torch.Generator seeded with `seed`: `torch.randint(N,
    (num_train,))`, then `torch.randint(N, (num_test,))`; the global generators are not touched."""
    gen, train_rows = _train_rows(mu, num_train, seed)
    test_rows = torch.randint(mu.shape[0], (int(num_test),), generator=gen, device=mu.device)
    return (train_rows, test_rows) + sap_labels(lat_sizes, train_rows, test_rows)


def _classes_table(present):
    """`sap_labels`' `present` [K', S] (host) as the helpers' "classes" int64 [K', S]: the values seen, -1 beyond."""
    K, S = present.shape
    classes = torch.sort(torch.where(present, torch.arange(S).expand(K, S), S), dim=1)[0]   # the values seen, then S
    return torch.where(classes < S, classes, -1)


def sap_score_matrix(mu, train_rows, test_rows, train_cls, test_cls, n_classes, counts, C, coef=None, iters=None):
    """`dv_sap_score_matrix` on `mu` [N, D] (any strides, a view of q_zCx included) -> the fp32 score [D, K'] of
    `sap_labels`' classes; optionally the fitted lines into fp64 `coef` [D, K', S, 2] and the Newton steps into int32
    `iters` [D, K', S]."""
    mu_args, d = _mu_args(mu), mu.shape[1]
    K, S = counts.shape
    _require_operands("sap_score_matrix", train_rows=(train_rows, torch.int64), test_rows=(test_rows, torch.int64),
                      train_cls=(train_cls, torch.int32), test_cls=(test_cls, torch.int32),
                      n_classes=(n_classes, torch.int32), counts=(counts, torch.int32), coef=(coef, torch.float64),
                      iters=(iters, torch.int32), optional=True)
    score = torch.empty(d, K, dtype=torch.float32, device=mu.device)
    N.call("dv_sap_score_matrix", *mu_args, N.ptr(train_rows), train_rows.numel(), N.ptr(test_rows), test_rows.numel(),
           N.ptr(train_cls), N.ptr(test_cls), N.ptr(n_classes), N.ptr(counts), K, S, float(C), N.ptr(score),
           N.ptr(coef), N.ptr(iters), N.stream())
    return score


def sap_from_matrix(score_matrix):
    """SAP of a score matrix [D, K'] (D >= 2): the mean over factors of the largest minus the second largest score of
    the factor's column, in fp64."""
    m = torch.sort(score_matrix.double().cpu(), dim=0, descending=True)[0]
    return float((m[0] - m[1]).mean())


def sap_score(mu, lat_sizes, num_train=10000, num_test=5000, C=0.01, seed=0):
    """SAP score of the encoder means `mu` [N, D] (CUDA fp32, dataset index order) of the full factor grid `lat_sizes`
    -> ({"SAP"}, helpers).  The rows and their classes are `_sap_draws`' (seeded with `seed`).  For every latent and
    scored factor `dv_sap_score_matrix` fits LinearSVC(C, class_weight="balanced") exactly and scores it on the test
    rows; SAP is `sap_from_matrix` of that table.
    helpers: "score_matrix" fp32 [D, K'], "factors" (the scored factor indices, ascending), "classes" int64 [K', S]
    (each factor's training values, ascending, -1 beyond), "coef" fp64 [D, K', S, 2] (w, b of each problem: class c's
    one-vs-rest problem in slot c, the two-class problem in slot 0, NaN beyond) and "solver_iterations" int32
    [D, K', S] (Newton steps, -1 for a fit that did not converge, which also raises a RuntimeWarning)."""
    lat_sizes = _check_sap_grid(lat_sizes, mu.shape[0], mu.shape[1], num_train, num_test, C)
    D = mu.shape[1]
    train_rows, test_rows, factors, train_cls, test_cls, n_classes, counts, present = _sap_draws(
        mu, lat_sizes, num_train, num_test, seed)
    K, S = counts.shape
    coef = torch.empty(D, K, S, 2, dtype=torch.float64, device=mu.device)
    iters = torch.empty(D, K, S, dtype=torch.int32, device=mu.device)
    matrix = sap_score_matrix(mu, train_rows, test_rows, train_cls, test_cls, n_classes, counts, C, coef, iters)
    matrix, coef, iters, present = matrix.cpu(), coef.cpu(), iters.cpu(), present.cpu()
    failed = int((iters < 0).sum())
    if failed:
        warnings.warn("SAP score: %d of the linear-SVM fits did not converge in the solver's step limit; see "
                      "helpers['solver_iterations'] (-1)" % failed, RuntimeWarning)
    helpers = {"score_matrix": matrix, "factors": torch.tensor(factors, dtype=torch.int64),
               "classes": _classes_table(present), "coef": coef, "solver_iterations": iters}
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
    mu_args, d = _mu_args(mu), mu.shape[1]
    V, L = rows_a.shape
    for name, t in (("rows_a", rows_a), ("rows_b", rows_b)):
        if t.dtype != torch.int64 or not t.is_contiguous() or t.shape != (V, L):
            raise ValueError("pair_abs_diff_mean: %s must be a contiguous int64 tensor of shape %s" % (name, (V, L)))
    x = torch.empty(V, d, dtype=torch.float64, device=mu.device)
    N.call("dv_pair_abs_diff_mean", *mu_args, N.ptr(rows_a), N.ptr(rows_b), V, L, N.ptr(x), N.stream())
    return x


def logistic_fit(x, labels, n_classes, K, num_train):
    """`dv_logistic_fit` on fp64 features `x` [V, D] (the first `num_train` rows train) with int32 class indices
    `labels` [num_train] and the class count in int32 `n_classes` [1] on the device -> (coef fp64 [K, D + 1], pred
    int32 [V], iters int32 [1]); see include/disvae_b200.h for the objective and the layout of coef."""
    V, D = x.shape
    _require_operands("logistic_fit", x=(x, torch.float64), labels=(labels, torch.int32),
                      n_classes=(n_classes, torch.int32))
    nbytes = N.lib().dv_logistic_fit_workspace_bytes(int(num_train), D, int(K))
    ws = _f64_workspace(nbytes, x.device)
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


# ---- DCI score (Eastwood & Williams 2018; disentanglement_lib's dci.py with GradientBoostingClassifier()) ----------
def check_dci_score(dataset, latent_dim, num_train=10000, num_test=5000):
    """ValueError unless the DCI score can be computed over `dataset` for a `latent_dim` model with these settings: the
    dataset has known factors (`lat_sizes`, `lat_names`), is their full grid and has at least 2 factors of more than
    one value.  No GPU work.  Returns lat_sizes as a list of ints."""
    return _check_dci_grid(_dataset_lat_sizes("DCI score", dataset), len(dataset), latent_dim, num_train, num_test)


def _check_dci_grid(lat_sizes, n, latent_dim, num_train, num_test):
    lat_sizes = _full_grid("DCI score", lat_sizes, n)
    scored = sum(s > 1 for s in lat_sizes)
    if scored < 2:
        raise ValueError("DCI score: %s has %d factors of more than one value; completeness is an entropy over the "
                         "factors and needs at least 2" % (lat_sizes, scored))
    if max(lat_sizes) > DCI_MAX_CLASSES:
        raise ValueError("DCI score: a factor of %s has more than the kernel's limit of %d values"
                         % (lat_sizes, DCI_MAX_CLASSES))
    if int(latent_dim) < 2:
        raise ValueError("DCI score: latent_dim must be at least 2 (disentanglement is an entropy over the latents), "
                         "got %d" % int(latent_dim))
    if int(latent_dim) > DCI_MAX_DIM:
        raise ValueError("DCI score: latent_dim %d is above the kernel's limit of %d" % (int(latent_dim), DCI_MAX_DIM))
    if int(num_train) < 1:
        raise ValueError("DCI score: num_train must be at least 1, got %d" % int(num_train))
    if int(num_train) > DCI_MAX_TRAIN:
        raise ValueError("DCI score: num_train %d is above the kernel's limit of %d" % (int(num_train), DCI_MAX_TRAIN))
    if int(num_test) < 1:
        raise ValueError("DCI score: num_test must be at least 1, got %d" % int(num_test))
    return lat_sizes


def dci_fit(mu, train_rows, test_rows, train_cls, n_classes, counts, stages=DCI_STAGES, trees=False):
    """`dv_dci_fit` on `mu` [N, D] (any strides, a view of q_zCx included) and `sap_labels`' classes -> (importance
    fp64 [D, K'], pred int32 [K', num_train + num_test] (class indices), trees), trees = None or (feature int32,
    threshold fp64, value fp64), each [K', S, stages, 15]; see include/disvae_b200.h for the fit."""
    mu_args, d = _mu_args(mu), mu.shape[1]
    K, S = counts.shape
    _require_operands("dci_fit", train_rows=(train_rows, torch.int64), test_rows=(test_rows, torch.int64),
                      train_cls=(train_cls, torch.int32), n_classes=(n_classes, torch.int32),
                      counts=(counts, torch.int32))
    num_train, num_test = train_rows.numel(), test_rows.numel()
    nbytes = N.lib().dv_dci_workspace_bytes(d, num_train, num_test, K, S)
    ws = _f64_workspace(nbytes, mu.device)
    importance = torch.empty(d, K, dtype=torch.float64, device=mu.device)
    pred = torch.empty(K, num_train + num_test, dtype=torch.int32, device=mu.device)
    out = None
    if trees:
        shape = (K, S, int(stages), 15)
        out = (torch.empty(shape, dtype=torch.int32, device=mu.device),
               torch.empty(shape, dtype=torch.float64, device=mu.device),
               torch.empty(shape, dtype=torch.float64, device=mu.device))
    N.call("dv_dci_fit", *mu_args, N.ptr(train_rows), num_train, N.ptr(test_rows), num_test, N.ptr(train_cls),
           N.ptr(n_classes), N.ptr(counts), K, S, int(stages), N.ptr(importance), N.ptr(pred),
           *(N.ptr(t) for t in (out or (None, None, None))), N.ptr(ws), nbytes, N.stream())
    return importance, pred, out


def _entropy(p, base):
    """scipy.stats.entropy(p, base=base) along axis 0 of a non-negative fp64 array."""
    p = p / p.sum(0)
    return -torch.where(p > 0, p * torch.log(p), torch.zeros_like(p)).sum(0) / math.log(base)


def dci_from_importance(importance):
    """(disentanglement, completeness) of an importance matrix R [D, K'] (D, K' >= 2), as dci.py computes them in
    fp64: disentanglement = sum_d rho_d (1 - H_K'(R[d, :] + 1e-11)), completeness = sum_k rho_k (1 - H_D(R[:, k] +
    1e-11)), rho the row (column) sums over the total, of a matrix of ones when R sums to 0."""
    R = importance.double().cpu()
    D, K = R.shape
    per_code = 1.0 - _entropy(R.t() + 1e-11, K)
    per_factor = 1.0 - _entropy(R + 1e-11, D)
    W = torch.ones_like(R) if float(R.sum()) == 0.0 else R
    return (float((per_code * (W.sum(1) / W.sum())).sum()), float((per_factor * (W.sum(0) / W.sum())).sum()))


def dci_score(mu, lat_sizes, num_train=10000, num_test=5000, seed=0):
    """DCI score of the encoder means `mu` [N, D] (CUDA fp32, dataset index order) of the full factor grid `lat_sizes`
    -> ({"disentanglement", "completeness", "informativeness_train", "informativeness_test"}, helpers).  The rows and
    their classes are `_sap_draws`' (seeded with `seed`), as SAP's are.  For every scored factor `dci_fit` grows
    GradientBoostingClassifier()'s 100 boosting stages on the training rows; a factor seen with one value in training
    has no trees, zero importance and predicts that value.  The informativeness scores are the mean accuracies over the
    factors (a test value unseen in training is never predicted right).
    helpers: "importance_matrix" fp64 [D, K'], "factors" (the scored factor indices, ascending), "classes" int64
    [K', S] (each factor's training values, ascending, -1 beyond), "train_accuracy" and "test_accuracy" fp64 [K']."""
    lat_sizes = _check_dci_grid(lat_sizes, mu.shape[0], mu.shape[1], num_train, num_test)
    num_train = int(num_train)
    train_rows, test_rows, factors, train_cls, test_cls, n_classes, counts, present = _sap_draws(
        mu, lat_sizes, num_train, num_test, seed)
    importance, pred, _ = dci_fit(mu, train_rows, test_rows, train_cls, n_classes, counts)
    right = pred == torch.cat([train_cls, test_cls], 1)
    train_acc = right[:, :num_train].double().mean(1).cpu()
    test_acc = right[:, num_train:].double().mean(1).cpu()
    importance, present = importance.cpu(), present.cpu()
    disentanglement, completeness = dci_from_importance(importance)
    helpers = {"importance_matrix": importance, "factors": torch.tensor(factors, dtype=torch.int64),
               "classes": _classes_table(present), "train_accuracy": train_acc, "test_accuracy": test_acc}
    score = {"disentanglement": disentanglement, "completeness": completeness,
             "informativeness_train": float(train_acc.mean()), "informativeness_test": float(test_acc.mean())}
    return score, helpers


# ---- modularity and explicitness (Ridgeway & Zemel 2018; disentanglement_lib's modularity_explicitness.py) --------
def check_modularity_explicitness(dataset, latent_dim, num_train=10000, num_test=5000):
    """ValueError unless modularity and explicitness can be computed over `dataset` for a `latent_dim` model with these
    settings: the dataset has known factors (`lat_sizes`, `lat_names`), is their full grid and has at least 2 factors
    of more than one value.  No GPU work.  Returns lat_sizes as a list of ints."""
    return _check_modularity_grid(_dataset_lat_sizes("modularity score", dataset), len(dataset), latent_dim, num_train,
                                  num_test)


def _check_modularity_grid(lat_sizes, n, latent_dim, num_train, num_test):
    lat_sizes = _full_grid("modularity score", lat_sizes, n)
    scored = sum(s > 1 for s in lat_sizes)
    if scored < 2:
        raise ValueError("modularity score: %s has %d factors of more than one value; modularity divides by the "
                         "factors less one and needs at least 2" % (lat_sizes, scored))
    if max(lat_sizes) > MODULARITY_MAX_CLASSES:
        raise ValueError("modularity score: a factor of %s has more than the kernel's limit of %d values"
                         % (lat_sizes, MODULARITY_MAX_CLASSES))
    if not 1 <= int(latent_dim) <= MODULARITY_MAX_DIM:
        raise ValueError("modularity score: latent_dim must be in [1, %d], got %d" % (MODULARITY_MAX_DIM,
                                                                                      int(latent_dim)))
    if not 1 <= int(num_train) <= MODULARITY_MAX_TRAIN:
        raise ValueError("modularity score: num_train must be in [1, %d], got %d" % (MODULARITY_MAX_TRAIN,
                                                                                     int(num_train)))
    if int(num_test) < 1:
        raise ValueError("modularity score: num_test must be at least 1, got %d" % int(num_test))
    return lat_sizes


def discrete_mutual_info(mu, train_rows, train_cls, n_classes, class_stride):
    """`dv_discrete_mutual_info` on `mu` [N, D] (any strides, a view of q_zCx included) and `sap_labels`' training
    classes -> (mi fp64 [D, K'], edges fp32 [D, 21]): sklearn's mutual_info_score of every factor's classes with every
    latent's 20-bin histogram discretisation over the training rows; see include/disvae_b200.h for the rules."""
    mu_args, d = _mu_args(mu), mu.shape[1]
    _require_operands("discrete_mutual_info", train_rows=(train_rows, torch.int64), train_cls=(train_cls, torch.int32),
                      n_classes=(n_classes, torch.int32))
    K = n_classes.numel()
    mi = torch.empty(d, K, dtype=torch.float64, device=mu.device)
    edges = torch.empty(d, MODULARITY_BINS + 1, dtype=torch.float32, device=mu.device)
    N.call("dv_discrete_mutual_info", *mu_args, N.ptr(train_rows), train_rows.numel(), N.ptr(train_cls),
           N.ptr(n_classes), K, int(class_stride), N.ptr(mi), N.ptr(edges), N.stream())
    return mi, edges


def explicitness_fit(mu, train_rows, test_rows, train_cls, test_cls, n_classes, class_stride, proba=False):
    """`dv_explicitness_fit` on `mu` [N, D] (any strides) and `sap_labels`' classes -> (coef fp64 [K', S, D + 1], auc
    fp64 [2, K', S] (training, test), iters int32 [K'], mean fp64 [D], std fp64 [D], proba): LogisticRegression(C=1)
    of every factor on the standardised latents and the ROC AUC of each class column; proba is None or fp64
    [K', S, num_train + num_test].  See include/disvae_b200.h for the rules."""
    mu_args, d = _mu_args(mu), mu.shape[1]
    _require_operands("explicitness_fit", train_rows=(train_rows, torch.int64), test_rows=(test_rows, torch.int64),
                      train_cls=(train_cls, torch.int32), test_cls=(test_cls, torch.int32),
                      n_classes=(n_classes, torch.int32))
    K, S = n_classes.numel(), int(class_stride)
    num_train, num_test = train_rows.numel(), test_rows.numel()
    nbytes = N.lib().dv_explicitness_workspace_bytes(d, num_train, num_test, K, S)
    ws = _f64_workspace(nbytes, mu.device)
    f64 = dict(dtype=torch.float64, device=mu.device)
    coef, auc = torch.empty(K, S, d + 1, **f64), torch.empty(2, K, S, **f64)
    iters = torch.empty(K, dtype=torch.int32, device=mu.device)
    mean, std = torch.empty(d, **f64), torch.empty(d, **f64)
    out = torch.empty(K, S, num_train + num_test, **f64) if proba else None
    N.call("dv_explicitness_fit", *mu_args, N.ptr(train_rows), num_train, N.ptr(test_rows), num_test, N.ptr(train_cls),
           N.ptr(test_cls), N.ptr(n_classes), K, S, N.ptr(coef), N.ptr(auc), N.ptr(iters), N.ptr(mean), N.ptr(std),
           N.ptr(out), N.ptr(ws), nbytes, N.stream())
    return coef, auc, iters, mean, std, out


def modularity_from_mutual_info(mi):
    """(modularity score, per-latent scores [D]) of a mutual-information matrix [D, K'] (K' >= 2), as
    modularity_explicitness.py's modularity() computes them in fp64: with m = max_k mi^2, a latent scores
    1 - (sum_k mi^2 - m) / (m (K' - 1)), or 0 where m = 0; the score is the mean over the latents."""
    sq = mi.double().cpu() ** 2
    m = sq.max(1)[0]
    delta = (sq.sum(1) - m) / (m * (sq.shape[1] - 1.0))
    per_latent = torch.where(m == 0, torch.zeros_like(m), 1.0 - delta)
    return float(per_latent.mean()), per_latent


def _explicitness_of(auc):
    """Mean AUC over the defined columns of every factor [K', S] -> [K'] (NaN for a factor without one)."""
    defined = ~torch.isnan(auc)
    count = defined.sum(1)
    total = torch.where(defined, auc, torch.zeros_like(auc)).sum(1)
    return torch.where(count > 0, total / count.clamp(min=1), torch.full_like(total, float("nan")))


def modularity_explicitness(mu, lat_sizes, num_train=10000, num_test=5000, seed=0):
    """Modularity and explicitness of the encoder means `mu` [N, D] (CUDA fp32, dataset index order) of the full factor
    grid `lat_sizes` -> ({"modularity_score", "explicitness_score_train", "explicitness_score_test"}, helpers).  The
    rows and their classes are `_sap_draws`' (seeded with `seed`), as SAP's are.  Modularity is
    `modularity_from_mutual_info` of `discrete_mutual_info` over the training rows.  Explicitness: `explicitness_fit`
    fits LogisticRegression(C=1) per scored factor on the standardised latents; a factor's value on a set is the mean
    ROC AUC over its class columns that have positives and negatives there, NaN for a factor of one training class or
    without such a column; each score is the mean over the factors with a value (NaN, with a RuntimeWarning, when none
    has one).
    helpers: "mutual_information" fp64 [D, K'], "bin_edges" fp32 [D, 21], "modularity_per_latent" fp64 [D],
    "factors" (the scored factor indices, ascending), "classes" int64 [K', S] (each factor's training values,
    ascending, -1 beyond), "feature_mean" and "feature_std" fp64 [D], "coef" fp64 [K', S, D + 1] (model rows in
    standardised features, NaN beyond), "train_auc" and "test_auc" fp64 [K', S] (NaN where undefined),
    "explicitness_train" and "explicitness_test" fp64 [K'], "solver_iterations" int32 [K'] (Newton steps, -1 for a
    fit that did not converge, which also raises a RuntimeWarning)."""
    lat_sizes = _check_modularity_grid(lat_sizes, mu.shape[0], mu.shape[1], num_train, num_test)
    train_rows, test_rows, factors, train_cls, test_cls, n_classes, counts, present = _sap_draws(
        mu, lat_sizes, num_train, num_test, seed)
    S = counts.shape[1]
    mi, edges = discrete_mutual_info(mu, train_rows, train_cls, n_classes, S)
    coef, auc, iters, mean, std, _ = explicitness_fit(mu, train_rows, test_rows, train_cls, test_cls, n_classes, S)
    mi, edges, coef, auc, iters = mi.cpu(), edges.cpu(), coef.cpu(), auc.cpu(), iters.cpu()
    mean, std, present = mean.cpu(), std.cpu(), present.cpu()
    modularity, per_latent = modularity_from_mutual_info(mi)
    failed = int((iters < 0).sum())
    if failed:
        warnings.warn("modularity score: %d of the logistic-regression fits did not converge in the solver's step "
                      "limit; see helpers['solver_iterations'] (-1)" % failed, RuntimeWarning)
    explicit = [_explicitness_of(auc[s]) for s in (0, 1)]
    score = {"modularity_score": modularity}
    for name, e in zip(("explicitness_score_train", "explicitness_score_test"), explicit):
        valued = e[~torch.isnan(e)]
        if valued.numel() == 0:
            warnings.warn("modularity score: no factor has an explicitness value on the %s rows; %s is NaN"
                          % (name.split("_")[-1], name), RuntimeWarning)
        score[name] = float(valued.mean()) if valued.numel() else float("nan")
    helpers = {"mutual_information": mi, "bin_edges": edges, "modularity_per_latent": per_latent,
               "factors": torch.tensor(factors, dtype=torch.int64), "classes": _classes_table(present),
               "feature_mean": mean, "feature_std": std, "coef": coef, "train_auc": auc[0].clone(),
               "test_auc": auc[1].clone(), "explicitness_train": explicit[0], "explicitness_test": explicit[1],
               "solver_iterations": iters}
    return score, helpers


# ---- downstream task (Locatello et al. 2019, section 6; disentanglement_lib's downstream_task.py) ------------------
def check_downstream_task(dataset, latent_dim, predictor="logistic_regression", num_train=(10, 100, 1000, 10000),
                          num_test=5000):
    """ValueError unless the downstream-task score can be computed over `dataset` for a `latent_dim` model with these
    settings: the dataset has known factors (`lat_sizes`, `lat_names`), is their full grid and has a factor of more
    than one value.  No GPU work.  Returns lat_sizes as a list of ints."""
    return _check_downstream_grid(_dataset_lat_sizes("downstream task", dataset), len(dataset), latent_dim, predictor,
                                  num_train, num_test)


def _check_downstream_grid(lat_sizes, n, latent_dim, predictor, num_train, num_test):
    lat_sizes = _full_grid("downstream task", lat_sizes, n)
    if all(s == 1 for s in lat_sizes):
        raise ValueError("downstream task: every factor of %s has one value; there is nothing to predict" % lat_sizes)
    if predictor not in DOWNSTREAM_PREDICTORS:
        raise ValueError("downstream task: predictor must be one of %s, got %r" % (DOWNSTREAM_PREDICTORS, predictor))
    limit = DOWNSTREAM_MAX_CLASSES if predictor == "logistic_regression" else DCI_MAX_CLASSES
    if max(lat_sizes) > limit:
        raise ValueError("downstream task: a factor of %s has more than the kernel's limit of %d values"
                         % (lat_sizes, limit))
    limit = DOWNSTREAM_MAX_DIM if predictor == "logistic_regression" else DCI_MAX_DIM
    if not 1 <= int(latent_dim) <= limit:
        raise ValueError("downstream task: latent_dim must be in [1, %d] for the %s predictor, got %d"
                         % (limit, predictor, int(latent_dim)))
    sizes = [num_train] if isinstance(num_train, int) else list(num_train)
    if not sizes:
        raise ValueError("downstream task: num_train must name at least one training size")
    for size in sizes:
        if not DOWNSTREAM_MIN_TRAIN <= int(size) <= DOWNSTREAM_MAX_TRAIN:
            raise ValueError("downstream task: every num_train must be in [%d, %d] (5 folds of at least one row), got "
                             "%d" % (DOWNSTREAM_MIN_TRAIN, DOWNSTREAM_MAX_TRAIN, int(size)))
    if int(num_test) < 1:
        raise ValueError("downstream task: num_test must be at least 1, got %d" % int(num_test))
    return lat_sizes


def downstream_logistic_cv(mu, train_rows, test_rows, train_cls, n_classes, class_stride, Cs=DOWNSTREAM_CS,
                           folds=False):
    """`dv_downstream_logistic_cv` on `mu` [N, D] (any strides, a view of q_zCx included) and `sap_labels`' training
    classes -> (fold_acc fp64 [K', 5, nC], chosen int32 [K'], coef fp64 [K', S, D + 1], pred int32 [K', num_train +
    num_test], iters int32 [K', 5 nC + 1], fold_coef, fold_pred): LogisticRegressionCV(Cs, cv=KFold(5)) of every factor
    on the raw latents.  With `folds`, fold_coef fp64 [K', 5, nC, S, D + 1] and fold_pred int32 [K', nC, num_train]
    hold every fold fit and its predictions, else they are None.  See include/disvae_b200.h for the rules."""
    mu_args, d = _mu_args(mu), mu.shape[1]
    _require_operands("downstream_logistic_cv", train_rows=(train_rows, torch.int64),
                      test_rows=(test_rows, torch.int64), train_cls=(train_cls, torch.int32),
                      n_classes=(n_classes, torch.int32))
    K, S = n_classes.numel(), int(class_stride)
    Cs = np.ascontiguousarray(Cs, dtype=np.float64)
    nC = Cs.size
    num_train, num_test = train_rows.numel(), test_rows.numel()
    nbytes = N.lib().dv_downstream_workspace_bytes(d, num_train, K, S, nC)
    ws = _f64_workspace(nbytes, mu.device)
    f64 = dict(dtype=torch.float64, device=mu.device)
    i32 = dict(dtype=torch.int32, device=mu.device)
    out = (torch.empty(K, DOWNSTREAM_FOLDS, nC, **f64), torch.empty(K, **i32), torch.empty(K, S, d + 1, **f64),
           torch.empty(K, num_train + num_test, **i32), torch.empty(K, DOWNSTREAM_FOLDS * nC + 1, **i32))
    fold = ((torch.empty(K, DOWNSTREAM_FOLDS, nC, S, d + 1, **f64), torch.empty(K, nC, num_train, **i32)) if folds
            else (None, None))
    N.call("dv_downstream_logistic_cv", *mu_args, N.ptr(train_rows), num_train, N.ptr(test_rows), num_test,
           N.ptr(train_cls), N.ptr(n_classes), K, S, Cs.ctypes.data, nC, *(N.ptr(t) for t in out + fold), N.ptr(ws),
           nbytes, N.stream())
    return out + fold


def downstream_task(mu, lat_sizes, predictor="logistic_regression", num_train=(10, 100, 1000, 10000), num_test=5000,
                    seed=0):
    """The downstream-task accuracies (Locatello et al. 2019, section 6) of the encoder means `mu` [N, D] (CUDA fp32,
    dataset index order) of the full factor grid `lat_sizes`, as disentanglement_lib's downstream_task.py computes
    them -> (score, helpers).  The draws come from a device torch.Generator seeded with `seed`: for each training size
    in order, `torch.randint(N, (size,))` training rows, then `torch.randint(N, (num_test,))` test rows; the global
    generators are not touched.  The classes are `sap_labels`' of each size's rows (a test value unseen in training is
    never predicted right).  For every scored factor (those of more than one value, ascending; factor i of the keys is
    the i-th of them) the predictor is fitted on the training rows and scored on both sets:
    - "logistic_regression": LogisticRegressionCV(Cs=10, cv=KFold(5)) on the raw means by `downstream_logistic_cv`;
      a factor seen with one value in training predicts it;
    - "boosted_trees": GradientBoostingClassifier() by `dci_fit`.
    score: for every size s, "{s}:mean_train_accuracy", "{s}:mean_test_accuracy", "{s}:min_train_accuracy",
    "{s}:min_test_accuracy" and "{s}:train_accuracy_factor_{i}", "{s}:test_accuracy_factor_{i}".
    helpers: "factors" int64 [K'] (the scored factor indices, ascending), "predictor", and per size s, helpers[s]:
    "classes" int64 [K', S] (each factor's training values, ascending, -1 beyond), "train_accuracy" and
    "test_accuracy" fp64 [K']; for the logistic predictor also "Cs" fp64 [10], "fold_accuracy" fp64 [K', 5, 10],
    "chosen_C" fp64 [K'], "coef" fp64 [K', S, D] and "intercept" fp64 [K', S] (the refit's model rows, NaN beyond),
    "solver_iterations" int32 [K', 51] (the fold fits' Newton steps, fold-major, then the refit's; -1 for a fit that
    did not converge, which also raises a RuntimeWarning)."""
    lat_sizes = _check_downstream_grid(lat_sizes, mu.shape[0], mu.shape[1], predictor, num_train, num_test)
    N.require_cuda_f32(mu)
    sizes = [int(num_train)] if isinstance(num_train, int) else [int(s) for s in num_train]
    gen = torch.Generator(device=mu.device)
    gen.manual_seed(int(seed))
    score, helpers = {}, {"predictor": predictor}
    failed = 0
    for size in sizes:
        train_rows = torch.randint(mu.shape[0], (size,), generator=gen, device=mu.device)
        test_rows = torch.randint(mu.shape[0], (int(num_test),), generator=gen, device=mu.device)
        factors, train_cls, test_cls, n_classes, counts, present = sap_labels(lat_sizes, train_rows, test_rows)
        S = counts.shape[1]
        h = {}
        if predictor == "boosted_trees":
            _, pred, _ = dci_fit(mu, train_rows, test_rows, train_cls, n_classes, counts)
        else:
            fold_acc, chosen, coef, pred, iters, _, _ = downstream_logistic_cv(mu, train_rows, test_rows, train_cls,
                                                                               n_classes, S)
            coef, iters, chosen = coef.cpu(), iters.cpu(), chosen.cpu().long()
            failed += int((iters < 0).sum())
            h.update({"Cs": torch.from_numpy(DOWNSTREAM_CS.copy()), "fold_accuracy": fold_acc.cpu(),
                      "chosen_C": torch.from_numpy(DOWNSTREAM_CS.copy())[chosen], "coef": coef[..., :-1].clone(),
                      "intercept": coef[..., -1].clone(), "solver_iterations": iters})
        right = pred == torch.cat([train_cls, test_cls], 1)
        train_acc = right[:, :size].double().mean(1).cpu()
        test_acc = right[:, size:].double().mean(1).cpu()
        h.update({"classes": _classes_table(present.cpu()), "train_accuracy": train_acc, "test_accuracy": test_acc})
        helpers[size] = h
        helpers["factors"] = torch.tensor(factors, dtype=torch.int64)
        s = str(size)
        score[s + ":mean_train_accuracy"] = float(train_acc.mean())
        score[s + ":mean_test_accuracy"] = float(test_acc.mean())
        score[s + ":min_train_accuracy"] = float(train_acc.min())
        score[s + ":min_test_accuracy"] = float(test_acc.min())
        for i in range(len(factors)):
            score[s + ":train_accuracy_factor_%d" % i] = float(train_acc[i])
            score[s + ":test_accuracy_factor_%d" % i] = float(test_acc[i])
    if failed:
        warnings.warn("downstream task: %d of the logistic-regression fits did not converge in the solver's step "
                      "limit; see helpers[size]['solver_iterations'] (-1)" % failed, RuntimeWarning)
    return score, helpers


# ---- IRS (Suter et al. 2019; disentanglement_lib's irs.py) -------------------------------------------------------
def check_irs_score(dataset, latent_dim, num_train=10000, diff_quantile=0.99):
    """ValueError unless IRS can be computed over `dataset` for a `latent_dim` model with these settings: the dataset
    has known factors (`lat_sizes`, `lat_names`), is their full grid and has a factor of more than one value.  No GPU
    work.  Returns lat_sizes as a list of ints."""
    return _check_irs_grid(_dataset_lat_sizes("IRS", dataset), len(dataset), latent_dim, num_train, diff_quantile)


def _check_irs_grid(lat_sizes, n, latent_dim, num_train, diff_quantile):
    lat_sizes = _full_grid("IRS", lat_sizes, n)
    if all(s == 1 for s in lat_sizes):
        raise ValueError("IRS: every factor of %s has one value; there is no factor to intervene on" % lat_sizes)
    if not 1 <= int(latent_dim) <= IRS_MAX_DIM:
        raise ValueError("IRS: latent_dim must be in [1, %d], got %d" % (IRS_MAX_DIM, int(latent_dim)))
    if not 1 <= int(num_train) <= IRS_MAX_TRAIN:
        raise ValueError("IRS: num_train must be in [1, %d], got %d" % (IRS_MAX_TRAIN, int(num_train)))
    if not 0.0 <= float(diff_quantile) <= 1.0:
        raise ValueError("IRS: diff_quantile must be in [0, 1], got %r" % (diff_quantile,))
    return lat_sizes


def irs_fit(mu, rows, values, diff_quantile):
    """`dv_irs_fit` on `mu` [N, D] (any strides, a view of q_zCx included), the drawn `rows` int64 [n] and the scored
    factors' `values` int32 [K', n] -> (max_deviation fp64 [D], active int32 [D], irs_matrix fp64 [D, K'],
    group_deviation fp64 [K', 20, D], group_count int32 [K', 20], edges fp64 [K', 21]); see include/disvae_b200.h for
    the rules."""
    mu_args, d = _mu_args(mu), mu.shape[1]
    _require_operands("irs_fit", rows=(rows, torch.int64), values=(values, torch.int32))
    n = rows.numel()
    K = values.shape[0]
    if values.dim() != 2 or values.shape[1] != n:
        raise ValueError("irs_fit: values must be [K', %d], got %s" % (n, tuple(values.shape)))
    nbytes = N.lib().dv_irs_workspace_bytes(d, n, K)
    ws = _f64_workspace(nbytes, mu.device)
    f64 = dict(dtype=torch.float64, device=mu.device)
    i32 = dict(dtype=torch.int32, device=mu.device)
    out = (torch.empty(d, **f64), torch.empty(d, **i32), torch.empty(d, K, **f64),
           torch.empty(K, IRS_BINS, d, **f64), torch.empty(K, IRS_BINS, **i32), torch.empty(K, IRS_BINS + 1, **f64))
    N.call("dv_irs_fit", *mu_args, N.ptr(rows), n, N.ptr(values), K, float(diff_quantile), *(N.ptr(t) for t in out),
           N.ptr(ws), nbytes, N.stream())
    return out


def irs_from_matrix(irs_matrix, max_deviations, active):
    """(IRS, per-latent scores [D], parents [D]) of `irs_fit`'s matrix [D, K'], in fp64 on the host, as irs.py's
    scalable_disentanglement_score finishes it over the active latents: a latent's score is its row's maximum and its
    parent that row's argmax (the lowest factor on a tie); IRS is the mean of the scores weighted by `max_deviations`,
    added in latent order.  Inactive latents score NaN with parent -1; with no active latent IRS is 0.0."""
    M = irs_matrix.double().cpu()
    dev = max_deviations.double().cpu().tolist()
    per_latent = torch.full((M.shape[0],), float("nan"), dtype=torch.float64)
    parents = torch.full((M.shape[0],), -1, dtype=torch.int64)
    num, den = 0.0, 0.0
    for d in torch.nonzero(active.cpu().bool())[:, 0].tolist():
        parents[d] = torch.argmax(M[d])                # the first of equal maxima
        per_latent[d] = M[d, parents[d]]
        num += dev[d] * float(per_latent[d])
        den += dev[d]
    return (num / den if den > 0.0 else 0.0), per_latent, parents


def irs_score(mu, lat_sizes, num_train=10000, diff_quantile=0.99, seed=0):
    """IRS (Suter et al. 2019) of the encoder means `mu` [N, D] (CUDA fp32, dataset index order) of the full factor
    grid `lat_sizes` -> ({"IRS", "num_active_dims"}, helpers).  The rows are `_train_rows`' draw seeded with `seed`,
    the training rows `_sap_draws` gives SAP, DCI and modularity; the scored factors are those of more than one value,
    ascending, each binned by disentanglement_lib's 20-bin histogram of its drawn values.  `irs_fit` gives the
    per-(latent, factor) matrix on the device, `irs_from_matrix` finishes it on the host.  "num_active_dims" counts the
    latents whose drawn values are not all equal.
    helpers: "irs_matrix" fp64 [D, K'] (NaN for an inactive latent), "disentanglement_scores" fp64 [D] (NaN when
    inactive), "parents" int64 [D] (-1 when inactive), "max_deviations" fp64 [D], "active_dims" bool [D], "factors"
    int64 [K'] (the scored factor indices, ascending), "bin_edges" fp64 [K', 21], "group_counts" int64 [K', 20] and
    "group_deviations" fp64 [K', 20, D] (NaN for an empty bin)."""
    lat_sizes = _check_irs_grid(lat_sizes, mu.shape[0], mu.shape[1], num_train, diff_quantile)
    _, rows = _train_rows(mu, num_train, seed)
    factors = [k for k, s in enumerate(lat_sizes) if s > 1]
    strides = [reduce(lambda x, y: x * y, lat_sizes[k + 1:], 1) for k in range(len(lat_sizes))]
    values = torch.stack([rows // strides[k] % lat_sizes[k] for k in factors]).int()
    max_dev, active, matrix, group_dev, group_count, edges = (t.cpu() for t in irs_fit(mu, rows, values,
                                                                                         diff_quantile))
    active = active.bool()
    irs, per_latent, parents = irs_from_matrix(matrix, max_dev, active)
    helpers = {"irs_matrix": matrix, "disentanglement_scores": per_latent, "parents": parents,
               "max_deviations": max_dev, "active_dims": active, "factors": torch.tensor(factors, dtype=torch.int64),
               "bin_edges": edges, "group_counts": group_count.long(), "group_deviations": group_dev}
    return {"IRS": irs, "num_active_dims": int(active.sum())}, helpers


# ---- UDR (Duan et al. 2020; disentanglement_lib's udr.py, compute_udr_sklearn) ------------------------------------
def udr_filenames(epoch=None):
    """(`udr.log`, `udr_helpers.pth`), or after training epoch `epoch` (`udr-{epoch}.log`, `udr_helpers-{epoch}.pth`)."""
    if epoch is None:
        return UDR_FILENAME, UDR_HELPERS_FILE
    return "udr-{}.log".format(epoch), "udr_helpers-{}.pth".format(epoch)


def check_udr(num_models, latent_dims, img_sizes=None, num_points=1000, correlation="lasso", groups=None):
    """ValueError unless UDR can score `num_models` models of latents `latent_dims` (one per model) taking images of
    `img_sizes` (one per model, or None) over `num_points` points with these settings: at least 2 models of one
    latent_dim D and one image shape, 1 <= D <= UDR_MAX_DIM, K D <= UDR_MAX_COLUMNS, 2 <= num_points <=
    UDR_MAX_POINTS, `correlation` one of UDR_CORRELATIONS, and `groups` (None: one group of every model) a partition of
    range(num_models) into groups of at least 2.  No GPU work.  Returns the groups as lists of ints."""
    K = int(num_models)
    if K < 2:
        raise ValueError("UDR: needs at least 2 models, got %d" % K)
    dims = [int(d) for d in latent_dims]
    if len(set(dims)) > 1:
        raise ValueError("UDR: the models have different latent_dim %s; UDR compares latents of one size" % dims)
    if img_sizes is not None and len({tuple(s) for s in img_sizes}) > 1:
        raise ValueError("UDR: the models take different image shapes %s; they must encode the same images"
                         % [tuple(s) for s in img_sizes])
    D = dims[0]
    if not 1 <= D <= UDR_MAX_DIM:
        raise ValueError("UDR: latent_dim must be in [1, %d], got %d" % (UDR_MAX_DIM, D))
    if K * D > UDR_MAX_COLUMNS:
        raise ValueError("UDR: %d models of %d latents are %d columns, above the kernel's limit of %d"
                         % (K, D, K * D, UDR_MAX_COLUMNS))
    if not 2 <= int(num_points) <= UDR_MAX_POINTS:
        raise ValueError("UDR: num_points must be in [2, %d], got %d" % (UDR_MAX_POINTS, int(num_points)))
    if correlation not in UDR_CORRELATIONS:
        raise ValueError("UDR: correlation must be one of %s, got %r" % (list(UDR_CORRELATIONS), correlation))
    if groups is None:
        return [list(range(K))]
    groups = [[int(k) for k in g] for g in groups]
    members = sorted(k for g in groups for k in g)
    if members != list(range(K)):
        raise ValueError("UDR: groups %s are not a partition of the models 0 .. %d" % (groups, K - 1))
    for g in groups:
        if len(g) < 2:
            raise ValueError("UDR: group %s has fewer than 2 models; a model's score is a median over the others of "
                             "its group" % g)
    return groups


def udr_fit(mu, logvar, correlation="lasso"):
    """`dv_udr_fit` on the encoder outputs `mu`, `logvar` (contiguous CUDA fp32 [K, n, D], the same points for every
    model) -> (raw fp64 [K, K, D, D], pair fp64 [K, K], kl fp64 [K, D], iters int32 [K, K]); see
    include/disvae_b200.h for the rules."""
    K, n, D = mu.shape
    _require_operands("udr_fit", mu=(mu, torch.float32), logvar=(logvar, torch.float32, (K, n, D)))
    check_udr(K, [D] * K, num_points=n, correlation=correlation)
    nbytes = N.lib().dv_udr_workspace_bytes(K, n, D)
    ws = _f64_workspace(nbytes, mu.device)
    f64 = dict(dtype=torch.float64, device=mu.device)
    raw, pair, kl = torch.empty(K, K, D, D, **f64), torch.empty(K, K, **f64), torch.empty(K, D, **f64)
    iters = torch.empty(K, K, dtype=torch.int32, device=mu.device)
    N.call("dv_udr_fit", N.ptr(mu), N.ptr(logvar), K, n, D, UDR_CORRELATIONS[correlation], UDR_LASSO_ALPHA,
           UDR_KL_THRESHOLD, N.ptr(raw), N.ptr(pair), N.ptr(kl), N.ptr(iters), N.ptr(ws), nbytes, N.stream())
    return raw, pair, kl, iters


def _median(values):
    """np.median of a 1-d fp64 tensor: the middle value, or the mean of the two middle values for an even count."""
    v = torch.sort(values)[0]
    m = v.numel()
    return float((v[(m - 1) // 2] + v[m // 2]) / 2)


def udr_from_pairs(pair, groups):
    """Every model's UDR from the pair scores [K, K] (pair[i, j]: i's latents the inputs, j's the targets): model k
    scores the median over the others j of its group of pair[j, k]."""
    scores = [0.0] * pair.shape[0]
    for g in groups:
        for k in g:
            scores[k] = _median(torch.stack([pair[j, k] for j in g if j != k]))
    return scores


def udr_score(mu, logvar, correlation="lasso", groups=None):
    """UDR of K models from their encoder outputs `mu`, `logvar` (contiguous CUDA fp32 [K, n, D] over the same points)
    -> ({"model_scores": [K] floats}, helpers).  `udr_fit` computes every ordered pair's score; `udr_from_pairs` takes
    each model's median within its group (`groups`, a partition of range(K); None: one group of every model).
    helpers: "pairwise" fp64 [K, K] (NaN on the diagonal), "raw_correlations" fp64 [K, K, D, D] (before the filter),
    "kl" fp64 [K, D], "informative" bool [K, D], "groups" (lists of model indices) and "solver_iterations" int32
    [K, K] (the Lasso's largest sweep count of each pair, -1 for a pair with a fit that did not converge, which also
    raises a RuntimeWarning; 0 for Spearman)."""
    K, n, D = mu.shape
    groups = check_udr(K, [D] * K, num_points=n, correlation=correlation, groups=groups)
    raw, pair, kl, iters = (t.cpu() for t in udr_fit(mu, logvar, correlation))
    failed = int((iters < 0).sum())
    if failed:
        warnings.warn("UDR: %d of the pairs have a Lasso fit that did not converge in the solver's sweep limit; see "
                      "helpers['solver_iterations'] (-1)" % failed, RuntimeWarning)
    helpers = {"pairwise": pair, "raw_correlations": raw, "kl": kl, "informative": kl > UDR_KL_THRESHOLD,
               "groups": groups, "solver_iterations": iters}
    return {"model_scores": udr_from_pairs(pair, groups)}, helpers


def udr_points(loader, num_points, seed):
    """The dataset rows UDR encodes: `torch.randint(len(dataset), (num_points,))` from a torch.Generator on
    `loader.device` seeded with `seed`; the global generators are not touched."""
    gen = torch.Generator(device=loader.device)
    gen.manual_seed(int(seed) & 0xFFFFFFFFFFFFFFFF)
    return torch.randint(loader.n, (int(num_points),), generator=gen, device=loader.device)


def udr(models, loader, num_points=1000, seed=0, correlation="lasso", groups=None):
    """UDR (Duan et al. 2020) of the trained `models` (any models with the same latent_dim and image shape, on
    `loader`'s device) over `loader` (a disvae.data.DeviceLoader) -> ({"model_scores": [K]}, helpers).  Every model
    encodes the same `num_points` rows (`udr_points`, seeded with `seed`), gathered from the loader's resident data, in
    eval mode (so the code is the encoder mean); each model's train / eval mode is kept.  No labels are read.  See
    `udr_score` for the score; helpers also hold "rows" int64 [num_points]."""
    from disvae.data import DeviceLoader
    models = list(models)
    if not isinstance(loader, DeviceLoader):
        raise ValueError("UDR: expected a disvae.data.DeviceLoader, got %s" % type(loader).__name__)
    groups = check_udr(len(models), [m.latent_dim for m in models], [m.img_size for m in models], num_points,
                       correlation, groups)
    if tuple(models[0].img_size) != tuple(loader.data.shape[1:]):
        raise ValueError("UDR: the loader holds %s images, the models take %s"
                         % (tuple(loader.data.shape[1:]), tuple(models[0].img_size)))
    rows = udr_points(loader, num_points, seed)
    mu, logvar = encode_resident_rows(models, loader, rows)
    scores, helpers = udr_score(mu, logvar, correlation, groups)
    helpers["rows"] = rows.cpu()
    return scores, helpers


def encode_resident_rows(models, loader, rows):
    """The encoder outputs (mu, logvar), fp32 [K, n, D], of the K `models` (one latent_dim) on the dataset rows `rows`
    (int64 [n] on the device), gathered from `loader`'s resident data (a DeviceLoader) UDR_ENCODE_BATCH at a time, in
    eval mode (so the code is the encoder mean); each model's train / eval mode is kept."""
    from disvae import ops
    K, n, D = len(models), rows.numel(), int(models[0].latent_dim)
    mu = torch.empty(K, n, D, dtype=torch.float32, device=loader.device)
    logvar = torch.empty_like(mu)
    with torch.no_grad():
        for k, model in enumerate(models):
            was_training = model.training
            model.eval()
            try:
                for a in range(0, n, UDR_ENCODE_BATCH):
                    x = ops.gather_u8_to_f32(loader.data, rows[a:a + UDR_ENCODE_BATCH])
                    mu[k, a:a + x.shape[0]], logvar[k, a:a + x.shape[0]] = model.encoder(x)
            finally:
                model.train(was_training)
    return mu, logvar


def write_udr(models, loader, save_dirs, seed, epoch=None, loggers=None, num_points=1000, correlation="lasso",
              groups=None):
    """`udr(models, loader, ...)` into every model's save_dir: `udr_filenames(epoch)`, the log {"UDR": its score} and
    the helpers with "member" = its index; each model's logger of `loggers` (or None) records its score."""
    scores, helpers = udr(models, loader, num_points=num_points, seed=seed, correlation=correlation, groups=groups)
    log_name, helpers_name = udr_filenames(epoch)
    for k, save_dir in enumerate(save_dirs):
        if loggers is not None:
            loggers[k].info("UDR: {}".format(scores["model_scores"][k]))
        save_metadata({"UDR": scores["model_scores"][k]}, save_dir, filename=log_name)
        torch.save(dict(helpers, member=k), os.path.join(save_dir, helpers_name))
    return scores, helpers


# ---- unsupervised scores (disentanglement_lib's unsupervised_metrics.py; Locatello et al. 2019, section 5.1) --------
def unsupervised_filenames(epoch=None):
    """(`unsupervised_scores.log`, `unsupervised_scores_helpers.pth`), or after training epoch `epoch`
    (`unsupervised_scores-{epoch}.log`, `unsupervised_scores_helpers-{epoch}.pth`)."""
    if epoch is None:
        return UNSUPERVISED_FILENAME, UNSUPERVISED_HELPERS_FILE
    return "unsupervised_scores-{}.log".format(epoch), "unsupervised_scores_helpers-{}.pth".format(epoch)


def check_unsupervised_scores(latent_dim, num_train=10000):
    """ValueError unless the unsupervised scores can be computed for codes of `latent_dim` latents over `num_train`
    drawn points: 2 <= latent_dim <= UNSUPERVISED_MAX_DIM (np.cov of one latent is 0-d and the mutual-information
    score divides by D^2 - D) and 2 <= num_train <= UNSUPERVISED_MAX_POINTS.  Needs no known factors; no GPU work."""
    D = int(latent_dim)
    if not 2 <= D <= UNSUPERVISED_MAX_DIM:
        raise ValueError("unsupervised scores: latent_dim must be in [2, %d], got %d" % (UNSUPERVISED_MAX_DIM, D))
    if not 2 <= int(num_train) <= UNSUPERVISED_MAX_POINTS:
        raise ValueError("unsupervised scores: num_train must be in [2, %d], got %d"
                         % (UNSUPERVISED_MAX_POINTS, int(num_train)))


def unsupervised_draws(n_items, num_train, latent_dim, seed, device):
    """(rows int64 [num_train], eps fp32 [num_train, latent_dim]) on `device`, from one torch.Generator seeded with
    `seed`: `torch.randint(n_items, (num_train,))` first, then `torch.randn(num_train, latent_dim)`.  The global
    generators are not touched."""
    gen = torch.Generator(device=device)
    gen.manual_seed(int(seed) & 0xFFFFFFFFFFFFFFFF)
    rows = torch.randint(int(n_items), (int(num_train),), generator=gen, device=device)
    eps = torch.randn(int(num_train), int(latent_dim), generator=gen, device=device)
    return rows, eps


def unsupervised_fit(mu, logvar, rows, eps):
    """`dv_unsupervised_fit` on `mu`, `logvar` [N, D] (CUDA fp32, the same strides, any of them: views of q_zCx
    included), the drawn `rows` int64 [n] and `eps` fp32 [n, D] -> (cov fp64 [2, D, D], eig fp64 [2, 2, D], sweeps
    int32 [2, 2], mi fp64 [2, D, D], edges fp32 [2, D, 21]), representation 0 the mean, 1 the sampled; see
    include/disvae_b200.h for the rules."""
    mu_args, d = _mu_args(mu), mu.shape[1]
    N.require_cuda_f32(logvar)
    if logvar.shape != mu.shape or logvar.stride() != mu.stride() or logvar.device != mu.device:
        raise ValueError("unsupervised_fit: logvar must have mu's shape, strides and device")
    n = rows.numel()
    _require_operands("unsupervised_fit", rows=(rows, torch.int64, (n,)), eps=(eps, torch.float32, (n, d)))
    check_unsupervised_scores(d, n)
    nbytes = N.lib().dv_unsupervised_workspace_bytes(n, d)
    ws = _f64_workspace(nbytes, mu.device)
    f64 = dict(dtype=torch.float64, device=mu.device)
    cov, eig, mi = torch.empty(2, d, d, **f64), torch.empty(2, 2, d, **f64), torch.empty(2, d, d, **f64)
    sweeps = torch.empty(2, 2, dtype=torch.int32, device=mu.device)
    edges = torch.empty(2, d, MODULARITY_BINS + 1, dtype=torch.float32, device=mu.device)
    N.call("dv_unsupervised_fit", mu_args[0], N.ptr(logvar), *mu_args[1:], N.ptr(rows), n, N.ptr(eps), N.ptr(cov),
           N.ptr(eig), N.ptr(sweeps), N.ptr(mi), N.ptr(edges), None, N.ptr(ws), nbytes, N.stream())
    return cov, eig, sweeps, mi, edges


def unsupervised_from_fit(cov, eig, mi):
    """The four scores of each representation from `unsupervised_fit`'s cov, eig and mi (fp64, combined on the host
    in fp64) -> {"mean": {...}, "sampled": {...}} under disentanglement_lib's keys:
    gaussian_total_correlation = -1/2 sum log eig(R) (+inf, with a RuntimeWarning, when eig_min(R) <= D DBL_EPSILON
    eig_max(R): linearly dependent latents); gaussian_wasserstein_correlation = 2 trace(C) - 2 sum sqrt(max(eig(S), 0));
    its _norm = that / trace(C) (0 when trace(C) = 0); mutual_info_score = the sum of mi off its diagonal / (D^2 - D)."""
    cov, eig, mi = cov.double().cpu(), eig.double().cpu(), mi.double().cpu()
    D = cov.shape[-1]
    scores = {}
    for r, name in enumerate(UNSUPERVISED_REPRESENTATIONS):
        lam_r, lam_s = eig[r, 0], eig[r, 1]
        if lam_r[0] <= D * UNSUPERVISED_DBL_EPSILON * lam_r[-1]:
            warnings.warn("unsupervised scores: the %s representation has linearly dependent latents (smallest "
                          "correlation eigenvalue %.3g); its gaussian_total_correlation is +inf" % (name, lam_r[0]),
                          RuntimeWarning)
            tc = math.inf
        else:
            tc = float(-0.5 * torch.log(lam_r).sum())
        trace = float(torch.diagonal(cov[r]).sum())
        w = 2.0 * trace - 2.0 * float(torch.sqrt(lam_s.clamp(min=0)).sum())
        off = mi[r] - torch.diag(torch.diagonal(mi[r]))
        scores[name] = {"gaussian_total_correlation": tc, "gaussian_wasserstein_correlation": w,
                        "gaussian_wasserstein_correlation_norm": w / trace if trace != 0 else 0.0,
                        "mutual_info_score": float(off.sum() / (D * D - D))}
    return scores


def _unsupervised_of(mu, logvar, fit_rows, eps, rows):
    """(scores, helpers) of `unsupervised_fit(mu, logvar, fit_rows, eps)`, `rows` the dataset rows drawn."""
    cov, eig, sweeps, mi, edges = (t.cpu() for t in unsupervised_fit(mu, logvar, fit_rows, eps))
    failed = int((sweeps < 0).sum())
    if failed:
        warnings.warn("unsupervised scores: %d of the eigensolves stopped at the sweep limit; see "
                      "helpers['solver_sweeps'] (-1)" % failed, RuntimeWarning)
    scores = unsupervised_from_fit(cov, eig, mi)
    eye = torch.eye(mi.shape[-1], dtype=torch.bool)
    helpers = {"rows": rows.cpu(), "cov": cov, "eigenvalues": eig,
               "constant": torch.diagonal(cov, dim1=1, dim2=2) == 0,
               "mutual_information": mi.masked_fill(eye, 0.0), "bin_edges": edges, "solver_sweeps": sweeps}
    return scores, helpers


def unsupervised_scores(mu, logvar, num_train=10000, seed=0):
    """The unsupervised scores of Locatello et al. 2019 (disentanglement_lib's unsupervised_metrics.py) of the encoder
    outputs `mu`, `logvar` [N, D] (CUDA fp32, the same strides, any of them; q_zCx views included) ->
    ({"mean": {4 keys}, "sampled": {4 keys}}, helpers).  `unsupervised_draws` (seeded with `seed`) draws num_train rows
    and the noise of the sampled representation mu + exp(logvar / 2) eps; `unsupervised_fit` computes each
    representation's covariance, the eigenvalues of its correlation matrix R and of diag(c)^1/2 C diag(c)^1/2, and the
    mutual information of every pair of latents; `unsupervised_from_fit` combines them.  No labels are read.
    helpers: "rows" int64 [num_train], "cov" fp64 [2, D, D], "eigenvalues" fp64 [2, 2, D] (R then S, ascending),
    "constant" bool [2, D] (latents of zero variance over the rows), "mutual_information" fp64 [2, D, D] (diagonal
    zeroed), "bin_edges" fp32 [2, D, 21] and "solver_sweeps" int32 [2, 2] (Jacobi sweeps, -1 for an eigensolve that
    reached the sweep limit, which also raises a RuntimeWarning); index 0 the mean representation, 1 the sampled."""
    n_items, D = mu.shape
    check_unsupervised_scores(D, num_train)
    rows, eps = unsupervised_draws(n_items, num_train, D, seed, mu.device)
    return _unsupervised_of(mu, logvar, rows, eps, rows)


def resident_unsupervised_scores(model, loader, num_train=10000, seed=0):
    """`unsupervised_scores` of `model` over the dataset of `loader` (a disvae.data.DeviceLoader), encoding only the
    drawn rows: the rows and noise are `unsupervised_draws(len(dataset), num_train, latent_dim, seed)`, the rows
    gathered from the resident data and encoded in eval mode (`encode_resident_rows`); the model keeps its train / eval
    mode.  Equals `unsupervised_scores` of the whole dataset's encodings in index order (up to the rounding of the
    encoder at another batch size)."""
    from disvae.data import DeviceLoader
    if not isinstance(loader, DeviceLoader):
        raise ValueError("unsupervised scores: expected a disvae.data.DeviceLoader, got %s" % type(loader).__name__)
    check_unsupervised_scores(model.latent_dim, num_train)
    if tuple(model.img_size) != tuple(loader.data.shape[1:]):
        raise ValueError("unsupervised scores: the loader holds %s images, the model takes %s"
                         % (tuple(loader.data.shape[1:]), tuple(model.img_size)))
    rows, eps = unsupervised_draws(loader.n, num_train, model.latent_dim, seed, loader.device)
    mu, logvar = encode_resident_rows([model], loader, rows)
    return _unsupervised_of(mu[0], logvar[0], torch.arange(rows.numel(), device=rows.device), eps, rows)


def write_unsupervised_scores(model, loader, save_dir, seed, epoch=None, logger=None, num_train=10000):
    """`resident_unsupervised_scores(model, loader, num_train, seed)` into `save_dir` as
    `unsupervised_filenames(epoch)`; `logger` (or None) records the scores."""
    scores, helpers = resident_unsupervised_scores(model, loader, num_train, seed)
    log_name, helpers_name = unsupervised_filenames(epoch)
    if logger is not None:
        logger.info("Unsupervised scores: {}".format(scores))
    save_metadata(scores, save_dir, filename=log_name)
    torch.save(helpers, os.path.join(save_dir, helpers_name))
    return scores, helpers


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

    def compute_dci_score(self, dataloader, num_train=10000, num_test=5000, seed=0):
        """DCI score (Eastwood & Williams 2018) of the model's encoder means over `dataloader` (the dataset in index
        order: DataLoader(shuffle=False) or DeviceLoader.in_order) -> {"disentanglement", "completeness",
        "informativeness_train", "informativeness_test"}; see `dci_score` for the definition and the order of the
        draws.  The Evaluator's __call__, training and sweeps do not write this score; score a sweep's members with
        `Evaluator(member.model, ...).compute_dci_score(sweep.loader.in_order(1000), seed=...)`."""
        return self._score(check_dci_score, dci_score, dataloader, seed, num_train=num_train, num_test=num_test)

    def compute_modularity_explicitness(self, dataloader, num_train=10000, num_test=5000, seed=0):
        """Modularity and explicitness (Ridgeway & Zemel 2018) of the model's encoder means over `dataloader` (the
        dataset in index order: DataLoader(shuffle=False) or DeviceLoader.in_order) -> {"modularity_score",
        "explicitness_score_train", "explicitness_score_test"}; see `modularity_explicitness` for the definition and
        the order of the draws.  The Evaluator's __call__, training and sweeps do not write this score; score a sweep's
        members with `Evaluator(member.model, ...).compute_modularity_explicitness(sweep.loader.in_order(1000),
        seed=...)`."""
        return self._score(check_modularity_explicitness, modularity_explicitness, dataloader, seed,
                           num_train=num_train, num_test=num_test)

    def compute_downstream_task(self, dataloader, predictor="logistic_regression", num_train=(10, 100, 1000, 10000),
                                num_test=5000, seed=0):
        """The downstream-task accuracies (Locatello et al. 2019, section 6) of the model's encoder means over
        `dataloader` (the dataset in index order: DataLoader(shuffle=False) or DeviceLoader.in_order) with the
        "logistic_regression" or "boosted_trees" predictor -> {"{size}:mean_train_accuracy", ...}; see
        `downstream_task` for the definition and the order of the draws.  The Evaluator's __call__, training and sweeps
        do not write this score; score a sweep's members with `Evaluator(member.model, None,
        device=...).compute_downstream_task(sweep.loader.in_order(1000), seed=...)`."""
        return self._score(check_downstream_task, downstream_task, dataloader, seed, predictor=predictor,
                           num_train=num_train, num_test=num_test)

    def compute_irs_score(self, dataloader, num_train=10000, diff_quantile=0.99, seed=0):
        """IRS (Suter et al. 2019) of the model's encoder means over `dataloader` (the dataset in index order:
        DataLoader(shuffle=False) or DeviceLoader.in_order) -> {"IRS", "num_active_dims"}; see `irs_score` for the
        definition and the draw.  The Evaluator's __call__, training and sweeps do not write this score; score a
        sweep's members with `Evaluator(member.model, None, device=...).compute_irs_score(sweep.loader.in_order(1000),
        seed=...)`."""
        return self._score(check_irs_score, irs_score, dataloader, seed, num_train=num_train,
                           diff_quantile=diff_quantile)

    def compute_unsupervised_scores(self, dataloader, num_train=10000, seed=0):
        """The unsupervised scores (Locatello et al. 2019, section 5.1) of the model's mean and sampled representations
        over `dataloader` (any dataset, with or without known factors, in index order: DataLoader(shuffle=False) or
        DeviceLoader.in_order) -> {"mean": {...}, "sampled": {...}}; see `unsupervised_scores` for the definition and
        the order of the draws.  The Evaluator's __call__ and training do not write these scores; a sweep writes them
        with `unsupervised_every` or `Sweep.unsupervised_scores`."""
        check_unsupervised_scores(self.model.latent_dim, num_train)
        dataset = getattr(dataloader, "dataset", None)
        if dataset is None or not hasattr(dataset, "__len__") or len(dataset) < 1:
            raise ValueError("unsupervised scores: expected a loader over a non-empty dataset, got %s"
                             % type(dataloader).__name__)
        mean, logvar = self._compute_q_zCx(dataloader)[1]
        return unsupervised_scores(mean, logvar, num_train=num_train, seed=seed)[0]

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
