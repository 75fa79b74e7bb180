"""Evaluator with the reference's API (disvae/evaluate.py:22-317).  Test losses run on the CUDA path; the MIG / AAM
disentanglement metrics run their one expensive piece -- the marginal-entropy estimator (evaluate.py:233-297), the
same pairwise Gaussian log-density pattern as the beta-TCVAE kernel -- in `dv_latent_entropy` instead of 1000
materialised [N, D, 10] tensors per call (SURVEY.md 8f-4).  Everything else (index bookkeeping, the two metric
formulas on a [n_factors, latent_dim] table) is host code that mirrors the reference line for line, quirks included.
"""
import contextlib
import inspect
import logging
import os
import tempfile
from collections import defaultdict
from functools import reduce
from timeit import default_timer

import torch
from tqdm import tqdm

from disvae import _native as N
from disvae.parallel import is_distributed
from disvae.utils.modelIO import save_metadata

TEST_LOSSES_FILE = "test_losses.log"
METRICS_FILENAME = "metrics.log"
METRIC_HELPERS_FILE = "metric_helpers.pth"
EVAL_SEED_STRIDE = 0x9E3779B97F4A7C15      # odd 64-bit constant: consecutive epochs get unrelated seeds


def epoch_metrics_filenames(epoch):
    """(`metrics-{epoch}.log`, `metric_helpers-{epoch}.pth`): the metrics written after training epoch `epoch`."""
    return "metrics-{}.log".format(epoch), "metric_helpers-{}.pth".format(epoch)


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


def write_epoch_metrics(model, loader, epoch, batch_size, save_dir, logger):
    """MIG / AAM of `model` over `loader.in_order(batch_size)` (a DeviceLoader) into `save_dir` as
    `epoch_metrics_filenames(epoch)`, with the index draws seeded by `evaluation_rng(.., model's noise key, epoch)`.
    The model's train / eval mode is kept."""
    device = loader.device
    key = model._noise_state(device)[0]           # fixed at the first training step; this fixes it the same way
    metrics_file, helpers_file = epoch_metrics_filenames(epoch)
    with tempfile.TemporaryDirectory(dir=save_dir) as tmp, evaluation_rng(device, key, epoch):
        Evaluator(model, None, device=device, logger=logger, save_dir=tmp, is_progress_bar=False)(
            loader.in_order(batch_size), is_metrics=True, is_losses=False)
        os.replace(os.path.join(tmp, METRICS_FILENAME), os.path.join(save_dir, metrics_file))
        os.replace(os.path.join(tmp, METRIC_HELPERS_FILE), os.path.join(save_dir, helpers_file))


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

    def __call__(self, data_loader, is_metrics=False, is_losses=True):
        """evaluate.py:59-96.  Like the reference, the first returned value is always None (it assigns the metrics to
        a differently named variable, :77-79); the metrics are logged and written to metrics.log."""
        start = default_timer()
        is_still_training = self.model.training
        self.model.eval()
        metric, losses = None, None
        if is_metrics:
            self.logger.info('Computing metrics...')
            metrics = self.compute_metrics(data_loader)
            self.logger.info('Losses: {}'.format(metrics))
            save_metadata(metrics, self.save_dir, filename=METRICS_FILENAME)
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
        try:
            lat_sizes = dataloader.dataset.lat_sizes
            lat_names = dataloader.dataset.lat_names
        except AttributeError:
            raise ValueError("Dataset needs to have known true factors of variations to compute the metric. This does not "
                             "seem to be the case for {}".format(type(dataloader.__dict__["dataset"]).__name__))
        self.logger.info("Computing the empirical distribution q(z|x).")
        samples_zCx, params_zCx = self._compute_q_zCx(dataloader)
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
