"""Training loop with the reference's Trainer API (disvae/training.py:17-196).

Differences from the reference are in HOW, not WHAT: the per-step `loss.item()` host sync
(training.py:164) is replaced by an on-device running sum read once per epoch plus an asynchronous
per-step copy of the loss into pinned host memory (the progress bar shows the latest value that has
already landed), host batches are uploaded one step ahead on a copy stream (`_Prefetcher`), and under
torch.distributed (one process per GPU) gradients are averaged with one flat all-reduce per step
(disvae.parallel).

A run can be stopped and continued at an epoch boundary: `training_state()` / `load_training_state()` (and
`trainer(..., save_state=True)`, which writes one at every checkpoint) carry everything a later step reads, so the
continued run is bit-identical to one that was never stopped.
"""
import logging
import os
from collections import defaultdict, namedtuple
from timeit import default_timer

import torch
import torch.distributed as dist
from tqdm import trange

from disvae import _native
from disvae.evaluate import check_epoch_scores, check_resident_metrics, select_scores, write_epoch_metrics
from disvae.fused import FusedAdam
from disvae.models.losses import DeviceLossLog
from disvae.parallel import GradAverage, broadcast_parameters, is_distributed
from disvae.utils.modelIO import TRAINING_STATE_PREFIX, save_model, save_training_state

TRAIN_LOSSES_LOGFILE = "train_losses.log"
TRAINING_STATE_FORMAT = 1                 # version of the dict `Trainer.training_state` returns


def training_state_filename(epoch):
    """`training-state-{epoch}.pt`; under data parallelism one file per rank, `training-state-{epoch}-rank{r}.pt`."""
    if is_distributed():
        return "{}{}-rank{}.pt".format(TRAINING_STATE_PREFIX, epoch, dist.get_rank())
    return "{}{}.pt".format(TRAINING_STATE_PREFIX, epoch)


class Trainer():
    """Trainer(model, optimizer, loss_f, device, logger, save_dir, gif_visualizer, is_progress_bar)
    -- training.py:46-62."""

    def __init__(self, model, optimizer, loss_f, device=torch.device("cpu"), logger=logging.getLogger(__name__),
                 save_dir="results", gif_visualizer=None, is_progress_bar=True):
        self.device = device
        self.model = model.to(self.device)
        self.loss_f = loss_f
        self.optimizer = optimizer
        self.save_dir = save_dir
        self.is_progress_bar = is_progress_bar
        self.logger = logger
        self.losses_logger = LossesLogger(os.path.join(self.save_dir, TRAIN_LOSSES_LOGFILE))
        self.gif_visualizer = gif_visualizer
        self.sync_every = 50                      # progress-bar refresh (host sync) period
        self._grad_avg = None                     # GradAverage of the data-parallel steps (`_setup_data_parallel`)
        self._fused = None                        # FusedAdam over `optimizer` (built lazily on the device)
        self.use_cuda_graph = os.environ.get("DISVAE_CUDA_GRAPH", "1") != "0"
        # DISVAE_DEVICE_DATA=1: a torch DataLoader passed to __call__ is replaced by a disvae.data.DeviceLoader over its
        # dataset (decoded once, kept on the GPU; its own shuffle stream, hence opt-in)
        self.device_data = os.environ.get("DISVAE_DEVICE_DATA", "0") == "1"
        self._device_loaders = {}                 # id(DataLoader) -> (DataLoader, its DeviceLoader)
        self._graphs = {}                         # (input shape, dtype) -> _Graph of the captured step
        self._eligible_steps = 0
        self._loss_log = None                     # DeviceLossLog of the training steps (built on the first GPU step)
        self._resident_input = None               # fp32 device batch a caller refills in place (disvae.sweep): a graph
                                                  # captured on it reads it directly instead of a copy
        self._next_epoch = 0                      # number of the epoch after the last one completed (training state)
        self._data_loader = None                  # the loader of the current / latest call (its data-order state)
        self._resume = None                       # (first epoch, loader state) of a loaded state, for the next call
        self._steps_at_load = 0                   # n_train_steps a loaded state restored
        self.logger.info("Training Device: {}".format(self.device))

    def __call__(self, data_loader, epochs=10, checkpoint_every=10, save_state=False, metrics_every=0,
                 metrics_batch_size=1000, factor_score=False, sap_score=False, beta_vae_score=False):
        """training.py:64-102.  `save_state=True` also writes the training state (`training_state_filename`) next to
        every checkpoint and after the last epoch.  After `load_training_state` the epochs are numbered on from the
        saved one and the loader continues the saved data order.  `metrics_every=k > 0` writes MIG / AAM of the model
        (`metrics-{epoch}.log`, `metric_helpers-{epoch}.pth`) after every epoch divisible by k and after the last one,
        computed from the loader's resident data (`disvae.evaluate.write_epoch_metrics`); `factor_score=True` adds the
        FactorVAE score of those epochs (`factor_vae_score-{epoch}.log`, `factor_vae_score_helpers-{epoch}.pth`),
        `sap_score=True` the SAP score (`sap_score-{epoch}.log`, `sap_score_helpers-{epoch}.pth`) and
        `beta_vae_score=True` the beta-VAE score (`beta_vae_score-{epoch}.log`, `beta_vae_score_helpers-{epoch}.pth`).
        Training itself is unchanged."""
        scores = select_scores(locals())
        start = default_timer()
        first, loader_state = (0, None) if self._resume is None else self._resume
        if loader_state is not None:
            check_loader_state(loader_state, data_loader, self.device_data)
        check_metrics_every(metrics_every)
        if metrics_every:
            check_resident_metrics(data_loader, metrics_batch_size, self.device_data)
        check_epoch_scores(scores, metrics_every, data_loader, self.model.latent_dim)
        self._resume = None
        if self.device_data and isinstance(data_loader, torch.utils.data.DataLoader):
            data_loader = self._device_loader(data_loader)
        if loader_state is not None:
            apply_loader_state(loader_state, data_loader)
        self._data_loader = data_loader
        self.model.train()
        last = first + epochs - 1
        for epoch in range(first, first + epochs):
            storer = defaultdict(list)
            mean_epoch_loss = self._train_epoch(data_loader, storer, epoch)
            self._end_epoch(epoch, storer, mean_epoch_loss, checkpoint_every,
                            save_state=save_state and (epoch % checkpoint_every == 0 or epoch == last))
            if metrics_every and (epoch % metrics_every == 0 or epoch == last):
                write_epoch_metrics(self.model, data_loader, epoch, metrics_batch_size, self.save_dir, self.logger,
                                    scores)
        self._end_training(start)

    def _end_epoch(self, epoch, storer, mean_epoch_loss, checkpoint_every, save_state=False):
        """training.py:84-90: epoch log line, train_losses.log rows, GIF frame, checkpoint; the training state when
        `save_state`."""
        self.logger.info('Epoch: {} Average loss per image: {:.2f}'.format(epoch + 1, mean_epoch_loss))
        self.losses_logger.log(epoch, storer)
        self._next_epoch = epoch + 1
        if self.gif_visualizer is not None:
            self.gif_visualizer()
        if epoch % checkpoint_every == 0:
            save_model(self.model, self.save_dir, filename="model-{}.pt".format(epoch))
        if save_state:
            save_training_state(self, self.save_dir, training_state_filename(epoch))

    # -- training state -------------------------------------------------------------------------
    def training_state(self):
        """The state a continued run needs, as CPU tensors and Python values (see INTEGRATION.md, "Resuming
        training").  Taken at an epoch end, where the optimizers' step counts have been written back (flush_state)."""
        model, lf = self.model, self.loss_f
        loader = self._resume[1] if self._resume is not None else loader_state(self._data_loader)
        state = dict(
            format=TRAINING_STATE_FORMAT, epoch=self._next_epoch,
            model=dict(model_type=getattr(model, "model_type", None), img_size=list(model.img_size),
                       latent_dim=int(model.latent_dim), state_dict=_cpu(model.state_dict())),
            optimizer=_cpu(self.optimizer.state_dict()),
            loss=dict(cls=type(lf).__name__, hparams=loss_hparams(lf), n_train_steps=int(lf.n_train_steps)),
            noise=_philox(getattr(model, "_rng_seed", None), getattr(model, "_rng_offset", None)),
            factor=None, loader=loader, log_rows=list(self.losses_logger.rows),
            world_size=dist.get_world_size() if is_distributed() else 1,
            rank=dist.get_rank() if is_distributed() else 0)
        if hasattr(lf, "call_optimize"):
            state["factor"] = dict(discriminator=_cpu(lf.discriminator.state_dict()),
                                   optimizer_d=_cpu(lf.optimizer_d.state_dict()),
                                   perm=_philox(getattr(lf, "_perm_seed", None), lf._perm_offset),
                                   global_perm=_philox(getattr(lf, "_gperm_seed", None), lf._gperm_offset))
        return state

    def load_training_state(self, state):
        """Continue from `state` (a `training_state()`): into a Trainer that has taken no step in this process, with
        the same model geometry, loss class and hyper-parameters and world size; raises ValueError naming the first
        field that differs, before anything is changed.  The loader is checked and set at the next call."""
        self._check_training_state(state)
        model, lf = self.model, self.loss_f
        dev = next(model.parameters()).device
        model.load_state_dict(state["model"]["state_dict"])
        self.optimizer.load_state_dict(state["optimizer"])   # FusedAdam, built at the first step, starts from its counts
        lf.n_train_steps = self._steps_at_load = state["loss"]["n_train_steps"]   # (_step_counter follows it)
        # the Philox keys and counters: the first steps (eager and captured alike) continue the saved streams
        if state["noise"]["key"] is not None:
            model.seed_noise(state["noise"]["key"], dev)
            model._rng_offset.fill_(state["noise"]["offset"])
        if state["factor"] is not None:
            f = state["factor"]
            lf.discriminator.load_state_dict(f["discriminator"])
            lf.optimizer_d.load_state_dict(f["optimizer_d"])
            if f["perm"]["key"] is not None:
                lf.seed_permutations(f["perm"]["key"], dev)
                lf._perm_offset.fill_(f["perm"]["offset"])
            if f["global_perm"]["key"] is not None:
                lf._gperm_seed = f["global_perm"]["key"]
                lf._gperm_offset = torch.full((1,), f["global_perm"]["offset"], dtype=torch.int64, device=dev)
        loader = state["loader"]
        if loader is not None and loader["kind"] == "host":
            torch.set_rng_state(loader["rng_state"])         # a RandomSampler draws its next orders from it
        self.losses_logger.restore(state["log_rows"])
        self._next_epoch = state["epoch"]
        self._resume = (state["epoch"], loader)

    def _check_training_state(self, state):
        def refuse(field, saved, here):
            raise ValueError("load_training_state: {} is {!r} in the saved state but {!r} here".format(field, saved, here))
        if not isinstance(state, dict) or state.get("format") != TRAINING_STATE_FORMAT:
            raise ValueError("load_training_state: unknown training-state format {!r} (this version reads {})".format(
                state.get("format") if isinstance(state, dict) else type(state).__name__, TRAINING_STATE_FORMAT))
        lf = self.loss_f
        if (self._graphs or self._eligible_steps or self._fused is not None or getattr(lf, "_fused_d", None) is not None
                or lf.n_train_steps != self._steps_at_load):
            raise ValueError("load_training_state: this Trainer has already taken training steps; load the state into "
                             "a new Trainer")
        m = state["model"]
        here = dict(model_type=getattr(self.model, "model_type", None), img_size=list(self.model.img_size),
                    latent_dim=int(self.model.latent_dim))
        for field in ("model_type", "img_size", "latent_dim"):
            if m[field] != here[field]:
                refuse(field, m[field], here[field])
        if state["loss"]["cls"] != type(lf).__name__:
            refuse("the loss class", state["loss"]["cls"], type(lf).__name__)
        saved, hp = state["loss"]["hparams"], loss_hparams(lf)
        for k in sorted(set(saved) | set(hp)):
            if saved.get(k) != hp.get(k):
                refuse("loss hyper-parameter " + k, saved.get(k), hp.get(k))
        world = dist.get_world_size() if is_distributed() else 1
        if state["world_size"] != world:
            refuse("the world size", state["world_size"], world)
        rank = dist.get_rank() if is_distributed() else 0
        if state["rank"] != rank:
            refuse("the rank", state["rank"], rank)
        if (state["factor"] is not None) != hasattr(lf, "call_optimize"):
            refuse("the discriminator state", state["factor"] is not None, hasattr(lf, "call_optimize"))
        if state["factor"] is not None:
            _check_shapes("discriminator", state["factor"]["discriminator"], lf.discriminator.state_dict())
        _check_shapes("model", m["state_dict"], self.model.state_dict())

    def _end_training(self, start):
        if self.gif_visualizer is not None:
            self.gif_visualizer.save_reset()
        self.model.eval()
        delta_time = (default_timer() - start) / 60
        self.logger.info('Finished training after {:.1f} min.'.format(delta_time))

    def _train_epoch(self, data_loader, storer, epoch):
        """training.py:104-135; the epoch loss is accumulated on the device."""
        on_gpu = self.device.type == "cuda"
        batches = _Prefetcher(data_loader, self.device) if on_gpu else data_loader
        tally = _EpochTally(self, len(data_loader), epoch)
        with tally.bar:
            for data, _ in batches:
                tally.add(self._step(data, storer))
        return tally.close()

    def _device_loader(self, loader):
        """The DeviceLoader standing in for `loader`, built (the dataset decoded and uploaded) once per loader."""
        entry = self._device_loaders.get(id(loader))
        if entry is None:
            from disvae.data import device_loader_for
            entry = self._device_loaders[id(loader)] = (loader, device_loader_for(loader, self.device))
        return entry[1]

    def _loss_ring(self):
        if getattr(self, "_ring", None) is None:
            self._ring = _HostLossRing(self.device)
        return self._ring

    # -- the pieces of a training step ----------------------------------------------------------
    def _device_batch(self, data, out=None):
        """`data` as the fp32 batch on the device, written into `out` when given.  uint8 batches (SURVEY.md 8f-3) are
        uploaded as bytes and converted by dv_u8_to_f32 (ToTensor's /255), float batches are copied."""
        if data.dtype == torch.uint8:
            from disvae import ops
            return ops.u8_to_f32(data.to(self.device, non_blocking=True), out=out)
        if out is None:
            return data.to(self.device, non_blocking=True)
        return out.copy_(data, non_blocking=True)

    def _discarded_forward(self, x):
        """FactorVAE: the full-batch forward pass whose result the reference discards (training.py:153), kept for its
        noise draw."""
        if hasattr(self.loss_f, "call_optimize"):
            with torch.no_grad():
                self.model(x)

    def _setup_data_parallel(self):
        """Once, before the first data-parallel forward pass: FactorVAE's discriminator is broadcast from rank 0
        (replicas must start from identical discriminators) and the GradAverage of the model's and the discriminator's
        parameters is built."""
        if self._grad_avg is not None or not is_distributed():
            return
        params = list(self.model.parameters())
        if hasattr(self.loss_f, "call_optimize"):
            broadcast_parameters(self.loss_f.discriminator)
            params += list(self.loss_f.discriminator.parameters())
        self._grad_avg = GradAverage(params)

    def _forward_backward(self, x, storer, **inject):
        """Forward pass, loss and backward pass of the fp32 device batch `x`; returns the detached loss.  Afterwards
        every `p.grad` (FactorVAE: the discriminator's too) holds this process's gradient.  `inject` forwards
        eps1/eps2/perms to FactorKLoss.call_optimize."""
        self._setup_data_parallel()
        if hasattr(self.loss_f, "call_optimize"):             # several optimizers (training.py:160-162): both backward passes
            loss = self.loss_f.call_optimize(x, self.model, self.optimizer, storer, step_optimizers=False, **inject)
        else:
            recon_batch, latent_dist, latent_sample = self.model(x)
            loss = self.loss_f(x, recon_batch, latent_dist, self.model.training, storer, latent_sample=latent_sample)
            self.optimizer.zero_grad()
            loss.backward()
        return loss.detach()

    def _average_grads(self):
        """-> the scale the optimizers apply to the gradients: 1.0 in one process.  Data parallel: every `p.grad` of
        the model and the discriminator becomes the sum over ranks (one flat all-reduce) and the scale is 1/world."""
        return self._grad_avg() if is_distributed() else 1.0

    def _optimizers(self):
        """(optimizer, its FusedAdam or False) of each network a step updates: the model and, for FactorVAE, the
        discriminator."""
        pairs = [(self.optimizer, FusedAdam.lazy(self, "_fused", self.optimizer))]
        lf = self.loss_f
        if hasattr(lf, "call_optimize"):
            pairs.append((lf.optimizer_d, FusedAdam.lazy(lf, "_fused_d", lf.optimizer_d)))
        return pairs

    def _optimizer_steps(self, grad_scale=1.0):
        """The Adam step of each network on its gradients times `grad_scale`: dv_adam_multi when FusedAdam takes the
        optimizer over (a plain torch.optim.Adam on CUDA parameters), else the optimizer's own step() after scaling its
        gradients in place."""
        for opt, fused in self._optimizers():
            if fused:
                fused.step(grad_scale)
                continue
            if grad_scale != 1.0:
                for group in opt.param_groups:
                    for p in group["params"]:
                        if p.grad is not None:
                            p.grad.mul_(grad_scale)
            opt.step()

    # -- whole-step CUDA graph ------------------------------------------------------------------
    def _graph_eligible(self, data):
        lf = self.loss_f
        if not (self.use_cuda_graph and self.device.type == "cuda" and self.model.training):
            return False
        if getattr(self.model, "_eps_queue", None):
            return False
        if hasattr(lf, "call_optimize"):
            # FactorVAE: both backward passes and both Adam steps fit one graph in a single process; under data
            # parallelism the graph ends after the second backward pass (gradient average + both Adam steps follow it)
            if getattr(lf, "_perm_queue", None):
                return False
            if not FusedAdam.lazy(lf, "_fused_d", lf.optimizer_d):
                return False
        if getattr(lf, "global_batch", False) and is_distributed():
            return False                                      # collectives inside the loss node: run eagerly
        # annealing and recording steps are eligible: the coefficients and the loss log follow the loss's device counter
        return bool(FusedAdam.lazy(self, "_fused", self.optimizer))

    def _capture(self, data):
        """The _Graph of a training step on batches like `data`: the discarded forward (FactorVAE), forward + loss +
        backward and, in one process, the Adam steps.  Capture executes nothing, so the host step counters that the
        step's code advances are put back; each replay advances them (`_graph_step`)."""
        if data is self._resident_input:
            static_x = data                                   # the caller refills this very tensor before each step
        else:
            static_x = self._device_batch(data, out=torch.empty(data.shape, dtype=torch.float32, device=self.device))
        lf, ddp = self.loss_f, is_distributed()
        adams = [fused for _, fused in self._optimizers()]
        lf._step_counter(static_x.device, False)             # exists and is in step before capture: nothing to re-write in it
        counters = (lf.n_train_steps, lf._step_dev_host, [f.host_steps for f in adams])
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        launches_before = _native.lib().dv_launch_count()
        with torch.cuda.graph(g):
            self._discarded_forward(static_x)
            static_loss = self._forward_backward(static_x, None)
            if not ddp:                                       # data parallel: the optimizers step after the average
                self._optimizer_steps()
        n_kernels = _native.lib().dv_launch_count() - launches_before
        lf.n_train_steps, lf._step_dev_host = counters[:2]
        for f, n in zip(adams, counters[2]):
            f.host_steps = n
        grads = tuple(p.grad for p in self._grad_avg.params) if ddp else None   # written by every replay
        return _Graph(g, static_x, static_loss, n_kernels, grads, () if ddp else tuple(adams))

    def _graph_step(self, data, storer):
        """fwd + loss + bwd (+ Adam when not data-parallel) of one batch as ONE CUDA graph launch (static
        shapes).  Data-parallel: the graph ends after the backward pass; `.grad` is bound to its static gradient
        tensors, then the gradient average and the Adam steps follow as in an eager step.  The loss's device step
        counter advances inside the graph (annealing coefficients, the device loss log of recording steps); the host
        counters follow here."""
        key = (tuple(data.shape), str(data.dtype))
        entry = self._graphs.get(key)
        if entry is None:
            entry = self._graphs[key] = self._capture(data)
        elif data is not entry.static_x:
            self._device_batch(data, out=entry.static_x)
        lf = self.loss_f
        lf._step_counter(entry.static_x.device, False)       # (re-written only if n_train_steps was set by hand)
        if self._loss_log is not None:
            self._loss_log.expect(lf.n_train_steps + 1, lf.record_loss_every, storer)   # before the replay writes its row
        entry.graph.replay()
        _native.GRAPH_LAUNCHES += entry.n_kernels
        if entry.grads is not None:
            for p, grad in zip(self._grad_avg.params, entry.grads):
                p.grad = grad
            self._optimizer_steps(self._average_grads())
        lf.n_train_steps += 1                                 # the replay's work on the host counters
        lf._step_dev_host += 1
        for f in entry.adams:
            f.host_steps += 1
        return entry.static_loss

    def _step(self, data, storer):
        """One optimisation step; returns the loss as a detached 0-dim device tensor.  On the GPU the scalars of a
        recording step go to the device loss log (eager and graph steps alike) and reach `storer` at the next flush:
        the end of the epoch, `_train_iteration`, or a full log."""
        if self.device.type != "cuda":
            return self._run_step(data, storer)
        if self._loss_log is None:
            self._loss_log = DeviceLossLog(self.device)
        self.loss_f._log = self._loss_log
        try:
            return self._run_step(data, storer)
        finally:
            self.loss_f._log = None

    def _run_step(self, data, storer):
        if self._graph_eligible(data):
            self._eligible_steps += 1
            if self._eligible_steps > 2 or (tuple(data.shape), str(data.dtype)) in self._graphs:   # 2 eager warm-up steps first
                return self._graph_step(data, storer)
        x = self._device_batch(data)
        self._discarded_forward(x)
        loss = self._forward_backward(x, storer)
        if self.model.training or not hasattr(self.loss_f, "call_optimize"):
            # (outside training FactorVAE only evaluates: no backward pass, no update, losses.py:276-278)
            self._optimizer_steps(self._average_grads())
        return loss

    def _train_iteration(self, data, storer):
        """training.py:137-164 (returns a Python float, i.e. synchronises; `storer` holds this step's scalars)."""
        loss = self._step(data, storer).item()
        self._flush_loss_log()
        return loss

    def _flush_loss_log(self):
        if self._loss_log is not None:
            self._loss_log.flush()

    def _grads_only(self, data, storer=None, **inject):
        """Forward + loss + backward (+ the data-parallel gradient average) of one batch WITHOUT an optimizer step:
        afterwards every `p.grad` (and, for FactorVAE, the discriminator's) holds the rank mean, which
        `_optimizer_steps()` consumes as it is.  Used by the parity checks (bench.py `parity` / `ddp_parity`, tests);
        `inject` forwards eps1/eps2/perms to FactorKLoss.call_optimize."""
        loss = self._forward_backward(self._device_batch(data), storer, **inject)
        scale = self._average_grads()
        if scale != 1.0:
            self._grad_avg.flat.mul_(scale)
        return loss


# -- training-state helpers -------------------------------------------------------------------------------------------
def _cpu(obj):
    """`obj` (a state_dict: nested dicts / lists of tensors and Python values) with every tensor copied to the host."""
    if torch.is_tensor(obj):
        return obj.detach().to("cpu", copy=True)
    if isinstance(obj, dict):
        return {k: _cpu(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(_cpu(v) for v in obj)
    return obj


def _philox(key, counter):
    """A Philox stream's key and counter value (None, None before its first draw)."""
    return dict(key=key, offset=None if counter is None else int(counter))


def loss_hparams(loss_f):
    """The loss's settings that a continued run must share: its public int / float / str / bool attributes
    (record_loss_every, rec_dist, steps_anneal, beta, gamma, ...), the step counter excepted."""
    return {k: v for k, v in sorted(vars(loss_f).items())
            if not k.startswith("_") and k != "n_train_steps" and isinstance(v, (bool, int, float, str))}


def _check_shapes(what, saved, here):
    if list(saved) != list(here):
        raise ValueError("load_training_state: the {} has parameters {} in the saved state but {} here".format(
            what, list(saved), list(here)))
    for k, v in saved.items():
        if tuple(v.shape) != tuple(here[k].shape):
            raise ValueError("load_training_state: {} parameter {} is {} in the saved state but {} here".format(
                what, k, tuple(v.shape), tuple(here[k].shape)))


def _loader_shape(loader):
    """(n, batch_size, shuffle, drop_last) of a DeviceLoader or a torch DataLoader."""
    from disvae.data import DeviceLoader
    if isinstance(loader, DeviceLoader):
        return loader.n, loader.batch_size, loader.shuffle, loader.drop_last
    return (len(loader.dataset), loader.batch_size, isinstance(loader.sampler, torch.utils.data.RandomSampler),
            loader.drop_last)


def loader_state(loader):
    """The data-order state of `loader` after the epochs it has run: a DeviceLoader's seed and epoch, or for a host
    loader the CPU RNG state its RandomSampler draws from.  None for no loader."""
    from disvae.data import DeviceLoader
    if loader is None:
        return None
    if isinstance(loader, DeviceLoader):
        n, b, shuffle, drop_last = _loader_shape(loader)
        return dict(kind="device", seed=loader.seed, epoch=loader.epoch, n=n, batch_size=b, shuffle=shuffle,
                    drop_last=drop_last)
    state = dict(kind="host", rng_state=torch.get_rng_state(), n=None, batch_size=None, shuffle=None, drop_last=None)
    if isinstance(loader, torch.utils.data.DataLoader):
        state.update(zip(("n", "batch_size", "shuffle", "drop_last"), _loader_shape(loader)))
    return state


def check_loader_state(saved, loader, device_data=False):
    """ValueError unless `loader` continues the data order `saved` describes: the same kind (a DeviceLoader, also one
    that DISVAE_DEVICE_DATA=1 builds from a DataLoader, or a host loader) over the same number of items, batch size,
    shuffling and drop_last.  No GPU work."""
    from disvae.data import DeviceLoader
    is_dl = isinstance(loader, torch.utils.data.DataLoader)
    kind = "device" if isinstance(loader, DeviceLoader) or (device_data and is_dl) else "host"
    if kind != saved["kind"]:
        raise ValueError("training state: the saved run read a {} loader but this call passes a {} one; the data order "
                         "would differ".format(saved["kind"], kind))
    if saved["n"] is None or not (is_dl or kind == "device"):
        return
    for field, want, got in zip(("n", "batch_size", "shuffle", "drop_last"),
                                (saved["n"], saved["batch_size"], saved["shuffle"], saved["drop_last"]),
                                _loader_shape(loader)):
        if want != got:
            raise ValueError("training state: the loader's {} is {!r} in the saved state but {!r} here".format(
                field, want, got))


def check_metrics_every(metrics_every):
    if isinstance(metrics_every, bool) or not isinstance(metrics_every, int) or metrics_every < 0:
        raise ValueError("metrics_every must be a non-negative integer (0: no metrics), got %r" % (metrics_every,))


def apply_loader_state(saved, loader):
    """A DeviceLoader continues the saved order (its seed and epoch); a host loader's RNG was restored at the load."""
    if saved["kind"] == "device":
        loader.seed, loader.epoch = saved["seed"], saved["epoch"]


# One captured training step (Trainer._graphs): the graph, its input buffer and loss, the native kernels one replay runs,
# under data parallelism the static gradient tensors the replay writes (in GradAverage order; None otherwise), and the
# FusedAdams whose steps the graph holds.
_Graph = namedtuple("_Graph", "graph static_x static_loss n_kernels grads adams")


class _EpochTally:
    """One epoch of a Trainer's bookkeeping: the running loss (on the device), the host loss ring behind the progress
    bar, and at the end the optimizer step counters and the device loss log brought up to date."""

    def __init__(self, trainer, n_batches, epoch):
        self.tr, self.n, self.i = trainer, n_batches, 0
        # own accumulator, updated in place: `loss` may be the CUDA graph's static output tensor, which the next
        # replay overwrites -- never keep a reference to it across steps
        self.loss = torch.zeros((), dtype=torch.float32, device=trainer.device)
        self.ring = trainer._loss_ring() if trainer.device.type == "cuda" else None
        self.bar = trange(n_batches, desc="Epoch {}".format(epoch + 1), leave=False, disable=not trainer.is_progress_bar)

    def add(self, loss):
        self.loss += loss
        if self.ring is not None:
            self.ring.push(loss)                              # async D2H of this step's loss (4 bytes)
        if self.tr.is_progress_bar and self.i % self.tr.sync_every == 0:
            self.bar.set_postfix(loss=self.ring.latest() if self.ring is not None else loss.item())
        self.bar.update()
        self.i += 1

    def close(self):
        """-> the mean loss of the epoch's batches (synchronises)."""
        self.bar.close()
        for fused in (self.tr._fused, getattr(self.tr.loss_f, "_fused_d", None)):
            if fused:
                fused.flush_state()                           # optimizer.state[p]["step"] follows the device counter
        self.tr._flush_loss_log()                             # this epoch's recorded scalars -> storer
        return self.loss.item() / self.n


class _Prefetcher:
    """Iterates a loader of (data, label) batches one step ahead: the host->device copy of batch i+1 is issued
    on a copy stream while step i runs (two device buffers, reused).  Pageable host tensors still work (the copy
    is then synchronous); batches already on the device pass through."""

    def __init__(self, loader, device):
        self.loader, self.device = loader, device
        self.stream = torch.cuda.Stream(device)
        self.bufs = [None, None]
        self.consumed = [None, None]              # main-stream events: buffer may be overwritten after this

    def _upload(self, item, slot):
        data, label = item
        if not torch.is_tensor(data) or data.device.type == "cuda":
            return data, label, None
        buf = self.bufs[slot]
        if buf is None or buf.shape != data.shape or buf.dtype != data.dtype:
            buf = self.bufs[slot] = torch.empty(data.shape, dtype=data.dtype, device=self.device)
        with torch.cuda.stream(self.stream):
            if self.consumed[slot] is not None:
                self.stream.wait_event(self.consumed[slot])
            buf.copy_(data, non_blocking=True)
            ready = torch.cuda.Event()
            ready.record(self.stream)
        return buf, label, ready

    def __iter__(self):
        it = iter(self.loader)
        slot = 0
        try:
            nxt = self._upload(next(it), slot)
        except StopIteration:
            return
        while nxt is not None:
            data, label, ready = nxt
            cur_slot = slot
            slot ^= 1
            try:
                nxt = self._upload(next(it), slot)            # overlaps with the step on `data`
            except StopIteration:
                nxt = None
            main = torch.cuda.current_stream(self.device)
            if ready is not None:
                main.wait_event(ready)
            yield data, label
            if ready is not None:                             # the step that read `data` has been enqueued
                ev = torch.cuda.Event()
                ev.record(main)
                self.consumed[cur_slot] = ev

    def __len__(self):
        return len(self.loader)


class _HostLossRing:
    """Per-step losses copied asynchronously into pinned host memory; `latest()` returns the newest value that
    has already arrived (never blocks)."""

    def __init__(self, device, size=64):
        self.host = torch.zeros(size, dtype=torch.float32).pin_memory()
        self.events = [None] * size
        self.n = 0
        self.size = size

    def push(self, loss):
        k = self.n % self.size
        self.host[k:k + 1].copy_(loss.detach().reshape(1), non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self.events[k] = ev
        self.n += 1

    def latest(self):
        for back in range(1, min(self.n, self.size) + 1):
            k = (self.n - back) % self.size
            if self.events[k] is not None and self.events[k].query():
                return float(self.host[k])
        return float("nan")


class LossesLogger(object):
    """CSV "Epoch,Loss,Value" writer (training.py:167-190).  `rows` keeps the rows written after the header, which a
    training state carries and `restore` writes back."""

    HEADER = ",".join(["Epoch", "Loss", "Value"])

    def __init__(self, file_path_name):
        if os.path.isfile(file_path_name):
            os.remove(file_path_name)
        self.file_path_name = file_path_name
        self.rows = []
        # a logger of its own, not the shared named one: several Trainers in one process (disvae.sweep) each write
        # only their own file
        self.logger = logging.Logger("losses_logger")
        self.logger.parent = logging.getLogger("losses_logger")
        self.logger.setLevel(1)
        self._open()
        self.logger.debug(self.HEADER)

    def _open(self):
        file_handler = logging.FileHandler(self.file_path_name)
        file_handler.setLevel(1)
        self.logger.addHandler(file_handler)

    def log(self, epoch, losses_storer):
        for k, v in losses_storer.items():
            row = ",".join(str(item) for item in [epoch, k, mean(v)])
            self.rows.append(row)
            self.logger.debug(row)

    def restore(self, rows):
        """Rewrite the file as the header and `rows` (a saved run's); later rows are appended to it."""
        for h in list(self.logger.handlers):
            self.logger.removeHandler(h)
            h.close()
        self.rows = list(rows)
        with open(self.file_path_name, "w") as f:
            f.write("".join(line + "\n" for line in [self.HEADER] + self.rows))
        self._open()


def mean(l):
    return sum(l) / len(l)
