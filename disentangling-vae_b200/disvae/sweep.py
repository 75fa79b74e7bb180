"""Train a sweep of models at once on one GPU: concurrent CUDA-graph steps over one resident dataset.

    members = [Trainer(model_k, optimizer_k, loss_k, device=dev, save_dir=dir_k) for k ...]
    Sweep(members, seeds=[seed_k ...])(loader, epochs=30, checkpoint_every=10)

Every member is an ordinary `Trainer` and keeps its own model, optimizer, loss, save_dir, train_losses.log,
checkpoints, GIF visualizer and progress output.  A member's loss may be any of `losses.LOSSES` (VAE, betaH, betaB,
factor, btcvae) or `losses.DIP_LOSSES` (dipI, dipII), with its own hyper-parameters.  All members read the same batches in the same order: one
`DeviceLoader` permutation per epoch and one gather per step, into one buffer that every member's captured graph reads.
Each member runs on its own stream (its two eager warm-up steps, its capture, then one graph replay per step), so the
replays of different members overlap on the GPU; the next gather waits for all of them.

Member k's result is bit-identical to a lone `Trainer` run with the same settings over the same loader seed after
`torch.manual_seed(seeds[k])`: the members share no scratch buffer, workspace or side stream (`ops.owner`), and their
Philox keys come from `seeds` (`philox_keys`) rather than from `torch.initial_seed()` at first use.

`Sweep.udr` (and `udr_every`) ranks the members against each other with the UDR score, which needs no known factors
of variation (`disvae.evaluate.udr`).  `Sweep.unsupervised_scores` (and `unsupervised_every`) writes every member's
unsupervised scores of its mean and sampled representations, which need none either
(`disvae.evaluate.unsupervised_scores`).

Limits: one process, one GPU, the CUDA-graph path.  Members must not have taken a training step yet (call the same
Sweep again to continue, or, in a new process, give every member the training state it saved with `save_state=True`
through `load_training_state`).  They must share the device and the input image shape, and
their optimizers (and FactorVAE's discriminator optimizer) must be ones `FusedAdam` takes over.  Anything else raises
`ValueError` before any GPU work.
"""
import contextlib
import itertools
import numbers
import weakref
from collections import defaultdict
from timeit import default_timer

import torch

from disvae import ops
from disvae.data import DeviceLoader, device_loader_for
from disvae.evaluate import (Evaluator, check_epoch_scores, check_resident_metrics, check_udr,
                             check_unsupervised_scores, evaluation_rng, evaluation_seed, score_evaluator_args,
                             select_scores, write_epoch_metrics, write_udr, write_unsupervised_scores)
from disvae.fused import FusedAdam
from disvae.models.losses import permutation_key
from disvae.models.vae import noise_key
from disvae.parallel import is_distributed
from disvae.training import Trainer, _EpochTally, apply_loader_state, check_loader_state, check_metrics_every

_tokens = itertools.count()          # ops.owner tokens: one per Trainer that ever joined a sweep


def philox_keys(seed):
    """(reparameterisation-noise key, FactorVAE permutation key) that a lone single-process run seeded with
    `torch.manual_seed(seed)` fixes at its first training step."""
    return noise_key(seed), permutation_key(seed)


def check_udr_every(udr_every):
    _check_every("udr_every", udr_every, "UDR")


def check_unsupervised_every(unsupervised_every):
    _check_every("unsupervised_every", unsupervised_every, "unsupervised scores")


def _check_every(name, every, what):
    if isinstance(every, bool) or not isinstance(every, int) or every < 0:
        raise ValueError("%s must be a non-negative integer (0: no %s), got %r" % (name, what, every))


class Sweep:
    """Sweep(members, seeds, udr_every=0, unsupervised_every=0): train the Trainers `members` together; `seeds[k]`
    plays the role of member k's `torch.manual_seed` for the draws made during training (reparameterisation noise,
    FactorVAE permutations).
    `udr_every` > 0 (the attribute of that name, which may be changed between calls) ranks the members with the UDR
    score during training: every call writes each member's `udr-{epoch}.log` and `udr_helpers-{epoch}.pth` after
    epochs 0, e, 2e, ... and its last, what `udr` writes after that epoch (UDR over all members, seeded with
    `evaluation_seed(loader.seed, epoch)`), independently of `metrics_every` and without known factors.
    `unsupervised_every` > 0 (an attribute too) writes each member's `unsupervised_scores-{epoch}.log` and
    `unsupervised_scores_helpers-{epoch}.pth` after the same epochs of its own count, what `unsupervised_scores` writes
    after that epoch (seeded per member, with `evaluation_seed(member's noise key, epoch)`), independently of
    `metrics_every` and `udr_every` and without known factors."""

    udr_every = 0
    unsupervised_every = 0

    def __init__(self, members, seeds, udr_every=0, unsupervised_every=0):
        check_udr_every(udr_every)
        check_unsupervised_every(unsupervised_every)
        self.udr_every = udr_every
        self.unsupervised_every = unsupervised_every
        self.members, self.seeds = list(members), list(seeds)
        if not self.members:
            raise ValueError("Sweep: no members")
        if len(self.seeds) != len(self.members):
            raise ValueError("Sweep: %d members but %d seeds" % (len(self.members), len(self.seeds)))
        for s in self.seeds:
            if not isinstance(s, numbers.Integral) or isinstance(s, bool):
                raise ValueError("Sweep: seeds must be integers, got %r" % (s,))
        if is_distributed():
            raise ValueError("Sweep: torch.distributed is not supported; a sweep trains its members in one process on "
                             "one GPU (run lone Trainers under data parallelism instead)")
        for k, m in enumerate(self.members):
            if not isinstance(m, Trainer):
                raise ValueError("Sweep: member %d is a %s, not a disvae.Trainer" % (k, type(m).__name__))
            if not m.use_cuda_graph:
                raise ValueError("Sweep: member %d has use_cuda_graph=False (DISVAE_CUDA_GRAPH=0); a sweep replays "
                                 "each member's captured CUDA graph and has no eager path" % k)
            if m._graphs or m._eligible_steps or m.loss_f.n_train_steps != m._steps_at_load:
                # its graph would read scratch shared with every other Trainer, and its Philox keys are already fixed
                # (a member that loaded a training state has taken no step in this process: it is accepted)
                raise ValueError("Sweep: member %d has already taken training steps; a sweep starts from members that "
                                 "have not (call the same Sweep again to continue training)" % k)
        for what in ("model", "optimizer", "loss_f"):
            if len({id(getattr(m, what)) for m in self.members}) < len(self.members):
                raise ValueError("Sweep: members share a %s object; each member needs its own" % what)
        img = tuple(self.members[0].model.img_size)
        for k, m in enumerate(self.members):
            if tuple(m.model.img_size) != img:
                raise ValueError("Sweep: member %d takes %s images but member 0 takes %s; members must share the "
                                 "input batch shape" % (k, tuple(m.model.img_size), img))
        self.img_size = img
        self._inputs = {}                 # kept across calls: the members' captured graphs read these buffers
        self._device_loaders = {}         # id(DataLoader) -> (DataLoader, its DeviceLoader), converted once
        self.loader = None                # the DeviceLoader of the latest call (what `evaluate` reads)
        self.streams = None               # one per member, made at the first call
        devs = {self._cuda_device(k, m) for k, m in enumerate(self.members)}
        if len(devs) > 1:
            raise ValueError("Sweep: members are on different devices %s; a sweep runs on one GPU" % sorted(map(str, devs)))
        self.device = devs.pop()
        if udr_every:
            self._check_udr()
        if unsupervised_every:
            self._check_unsupervised()
        for k, m in enumerate(self.members):
            opts = [("optimizer", m.optimizer)]
            if hasattr(m.loss_f, "call_optimize"):
                opts.append(("discriminator optimizer", m.loss_f.optimizer_d))
            for what, opt in opts:
                if not FusedAdam.supports(opt):
                    raise ValueError("Sweep: member %d's %s (%s) is not a plain torch.optim.Adam over CUDA fp32 "
                                     "parameters (no amsgrad, weight decay or maximize), which the graph path needs"
                                     % (k, what, type(opt).__name__))
            if m.model._eps_queue or getattr(m.loss_f, "_perm_queue", None):
                raise ValueError("Sweep: member %d has injected noise or permutations queued" % k)

    @staticmethod
    def _cuda_device(k, m):
        dev = torch.device(m.device)
        if dev.type != "cuda":
            raise ValueError("Sweep: member %d is on %s; a sweep runs on a CUDA device" % (k, dev))
        return torch.device("cuda", torch.cuda.current_device() if dev.index is None else dev.index)

    def _loader(self, data_loader):
        """The DeviceLoader of the sweep, after the checks that need no GPU work."""
        if isinstance(data_loader, DeviceLoader):
            shape = tuple(data_loader.data.shape[1:])
            if data_loader.device != self.device:
                raise ValueError("Sweep: the DeviceLoader holds its data on %s, the members are on %s"
                                 % (data_loader.device, self.device))
        elif isinstance(data_loader, torch.utils.data.DataLoader):
            shape = tuple(data_loader.dataset[0][0].shape)
        else:
            raise ValueError("Sweep: expected a disvae.data.DeviceLoader or a torch DataLoader, got %s"
                             % type(data_loader).__name__)
        if shape != self.img_size:
            raise ValueError("Sweep: the loader yields %s images, the members take %s" % (shape, self.img_size))
        if isinstance(data_loader, DeviceLoader):
            return data_loader
        entry = self._device_loaders.get(id(data_loader))
        if entry is None:                 # later calls continue its epochs, as a Trainer with DISVAE_DEVICE_DATA=1 does
            entry = self._device_loaders[id(data_loader)] = (data_loader, device_loader_for(data_loader, self.device))
        return entry[1]

    def __call__(self, data_loader, epochs=10, checkpoint_every=10, save_state=False, metrics_every=0,
                 metrics_batch_size=1000, factor_score=False, sap_score=False, beta_vae_score=False):
        """Train every member for `epochs` epochs over `data_loader` (a DeviceLoader, or a DataLoader converted to one
        once per Sweep), like `Trainer.__call__` for each.  Calling again continues as a lone Trainer called again
        does: step counters, Adam state, Philox counters and the loader's epochs carry on.  `save_state=True` writes
        each member's training state into its own save_dir; members that loaded one continue from it.
        `metrics_every` writes each member's `metrics-{epoch}.log` as `Trainer.__call__` does, one member after
        another on the caller's stream, over the one resident copy; `factor_score=True`, `sap_score=True` and
        `beta_vae_score=True` add each member's FactorVAE, SAP and beta-VAE scores of those epochs.  With
        `self.udr_every` > 0 the members' UDR files of those epochs are written too, and with
        `self.unsupervised_every` > 0 their unsupervised scores (see the class)."""
        scores = select_scores(locals())
        first, loader_state = self._resume()
        if loader_state is not None:
            check_loader_state(loader_state, data_loader, device_data=True)
        check_metrics_every(metrics_every)
        udr_every = self.udr_every
        check_udr_every(udr_every)
        if udr_every:
            self._check_udr()
        unsupervised_every = self.unsupervised_every
        check_unsupervised_every(unsupervised_every)
        if unsupervised_every:
            self._check_unsupervised()
        if metrics_every:
            check_resident_metrics(data_loader, metrics_batch_size, device_data=True)
        for m in self.members:
            check_epoch_scores(scores, metrics_every, data_loader, m.model.latent_dim)
        loader = self._loader(data_loader)
        for m in self.members:
            m._resume = None
        if loader_state is not None:
            apply_loader_state(loader_state, loader)
        self.loader = loader
        start = default_timer()
        with torch.cuda.device(self.device):
            self._run(loader, first, epochs, checkpoint_every, save_state, start, metrics_every, metrics_batch_size,
                      scores, udr_every, unsupervised_every)

    def evaluate(self, is_metrics=True, is_losses=True, batch_size=1000, is_factor_score=False, is_sap_score=False,
                 is_beta_vae_score=False):
        """Every member's `Evaluator(...)(loader.in_order(batch_size), is_metrics, is_losses)` over the loader of the
        latest call, into its save_dir (`metrics.log`, `metric_helpers.pth`, `test_losses.log`, as `main.py
        --is-eval-only` writes them), with the index draws seeded as the metrics after its latest epoch
        (`disvae.evaluate.evaluation_rng`); its `metrics.log` equals that epoch's `metrics-{epoch}.log`.
        `is_factor_score=True` also writes `factor_vae_score.log` and `factor_vae_score_helpers.pth`, seeded as the score
        after its latest epoch (`disvae.evaluate.evaluation_seed`), `is_sap_score=True` `sap_score.log` and
        `sap_score_helpers.pth`, and `is_beta_vae_score=True` `beta_vae_score.log` and `beta_vae_score_helpers.pth`,
        seeded the same way.  The UDR files of the members come from `udr`."""
        scores = select_scores(locals(), "is_")
        if self.loader is None:
            raise ValueError("Sweep.evaluate: the sweep has no loader yet; train it first (sweep(loader, ...))")
        if is_metrics:
            check_resident_metrics(self.loader, batch_size, device_data=True)
        elif int(batch_size) < 1:
            raise ValueError("Sweep.evaluate: batch_size must be positive, got %d" % int(batch_size))
        for s in scores:
            for m in self.members:
                s.check(self.loader.dataset, m.model.latent_dim)
        with torch.cuda.device(self.device):
            for m in self.members:
                key, epoch = m.model._noise_state(self.device)[0], m._next_epoch - 1
                score_args = score_evaluator_args(scores, evaluation_seed(key, epoch))
                with evaluation_rng(self.device, key, epoch):
                    Evaluator(m.model, m.loss_f, device=self.device, logger=m.logger, save_dir=m.save_dir,
                              is_progress_bar=m.is_progress_bar)(self.loader.in_order(batch_size), is_metrics=is_metrics,
                                                                 is_losses=is_losses, **score_args)

    def udr(self, num_points=1000, seed=None, correlation="lasso", groups=None):
        """UDR (Duan et al. 2020) of the members over the loader of the latest call -> (scores, helpers) of
        `disvae.evaluate.udr`; member k's score is `scores["model_scores"][k]`.  Every member's save_dir gets `udr.log`
        ({"UDR": its score}) and `udr_helpers.pth` (the helpers with "member" = k and the drawn "rows").  The points
        are drawn with `seed`, by default `evaluation_seed(loader.seed, latest epoch)`, which depends on neither the
        order of the members nor their seeds.  `groups` partitions the member indices (None: one group of all)."""
        if self.loader is None:
            raise ValueError("Sweep.udr: the sweep has no loader yet; train it first (sweep(loader, ...))")
        groups = self._check_udr(num_points, correlation, groups)
        if seed is None:
            seed = evaluation_seed(self.loader.seed, self.members[0]._next_epoch - 1)
        with torch.cuda.device(self.device):
            return write_udr([m.model for m in self.members], self.loader, [m.save_dir for m in self.members], seed,
                             loggers=[m.logger for m in self.members], num_points=num_points,
                             correlation=correlation, groups=groups)

    def unsupervised_scores(self, num_train=10000, seed=None):
        """Every member's unsupervised scores (`disvae.evaluate.unsupervised_scores`) over the loader of the latest
        call -> [(scores, helpers)] in member order.  Member k's save_dir gets `unsupervised_scores.log` and
        `unsupervised_scores_helpers.pth`.  Each member encodes only its own drawn rows, seeded with `seed`, by default
        `evaluation_seed(its noise key, latest epoch)` -- the rule of the metrics, so a member's files do not depend on
        the other members."""
        if self.loader is None:
            raise ValueError("Sweep.unsupervised_scores: the sweep has no loader yet; train it first (sweep(loader, ...))")
        self._check_unsupervised(num_train)
        out = []
        with torch.cuda.device(self.device):
            for m in self.members:
                s = self._unsupervised_seed(m, m._next_epoch - 1) if seed is None else seed
                out.append(write_unsupervised_scores(m.model, self.loader, m.save_dir, s, logger=m.logger,
                                                     num_train=num_train))
        return out

    def _unsupervised_seed(self, m, epoch):
        return evaluation_seed(m.model._noise_state(self.device)[0], epoch)

    def _check_unsupervised(self, num_train=10000):
        for m in self.members:
            check_unsupervised_scores(m.model.latent_dim, num_train)

    def _check_udr(self, num_points=1000, correlation="lasso", groups=None):
        return check_udr(len(self.members), [m.model.latent_dim for m in self.members],
                         [m.model.img_size for m in self.members], num_points, correlation, groups)

    def _resume(self):
        """(first epoch, saved loader state) of the members' loaded training states, (0, None) if none has one.
        Members that loaded states must all have stopped at the same epoch of the same data order."""
        pending = [m._resume for m in self.members]
        if all(r is None for r in pending):
            return 0, None
        for k, r in enumerate(pending):
            if r is None:
                raise ValueError("Sweep: member %d has not loaded a training state but others have; resume every "
                                 "member or none" % k)
            epoch, loader = r
            if loader is None or loader["kind"] != "device":
                raise ValueError("Sweep: member %d's training state was not saved over a DeviceLoader; a sweep "
                                 "continues only the data order of one" % k)
            if epoch != pending[0][0] or loader != pending[0][1]:
                raise ValueError("Sweep: member %d's training state (epoch %d, loader %r) is not where member 0's "
                                 "(epoch %d, loader %r) stopped" % (k, epoch, loader, pending[0][0], pending[0][1]))
        return pending[0]

    @contextlib.contextmanager
    def _member(self, k):
        """Member k's stream is current and its kernels use its own scratch, workspaces and side stream."""
        with torch.cuda.stream(self.streams[k]), ops.owner(self.members[k]._sweep_token):
            yield

    def _run(self, loader, first, epochs, checkpoint_every, save_state, start, metrics_every, metrics_batch_size,
             scores, udr_every=0, unsupervised_every=0):
        members = self.members
        main = torch.cuda.current_stream(self.device)
        if self.streams is None:
            self.streams = [torch.cuda.Stream(self.device) for _ in members]
        for m, seed in zip(members, self.seeds):
            if getattr(m, "_sweep_token", None) is None:
                m._sweep_token = ("sweep", next(_tokens))
                weakref.finalize(m, ops.release, m._sweep_token)     # with the member go its graphs and their scratch
            # The keys are fixed before the member's first draw and never again: its graph bakes in the address of
            # each Philox counter, and a later call continues the counters as a lone Trainer called again does.
            noise, perm = philox_keys(seed)
            if m.model._rng_offset is None:
                m.model.seed_noise(noise, self.device)
            if hasattr(m.loss_f, "seed_permutations") and m.loss_f._perm_offset is None:
                m.loss_f.seed_permutations(perm, self.device)
            m._data_loader = loader
            m.model.train()
        done = [None] * len(members)      # each member's stream after its latest step
        inputs = self._inputs             # batch size -> the buffer the gather writes and every member's graph reads
        last = first + epochs - 1
        try:
            for epoch in range(first, first + epochs):
                storers = [defaultdict(list) for _ in members]
                tallies = []
                for k, m in enumerate(members):
                    with self._member(k):
                        tallies.append(_EpochTally(m, len(loader), epoch))
                for idx in loader.epoch_indices():
                    x = inputs.get(idx.numel())
                    if x is None:
                        x = inputs[idx.numel()] = torch.empty((idx.numel(),) + self.img_size, dtype=torch.float32,
                                                              device=self.device)
                    for ev in done:                                # the members have read the previous batch
                        if ev is not None:
                            main.wait_event(ev)
                    ops.gather_u8_to_f32(loader.data, idx, out=x)
                    gathered = torch.cuda.Event()
                    gathered.record(main)
                    for k, m in enumerate(members):
                        self.streams[k].wait_event(gathered)
                        with self._member(k):
                            m._resident_input = x
                            tallies[k].add(m._step(x, storers[k]))
                            done[k] = torch.cuda.Event()
                            done[k].record()
                for k, m in enumerate(members):
                    with self._member(k):
                        m._end_epoch(epoch, storers[k], tallies[k].close(), checkpoint_every,
                                     save_state=save_state and (epoch % checkpoint_every == 0 or epoch == last))
                        done[k] = torch.cuda.Event()
                        done[k].record()
                if metrics_every and (epoch % metrics_every == 0 or epoch == last):
                    for ev in done:                                # every member has ended the epoch
                        main.wait_event(ev)
                    for m in members:                              # the next gather, on `main`, waits for these
                        write_epoch_metrics(m.model, loader, epoch, metrics_batch_size, m.save_dir, m.logger, scores)
                if udr_every and (epoch % udr_every == 0 or epoch == last):
                    for ev in done:                                # every member has ended the epoch
                        main.wait_event(ev)
                    write_udr([m.model for m in members], loader, [m.save_dir for m in members],
                              evaluation_seed(loader.seed, epoch), epoch, [m.logger for m in members])
                if unsupervised_every and (epoch % unsupervised_every == 0 or epoch == last):
                    for ev in done:                                # every member has ended the epoch
                        main.wait_event(ev)
                    for m in members:
                        write_unsupervised_scores(m.model, loader, m.save_dir, self._unsupervised_seed(m, epoch), epoch,
                                                  m.logger)
        finally:
            for ev in done:
                if ev is not None:
                    main.wait_event(ev)
            for m in members:
                m._resident_input = None
        for k, m in enumerate(members):
            with self._member(k):
                m._end_training(start)
