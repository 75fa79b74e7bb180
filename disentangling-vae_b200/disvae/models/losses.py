"""Disentanglement losses with the reference's API (disvae/models/losses.py) on the sm_90a
kernels: one fused reconstruction+KL kernel (ops.VaeLossFn), the beta-TCVAE decomposition kernel
(ops.BtcvaeFn), the FactorVAE heads and, beyond the reference, the DIP-VAE covariance penalty (ops.DipFn).  Logged scalars are fetched with ONE device->host copy
per recorded step instead of one `.item()` per value (losses.py:151,384-389,447,476-478).
"""
import abc

import torch
from torch import optim

from disvae import ops
from disvae._native import DIST
from .discriminator import Discriminator

LOSSES = ["VAE", "betaH", "betaB", "factor", "btcvae"]
DIP_LOSSES = ["dipI", "dipII"]      # not in LOSSES (the reference's `main.py -l` choices): reachable from Python
RECON_DIST = ["bernoulli", "laplace", "gaussian"]


def get_loss_f(loss_name, **kwargs_parse):
    """Return the loss object for the argparse dictionary (losses.py:22-49)."""
    kwargs_all = dict(rec_dist=kwargs_parse["rec_dist"], steps_anneal=kwargs_parse["reg_anneal"])
    if loss_name == "betaH":
        return BetaHLoss(beta=kwargs_parse["betaH_B"], **kwargs_all)
    elif loss_name == "VAE":
        return BetaHLoss(beta=1, **kwargs_all)
    elif loss_name == "betaB":
        return BetaBLoss(C_init=kwargs_parse["betaB_initC"], C_fin=kwargs_parse["betaB_finC"],
                         gamma=kwargs_parse["betaB_G"], **kwargs_all)
    elif loss_name == "factor":
        return FactorKLoss(kwargs_parse["device"], gamma=kwargs_parse["factor_G"],
                           disc_kwargs=dict(latent_dim=kwargs_parse["latent_dim"]),
                           optim_kwargs=dict(lr=kwargs_parse["lr_disc"], betas=(0.5, 0.9)), **kwargs_all)
    elif loss_name == "btcvae":
        return BtcvaeLoss(kwargs_parse["n_data"], alpha=kwargs_parse["btcvae_A"], beta=kwargs_parse["btcvae_B"],
                          gamma=kwargs_parse["btcvae_G"], **kwargs_all)
    elif loss_name in DIP_LOSSES:
        return DipVAELoss(loss_name[len("dip"):], lambda_od=kwargs_parse.get("dip_lambda_od", 10.),
                          lambda_d=kwargs_parse.get("dip_lambda_d"), **kwargs_all)
    else:
        assert loss_name not in LOSSES
        raise ValueError("Uknown loss : {}".format(loss_name))


def _dist_id(distribution):
    if distribution not in DIST:
        assert distribution not in RECON_DIST
        raise ValueError("Unkown distribution: {}".format(distribution))
    return DIST[distribution]


def linear_annealing(init, fin, step, annealing_steps):
    """losses.py:511-518"""
    if annealing_steps == 0:
        return fin
    assert fin > init
    return min(init + (fin - init) * step / annealing_steps, fin)


def _record(storer, names, values):
    """ONE device->host transfer for every logged scalar of this step."""
    if storer is None:
        return
    flat = torch.cat([v.detach().reshape(-1) for v in values]).tolist()
    i = 0
    for name, v in zip(names, values):
        n = v.numel()
        if isinstance(name, str):
            storer[name].append(flat[i])
        else:                       # a list of names for a vector
            for nm, x in zip(name, flat[i:i + n]):
                storer[nm].append(x)
        i += n


def _kl_names(latent_dim):
    return ['kl_loss_' + str(i) for i in range(latent_dim)]


def _flat_names(names, lens):
    """The storer keys `_record` appends to, in its order, for values of `lens` entries each."""
    flat = []
    for name, n in zip(names, lens):
        flat += [name] if isinstance(name, str) else list(name)[:n]
    return flat


class DeviceLossLog:
    """The scalars of recording training steps kept on the device until the host asks for them.

    A recording step's kernels write its values into one row of a device ring (ops: the `log` of the loss kernels,
    dv_loss_record), so the step has no host synchronisation and can be replayed from a CUDA graph.  The host side knows
    which steps record (`expect`: the reference's rule on n_train_steps) and for which storer; `flush` copies the ring
    back once and appends every pending row to its storer with exactly the keys, order and values `_record` appends.
    The ring is flushed before a new row could overwrite a pending one (every `capacity` recording steps at most)."""

    def __init__(self, device, capacity=256):
        self.device, self.capacity = device, capacity
        self.ring = self.host = None
        self.names = None               # keys of one row, in `_record`'s order
        self.pending = []               # (row, storer) in step order

    def spec(self, every, names, values):
        """The _native.LossLog of one step: `values` as `_record` takes them, None for the loss the launch computes."""
        from disvae import _native
        lens = [1 if v is None else v.numel() for v in values]
        self.layout(_flat_names(names, lens))
        flat = self.names
        if len(values) > _native.LOSS_LOG_MAX_SRC:
            raise ValueError("at most %d logged values per step" % _native.LOSS_LOG_MAX_SRC)
        log = _native.LossLog()
        log.ring, log.cap, log.ncols, log.every, log.nsrc = self.ring.data_ptr(), self.capacity, len(flat), every, len(values)
        for k, (v, n) in enumerate(zip(values, lens)):
            if v is not None:
                _native.require_cuda_f32(v)
                if not v.is_contiguous():
                    raise ValueError("logged values must be contiguous")
            log.src[k] = None if v is None else v.data_ptr()
            log.len[k] = n
        return log

    def layout(self, names):
        """Keys of one row (the ring is allocated with the first layout; one log serves one loss)."""
        if self.ring is None:
            self.ring = torch.zeros(self.capacity, len(names), dtype=torch.float32, device=self.device)
            self.host = torch.zeros(self.capacity, len(names), dtype=torch.float32)
            if self.ring.is_cuda:
                self.host = self.host.pin_memory()
        if self.names is not None and names != self.names:
            raise ValueError("one DeviceLossLog serves one loss: got keys %s after %s" % (names, self.names))
        self.names = names

    def expect(self, step, every, storer):
        """Training step `step` is about to run with `storer`: note its row if it records.  The device writes the row of
        every recording step, storer or not, so a row still pending is read back before it can be overwritten."""
        if step % every != 1:
            return
        row = (step - 1) // every % self.capacity
        if any(r == row for r, _ in self.pending):
            self.flush()
        if storer is not None:
            self.pending.append((row, storer))

    def flush(self):
        """One copy of the ring to the host (after everything enqueued so far), then the pending rows into their storers."""
        if not self.pending:
            return
        self.host.copy_(self.ring, non_blocking=True)
        if self.ring.is_cuda:
            done = torch.cuda.Event()
            done.record()
            done.synchronize()
        rows = self.host.tolist()
        for row, storer in self.pending:
            for name, v in zip(self.names, rows[row]):
                storer[name].append(v)
        self.pending.clear()


def permutation_key(seed, salt=0):
    """Philox key of FactorVAE's latent permutations in a process seeded with `seed` (`salt`: parallel.rank_salt())."""
    return ((int(seed) ^ 0x9E3779B97F4A7C15) + salt) & 0xFFFFFFFFFFFFFFFF


class BaseLoss(abc.ABC):
    """losses.py:52-114: step counter, record-every-50 policy, common options.

    Besides the host counter `n_train_steps` each loss owns an int64 device copy of it, advanced by the loss kernel of
    every training step (ops.LossCombineSchedFn / BetaBLossFn), from which the annealing coefficients and the device
    loss log are computed: a step replayed from a CUDA graph anneals and records like an eager one.  `_log` is the
    DeviceLossLog of the Trainer step in progress (None otherwise: scalars go to the storer through `_record`)."""

    def __init__(self, record_loss_every=50, rec_dist="bernoulli", steps_anneal=0):
        self.n_train_steps = 0
        self.record_loss_every = record_loss_every
        self.rec_dist = rec_dist
        self.steps_anneal = steps_anneal
        self._step_dev = None           # the device counter (created on the first training call)
        self._step_dev_host = 0         # its value once the work enqueued so far has run
        self._log = None

    @abc.abstractmethod
    def __call__(self, data, recon_data, latent_dist, is_train, storer, **kwargs):
        """Loss of a batch: data/recon_data [B,C,H,W], latent_dist = (mean, logvar) [B,D]."""

    def _pre_call(self, is_train, storer):
        if is_train:
            self.n_train_steps += 1
            if self._log is not None:                       # recorded on the device, handed to `storer` by the flush
                self._log.expect(self.n_train_steps, self.record_loss_every, storer)
                return None
        if not is_train or self.n_train_steps % self.record_loss_every == 1:
            return storer
        return None

    def _step_counter(self, device, advancing):
        """The device step counter, holding what the host counter held before this step: n_train_steps - 1 when the
        launch about to be enqueued advances it (`advancing`, after _pre_call), n_train_steps otherwise.  Re-written
        only when the two have drifted apart (n_train_steps set by hand), so never inside a captured step."""
        want = self.n_train_steps - 1 if advancing else self.n_train_steps
        if self._step_dev is None or self._step_dev.device != device:
            self._step_dev = torch.full((1,), want, dtype=torch.int64, device=device)
        elif self._step_dev_host != want:
            self._step_dev.fill_(want)
        self._step_dev_host = self.n_train_steps
        return self._step_dev

    def _log_spec(self, is_train, names, values):
        """The device loss log of this call (None: none -- outside a Trainer step, or not training)."""
        if not is_train or self._log is None:
            return None
        return self._log.spec(self.record_loss_every, names, values)

    def _combine(self, out, b, coef_a, coef_b, annealed, is_train, log):
        """ops.LossCombineSchedFn: coefficient number `annealed` (coef_a, then coef_b; or each number of a tuple) is
        multiplied by linear_annealing(0, 1, step, steps_anneal) on the device."""
        step = self._step_counter(out.device, True) if is_train else None
        mask = sum(1 << k for k in annealed) if isinstance(annealed, tuple) else 1 << annealed
        loss, _ = ops.LossCombineSchedFn.apply(out, b, coef_a, coef_b, mask, (0, 1, self.steps_anneal),
                                               is_train, step, log)
        return loss

    def _rec_kl(self, data, recon_data, latent_dist):
        """(recon_loss, kl_total, per-dim kl vector) from the fused kernel."""
        out = self._rec_kl_vec(data, recon_data, latent_dist)
        return out[0], out[1], out[2:]

    def _rec_kl_vec(self, data, recon_data, latent_dist):
        """The fused kernel's whole output [2 + D] = (recon_loss, kl_total, kl_dim_0 ..): for ops.LossCombineFn."""
        return ops.VaeLossFn.apply(recon_data, data, latent_dist[0], latent_dist[1], _dist_id(self.rec_dist))


class BetaHLoss(BaseLoss):
    """beta-VAE (Higgins et al.), losses.py:117-153: rec + anneal * beta * KL."""

    def __init__(self, beta=4, **kwargs):
        super().__init__(**kwargs)
        self.beta = beta

    def __call__(self, data, recon_data, latent_dist, is_train, storer, **kwargs):
        storer = self._pre_call(is_train, storer)
        out = self._rec_kl_vec(data, recon_data, latent_dist)
        rec_loss, kl_loss, kl_dims = out[0], out[1], out[2:]
        names = ['recon_loss', 'kl_loss', _kl_names(kl_dims.numel()), 'loss']
        log = self._log_spec(is_train, names, [rec_loss, kl_loss, kl_dims, None])
        loss = self._combine(out, None, [1.0, self.beta], None, 1, is_train, log)     # rec + anneal * (beta * kl)
        _record(storer, names, [rec_loss, kl_loss, kl_dims, loss])
        return loss


class BetaBLoss(BaseLoss):
    """beta-VAE with capacity annealing (Burgess et al.), losses.py:156-202."""

    def __init__(self, C_init=0., C_fin=20., gamma=100., **kwargs):
        super().__init__(**kwargs)
        self.gamma = gamma
        self.C_init = C_init
        self.C_fin = C_fin

    def __call__(self, data, recon_data, latent_dist, is_train, storer, **kwargs):
        storer = self._pre_call(is_train, storer)
        out = self._rec_kl_vec(data, recon_data, latent_dist)
        rec_loss, kl_loss, kl_dims = out[0], out[1], out[2:]
        names = ['recon_loss', 'kl_loss', _kl_names(kl_dims.numel()), 'loss']
        log = self._log_spec(is_train, names, [rec_loss, kl_loss, kl_dims, None])
        assert not (is_train and self.steps_anneal) or self.C_fin > self.C_init     # linear_annealing's own check
        step = self._step_counter(out.device, True) if is_train else None
        # rec + gamma * |kl - C| with C = linear_annealing(C_init, C_fin, step, steps_anneal) (C_fin outside training)
        loss, _ = ops.BetaBLossFn.apply(out, self.gamma, (self.C_init, self.C_fin, self.steps_anneal), is_train, step, log)
        _record(storer, names, [rec_loss, kl_loss, kl_dims, loss])
        return loss


class FactorKLoss(BaseLoss):
    """FactorVAE, Algorithm 2 of Kim & Mnih (losses.py:205-313)."""

    def __init__(self, device, gamma=10., disc_kwargs={}, optim_kwargs=dict(lr=5e-5, betas=(0.5, 0.9)), **kwargs):
        super().__init__(**kwargs)
        self.gamma = gamma
        self.device = device
        self.discriminator = Discriminator(**disc_kwargs).to(self.device)
        self.optimizer_d = optim.Adam(self.discriminator.parameters(), **optim_kwargs)
        self._perm_offset = None
        self._perm_queue = []          # injected permutations (parity tests), consumed FIFO
        self._fused_d = None           # FusedAdam over optimizer_d (built lazily once the discriminator is on CUDA)
        # Data parallel only (no meaning for one process): False = every rank permutes its own second half-batch (the
        # reference handed that shard as its batch, SURVEY.md 8e); True = every rank takes its rows of ONE permutation of
        # the all-gathered second halves, so the "product of marginals" samples no longer depend on the number of ranks.
        # DISVAE_GLOBAL_FACTOR=1 turns it on without touching main.py.
        import os
        self.global_batch = os.environ.get("DISVAE_GLOBAL_FACTOR") == "1"
        self._gperm_offset = None

    def _step_d(self):
        """Discriminator Adam step: dv_adam_multi when optimizer_d is a plain CUDA Adam."""
        from disvae.fused import FusedAdam
        fused = FusedAdam.lazy(self, "_fused_d", self.optimizer_d)
        if fused:
            fused.step()
        else:
            self.optimizer_d.step()

    def __call__(self, *args, **kwargs):
        raise ValueError("Use `call_optimize` to also train the discriminator")

    def _perm_state(self, device):
        if self._perm_offset is None or self._perm_offset.device != device:
            from disvae.parallel import rank_salt
            self.seed_permutations(permutation_key(torch.initial_seed(), rank_salt()), device)
        return self._perm_seed, self._perm_offset

    def seed_permutations(self, key, device):
        """Fix the Philox key of the latent permutations (what the first training step would take from
        torch.initial_seed(); permutation_key) and start its counter at 0 on `device`."""
        self._perm_seed = int(key)
        self._perm_offset = torch.zeros(1, dtype=torch.int64, device=device)

    def _global_perm_state(self, device):
        """Key of the global permutation: rank 0's seed, unsalted (one process with the same seed draws the same
        permutation), and an offset that advances by world*h*D on every rank."""
        if self._gperm_offset is None or self._gperm_offset.device != device:
            from disvae.parallel import broadcast_u64
            self._gperm_seed = broadcast_u64(int(torch.initial_seed()) ^ 0x9E3779B97F4A7C15)
            self._gperm_offset = torch.zeros(1, dtype=torch.int64, device=device)
        return self._gperm_seed, self._gperm_offset

    def _permute_global(self, latent_sample2, perms=None):
        """This rank's rows [rank*h, (rank+1)*h) of the permutation of the second halves of all ranks, rank-major.
        `perms`: injected global permutations [D, world*h]."""
        import torch.distributed as dist
        from disvae.parallel import all_gather_rows, check_equal_rows
        h = latent_sample2.size(0)
        check_equal_rows(h)                                      # before the gather: unequal sizes would hang it
        z2_all = all_gather_rows(latent_sample2)
        row0 = dist.get_rank() * h
        if perms is not None:
            return ops.permute_dims_rows(z2_all, row0, h, perms)
        seed, off = self._global_perm_state(latent_sample2.device)
        return ops.permute_dims_rows(z2_all, row0, h, None, seed, off)

    def call_optimize(self, data, model, optimizer, storer, eps1=None, eps2=None, perms=None, step_optimizers=True):
        """losses.py:243-313.  `eps1`/`eps2`/`perms` optionally inject the noise of the two
        halves and the per-dimension permutations ([D, B/2] int64; [D, world*B/2] in global-batch mode) for parity tests.
        `step_optimizers=False`: both backward passes run, neither optimizer steps -- the Trainer steps them
        itself (under data parallelism after the gradients of all ranks are averaged)."""
        storer = self._pre_call(model.training, storer)
        half = data.size(0) // 2
        parts = data.split(half)
        data1, data2 = parts[0], parts[1]

        recon_batch, latent_dist, latent_sample1 = model(data1, eps=eps1)
        out = self._rec_kl_vec(data1, recon_batch, latent_dist)
        rec_loss, kl_loss, kl_dims = out[0], out[1], out[2:]

        if not model.training:
            d_z = self.discriminator(latent_sample1)
            tc_loss = ops.FactorTcFn.apply(d_z)
            vae_loss = self._combine(out, tc_loss, [1.0, 1.0], [self.gamma], 2, False, None)
            _record(storer, ['recon_loss', 'kl_loss', _kl_names(kl_dims.numel()), 'loss', 'tc_loss'],
                    [rec_loss, kl_loss, kl_dims, vae_loss, tc_loss])
            return vae_loss

        # The reference evaluates the discriminator twice (losses.py:262 on z of the first half, :286 on the permuted z of
        # the second half) with a backward pass in between.  Nothing in that backward pass feeds the second evaluation, so
        # the second half is encoded and permuted first (same order of noise draws: eps1, eps2, permutation) and the
        # discriminator sees [z1; z_perm] in ONE pass of 2 x half rows: its layers are launch-latency bound at these sizes,
        # so one forward and one backward pass through it disappear from the step.  Rows are independent in every layer:
        # d_z and d_z_perm are bit-identical to the two separate evaluations.
        with torch.no_grad():                                    # (the reference detaches z_perm: no graph is needed)
            latent_sample2 = model.sample_latent(data2, eps=eps2)
            if perms is None and self._perm_queue:
                perms = self._perm_queue.pop(0)
            from disvae.parallel import is_distributed
            if self.global_batch and is_distributed():
                z_perm = self._permute_global(latent_sample2, perms)
            elif perms is None:
                seed, off = self._perm_state(latent_sample2.device)
                z_perm = ops.permute_dims(latent_sample2, None, seed, off)
            else:
                z_perm = ops.permute_dims(latent_sample2, perms)
        with ops.mlp_note_parts(2):
            d_all = self.discriminator(torch.cat([latent_sample1, z_perm]))
        d_z, d_z_perm = d_all[:half], d_all[half:]
        tc_loss = ops.FactorTcFn.apply(d_z)                      # mean(d_z[:,0] - d_z[:,1])
        vae_loss = self._combine(out, tc_loss, [1.0, 1.0], [self.gamma], 2, True, None)   # rec + kl + anneal*gamma*tc

        optimizer.zero_grad()
        with ops.mlp_input_grad_only():                          # the discriminator's own gradients of this pass are zeroed below
            vae_loss.backward(retain_graph=True)

        d_tc_loss = ops.FactorCeFn.apply(d_z, d_z_perm)           # 0.5 * (CE(d_z, 0) + CE(d_z_perm, 1))

        self.optimizer_d.zero_grad()
        d_tc_loss.backward()                                     # also reaches the encoder through d_z (trap T5)
        if step_optimizers:
            optimizer.step()
            self._step_d()

        names = ['recon_loss', 'kl_loss', _kl_names(kl_dims.numel()), 'loss', 'tc_loss', 'discrim_loss']
        values = [rec_loss, kl_loss, kl_dims, vae_loss, tc_loss, d_tc_loss]
        log = self._log_spec(True, names, values)
        if log is not None:                                      # the discriminator loss exists only now: own launch
            ops.loss_record(self._step_dev, log)
        _record(storer, names, values)
        return vae_loss


class BtcvaeLoss(BaseLoss):
    """beta-TCVAE (Chen et al.), losses.py:316-391: rec + alpha*MI + beta*TC + anneal*gamma*dwKL,
    minibatch-stratified sampling by default (is_mss, trap T4)."""

    def __init__(self, n_data, alpha=1., beta=6., gamma=1., is_mss=True, **kwargs):
        super().__init__(**kwargs)
        self.n_data = n_data
        self.beta = beta
        self.alpha = alpha
        self.gamma = gamma
        self.is_mss = is_mss
        # Data parallel only (no meaning for one process): False = every rank applies the estimator to its own shard
        # (the reference handed that shard as its batch, SURVEY.md 8e); True = the estimator of the GLOBAL batch
        # (all-gather of z/mu/logvar, row-block kernel, reduce-scatter of the column gradients; SURVEY.md 8f-1), whose
        # value no longer depends on the number of ranks.  DISVAE_GLOBAL_BTCVAE=1 turns it on without touching main.py.
        import os
        self.global_batch = os.environ.get("DISVAE_GLOBAL_BTCVAE", "0") == "1"

    def __call__(self, data, recon_batch, latent_dist, is_train, storer, latent_sample=None):
        storer = self._pre_call(is_train, storer)
        out = self._rec_kl_vec(data, recon_batch, latent_dist)
        rec_loss, kl_loss, kl_dims = out[0], out[1], out[2:]
        from disvae.parallel import is_distributed
        if self.global_batch and is_train and is_distributed():
            terms = ops.BtcvaeGlobalFn.apply(latent_sample, latent_dist[0], latent_dist[1], self.n_data, self.is_mss, None)
        else:
            terms = ops.btcvae_terms(latent_sample, latent_dist[0], latent_dist[1], self.n_data, self.is_mss)
        mi_loss, tc_loss, dw_kl_loss = terms[0], terms[1], terms[2]
        names = ['recon_loss', 'loss', 'mi_loss', 'tc_loss', 'dw_kl_loss', 'kl_loss', _kl_names(kl_dims.numel())]
        log = self._log_spec(is_train, names, [rec_loss, None, mi_loss, tc_loss, dw_kl_loss, kl_loss, kl_dims])
        # rec + (alpha*mi + beta*tc + anneal*gamma*dw_kl) as one launch (the kl entries of `out` only feed the log)
        loss = self._combine(out, terms, [1.0], [self.alpha, self.beta, self.gamma], 3, is_train, log)
        _record(storer, names, [rec_loss, loss, mi_loss, tc_loss, dw_kl_loss, kl_loss, kl_dims])
        return loss


class DipVAELoss(BaseLoss):
    """DIP-VAE-I / DIP-VAE-II (Kumar et al. 2018, eq. 6 and section 3; not in the reference):
    rec + kl + anneal * (lambda_od * od + lambda_d * dd) with od = sum_{i != j} C_ij^2, dd = sum_i (C_ii - 1)^2 and
    C = Cov_mu (dip_type "I") or Cov_mu + diag(mean exp(logvar)) ("II"), the biased covariance of the batch's encoder
    means (ops.DipFn).  lambda_d=None takes the ratios of Locatello et al. 2019: 10 * lambda_od for I, lambda_od for II.
    Under torch.distributed the penalty is that of each rank's shard (the gradient average follows it)."""

    def __init__(self, dip_type="I", lambda_od=10., lambda_d=None, **kwargs):
        import math
        import numbers
        if dip_type not in ops.DIP_TYPES:
            raise ValueError("Unknown DIP-VAE type {!r}: expected one of {}".format(dip_type, sorted(ops.DIP_TYPES)))
        if lambda_d is None and isinstance(lambda_od, numbers.Real):
            lambda_d = 10. * lambda_od if dip_type == "I" else lambda_od
        for name, v in (("lambda_od", lambda_od), ("lambda_d", lambda_d)):
            if isinstance(v, bool) or not isinstance(v, numbers.Real) or not math.isfinite(v) or v < 0:
                raise ValueError("DIP-VAE {} must be a finite number >= 0, got {!r}".format(name, v))
        super().__init__(**kwargs)
        self.dip_type = dip_type
        self.lambda_od = float(lambda_od)
        self.lambda_d = float(lambda_d)

    def __call__(self, data, recon_batch, latent_dist, is_train, storer, **kwargs):
        storer = self._pre_call(is_train, storer)
        out = self._rec_kl_vec(data, recon_batch, latent_dist)
        rec_loss, kl_loss, kl_dims = out[0], out[1], out[2:]
        terms = ops.dip_terms(latent_dist[0], latent_dist[1], self.dip_type)
        od, dd = terms[0], terms[1]
        names = ['recon_loss', 'kl_loss', _kl_names(kl_dims.numel()), 'dip_od_loss', 'dip_d_loss', 'loss']
        log = self._log_spec(is_train, names, [rec_loss, kl_loss, kl_dims, od, dd, None])
        # rec + kl + anneal * (lambda_od * od + lambda_d * dd) as one launch
        loss = self._combine(out, terms, [1.0, 1.0], [self.lambda_od, self.lambda_d], (2, 3), is_train, log)
        _record(storer, names, [rec_loss, kl_loss, kl_dims, od, dd, loss])
        return loss


# ---- functional forms kept for API parity with the reference module ---------------------
def _reconstruction_loss(data, recon_data, distribution="bernoulli", storer=None):
    """losses.py:394-449"""
    b, d = recon_data.size(0), 1
    zeros = torch.zeros(b, d, dtype=torch.float32, device=recon_data.device)
    out = ops.VaeLossFn.apply(recon_data, data, zeros, zeros, _dist_id(distribution))
    _record(storer, ['recon_loss'], [out[0]])
    return out[0]


def _kl_normal_loss(mean, logvar, storer=None):
    """losses.py:452-480"""
    dummy = torch.full((mean.size(0), 4), 0.5, dtype=torch.float32, device=mean.device)
    out = ops.VaeLossFn.apply(dummy, dummy, mean, logvar, DIST["gaussian"])
    _record(storer, ['kl_loss', _kl_names(mean.size(1))], [out[1], out[2:]])
    return out[1]


def _permute_dims(latent_sample, perms=None):
    """losses.py:483-508; without `perms` the per-dimension permutations follow the reference's
    CPU `torch.randperm` stream (trap T7)."""
    b, d = latent_sample.shape
    if perms is None:
        perms = torch.stack([torch.randperm(b) for _ in range(d)])
    return ops.permute_dims(latent_sample, perms)


def _get_log_pz_qz_prodzi_qzCx(latent_sample, latent_dist, n_data, is_mss=True):
    """losses.py:523-544 (values only)."""
    return ops.btcvae_rowstats(latent_sample, latent_dist[0], latent_dist[1], n_data, is_mss)
