"""Host-side checks of the annealed, graph-capturable training step (no GPU needed).

* `device_coef` restates the arithmetic of the device annealing coefficient (dv_glue.cu `anneal_value` and the
  coefficient rounding of dv_loss_combine_sched_fwd / dv_betab_loss_fwd): it must equal, bit for bit, what the host path
  handed to the kernels -- Python's linear_annealing(...) * coefficient rounded to float32 -- at every step of the
  schedules the reference ships.
* DeviceLossLog's record selection, ring rows and flush order against BaseLoss._pre_call + _record (the host path).
"""
from collections import defaultdict

import numpy as np
import pytest
import torch

from disvae.models import losses as L


def device_coef(base, init, fin, steps, steps_anneal, is_train=True):
    """float32 coefficients of the device path for an array of steps: A = min(init + (fin - init) * step / steps_anneal,
    fin) in double, in that operation order (A = fin when steps_anneal == 0 or outside training), then float32(A * base)
    -- or float32(A) for beta-VAE_B's capacity C (base None)."""
    steps = np.asarray(steps, dtype=np.int64)
    f64 = np.float64
    if not is_train or steps_anneal == 0:
        a = np.full(steps.shape, f64(fin))
    else:
        x = f64(init) + (f64(fin) - f64(init)) * steps.astype(np.float64) / f64(steps_anneal)
        a = np.where(f64(fin) < x, f64(fin), x)
    return (a if base is None else a * f64(base)).astype(np.float32)


def host_coef(base, init, fin, step, steps_anneal, is_train=True):
    """What the host path computed: the Python value that ctypes / torch rounded to float32."""
    a = L.linear_annealing(init, fin, step, steps_anneal) if is_train else fin
    return np.float32(a if base is None else a * base)


# (base, init, fin, steps_anneal): linear_annealing(0, 1, step, reg_anneal) times beta (β-VAE_H: 4, 10), gamma (FactorVAE
# 6.4, β-TCVAE 1) -- and β-VAE_B's capacity C = linear_annealing(C_init, C_fin, step, reg_anneal), no coefficient
SCHEDULES = [(4, 0, 1, 10000), (10, 0, 1, 10000), (6.4, 0, 1, 10000), (1, 0, 1, 10000),
             (4, 0, 1, 1), (10, 0, 1, 1), (6.4, 0, 1, 1),
             (None, 0, 25, 100000), (None, 0, 50, 100000), (None, 0., 25., 100000), (None, 0.5, 30., 7),
             (4, 0, 1, 7), (6.4, 0, 1, 7), (None, 0, 25, 7)]


@pytest.mark.parametrize("base,init,fin,steps_anneal", SCHEDULES)
def test_device_coefficient_formula_is_bit_identical_to_host(base, init, fin, steps_anneal):
    steps = np.arange(0, steps_anneal + 3)
    got = device_coef(base, init, fin, steps, steps_anneal)
    want = np.array([host_coef(base, init, fin, int(s), steps_anneal) for s in steps], dtype=np.float32)
    bad = np.nonzero(got.view(np.uint32) != want.view(np.uint32))[0]
    assert bad.size == 0, [(int(steps[i]), float(got[i]), float(want[i])) for i in bad[:5]]
    assert got[-1] == np.float32(fin if base is None else fin * base)        # annealing has ended


@pytest.mark.parametrize("base,init,fin", [(4, 0, 1), (10, 0, 1), (6.4, 0, 1), (None, 0, 25), (None, 0, 50)])
def test_device_coefficient_without_annealing_and_outside_training(base, init, fin):
    steps = np.arange(0, 60)
    for is_train in (True, False):
        got = device_coef(base, init, fin, steps, 0 if is_train else 10000, is_train)
        want = [host_coef(base, init, fin, int(s), 0 if is_train else 10000, is_train) for s in steps]
        assert got.view(np.uint32).tolist() == np.array(want, dtype=np.float32).view(np.uint32).tolist()


class _Logged(L.BaseLoss):
    """A loss whose logged values are a function of the step: `_record` (host path) or the device log (rows written
    by a stand-in for the kernel, which records on the counter value exactly like dv_glue.cu's log_record)."""
    D = 3

    def values(self):
        s = float(self.n_train_steps)
        return [torch.tensor(s + 0.25), torch.tensor(-s), torch.arange(self.D, dtype=torch.float32) + s / 8]

    def names(self):
        return ['recon_loss', 'loss', L._kl_names(self.D)]

    def __call__(self, data, recon_data, latent_dist, is_train, storer, **kwargs):
        storer = self._pre_call(is_train, storer)
        vals = self.values()
        if is_train and self._log is not None:
            log = self._log
            log.layout(L._flat_names(self.names(), [v.numel() for v in vals]))
            s, every = self.n_train_steps, self.record_loss_every
            if s % every == 1:                                # the kernel: predicated on the counter, not on the storer
                log.ring[(s - 1) // every % log.capacity] = torch.cat([v.reshape(-1) for v in vals])
        L._record(storer, self.names(), vals)


@pytest.mark.parametrize("every,capacity", [(5, 256), (5, 3), (50, 2), (1, 4), (2, 1), (7, 5)])
def test_device_log_selection_and_flush_order_match_pre_call(every, capacity):
    """Steps 1..200 over four 'epochs' (storers), some steps without a storer, flushes at epoch ends and whenever the
    ring fills: every storer gets exactly the keys, order and values of the host path."""
    host, dev = _Logged(record_loss_every=every), _Logged(record_loss_every=every)
    dev._log = L.DeviceLossLog(torch.device("cpu"), capacity=capacity)
    sh, sd = [], []
    for step in range(1, 201):
        if (step - 1) % 50 == 0:
            sh.append(defaultdict(list))
            sd.append(defaultdict(list))
        use = step % 11 != 4                                  # a caller without a storer now and then
        host(None, None, None, True, sh[-1] if use else None)
        dev(None, None, None, True, sd[-1] if use else None)
        assert len(dev._log.pending) <= capacity
        if step % 50 == 0:
            dev._log.flush()                                  # epoch end
        if step % 37 == 0:                                    # evaluation calls: always logged, never counted
            ev_h, ev_d = defaultdict(list), defaultdict(list)
            host(None, None, None, False, ev_h)
            dev(None, None, None, False, ev_d)
            assert list(ev_h.items()) == list(ev_d.items()) and len(ev_h) == 2 + _Logged.D
    assert host.n_train_steps == dev.n_train_steps == 200
    for a, b in zip(sh, sd):
        assert list(a.items()) == list(b.items())             # keys in insertion order, every value bit for bit
    assert sum(len(st["loss"]) for st in sh) == sum(1 for s in range(1, 201) if s % every == 1 and s % 11 != 4)


def test_flat_names_follow_record():
    names = ['recon_loss', 'loss', 'mi_loss', 'tc_loss', 'dw_kl_loss', 'kl_loss', L._kl_names(4)]
    assert L._flat_names(names, [1] * 6 + [4]) == names[:6] + ['kl_loss_0', 'kl_loss_1', 'kl_loss_2', 'kl_loss_3']
