#!/usr/bin/env python
"""Cost of the unsupervised scores on the GPU: `dv_unsupervised_fit` at the default shape and at its limits with the
time of each launch, a whole `Sweep.unsupervised_scores` of a c2 sweep, and a c2 sweep epoch with
`unsupervised_every=1` against 0; for comparison, the same scores with numpy / scipy / sklearn on the host.

    python scripts/unsupervised_rate.py [--rounds 3] [--steps 150] [--out FILE]

Fits (correlated Gaussian codes, logvar -2, rows drawn with replacement):
  (D, n) = (10, 10000) and (128, 32768): CUDA-event ms per call, the median of 20 calls after a warm-up, the Jacobi
  sweep counts, and each kernel's device time from torch.profiler over 5 further calls (a run of its own)
Sweep (bench.py's c2 members, seeds 1234 .., over a DeviceLoader of random byte images, `--steps` batches per epoch):
  Sweep.unsupervised_scores   K = 8 members after one training epoch: host clock around the call (draws, gathers, 8
                              encoder passes of 10,000 points, 8 fits, copies, the 16 files), which ends in a synchronise
  epoch, unsupervised_every   one epoch with `sweep.unsupervised_every` = 1 against 0, alternating, after an untimed
                              first epoch
Host: unsupervised_metrics.py's lines (np.cov, slogdet, scipy's sqrtm, np.histogram / np.digitize and sklearn's
mutual_info_score for every pair of latents) for both representations of the same shapes, one process.
Prints the card, its power limit and SM clocks first, then one JSON line per measurement.
"""
import argparse
import json
import logging
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [os.path.join(ROOT, "disentangling-vae_b200"), ROOT, HERE]

import torch  # noqa: E402

SHAPES = [(10, 10000), (128, 32768)]
KERNELS = ("uns_gather", "uns_column", "uns_cov", "uns_eig", "discrete_mi")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return {"torch_name": torch.cuda.get_device_name(),
            "nvidia_smi name, power.limit, clocks.sm, clocks.max.sm": q[torch.cuda.current_device()] if q else None}


def codes(N, D, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    mix = torch.eye(D, device=dev) + 0.6 / D ** 0.5 * torch.randn(D, D, generator=g, device=dev)
    mu = torch.randn(N, D, generator=g, device=dev) @ mix
    return mu.contiguous(), torch.full_like(mu, -2.0)


def event_ms(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e)


def kernel_split(fn, calls=5):
    """Device ms per call of each kernel of KERNELS, from torch.profiler's CUDA activities over `calls` calls."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    split = {k: 0.0 for k in KERNELS}
    for ev in prof.key_averages():
        for k in KERNELS:
            if k in ev.key:
                split[k] += ev.device_time_total / 1e3 / calls
    return split


def host_seconds(x, lv, eps):
    """unsupervised_metrics.py's lines for both representations of the codes x [n, D]."""
    import scipy.linalg
    from sklearn.metrics import mutual_info_score
    t = time.perf_counter()
    for mus in (x.T, (x + np.exp(lv / 2) * eps).T):
        cov = np.cov(mus)
        0.5 * (np.sum(np.log(np.diag(cov))) - np.linalg.slogdet(cov)[1])
        2 * np.trace(cov) - 2 * np.trace(scipy.linalg.sqrtm(cov * np.expand_dims(np.diag(cov), axis=1)))
        d = np.stack([np.digitize(m, np.histogram(m, 20)[1][:-1]) for m in mus])
        for i in range(len(d)):
            for j in range(len(d)):
                mutual_info_score(d[j], d[i])
    return time.perf_counter() - t


def emit(rec, out):
    print(json.dumps(rec), flush=True)
    out.append(rec)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=150, help="batches per c2 epoch")
    ap.add_argument("--out", default=None, help="also write the records as JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("unsupervised_rate.py needs a CUDA device")
    from disvae.data import DeviceLoader
    from disvae.evaluate import unsupervised_draws, unsupervised_fit
    from disvae.sweep import Sweep
    from sweep_rate import ByteImages, members
    import bench
    dev = torch.device("cuda", 0)
    recs = []
    emit({"card": card()}, recs)

    host_inputs = []
    for D, n in SHAPES:
        mu, lv = codes(n, D, 0, dev)
        rows, eps = unsupervised_draws(n, n, D, 1, dev)
        fit = lambda: unsupervised_fit(mu, lv, rows, eps)   # noqa: E731
        fit()
        ms = [event_ms(fit) for _ in range(20)]
        sweeps = unsupervised_fit(mu, lv, rows, eps)[2].cpu().tolist()
        emit({"fit": "D%d_n%d" % (D, n), "D": D, "n": n, "ms_median": statistics.median(ms),
              "jacobi_sweeps [mean R, mean S], [sampled R, sampled S]": sweeps,
              "kernel_ms_per_call": kernel_split(fit)}, recs)
        r = rows.cpu().numpy()
        host_inputs.append((D, n, mu.cpu().numpy()[r].astype(np.float64), lv.cpu().numpy()[r].astype(np.float64),
                            eps.cpu().numpy().astype(np.float64)))
        del mu, lv
        torch.cuda.empty_cache()

    _, img, B, *_ = bench.WORKLOADS["c2"]
    loader = DeviceLoader(ByteImages(args.steps * B, img), B, seed=1234, device=dev)
    logging.getLogger("unsupervised_rate").setLevel(logging.WARNING)
    with tempfile.TemporaryDirectory() as root:
        sweep = Sweep(members("c2", 8, dev, root), seeds=[1234 + j for j in range(8)])
        sweep(loader, epochs=1, checkpoint_every=1000)
        sweep.unsupervised_scores()
        sec = []
        for _ in range(args.rounds):
            torch.cuda.synchronize()
            t = time.perf_counter()
            sweep.unsupervised_scores()
            torch.cuda.synchronize()
            sec.append(time.perf_counter() - t)
        emit({"sweep_unsupervised_scores": "c2", "K": 8, "n": 10000, "ms_median": 1e3 * statistics.median(sec)},
             recs)
        epoch = {0: [], 1: []}
        for _ in range(args.rounds):
            for every in (0, 1):
                torch.cuda.synchronize()
                t = time.perf_counter()
                sweep.unsupervised_every = every
                sweep(loader, epochs=1, checkpoint_every=1000)
                torch.cuda.synchronize()
                epoch[every].append(time.perf_counter() - t)
        emit({"sweep_epoch": "c2", "K": 8, "steps": args.steps,
              "s_unsupervised_every_0": statistics.median(epoch[0]),
              "s_unsupervised_every_1": statistics.median(epoch[1])}, recs)

    for D, n, x, lv, eps in host_inputs:
        emit({"host": "numpy/scipy/sklearn", "D": D, "n": n, "s": host_seconds(x, lv, eps)}, recs)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(recs, f, indent=1)


if __name__ == "__main__":
    main()
