#!/usr/bin/env python
"""Cost of the UDR score on the GPU: `dv_udr_fit` at the default shape and at its limits, a whole `Sweep.udr` of a c2
sweep, and a c2 sweep epoch with `udr_every=1` against 0; for comparison, the same pair fits with sklearn / scipy on
the host.

    python scripts/udr_rate.py [--rounds 3] [--steps 150] [--host-k 8,16] [--out FILE]

Fits (synthetic codes: each model a signed permutation of shared Gaussian factors, mixed slightly, plus noise):
  default  K = 8, D = 10, n = 1000, Lasso and Spearman: CUDA-event ms per call, the median of 20 calls after a warm-up
  limits   (K, D, n) = (32, 128, 1000), (409, 10, 1000), (4096, 1, 1000) and (8, 10, 16384), both modes: one call per
           round after a warm-up, median over the rounds
Sweep (bench.py's c2 members, seeds 1234 .., over a DeviceLoader of random byte images, `--steps` batches per epoch):
  Sweep.udr           K = 8 members after one training epoch: host clock around the call (draw, gather, 8 encoder
                      passes of 1000 points, dv_udr_fit, copies, the 16 files), which ends in a synchronise
  epoch, udr_every    one epoch with `sweep.udr_every` = 1 against 0, alternating, after an untimed first epoch
Host: sklearn's Lasso(alpha=0.1) (its default tol, as udr.py uses it) and scipy's spearmanr for every ordered pair of
K models in `--host-k`, D = 10, n = 1000, one process.
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

LIMITS = [(32, 128, 1000), (409, 10, 1000), (4096, 1, 1000), (8, 10, 16384)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return {"torch_name": torch.cuda.get_device_name(),
            "nvidia_smi name, power.limit, clocks.sm, clocks.max.sm": q[torch.cuda.current_device()] if q else None}


def codes(K, n, D, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    F = torch.randn(n, D, generator=g, device=dev)
    mu = torch.empty(K, n, D, device=dev)
    for k in range(K):
        perm = torch.randperm(D, generator=g, device=dev)
        sign = torch.where(torch.rand(D, generator=g, device=dev) < 0.5, -1.0, 1.0)
        mix = torch.eye(D, device=dev)[perm] * sign + 0.2 * torch.randn(D, D, generator=g, device=dev)
        mu[k] = F @ mix + 0.3 * torch.randn(n, D, generator=g, device=dev)
    return mu.contiguous(), torch.full_like(mu, -2.0)


def event_ms(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e)


def host_seconds(mu, kind):
    from scipy.stats import spearmanr
    from sklearn.linear_model import Lasso
    from sklearn.preprocessing import StandardScaler
    K = mu.shape[0]
    z = [StandardScaler().fit_transform(mu[k]) for k in range(K)]
    t = time.perf_counter()
    for i in range(K):
        for j in range(K):
            if i == j:
                continue
            if kind == "lasso":
                Lasso(alpha=0.1).fit(z[i], z[j])
            else:
                spearmanr(mu[i], mu[j])
    return time.perf_counter() - t


def emit(rec, out):
    print(json.dumps(rec), flush=True)
    out.append(rec)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=150, help="batches per c2 epoch")
    ap.add_argument("--host-k", default="8,16")
    ap.add_argument("--out", default=None, help="also write the records as JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("udr_rate.py needs a CUDA device")
    from disvae.data import DeviceLoader
    from disvae.evaluate import udr_fit
    from disvae.sweep import Sweep
    from sweep_rate import ByteImages, members
    import bench
    dev = torch.device("cuda", 0)
    recs = []
    emit({"card": card()}, recs)

    mu, lv = codes(8, 1000, 10, 0, dev)
    for mode in ("lasso", "spearman"):
        udr_fit(mu, lv, mode)
        ms = [event_ms(lambda: udr_fit(mu, lv, mode)) for _ in range(20)]
        iters = int(udr_fit(mu, lv, mode)[3].max())
        emit({"fit": "default", "K": 8, "D": 10, "n": 1000, "mode": mode, "ms_median": statistics.median(ms),
              "max_sweeps": iters}, recs)
    for K, D, n in LIMITS:
        mu, lv = codes(K, n, D, 1, dev)
        for mode in ("lasso", "spearman"):
            udr_fit(mu, lv, mode)
            ms = [event_ms(lambda: udr_fit(mu, lv, mode)) for _ in range(args.rounds)]
            emit({"fit": "limit", "K": K, "D": D, "n": n, "mode": mode, "ms_median": statistics.median(ms),
                  "max_sweeps": int(udr_fit(mu, lv, mode)[3].max())}, recs)
        del mu, lv
        torch.cuda.empty_cache()

    _, img, B, *_ = bench.WORKLOADS["c2"]
    loader = DeviceLoader(ByteImages(args.steps * B, img), B, seed=1234, device=dev)
    logging.getLogger("udr_rate").setLevel(logging.WARNING)
    with tempfile.TemporaryDirectory() as root:
        sweep = Sweep(members("c2", 8, dev, root), seeds=[1234 + j for j in range(8)])
        sweep(loader, epochs=1, checkpoint_every=1000)
        sweep.udr()
        sec = []
        for _ in range(args.rounds):
            torch.cuda.synchronize()
            t = time.perf_counter()
            sweep.udr()
            torch.cuda.synchronize()
            sec.append(time.perf_counter() - t)
        emit({"sweep_udr": "c2", "K": 8, "n": 1000, "ms_median": 1e3 * statistics.median(sec)}, recs)
        epoch = {0: [], 1: []}
        for _ in range(args.rounds):
            for every in (0, 1):
                torch.cuda.synchronize()
                t = time.perf_counter()
                sweep.udr_every = every
                sweep(loader, epochs=1, checkpoint_every=1000)
                torch.cuda.synchronize()
                epoch[every].append(time.perf_counter() - t)
        emit({"sweep_epoch": "c2", "K": 8, "steps": args.steps, "s_udr_every_0": statistics.median(epoch[0]),
              "s_udr_every_1": statistics.median(epoch[1])}, recs)

    for K in (int(k) for k in args.host_k.split(",")):
        mu, _ = codes(K, 1000, 10, 2, dev)
        mu = mu.cpu().numpy().astype(np.float64)
        for kind in ("lasso", "spearman"):
            emit({"host": kind, "K": K, "D": 10, "n": 1000, "pairs": K * (K - 1), "s": host_seconds(mu, kind)}, recs)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(recs, f, indent=1)


if __name__ == "__main__":
    main()
