#!/usr/bin/env python
"""Cost of the IRS score on the GPU, at the dSprites shape and at the limits of `dv_irs_fit`, against the numpy
restatement on the host.

    python scripts/irs_score_rate.py [--calls 20] [--out FILE]

Codes are synthetic (no model): on dSprites' factor grid (1, 3, 6, 40, 32, 32; 737,280 items) latent d follows scored
factor d plus noise and the other latents are noise, D = 10, 10,000 drawn rows; at the limits, a grid of eight factors
(4, 5, 6, 7, 8, 9, 10, 4 values; 2,419,200 items, 9.9 GB of fp32 codes), D = 1,024 latents and 32,768 drawn rows.
  * fit:    CUDA-event ms of one `dv_irs_fit` (3 launches), median of --calls after a warm-up call;
  * score:  ms of the whole `disvae.evaluate.irs_score` (draw, factor values, fit, copies, host finish), host clock
            ending in a device synchronise, median of --calls;
  * host:   seconds of tests/irs_reference.py's fp64 restatement of the same fit in numpy, once;
and the largest difference between the GPU and host IRS matrices.  Prints the card and its power limit.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [os.path.join(ROOT, "disentangling-vae_b200"), os.path.join(ROOT, "tests"), HERE]
from eval_rate import card, timed  # noqa: E402

SHAPES = {"dsprites": ([1, 3, 6, 40, 32, 32], 10, 10000),
          "limit": ([4, 5, 6, 7, 8, 9, 10, 4], 1024, 32768)}


def codes(lat_sizes, D, dev, seed=0):
    """mu [N, D] on `dev`: latent d = scored factor d / its size + 0.2 noise, further latents noise."""
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    n = int(np.prod(lat_sizes))
    x = torch.randn(n, D, generator=g, device=dev)
    idx = torch.arange(n, device=dev)
    scored = [k for k, s in enumerate(lat_sizes) if s > 1]
    for d, k in enumerate(scored[:D]):
        stride = int(np.prod(lat_sizes[k + 1:]))
        x[:, d] = (idx // stride % lat_sizes[k]).float() / lat_sizes[k] + 0.2 * x[:, d]
    return x


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the summary JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("irs_score_rate.py needs a CUDA device")
    import irs_reference as R
    from disvae.evaluate import _train_rows, irs_fit, irs_score
    dev = torch.device("cuda", 0)
    summary = {"card": card(), "shapes": {}}
    print(json.dumps({"card": summary["card"]}), flush=True)
    for name, (lat, D, n) in SHAPES.items():
        mu = codes(lat, D, dev)
        _, rows = _train_rows(mu, n, 0)
        factors, values = R.draw_values(lat, rows.cpu().numpy())
        values = torch.from_numpy(values).int().to(dev)
        got = irs_fit(mu, rows, values, 0.99)
        fit_ms = []
        for _ in range(args.calls):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            irs_fit(mu, rows, values, 0.99)
            e1.record()
            torch.cuda.synchronize()
            fit_ms.append(e0.elapsed_time(e1))
        irs_score(mu, lat, num_train=n, seed=0)
        score_ms = [timed(lambda: irs_score(mu, lat, num_train=n, seed=0)) * 1000 for _ in range(args.calls)]
        x = mu[rows].cpu().numpy()
        t0 = time.perf_counter()
        want = R.fit(x, values.cpu().numpy(), 0.99)
        host_s = time.perf_counter() - t0
        M = got[2].cpu().numpy()
        act = want["active"]
        row = {"lat_sizes": lat, "D": D, "n": n, "K": len(factors), "fit_ms": round(float(np.median(fit_ms)), 3),
               "fit_ms_min": round(float(np.min(fit_ms)), 3), "score_ms": round(float(np.median(score_ms)), 3),
               "numpy_s": round(host_s, 2), "IRS": irs_score(mu, lat, num_train=n, seed=0)[0]["IRS"],
               "max_abs_matrix_diff": float(np.abs(M[act] - want["irs_matrix"][act]).max())}
        summary["shapes"][name] = row
        print(json.dumps({name: row}), flush=True)
        del mu
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(summary, fh, indent=1)


if __name__ == "__main__":
    main()
