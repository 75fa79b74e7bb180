#!/usr/bin/env python
"""Cost of modularity and explicitness on the GPU, at the dSprites shape and at the limits of `dv_explicitness_fit`.

    python scripts/modularity_explicitness_rate.py [--rounds 3] [--shapes dsprites,dsprites_d128,limit] [--out FILE]

Shapes (fp32 codes whose first latents follow the factors, plus Gaussian noise; the rest noise):
  dsprites       lat_sizes [1, 3, 6, 40, 32, 32] (737,280 rows), D = 10, 10,000 training / 5,000 test rows
  dsprites_d128  the same with D = 128, the latent limit
  limit          lat_sizes [256, 2, 64] (32,768 rows), D = 128, 32,768 training / 5,000 test rows: every limit at once
                 (256 classes, 128 latents, 32,768 training rows), one round
Per shape: the CUDA-event time of one `dv_discrete_mutual_info` and of one `dv_explicitness_fit` (three launches),
then of the whole `modularity_explicitness` (draws, labels, both entry points, copies) ended by a device synchronise,
after one untimed warm-up call of each (none at the limit, where one call is the measurement); the Newton steps of
every fit; then, in a run of its own under torch.profiler, the device time of each of the four kernels.  Prints the
card and its power limit first, then one JSON line per shape, and the medians over the rounds.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.join(os.path.dirname(HERE), "disentangling-vae_b200"), HERE]
from eval_rate import card  # noqa: E402

SHAPES = {"dsprites": ([1, 3, 6, 40, 32, 32], 10, 10000, 5000, 3),
          "dsprites_d128": ([1, 3, 6, 40, 32, 32], 128, 10000, 5000, 3),
          "limit": ([256, 2, 64], 128, 32768, 5000, 1)}
KERNELS = ("discrete_mi_kernel", "standardise_kernel", "explicitness_fit_kernel", "auc_kernel")


def code(lat_sizes, D, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    n = int(np.prod(lat_sizes))
    v = torch.from_numpy(np.stack(np.unravel_index(np.arange(n), lat_sizes), 1)).float().to(dev)
    x = torch.randn(n, D, generator=g, device=dev)
    K = min(D, len(lat_sizes))
    x[:, :K] = v[:, :K] / torch.tensor(lat_sizes[:K], device=dev).float() + 0.2 * x[:, :K]
    return x


def event_ms(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=None, help="rounds per shape (default: 3, 1 at the limit)")
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("modularity_explicitness_rate.py needs a CUDA device")
    from disvae import evaluate
    dev = torch.device("cuda", 0)
    results = {"card": card()}
    print(json.dumps(results), flush=True)
    for name in args.shapes.split(","):
        lat, D, n, m, rounds = SHAPES[name]
        rounds = args.rounds or rounds
        x = code(lat, D, 1, dev)
        g = torch.Generator(device=dev).manual_seed(2)
        tr = torch.randint(x.shape[0], (n,), generator=g, device=dev)
        te = torch.randint(x.shape[0], (m,), generator=g, device=dev)
        factors, train_cls, test_cls, n_classes, counts, _ = evaluate.sap_labels(lat, tr, te)
        S = counts.shape[1]

        def mi():
            evaluate.discrete_mutual_info(x, tr, train_cls, n_classes, S)

        out = {}

        def fit():
            out["fit"] = evaluate.explicitness_fit(x, tr, te, train_cls, test_cls, n_classes, S)

        def score():
            evaluate.modularity_explicitness(x, lat, num_train=n, num_test=m, seed=3)

        if name != "limit":
            mi(), fit(), score()
            torch.cuda.synchronize()
        rows = []
        for r in range(rounds):
            row = {"shape": name, "round": r, "mi_ms": event_ms(mi), "fit_ms": event_ms(fit)}
            row["newton_steps"] = out["fit"][2].tolist()
            if name != "limit":
                row["score_ms"] = event_ms(score)
            rows.append(row)
            print(json.dumps(row), flush=True)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            mi(), fit()
            torch.cuda.synchronize()
        per = {}
        for ev in prof.key_averages():
            for k in KERNELS:
                if k in ev.key:
                    per[k] = per.get(k, 0.0) + ev.device_time_total / 1000.0
        summary = {"shape": name, "lat_sizes": lat, "D": D, "num_train": n, "num_test": m, "rounds": rounds,
                   "kernel_ms": per}
        for key in ("mi_ms", "fit_ms", "score_ms"):
            if key in rows[0]:
                summary["median_" + key] = float(np.median([r[key] for r in rows]))
        print(json.dumps(summary), flush=True)
        results[name] = {"rounds": rows, "summary": summary}
        del out["fit"]
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
