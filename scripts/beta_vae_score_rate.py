#!/usr/bin/env python
"""Cost of the beta-VAE score on the dSprites-shaped dataset of `eval_rate.py` (737,280 x 1x64x64, lat_sizes
[1, 3, 6, 40, 32, 32]) with a c2 model (beta-TCVAE, batch 1024, latent 10) after one untimed training epoch.

    python scripts/beta_vae_score_rate.py [--rounds 3] [--batch 1000] [--out FILE]

Per round, in this order:
  * features: CUDA-event time of one `dv_pair_abs_diff_mean` launch (15,000 points of L = 64 pairs, D = 10) on the
              encoder means the Evaluator reads (the interleaved q_zCx), 20 launches;
  * fit:      CUDA-event time of one `dv_logistic_fit` launch on those features (the 5 factors of more than one value,
              10,000 training rows), 20 launches;
  * fit_limit: the same at the kernel's limits (D = 128, 32 classes, 10,000 training rows of synthetic features),
              3 launches;
  * score:    `disvae.evaluate.beta_vae_score` from the encodings (draws, both launches, copies), 10 calls;
  * eval:     Evaluator(...)(DeviceLoader.in_order(batch), is_metrics=True) without and with is_beta_vae_score=True;
  * epoch:    one c2 training epoch with metrics_every=1, without and with beta_vae_score=True.
Every host timing ends in a device synchronise.  Prints the card and its power limit (read in the same run), each
round, and the medians over the rounds, with the Newton steps of the fits.
"""
import argparse
import json
import logging
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.join(os.path.dirname(HERE), "disentangling-vae_b200"), HERE]
from eval_rate import ProceduralDSprites, card, timed  # noqa: E402

KEYS = ("features_us", "fit_us", "fit_limit_us", "score_ms", "eval_metrics_s", "eval_metrics_bvae_s", "epoch_metrics_s",
        "epoch_metrics_bvae_s")


def kernel_us(fn, n=20):
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1000 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=1000)
    ap.add_argument("--out", default=None, help="also write the summary JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("beta_vae_score_rate.py needs a CUDA device")
    import disvae
    from disvae.data import DeviceLoader
    from disvae.evaluate import beta_vae_points, beta_vae_score, logistic_fit, pair_abs_diff_mean
    from disvae.models.losses import get_loss_f
    dev = torch.device("cuda", 0)
    print(json.dumps({"card": card()}), flush=True)
    ds = ProceduralDSprites()
    lat_sizes = [int(s) for s in ds.lat_sizes]

    torch.manual_seed(1234)
    model = disvae.init_specific_model("Burgess", (1, 64, 64), 10).to(dev)
    opt = torch.optim.Adam(model.parameters(), lr=5e-4)
    lf = get_loss_f("btcvae", rec_dist="bernoulli", reg_anneal=0, btcvae_A=1, btcvae_B=6, btcvae_G=1, n_data=len(ds))
    save_dir = tempfile.mkdtemp(prefix="dvbvae")
    log = logging.getLogger("beta_vae_score_rate")
    tr = disvae.Trainer(model, opt, lf, device=dev, logger=log, save_dir=save_dir, is_progress_bar=False)
    ev = disvae.Evaluator(model, lf, device=dev, logger=log, save_dir=save_dir, is_progress_bar=False)
    dl = DeviceLoader(ds, 1024, shuffle=True, device=dev)
    tr(dl, epochs=1, checkpoint_every=10 ** 9)                           # warm-up: graph capture, allocator
    ev(dl.in_order(args.batch), is_metrics=True, is_losses=False, is_beta_vae_score=True)

    model.eval()
    mean = ev._compute_q_zCx(dl.in_order(args.batch))[1][0]            # the interleaved view the Evaluator reads
    model.train()
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    (tl, ta, tb), (el, ea, eb) = [beta_vae_points(lat_sizes, c, 64, gen) for c in (10000, 5000)]
    rows_a, rows_b = torch.cat([ta, ea]), torch.cat([tb, eb])
    x = pair_abs_diff_mean(mean, rows_a, rows_b)
    K = sum(s > 1 for s in lat_sizes)
    labels, n_classes = tl.int(), torch.tensor([K], dtype=torch.int32, device=dev)     # every factor is drawn
    # the limits: D = 128, 32 classes, features like the score's (non-negative, one raised dim per class)
    g = torch.Generator(device=dev)
    g.manual_seed(1)
    y_lim = torch.randint(32, (15000,), generator=g, device=dev)
    x_lim = 0.5 * torch.randn(15000, 128, generator=g, device=dev, dtype=torch.float64).abs()
    x_lim[torch.arange(15000, device=dev), y_lim * 4] += 0.2
    nc_lim = torch.tensor([32], dtype=torch.int32, device=dev)
    steps = {"fit": int(logistic_fit(x, labels, n_classes, K, 10000)[2]),
             "fit_limit": int(logistic_fit(x_lim, y_lim[:10000].int(), nc_lim, 32, 10000)[2])}

    rounds = []
    for r in range(args.rounds):
        row = {"round": r}
        row["features_us"] = kernel_us(lambda: pair_abs_diff_mean(mean, rows_a, rows_b))
        row["fit_us"] = kernel_us(lambda: logistic_fit(x, labels, n_classes, K, 10000))
        row["fit_limit_us"] = kernel_us(lambda: logistic_fit(x_lim, y_lim[:10000].int(), nc_lim, 32, 10000), n=3)
        row["score_ms"] = timed(lambda: [beta_vae_score(mean, lat_sizes, seed=s) for s in range(10)]) * 1000 / 10
        row["eval_metrics_s"] = timed(lambda: ev(dl.in_order(args.batch), is_metrics=True, is_losses=False))
        row["eval_metrics_bvae_s"] = timed(lambda: ev(dl.in_order(args.batch), is_metrics=True, is_losses=False,
                                                      is_beta_vae_score=True))
        row["epoch_metrics_s"] = timed(lambda: tr(dl, epochs=1, checkpoint_every=10 ** 9, metrics_every=1,
                                                  metrics_batch_size=args.batch))
        row["epoch_metrics_bvae_s"] = timed(lambda: tr(dl, epochs=1, checkpoint_every=10 ** 9, metrics_every=1,
                                                       metrics_batch_size=args.batch, beta_vae_score=True))
        row = {k: (round(v, 4) if isinstance(v, float) else v) for k, v in row.items()}
        rounds.append(row)
        print(json.dumps(rounds[-1]), flush=True)
    med = {k: float(np.median([x[k] for x in rounds])) for k in KEYS}
    score, helpers = beta_vae_score(mean, lat_sizes, seed=0)
    summary = {"card": card(), "n": len(ds), "batch": args.batch, "median": med, "rounds": rounds, "score": score,
               "newton_steps": dict(steps, score=int(helpers["solver_iterations"]))}
    print(json.dumps(summary), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
