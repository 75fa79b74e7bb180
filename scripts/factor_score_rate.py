#!/usr/bin/env python
"""Cost of the FactorVAE score on the dSprites-shaped dataset of `eval_rate.py` (737,280 x 1x64x64, lat_sizes
[1, 3, 6, 40, 32, 32]) with a c2 model (beta-TCVAE, batch 1024, latent 10) after one untimed training epoch.

    python scripts/factor_score_rate.py [--rounds 3] [--batch 1000] [--out FILE]

Per round, in this order:
  * kernels:  CUDA-event time of the global-variance launch (1 group of 10,000 rows) and of the vote launch (15,000
              groups of 64 rows), 50 launches each, on the encoder means the Evaluator reads (the interleaved q_zCx);
  * score:    `disvae.evaluate.factor_vae_score` from those encodings (draws, both launches, vote tables), 20 calls;
  * eval:     Evaluator(...)(DeviceLoader.in_order(batch), is_metrics=True) without and with is_factor_score=True;
  * epoch:    one c2 training epoch with metrics_every=1, without and with factor_score=True.
Every host timing ends in a device synchronise.  Prints the card and its power limit (read in the same run), each
round, and the medians over the rounds.
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

KEYS = ("global_var_us", "votes_us", "score_ms", "eval_metrics_s", "eval_metrics_score_s", "epoch_metrics_s",
        "epoch_metrics_score_s")


def kernel_us(fn, n=50):
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
        raise SystemExit("factor_score_rate.py needs a CUDA device")
    import disvae
    from disvae.data import DeviceLoader
    from disvae.evaluate import factor_vae_score, factor_vote_rows, group_variance
    from disvae.models.losses import get_loss_f
    dev = torch.device("cuda", 0)
    print(json.dumps({"card": card()}), flush=True)
    ds = ProceduralDSprites()
    lat_sizes = [int(s) for s in ds.lat_sizes]

    torch.manual_seed(1234)
    model = disvae.init_specific_model("Burgess", (1, 64, 64), 10).to(dev)
    opt = torch.optim.Adam(model.parameters(), lr=5e-4)
    lf = get_loss_f("btcvae", rec_dist="bernoulli", reg_anneal=0, btcvae_A=1, btcvae_B=6, btcvae_G=1, n_data=len(ds))
    save_dir = tempfile.mkdtemp(prefix="dvfactor")
    log = logging.getLogger("factor_score_rate")
    tr = disvae.Trainer(model, opt, lf, device=dev, logger=log, save_dir=save_dir, is_progress_bar=False)
    ev = disvae.Evaluator(model, lf, device=dev, logger=log, save_dir=save_dir, is_progress_bar=False)
    dl = DeviceLoader(ds, 1024, shuffle=True, device=dev)
    tr(dl, epochs=1, checkpoint_every=10 ** 9)                           # warm-up: graph capture, allocator
    ev(dl.in_order(args.batch), is_metrics=True, is_losses=False, is_factor_score=True)

    model.eval()
    mean = ev._compute_q_zCx(dl.in_order(args.batch))[1][0]            # the interleaved view the Evaluator reads
    model.train()
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    var_rows = torch.randint(len(ds), (1, 10000), generator=gen, device=dev)
    global_var = torch.empty(1, mean.size(1), device=dev)
    group_variance(mean, var_rows, var_out=global_var)
    rows = torch.cat([factor_vote_rows(lat_sizes, n, 64, gen)[1] for n in (10000, 5000)])
    dims = torch.empty(rows.size(0), dtype=torch.int32, device=dev)

    rounds = []
    for r in range(args.rounds):
        row = {"round": r}
        row["global_var_us"] = kernel_us(lambda: group_variance(mean, var_rows, var_out=global_var))
        row["votes_us"] = kernel_us(lambda: group_variance(mean, rows, global_var=global_var[0], argmin_out=dims))
        row["score_ms"] = timed(lambda: [factor_vae_score(mean, lat_sizes, seed=s) for s in range(20)]) * 1000 / 20
        row["eval_metrics_s"] = timed(lambda: ev(dl.in_order(args.batch), is_metrics=True, is_losses=False))
        row["eval_metrics_score_s"] = timed(lambda: ev(dl.in_order(args.batch), is_metrics=True, is_losses=False,
                                                       is_factor_score=True))
        row["epoch_metrics_s"] = timed(lambda: tr(dl, epochs=1, checkpoint_every=10 ** 9, metrics_every=1,
                                                  metrics_batch_size=args.batch))
        row["epoch_metrics_score_s"] = timed(lambda: tr(dl, epochs=1, checkpoint_every=10 ** 9, metrics_every=1,
                                                        metrics_batch_size=args.batch, factor_score=True))
        row = {k: (round(v, 4) if isinstance(v, float) else v) for k, v in row.items()}
        rounds.append(row)
        print(json.dumps(rounds[-1]), flush=True)
    med = {k: float(np.median([x[k] for x in rounds])) for k in KEYS}
    summary = {"card": card(), "n": len(ds), "batch": args.batch, "median": med, "rounds": rounds,
               "score": factor_vae_score(mean, lat_sizes, seed=0)[0]}
    print(json.dumps(summary), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
