#!/usr/bin/env python
"""Cost of the SAP score on the dSprites-shaped dataset of `eval_rate.py` (737,280 x 1x64x64, lat_sizes
[1, 3, 6, 40, 32, 32]) with a c2 model (beta-TCVAE, batch 1024, latent 10) after one untimed training epoch.

    python scripts/sap_score_rate.py [--rounds 3] [--batch 1000] [--out FILE]

Per round, in this order:
  * kernel:   CUDA-event time of one `dv_sap_score_matrix` launch (D = 10, the 5 factors of more than one value,
              10,000 training and 5,000 test rows), 20 launches, on the encoder means the Evaluator reads (the
              interleaved q_zCx);
  * score:    `disvae.evaluate.sap_score` from those encodings (draws, labels, the launch, copies), 10 calls;
  * eval:     Evaluator(...)(DeviceLoader.in_order(batch), is_metrics=True) without and with is_sap_score=True;
  * epoch:    one c2 training epoch with metrics_every=1, without and with sap_score=True.
Every host timing ends in a device synchronise.  Prints the card and its power limit (read in the same run), each
round, and the medians over the rounds, with the solver's largest Newton step count.
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

KEYS = ("kernel_us", "score_ms", "eval_metrics_s", "eval_metrics_sap_s", "epoch_metrics_s", "epoch_metrics_sap_s")


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
        raise SystemExit("sap_score_rate.py needs a CUDA device")
    import disvae
    from disvae.data import DeviceLoader
    from disvae.evaluate import sap_labels, sap_score, sap_score_matrix
    from disvae.models.losses import get_loss_f
    dev = torch.device("cuda", 0)
    print(json.dumps({"card": card()}), flush=True)
    ds = ProceduralDSprites()
    lat_sizes = [int(s) for s in ds.lat_sizes]

    torch.manual_seed(1234)
    model = disvae.init_specific_model("Burgess", (1, 64, 64), 10).to(dev)
    opt = torch.optim.Adam(model.parameters(), lr=5e-4)
    lf = get_loss_f("btcvae", rec_dist="bernoulli", reg_anneal=0, btcvae_A=1, btcvae_B=6, btcvae_G=1, n_data=len(ds))
    save_dir = tempfile.mkdtemp(prefix="dvsap")
    log = logging.getLogger("sap_score_rate")
    tr = disvae.Trainer(model, opt, lf, device=dev, logger=log, save_dir=save_dir, is_progress_bar=False)
    ev = disvae.Evaluator(model, lf, device=dev, logger=log, save_dir=save_dir, is_progress_bar=False)
    dl = DeviceLoader(ds, 1024, shuffle=True, device=dev)
    tr(dl, epochs=1, checkpoint_every=10 ** 9)                           # warm-up: graph capture, allocator
    ev(dl.in_order(args.batch), is_metrics=True, is_losses=False, is_sap_score=True)

    model.eval()
    mean = ev._compute_q_zCx(dl.in_order(args.batch))[1][0]            # the interleaved view the Evaluator reads
    model.train()
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    train_rows = torch.randint(len(ds), (10000,), generator=gen, device=dev)
    test_rows = torch.randint(len(ds), (5000,), generator=gen, device=dev)
    _, train_cls, test_cls, n_classes, counts, _ = sap_labels(lat_sizes, train_rows, test_rows)

    rounds = []
    for r in range(args.rounds):
        row = {"round": r}
        row["kernel_us"] = kernel_us(lambda: sap_score_matrix(mean, train_rows, test_rows, train_cls, test_cls,
                                                              n_classes, counts, 0.01))
        row["score_ms"] = timed(lambda: [sap_score(mean, lat_sizes, seed=s) for s in range(10)]) * 1000 / 10
        row["eval_metrics_s"] = timed(lambda: ev(dl.in_order(args.batch), is_metrics=True, is_losses=False))
        row["eval_metrics_sap_s"] = timed(lambda: ev(dl.in_order(args.batch), is_metrics=True, is_losses=False,
                                                     is_sap_score=True))
        row["epoch_metrics_s"] = timed(lambda: tr(dl, epochs=1, checkpoint_every=10 ** 9, metrics_every=1,
                                                  metrics_batch_size=args.batch))
        row["epoch_metrics_sap_s"] = timed(lambda: tr(dl, epochs=1, checkpoint_every=10 ** 9, metrics_every=1,
                                                      metrics_batch_size=args.batch, sap_score=True))
        row = {k: (round(v, 4) if isinstance(v, float) else v) for k, v in row.items()}
        rounds.append(row)
        print(json.dumps(rounds[-1]), flush=True)
    med = {k: float(np.median([x[k] for x in rounds])) for k in KEYS}
    score, helpers = sap_score(mean, lat_sizes, seed=0)
    summary = {"card": card(), "n": len(ds), "batch": args.batch, "median": med, "rounds": rounds, "score": score,
               "max_newton_steps": int(helpers["solver_iterations"].max())}
    print(json.dumps(summary), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
