#!/usr/bin/env python
"""Cost of the DCI score on the dSprites-shaped dataset of `eval_rate.py` (737,280 x 1x64x64, lat_sizes
[1, 3, 6, 40, 32, 32]) with a c2 model (beta-TCVAE, batch 1024, latent 10) after one untimed training epoch, and its
agreement with sklearn's GradientBoostingClassifier() on the host.

    python scripts/dci_score_rate.py [--rounds 3] [--batch 1000] [--host-factors 3,6] [--out FILE]

Per round, in this order:
  * fit:      CUDA-event time of one `dv_dci_fit` (D = 10, the 5 factors of more than one value = 113 columns,
              10,000 training and 5,000 test rows, 100 stages: 204 launches), on the encoder means the Evaluator reads
              (the interleaved q_zCx);
  * score:    `disvae.evaluate.dci_score` from those encodings (draws, labels, the fit, copies);
  * eval:     Evaluator(...)(DeviceLoader.in_order(batch), is_metrics=True), MIG / AAM alone, for scale.
Every host timing ends in a device synchronise.  Then, once, on the host: GradientBoostingClassifier(random_state=0)
fitted to the same rows of every factor whose size is in --host-factors (by default the 3- and 6-value factors; the
others take minutes each), with its time, the time projected to all 113 columns at the per-column cost of those fits
(labelled as projected), and its agreement with the GPU fit on those factors: the largest importance difference, the
differing predictions, and the accuracies side by side.  Prints the card and its power limit, each round, and the
medians over the rounds.
"""
import argparse
import json
import logging
import os
import sys
import tempfile
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.join(os.path.dirname(HERE), "disentangling-vae_b200"), HERE]
from eval_rate import ProceduralDSprites, card, timed  # noqa: E402

KEYS = ("fit_ms", "score_ms", "eval_metrics_s")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=1000)
    ap.add_argument("--host-factors", default="3,6", help="sizes of the factors fitted by sklearn on the host")
    ap.add_argument("--out", default=None, help="also write the summary JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dci_score_rate.py needs a CUDA device")
    import disvae
    from disvae.data import DeviceLoader
    from disvae.evaluate import dci_fit, dci_score, sap_labels
    from disvae.models.losses import get_loss_f
    dev = torch.device("cuda", 0)
    print(json.dumps({"card": card()}), flush=True)
    ds = ProceduralDSprites()
    lat_sizes = [int(s) for s in ds.lat_sizes]

    torch.manual_seed(1234)
    model = disvae.init_specific_model("Burgess", (1, 64, 64), 10).to(dev)
    opt = torch.optim.Adam(model.parameters(), lr=5e-4)
    lf = get_loss_f("btcvae", rec_dist="bernoulli", reg_anneal=0, btcvae_A=1, btcvae_B=6, btcvae_G=1, n_data=len(ds))
    save_dir = tempfile.mkdtemp(prefix="dvdci")
    log = logging.getLogger("dci_score_rate")
    tr = disvae.Trainer(model, opt, lf, device=dev, logger=log, save_dir=save_dir, is_progress_bar=False)
    ev = disvae.Evaluator(model, lf, device=dev, logger=log, save_dir=save_dir, is_progress_bar=False)
    dl = DeviceLoader(ds, 1024, shuffle=True, device=dev)
    tr(dl, epochs=1, checkpoint_every=10 ** 9)
    ev(dl.in_order(args.batch), is_metrics=True, is_losses=False)

    model.eval()
    mean = ev._compute_q_zCx(dl.in_order(args.batch))[1][0]            # the interleaved view the Evaluator reads
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    train_rows = torch.randint(len(ds), (10000,), generator=gen, device=dev)
    test_rows = torch.randint(len(ds), (5000,), generator=gen, device=dev)
    factors, train_cls, test_cls, n_classes, counts, _ = sap_labels(lat_sizes, train_rows, test_rows)
    dci_fit(mean, train_rows, test_rows, train_cls, n_classes, counts)

    rounds = []
    for r in range(args.rounds):
        row = {"round": r}
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        importance, pred, _ = dci_fit(mean, train_rows, test_rows, train_cls, n_classes, counts)
        e1.record()
        torch.cuda.synchronize()
        row["fit_ms"] = e0.elapsed_time(e1)
        row["score_ms"] = timed(lambda: dci_score(mean, lat_sizes, seed=0)) * 1000
        row["eval_metrics_s"] = timed(lambda: ev(dl.in_order(args.batch), is_metrics=True, is_losses=False))
        row = {k: (round(v, 4) if isinstance(v, float) else v) for k, v in row.items()}
        rounds.append(row)
        print(json.dumps(rounds[-1]), flush=True)
    med = {k: float(np.median([x[k] for x in rounds])) for k in KEYS}
    score, helpers = dci_score(mean, lat_sizes, seed=0)
    summary = {"card": card(), "n": len(ds), "batch": args.batch, "median": med, "rounds": rounds, "score": score,
               "train_accuracy": helpers["train_accuracy"].tolist(), "test_accuracy": helpers["test_accuracy"].tolist()}

    from sklearn.ensemble import GradientBoostingClassifier
    sizes = [int(s) for s in args.host_factors.split(",") if s]
    x = mean.float().cpu().numpy()
    tr_rows, te_rows = train_rows.cpu().numpy(), test_rows.cpu().numpy()
    y_tr, y_te = train_cls.cpu().numpy(), test_cls.cpu().numpy()
    imp, prd = importance.cpu().numpy(), pred.cpu().numpy()
    host, seconds, columns = [], 0.0, 0
    for j, k in enumerate(factors):
        if lat_sizes[k] not in sizes:
            continue
        t0 = time.perf_counter()
        clf = GradientBoostingClassifier(random_state=0).fit(x[tr_rows], y_tr[j])
        dt = time.perf_counter() - t0
        nc = int(n_classes[j])
        seconds += dt
        columns += nc if nc > 2 else 1
        p_tr, p_te = clf.predict(x[tr_rows]), clf.predict(x[te_rows])
        host.append({"factor": k, "classes": nc, "sklearn_s": round(dt, 2),
                     "max_importance_diff": float(np.abs(clf.feature_importances_ - imp[:, j]).max()),
                     "differing_train_predictions": int((p_tr != prd[j, :10000]).sum()),
                     "differing_test_predictions": int((p_te != prd[j, 10000:]).sum()),
                     "train_accuracy": [float(np.mean(p_tr == y_tr[j])), float(helpers["train_accuracy"][j])],
                     "test_accuracy": [float(np.mean(p_te == y_te[j])), float(helpers["test_accuracy"][j])]})
        print(json.dumps(host[-1]), flush=True)
    total_columns = int(sum(int(c) if c > 2 else int(c > 1) for c in n_classes.tolist()))
    summary["host"] = {"fits": host, "sklearn_s": round(seconds, 2),
                       "projected_all_factors_s": round(seconds / max(columns, 1) * total_columns, 1),
                       "columns": columns, "total_columns": total_columns}
    print(json.dumps(summary), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
