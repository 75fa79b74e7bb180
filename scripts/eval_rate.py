#!/usr/bin/env python
"""Time of one MIG / AAM evaluation through the host DataLoader against the resident data, on a dSprites-shaped dataset.

    python scripts/eval_rate.py [--rounds 3] [--batch 1000] [--out FILE]

The dataset is 737,280 binary 1x64x64 images with procedural factors (lat_sizes [1, 3, 6, 40, 32, 32], the order and
sizes of dSprites': shape, scale, orientation, posX, posY; orientation does not change the image) and a per-item
`__getitem__` like the reference's DSprites (bytes x 255, then ToTensor's HWC -> CHW and /255).  The model is a c2
Trainer's (beta-TCVAE, 1x64x64, batch 1024, latent 10, Adam lr 5e-4) after one untimed training epoch.  Per round, in
this order:
  * host:     Evaluator(...)(DataLoader(dataset, batch_size, shuffle=False), is_metrics=True, is_losses=False);
  * resident: the same over DeviceLoader.in_order(batch_size);
  * epoch:    one c2 training epoch with metrics_every=0, then one with metrics_every=1 (the difference is the added
              time per epoch).
Every timing ends in a device synchronise.  Prints the card and its power limit (read in the same run), each round,
and the medians over the rounds.
"""
import argparse
import json
import logging
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "disentangling-vae_b200"))


class ProceduralDSprites(torch.utils.data.Dataset):
    """dSprites-shaped: 737,280 binary 64x64 images, the last factor fastest, served like DSprites.__getitem__."""
    lat_names = ("color", "shape", "scale", "orientation", "posX", "posY")
    lat_sizes = np.array([1, 3, 6, 40, 32, 32])

    def __init__(self):
        n = int(np.prod(self.lat_sizes))
        self.imgs = np.empty((n, 64, 64), dtype=np.uint8)
        ar = np.arange(64)
        for a in range(0, n, 32768):
            idx = np.arange(a, min(a + 32768, n))
            _, shape, scale, _, px, py = np.unravel_index(idx, self.lat_sizes)
            side = 6 + 2 * scale                                       # 6 .. 16 pixels
            w = np.where(shape == 1, side // 2, side)                  # square, tall bar, wide bar
            h = np.where(shape == 2, side // 2, side)
            x0, y0 = 8 + px, 8 + py
            col = (ar >= x0[:, None]) & (ar < (x0 + w)[:, None])
            row = (ar >= y0[:, None]) & (ar < (y0 + h)[:, None])
            self.imgs[a:a + len(idx)] = row[:, :, None] & col[:, None, :]

    def __len__(self):
        return len(self.imgs)

    def __getitem__(self, i):
        img = np.expand_dims(self.imgs[i] * 255, -1)                    # HxWx1 bytes, as the reference hands ToTensor
        return torch.from_numpy(img.transpose(2, 0, 1).copy()).float().div(255), 0


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return {"torch_name": torch.cuda.get_device_name(), "nvidia_smi": q[torch.cuda.current_device()] if q else None}


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=1000)
    ap.add_argument("--out", default=None, help="also write the summary JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_rate.py needs a CUDA device")
    import disvae
    from disvae.data import DeviceLoader
    from disvae.models.losses import get_loss_f
    dev = torch.device("cuda", 0)
    print(json.dumps({"card": card()}), flush=True)
    t0 = time.perf_counter()
    ds = ProceduralDSprites()
    print(json.dumps({"dataset_build_s": round(time.perf_counter() - t0, 1), "n": len(ds)}), flush=True)

    torch.manual_seed(1234)
    model = disvae.init_specific_model("Burgess", (1, 64, 64), 10).to(dev)
    opt = torch.optim.Adam(model.parameters(), lr=5e-4)
    lf = get_loss_f("btcvae", rec_dist="bernoulli", reg_anneal=0, btcvae_A=1, btcvae_B=6, btcvae_G=1, n_data=len(ds))
    save_dir = tempfile.mkdtemp(prefix="dveval")
    log = logging.getLogger("eval_rate")
    tr = disvae.Trainer(model, opt, lf, device=dev, logger=log, save_dir=save_dir, is_progress_bar=False)
    ev = disvae.Evaluator(model, lf, device=dev, logger=log, save_dir=save_dir, is_progress_bar=False)

    t0 = time.perf_counter()
    dl = DeviceLoader(ds, 1024, shuffle=True, device=dev)
    torch.cuda.synchronize()
    print(json.dumps({"materialise_s": round(time.perf_counter() - t0, 1)}), flush=True)
    host = torch.utils.data.DataLoader(ds, batch_size=args.batch, shuffle=False)

    tr(dl, epochs=1, checkpoint_every=10 ** 9)                           # warm-up: graph capture, allocator
    ev(dl.in_order(args.batch), is_metrics=True, is_losses=False)       # warm-up of the evaluation shapes
    rounds = []
    for r in range(args.rounds):
        row = {"round": r}
        row["host_s"] = timed(lambda: ev(host, is_metrics=True, is_losses=False))
        row["resident_s"] = timed(lambda: ev(dl.in_order(args.batch), is_metrics=True, is_losses=False))
        row["epoch_s"] = timed(lambda: tr(dl, epochs=1, checkpoint_every=10 ** 9))
        row["epoch_metrics_s"] = timed(lambda: tr(dl, epochs=1, checkpoint_every=10 ** 9, metrics_every=1,
                                                  metrics_batch_size=args.batch))
        row = {k: (round(v, 3) if isinstance(v, float) else v) for k, v in row.items()}
        rounds.append(row)
        print(json.dumps(rounds[-1]), flush=True)
    med = {k: float(np.median([x[k] for x in rounds])) for k in ("host_s", "resident_s", "epoch_s", "epoch_metrics_s")}
    med["added_per_epoch_s"] = float(np.median([x["epoch_metrics_s"] - x["epoch_s"] for x in rounds]))
    summary = {"card": card(), "n": len(ds), "batch": args.batch, "median": med, "rounds": rounds}
    print(json.dumps(summary), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
