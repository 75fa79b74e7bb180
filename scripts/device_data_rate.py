#!/usr/bin/env python
"""Training throughput with the host DataLoader against disvae.data.DeviceLoader on a dSprites-shaped dataset.

    python scripts/device_data_rate.py [--n 737280] [--host-steps 60] [--rounds 3]

The dataset is 737,280 binary 1x64x64 images with a per-item `__getitem__` like the reference's DSprites (bytes x 255,
then ToTensor's HWC -> CHW and /255), trained with the c2 settings of bench.py (beta-TCVAE, batch 1024, latent 10,
Adam lr 5e-4).  Prints the card and its power limit, the materialisation time of the DeviceLoader (every item through
`__getitem__` once, uploaded as uint8), and per round: images/s of `--host-steps` Trainer steps fed by
DataLoader(num_workers=0, pin_memory=True, shuffle=True), then images/s of one whole DeviceLoader epoch.  A first
DeviceLoader epoch and a few host steps run before the rounds (graph capture, allocator, loader start-up).
"""
import argparse
import itertools
import json
import logging
import os
import subprocess
import sys
import tempfile
import time
from collections import defaultdict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "disentangling-vae_b200"))


class SyntheticDSprites(torch.utils.data.Dataset):
    """dSprites-shaped: binary 64x64 images stored as 0/1 bytes, served like the reference's DSprites.__getitem__."""
    lat_sizes = np.array([3, 6, 40, 32, 32])

    def __init__(self, n, seed=0):
        rng = np.random.default_rng(seed)
        self.imgs = np.empty((n, 64, 64), dtype=np.uint8)
        for a in range(0, n, 65536):
            self.imgs[a:a + 65536] = rng.random((min(65536, n - a), 64, 64), dtype=np.float32) > 0.8

    def __len__(self):
        return len(self.imgs)

    def __getitem__(self, i):
        img = np.expand_dims(self.imgs[i] * 255, -1)                    # HxWx1 bytes, as the reference hands ToTensor
        return torch.from_numpy(img.transpose(2, 0, 1).copy()).float().div(255), 0


class FirstSteps:
    """The first `k` batches of a loader (a fixed number of Trainer steps)."""

    def __init__(self, loader, k):
        self.loader, self.k = loader, k

    def __iter__(self):
        return itertools.islice(iter(self.loader), self.k)

    def __len__(self):
        return self.k


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return {"torch_name": torch.cuda.get_device_name(), "nvidia_smi": q[torch.cuda.current_device()] if q else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=737280)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--host-steps", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("device_data_rate.py needs a CUDA device")
    import disvae
    from disvae.data import DeviceLoader
    from disvae.models.losses import get_loss_f
    dev = torch.device("cuda", 0)
    print(json.dumps({"card": card()}), flush=True)
    ds = SyntheticDSprites(args.n)

    torch.manual_seed(1234)
    model = disvae.init_specific_model("Burgess", (1, 64, 64), 10).to(dev)
    opt = torch.optim.Adam(model.parameters(), lr=5e-4)
    lf = get_loss_f("btcvae", rec_dist="bernoulli", reg_anneal=0, btcvae_A=1, btcvae_B=6, btcvae_G=1, n_data=args.n)
    tr = disvae.Trainer(model, opt, lf, device=dev, logger=logging.getLogger("rate"),
                        save_dir=tempfile.mkdtemp(prefix="dvrate"), is_progress_bar=False)
    model.train()

    t0 = time.perf_counter()
    dl = DeviceLoader(ds, args.batch, shuffle=True, device=dev)
    torch.cuda.synchronize()
    materialise_s = time.perf_counter() - t0
    print(json.dumps({"materialise_s": round(materialise_s, 2), "items": args.n,
                      "device_bytes": dl.data.numel()}), flush=True)
    host = torch.utils.data.DataLoader(ds, batch_size=args.batch, shuffle=True, num_workers=0, pin_memory=True)

    epoch = [0]

    def timed(loader, images):
        torch.cuda.synchronize()
        t = time.perf_counter()
        tr._train_epoch(loader, defaultdict(list), epoch[0])
        torch.cuda.synchronize()
        epoch[0] += 1
        return images / (time.perf_counter() - t)

    timed(dl, 0)                                                         # warm-up: graph capture of both shapes
    timed(FirstSteps(host, 5), 0)
    full_epoch_images = sum(size for _, size in dl.windows)
    rounds = []
    for r in range(args.rounds):
        h = timed(FirstSteps(host, args.host_steps), args.host_steps * args.batch)
        d = timed(dl, full_epoch_images)
        rounds.append({"round": r, "host_loader_img_s": round(h), "device_loader_img_s": round(d)})
        print(json.dumps(rounds[-1]), flush=True)
    print(json.dumps({"card": card(), "materialise_s": round(materialise_s, 2), "batch": args.batch, "n": args.n,
                      "host_steps": args.host_steps, "device_epoch_images": full_epoch_images,
                      "host_loader_img_s_median": float(np.median([x["host_loader_img_s"] for x in rounds])),
                      "device_loader_img_s_median": float(np.median([x["device_loader_img_s"] for x in rounds])),
                      "rounds": rounds}))


if __name__ == "__main__":
    main()
