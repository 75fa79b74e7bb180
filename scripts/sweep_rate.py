#!/usr/bin/env python
"""Throughput of a sweep (disvae.sweep.Sweep: K members, concurrent graph replays) against the same K members trained
one after another as lone Trainers, in one process over one resident dataset.

    python scripts/sweep_rate.py [--workloads c1,c2,c3] [--ks 1,2,4,8] [--reps 3] [--steps S]

Members are bench.py's model, loss and optimizer for the workload (seeds 1234, 1235, ..), over one DeviceLoader of
random byte images (S batches of the workload's batch size).  Each arm first trains one untimed epoch (the eager
warm-up steps and the capture), then two timed epochs: host clock around the call, which ends in a synchronisation.
Arms alternate --reps times; the medians are reported: images/s summed over the members, ms per sweep step (the time
to advance every member by one step) and device memory per member (growth of the allocator's reserved memory while
the arm's members were built and trained, over K).  One JSON line, with the card's name and power limit read in the
same run, then a Markdown table of the medians.
"""
import argparse
import json
import logging
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "disentangling-vae_b200"))

import torch  # noqa: E402

import bench  # noqa: E402
from anneal_graph_rate import card  # noqa: E402

TIMED_EPOCHS = 2
DEFAULT_STEPS = {"c1": 400, "c2": 150, "c3": 150}


class ByteImages(torch.utils.data.Dataset):
    """n random byte images, returned as ToTensor would (float32 k/255)."""

    def __init__(self, n, img, seed=1234):
        g = torch.Generator().manual_seed(seed)
        self.imgs = torch.randint(0, 256, (n,) + tuple(img), dtype=torch.uint8, generator=g)

    def __len__(self):
        return len(self.imgs)

    def __getitem__(self, i):
        return self.imgs[i].float().div(255), 0


def members(workload, k, device, root):
    import disvae
    from disvae.models.losses import get_loss_f
    loss_name, img, B, z, n_data, lkw, lr, _ = bench.WORKLOADS[workload]
    out = []
    for j in range(k):
        torch.manual_seed(1234 + j)
        model = disvae.init_specific_model("Burgess", img, z)
        opt = torch.optim.Adam(model.parameters(), lr=lr)
        out.append(disvae.Trainer(model, opt, get_loss_f(loss_name, **bench.loss_kwargs(workload, device)), device=device,
                                  logger=logging.getLogger("sweep_rate"), save_dir=tempfile.mkdtemp(dir=root),
                                  is_progress_bar=False))
    return out


def arm(workload, k, swept, loader, device, root):
    """-> (seconds of the timed epochs, reserved bytes per member)."""
    from disvae.sweep import Sweep
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    reserved0 = torch.cuda.memory_reserved(device)
    trs = members(workload, k, device, root)
    if swept:
        sweep = Sweep(trs, seeds=[1234 + j for j in range(k)])
        runs = [lambda e: sweep(loader, epochs=e, checkpoint_every=1000)]
    else:
        runs = [lambda e, t=t: t(loader, epochs=e, checkpoint_every=1000) for t in trs]
    for run in runs:                                           # untimed: warm-up steps and capture
        run(1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for run in runs:
        run(TIMED_EPOCHS)
    torch.cuda.synchronize()
    sec = time.perf_counter() - t0
    assert all(len(t._graphs) == 1 for t in trs)
    per_member = (torch.cuda.memory_reserved(device) - reserved0) / k
    del trs, runs
    return sec, per_member


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c1,c2,c3")
    ap.add_argument("--ks", default="1,2,4,8")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=None, help="batches per epoch (default: c1 400, c2 and c3 150)")
    args = ap.parse_args()
    logging.getLogger("sweep_rate").setLevel(logging.WARNING)
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    from disvae.data import DeviceLoader
    res = {"card": card(device), "reps": args.reps, "timed_epochs": TIMED_EPOCHS, "workloads": {}}
    rows = []
    with tempfile.TemporaryDirectory(prefix="dvsweep") as root:
        for w in args.workloads.split(","):
            _, img, B, *_ = bench.WORKLOADS[w]
            steps = args.steps or DEFAULT_STEPS.get(w, 100)
            loader = DeviceLoader(ByteImages(steps * B, img), B, seed=1234, device=device)
            arm(w, 1, True, loader, device, root)                 # untimed: first-use costs (library, allocator)
            res["workloads"][w] = {"what": bench.WORKLOAD_NAMES[w], "batch": B, "steps_per_epoch": steps, "k": {}}
            for k in (int(s) for s in args.ks.split(",")):
                runs = {"sweep": [], "sequential": []}
                for _ in range(args.reps):
                    for name in ("sweep", "sequential"):
                        runs[name].append(arm(w, k, name == "sweep", loader, device, root))
                entry = {}
                for name, rs in runs.items():
                    sec = sorted(r[0] for r in rs)[len(rs) // 2]
                    mem = sorted(r[1] for r in rs)[len(rs) // 2]
                    n_steps = TIMED_EPOCHS * steps
                    entry[name] = {"images_per_s": round(k * B * n_steps / sec), "ms_per_sweep_step": round(1e3 * sec / n_steps, 4),
                                   "mib_per_member": round(mem / 2 ** 20, 1), "seconds_runs": [round(r[0], 4) for r in rs]}
                entry["sweep_over_sequential"] = round(entry["sweep"]["images_per_s"] / entry["sequential"]["images_per_s"], 3)
                res["workloads"][w]["k"][k] = entry
                rows.append((w, k, entry))
            del loader
            torch.cuda.empty_cache()
    print(json.dumps(res), flush=True)
    print("| workload | K | sweep img/s | sequential img/s | sweep / sequential | sweep ms/step | sequential ms/step | "
          "MiB/member (sweep, sequential) |")
    print("|---|---|---|---|---|---|---|---|")
    for w, k, e in rows:
        s, q = e["sweep"], e["sequential"]
        print("| %s | %d | %d | %d | %.2f | %.3f | %.3f | %.0f, %.0f |" % (w, k, s["images_per_s"], q["images_per_s"],
              e["sweep_over_sequential"], s["ms_per_sweep_step"], q["ms_per_sweep_step"], s["mib_per_member"],
              q["mib_per_member"]))


if __name__ == "__main__":
    main()
