#!/usr/bin/env python
"""Step time of an annealed run's first steps: eager (use_cuda_graph=False -- how those steps ran before the annealing
coefficient and the loss log moved to the device) against the Trainer's CUDA-graph path.

    python scripts/anneal_graph_rate.py [--workloads c1,c2] [--steps 2000] [--reps 3] [--reg-anneal 10000]

Each arm is a fresh Trainer (bench.py's model, loss and optimizer for the workload, seed 1234) with reg_anneal = 10000
running --steps steps of one epoch through Trainer._train_epoch with a real storer (every 50th step records), over 8
resident batches rotated; the whole epoch is timed with CUDA events, so the graph arm includes its two eager warm-up
steps and the capture.  Arms alternate --reps times; the median ms/step of each is reported, with the card's name and
power limit read in the same run.  One JSON line.
"""
import argparse
import json
import logging
import os
import subprocess
import sys
import tempfile
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "disentangling-vae_b200"))

import torch  # noqa: E402

import bench  # noqa: E402


def card(device):
    idx = device.index or 0
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(idx)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:                                     # the measurement stands without it, marked
        return {"name": torch.cuda.get_device_name(device), "power_limit": "unavailable (%r)" % e}


def arm(workload, use_graph, steps, reg_anneal, device):
    import disvae
    from disvae.models.losses import get_loss_f
    loss_name, img, B, z, n_data, lkw, lr, _ = bench.WORKLOADS[workload]
    torch.manual_seed(1234)
    model = disvae.init_specific_model("Burgess", img, z).to(device)
    opt = torch.optim.Adam(model.parameters(), lr=lr)
    kw = bench.loss_kwargs(workload, device)
    kw["reg_anneal"] = reg_anneal
    tr = disvae.Trainer(model, opt, get_loss_f(loss_name, **kw), device=device, logger=logging.getLogger("anneal"),
                        save_dir=tempfile.mkdtemp(prefix="dvanneal"), is_progress_bar=False)
    tr.use_cuda_graph = use_graph
    model.train()
    g = torch.Generator().manual_seed(1234)
    batches = [torch.rand(B, *img, generator=g).to(device) for _ in range(bench.N_ROTATE)]
    loader = [(batches[i % len(batches)], None) for i in range(steps)]
    storer = defaultdict(list)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    tr._train_epoch(loader, storer, 0)
    e1.record()
    torch.cuda.synchronize()
    assert tr.loss_f.n_train_steps == steps and bool(tr._graphs) == use_graph
    ms = e0.elapsed_time(e1) / steps
    del tr, model, opt, batches, loader
    torch.cuda.empty_cache()
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c1,c2")
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--reg-anneal", type=int, default=10000)
    args = ap.parse_args()
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    res = {"card": card(device), "steps": args.steps, "reg_anneal": args.reg_anneal, "reps": args.reps, "workloads": {}}
    for w in args.workloads.split(","):
        arm(w, True, 20, args.reg_anneal, device)              # untimed: first-use costs (library, allocator, capture)
        runs = {"eager": [], "graph": []}
        for _ in range(args.reps):
            for name in ("eager", "graph"):
                runs[name].append(arm(w, name == "graph", args.steps, args.reg_anneal, device))
        med = {k: sorted(v)[len(v) // 2] for k, v in runs.items()}
        res["workloads"][w] = {"what": bench.WORKLOAD_NAMES[w], "ms_per_step_runs": {k: [round(x, 4) for x in v]
                                                                                     for k, v in runs.items()},
                               "ms_per_step_median": {k: round(v, 4) for k, v in med.items()},
                               "eager_over_graph": round(med["eager"] / med["graph"], 3)}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
