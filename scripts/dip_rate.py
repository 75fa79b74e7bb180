#!/usr/bin/env python
"""Cost of the DIP-VAE covariance penalty: the kernels on their own, and a c2-shaped training step with it.

    python scripts/dip_rate.py [--reps 3] [--steps 60]

1. dv_dip_fwd + dv_dip_bwd (DIP-VAE-II, the type that also reads logvar) at (B, D) = (1024, 10), (256, 64),
   (2048, 64) on the encoder's interleaved layout: 200 back-to-back pairs captured in one CUDA graph, replayed 10 times
   between CUDA events; µs per pair, median of --reps.
2. Steps per second of a c2-shaped Trainer (1x64x64, B = 1024, z = 10, Adam 5e-4, resident data, CUDA-graph path) for
   betaH, dipI and dipII: each arm trains one untimed epoch (warm-up steps and capture), then one timed epoch of
   --steps steps (host clock around the call, which ends in a synchronisation).  The three losses alternate --reps
   times in one process; the medians are reported.
One JSON line, with the card's name and power limit read in the same run, then a Markdown table.
"""
import argparse
import json
import logging
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "disentangling-vae_b200"))

import torch  # noqa: E402

from anneal_graph_rate import card  # noqa: E402
from sweep_rate import ByteImages  # noqa: E402

KERNEL_SHAPES = [(1024, 10), (256, 64), (2048, 64)]
LOSSES = ["betaH", "dipI", "dipII"]
PAIRS, REPLAYS = 200, 10


def kernel_us(B, D, device):
    """µs per dv_dip_fwd + dv_dip_bwd pair, device time of a replayed graph of PAIRS pairs."""
    from disvae import _native as N
    L = N.lib()
    g = torch.Generator(device=device).manual_seed(B + D)
    ml = torch.randn(B, D, 2, device=device, generator=g)
    mu, lv = ml[..., 0], ml[..., 1]
    ws = torch.empty((L.dv_dip_workspace_bytes(B, D) + 3) // 4, device=device)
    terms = torch.empty(2, device=device)
    g_terms = torch.tensor([10.0, 10.0], device=device)
    g_mu, g_lv = torch.empty(B, D, device=device), torch.empty(B, D, device=device)
    s = torch.cuda.Stream(device)

    def pair():
        N.call("dv_dip_fwd", mu.data_ptr(), lv.data_ptr(), 2, 2 * D, B, D, 2, terms.data_ptr(), ws.data_ptr(), N.stream())
        N.call("dv_dip_bwd", mu.data_ptr(), lv.data_ptr(), 2, 2 * D, B, D, 2, g_terms.data_ptr(), g_mu.data_ptr(),
               g_lv.data_ptr(), ws.data_ptr(), N.stream())
    with torch.cuda.stream(s):
        pair()                                                   # first use outside the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        for _ in range(PAIRS):
            pair()
    graph.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(REPLAYS):
        graph.replay()
    e1.record()
    e1.synchronize()
    return 1e3 * e0.elapsed_time(e1) / (PAIRS * REPLAYS)


def step_ms(loss_name, loader, steps, device, root):
    """ms per training step of one timed epoch (after an untimed one)."""
    import disvae
    from disvae.models.losses import get_loss_f
    torch.manual_seed(1234)
    model = disvae.init_specific_model("Burgess", (1, 64, 64), 10)
    opt = torch.optim.Adam(model.parameters(), lr=5e-4)
    lf = get_loss_f(loss_name, rec_dist="bernoulli", reg_anneal=0, betaH_B=4)
    tr = disvae.Trainer(model, opt, lf, device=device, logger=logging.getLogger("dip_rate"),
                        save_dir=tempfile.mkdtemp(dir=root), is_progress_bar=False)
    tr(loader, epochs=1, checkpoint_every=1000)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    tr(loader, epochs=1, checkpoint_every=1000)
    torch.cuda.synchronize()
    sec = time.perf_counter() - t0
    assert len(tr._graphs) == 1
    return 1e3 * sec / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=60, help="batches of 1024 per epoch")
    args = ap.parse_args()
    logging.getLogger("dip_rate").setLevel(logging.WARNING)
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    from disvae.data import DeviceLoader
    res = {"card": card(device), "reps": args.reps, "kernel_us_per_fwd_bwd": {}, "c2_step": {}}
    for B, D in KERNEL_SHAPES:
        runs = [kernel_us(B, D, device) for _ in range(args.reps)]
        res["kernel_us_per_fwd_bwd"]["%dx%d" % (B, D)] = {"median": round(statistics.median(runs), 3),
                                                          "runs": [round(r, 3) for r in runs]}
    loader = DeviceLoader(ByteImages(args.steps * 1024, (1, 64, 64)), 1024, seed=1234, device=device)
    runs = {name: [] for name in LOSSES}
    with tempfile.TemporaryDirectory(prefix="dvdip") as root:
        step_ms("betaH", loader, args.steps, device, root)    # untimed: first-use costs (library, allocator)
        for _ in range(args.reps):
            for name in LOSSES:
                runs[name].append(step_ms(name, loader, args.steps, device, root))
    for name, rs in runs.items():
        med = statistics.median(rs)
        res["c2_step"][name] = {"ms_per_step": round(med, 4), "steps_per_s": round(1e3 / med, 1),
                                "runs_ms": [round(r, 4) for r in rs]}
    for name in ("dipI", "dipII"):
        res["c2_step"][name]["us_over_betaH"] = round(1e3 * (res["c2_step"][name]["ms_per_step"]
                                                            - res["c2_step"]["betaH"]["ms_per_step"]), 1)
    print(json.dumps(res), flush=True)
    print("card: %s, power limit %s" % (res["card"]["name"], res["card"]["power_limit"]))
    print("| (B, D) | µs per fwd + bwd |")
    print("|---|---|")
    for k, v in res["kernel_us_per_fwd_bwd"].items():
        print("| %s | %.2f |" % (k, v["median"]))
    print("| c2 loss | ms / step | steps / s | µs over betaH |")
    print("|---|---|---|---|")
    for name in LOSSES:
        e = res["c2_step"][name]
        print("| %s | %.4f | %.1f | %s |" % (name, e["ms_per_step"], e["steps_per_s"], e.get("us_over_betaH", "")))


if __name__ == "__main__":
    main()
