#!/usr/bin/env python
"""Cost of the FactorVAE permutation entry point dv_permute_dims_rows, and of the global-batch FactorVAE mode.

    python scripts/permute_cost.py [--iters 200]

Prints one JSON line per measurement: the CUDA-event median of dv_permute_dims_rows (device permutations) over
`--iters` launches after warm-up, for the full window and a 1/8 window, at B rows x D=10 across the single-CTA
(B <= 4096) and multi-CTA sort.  With two or more GPUs it also times eager BASELINE.json configs[3] (c4: FactorVAE,
3x64x64, 512 images per GPU) steps on two ranks with local and with global-batch permutations.  The GPU name and power
limit are read in the same run.
"""
import argparse
import json
import os
import socket
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "disentangling-vae_b200"))

import torch  # noqa: E402

SIZES = [(256, 10), (2048, 10), (4096, 10), (8192, 10), (65536, 10)]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q[0] if q else "unavailable"}


def time_permutations(iters):
    from disvae import ops
    info = gpu_info()
    for B, D in SIZES:
        z = torch.randn(B, D, device="cuda")
        off = torch.zeros(1, dtype=torch.int64, device="cuda")
        for label, row0, nrows in [("full", 0, B), ("1/8", B // 2, B // 8)]:
            for _ in range(20):
                ops.permute_dims_rows(z, row0, nrows, None, 1, off)
            torch.cuda.synchronize()
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
            for e0, e1 in ev:
                e0.record()
                ops.permute_dims_rows(z, row0, nrows, None, 1, off)
                e1.record()
            torch.cuda.synchronize()
            ts = sorted(e0.elapsed_time(e1) * 1e3 for e0, e1 in ev)
            print(json.dumps(dict(what="dv_permute_dims_rows", B=B, D=D, window=label, nrows=nrows, launches=iters,
                                  median_us=round(ts[len(ts) // 2], 2), min_us=round(ts[0], 2), **info)), flush=True)


def c4_rank(steps, warmup):
    """One rank of the two-GPU c4 comparison (run under torch.distributed.run)."""
    import logging
    import tempfile
    import torch.distributed as dist
    import disvae
    from disvae.models.losses import get_loss_f
    from disvae.parallel import broadcast_parameters
    rank, local = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"])
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    res = {}
    for mode in ("local", "global"):
        torch.manual_seed(1234)
        model = disvae.init_specific_model("Burgess", (3, 64, 64), 10).to(dev)
        broadcast_parameters(model)
        opt = torch.optim.Adam(model.parameters(), lr=1e-4)
        lf = get_loss_f("factor", rec_dist="bernoulli", reg_anneal=0, factor_G=6.4, latent_dim=10, lr_disc=1e-5,
                        device=dev)
        lf.global_batch = mode == "global"
        tr = disvae.Trainer(model, opt, lf, device=dev, logger=logging.getLogger("c4"), save_dir=tempfile.mkdtemp(),
                            is_progress_bar=False)
        tr.use_cuda_graph = False                    # both modes eager: the global mode always is
        model.train()
        xs = [torch.rand(512, 3, 64, 64, device=dev) for _ in range(4)]
        for i in range(warmup):
            tr._step(xs[i % 4], None)
        torch.cuda.synchronize()
        dist.barrier()
        t0 = time.perf_counter()
        for i in range(steps):
            tr._step(xs[i % 4], None)
        torch.cuda.synchronize()
        res[mode] = (time.perf_counter() - t0) * 1e3 / steps
    allr = [None] * dist.get_world_size()
    dist.all_gather_object(allr, res)
    if rank == 0:
        info = gpu_info()
        for mode in ("local", "global"):
            print(json.dumps(dict(what="c4 eager step, 2 ranks, 512 images per GPU", mode=mode, steps=steps,
                                  ms_per_step=[round(r[mode], 3) for r in allr], **info)), flush=True)
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--c4-rank", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.c4_rank:
        return c4_rank(args.steps, args.warmup)
    assert torch.cuda.is_available(), "permute_cost.py measures on a GPU"
    time_permutations(max(args.iters, 200))
    if torch.cuda.device_count() < 2:
        print(json.dumps(dict(what="c4 eager step, 2 ranks", result="not measured: fewer than two GPUs")), flush=True)
        return
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                    "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.abspath(__file__), "--c4-rank",
                    "--steps", str(args.steps), "--warmup", str(args.warmup)], check=True)


if __name__ == "__main__":
    main()
