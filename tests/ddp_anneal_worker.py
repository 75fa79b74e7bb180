#!/usr/bin/env python
"""One rank of the annealed graph-vs-eager check under data parallelism; launched by tests/test_anneal_graph_gpu.py as

    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port P tests/ddp_anneal_worker.py \
        --loss btcvae|factor

Each rank trains the same replica twice from the same seed -- once with the Trainer's CUDA graph, once eagerly -- for one
epoch of annealed steps (reg_anneal 7) that record every 5th step.  On every rank the two runs must agree bit for bit:
parameters, Adam moments (FactorVAE: the discriminator's too) and every storer list.  With fewer GPUs than ranks all
ranks share cuda:0 and the collectives run over gloo on CUDA tensors.  Prints one "DDP_ANNEAL {json}" line on rank 0.
"""
import argparse
import json
import logging
import os
import sys
import tempfile
from collections import defaultdict

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "disentangling-vae_b200"))


def run(loss_name, use_graph, dev, rank, world, steps, per, img):
    import disvae
    from disvae.models.losses import get_loss_f
    from disvae.parallel import broadcast_parameters
    torch.manual_seed(1234)
    model = disvae.init_specific_model("Burgess", img, 10).to(dev)
    broadcast_parameters(model)
    opt = torch.optim.Adam(model.parameters(), lr=5e-4)
    lf = get_loss_f(loss_name, rec_dist="bernoulli", reg_anneal=7, btcvae_A=1, btcvae_B=6, btcvae_G=1, n_data=202599,
                    factor_G=6.4, latent_dim=10, lr_disc=1e-4, device=dev)
    lf.record_loss_every = 5
    tr = disvae.Trainer(model, opt, lf, device=dev, logger=logging.getLogger("ddp"), save_dir=tempfile.mkdtemp(),
                        is_progress_bar=False)
    tr.use_cuda_graph = use_graph
    model.train()
    g = torch.Generator().manual_seed(7 + rank)
    loader = [(torch.rand(per, *img, generator=g).to(dev), None) for _ in range(steps)]
    storer = defaultdict(list)
    tr._train_epoch(loader, storer, 0)
    torch.cuda.synchronize()
    state = {}
    nets = [("vae", model, opt)] + ([("disc", lf.discriminator, lf.optimizer_d)] if loss_name == "factor" else [])
    for tag, net, o in nets:
        for k, p in net.named_parameters():
            state["%s.%s" % (tag, k)] = p.detach().clone()
            state["%s.%s.m" % (tag, k)] = o.state[p]["exp_avg"].clone()
            state["%s.%s.v" % (tag, k)] = o.state[p]["exp_avg_sq"].clone()
    return state, storer, bool(tr._graphs), lf.n_train_steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--loss", default="btcvae")
    ap.add_argument("--steps", type=int, default=24)
    args = ap.parse_args()
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    shared = torch.cuda.device_count() < world
    dev = torch.device("cuda", 0 if shared else local)
    torch.cuda.set_device(dev)
    if shared:
        dist.init_process_group("gloo")
    else:
        dist.init_process_group("nccl", device_id=dev)
    per = 64 if args.loss == "factor" else 32
    img = (1, 64, 64)
    s_g, st_g, graphed, n_g = run(args.loss, True, dev, rank, world, args.steps, per, img)
    s_e, st_e, _, n_e = run(args.loss, False, dev, rank, world, args.steps, per, img)
    differ = [k for k in s_g if not torch.equal(s_g[k], s_e[k])]
    rep = {"rank": rank, "backend": "gloo(shared cuda:0)" if shared else "nccl", "graph_path": graphed,
           "steps": [n_g, n_e], "differ": differ[:8], "records": len(st_g["loss"]),
           "storer_equal": list(st_g.items()) == list(st_e.items())}
    rep["ok"] = bool(graphed and not differ and rep["storer_equal"] and n_g == n_e == args.steps
                     and rep["records"] == len(range(1, args.steps + 1, 5)))
    reps = [None] * world
    dist.all_gather_object(reps, rep)
    if rank == 0:
        print("DDP_ANNEAL " + json.dumps({"ok": all(r["ok"] for r in reps), "world": world, "loss": args.loss,
                                          "ranks": reps}), flush=True)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if rep["ok"] else 1)


if __name__ == "__main__":
    main()
