#!/usr/bin/env python
"""One rank of the data-parallel parity check (SURVEY.md 8e); launched by tests/test_ddp_gpu.py and
scripts/gpu_multi.sh as

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 --master-port P tests/ddp_worker.py \
        --loss btcvae|factor|betaH [--per 32] [--z 10]

With N visible GPUs every rank takes its own device over NCCL; with fewer GPUs than ranks (the single-GPU test box) all
ranks share cuda:0 and the collectives run over gloo on CUDA tensors -- the host-side logic under test (the FactorVAE
discriminator broadcast, and the one gradient average, `GradAverage` via Trainer._average_grads, that eager and replayed
steps share before the fused Adam takes the 1/world scale) is the same.

Checked on every rank, verdict gathered on rank 0 (exit code 0/1, one "DDP_WORKER {json}" line):
  * rank r's loss == oracle loss on shard r                                   (1e-4)
  * rank-averaged gradients of every parameter (FactorVAE: also the discriminator's) == mean over shards of the
    oracle's gradients                                                        (3e-3 of the tensor's max: plumbing check)
  * after one real optimisation step: Adam's exp_avg == (1-beta1) * that mean gradient, exp_avg_sq == (1-beta2) * its
    square (linear / quadratic in the gradient -- unlike the parameters, which move by +-lr whatever the gradient is)
  * replicas stay bit-identical over further steps (device noise, CUDA-graph path where eligible), loss decreases
  * every one of those steps, eager or replayed, FactorVAE included, makes exactly one all-reduce of the gradient
    buffer (other all-reduces, e.g. the global-batch estimator's, are not counted)
  * after the first (eager) step and after the last one, every `p.grad` (FactorVAE: the discriminator's too) lies in
    that one buffer
"""
import argparse
import json
import logging
import os
import sys
import tempfile
from collections import OrderedDict

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "disentangling-vae_b200"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--loss", default="btcvae")
    ap.add_argument("--per", type=int, default=32, help="images per rank (FactorVAE: two halves of per/2)")
    ap.add_argument("--z", type=int, default=10)
    ap.add_argument("--img", default="1,64,64")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--global-btcvae", action="store_true",
                    help="SURVEY.md 8f-1: the estimator of the all-gathered GLOBAL batch; the oracle is then ONE process on "
                         "the whole batch: mean of the ranks' losses == its loss, averaged gradients == its gradients")
    args = ap.parse_args()
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    ngpu = torch.cuda.device_count()
    shared = ngpu < world
    dev = torch.device("cuda", 0 if shared else local)
    torch.cuda.set_device(dev)
    if shared:
        dist.init_process_group("gloo")
    else:
        dist.init_process_group("nccl", device_id=dev)

    import disvae
    from disvae.models.losses import get_loss_f
    from disvae.parallel import broadcast_parameters, shard_batch
    from oracle import disvae_oracle as O

    img, z, per = tuple(int(v) for v in args.img.split(",")), args.z, args.per
    n_data, lr, lr_d = 202599, 5e-4, 1e-4
    factor = args.loss == "factor"
    torch.manual_seed(1234 + rank)                     # different init per rank: the broadcast must fix it
    model = disvae.init_specific_model("Burgess", img, z).to(dev)
    broadcast_parameters(model)
    opt = torch.optim.Adam(model.parameters(), lr=lr)
    kw = dict(rec_dist="bernoulli", reg_anneal=0, betaH_B=4, btcvae_A=1, btcvae_B=6, btcvae_G=1, n_data=n_data,
              factor_G=6.4, latent_dim=z, lr_disc=lr_d, device=dev)
    lf = get_loss_f(args.loss, **kw)                   # factor: every rank draws its OWN discriminator here ...
    glob = args.global_btcvae
    if glob:
        assert args.loss == "btcvae"
        lf.global_batch = True
    tr = disvae.Trainer(model, opt, lf, device=dev, logger=logging.getLogger("ddp"), save_dir=tempfile.mkdtemp(),
                        is_progress_bar=False)
    model.train()
    if factor:
        broadcast_parameters(lf.discriminator)         # ... (the Trainer broadcasts it too, at its first factor step)
    p0 = OrderedDict((k, v.detach().cpu().clone()) for k, v in model.state_dict().items())
    d0 = OrderedDict((k, v.detach().cpu().clone()) for k, v in lf.discriminator.state_dict().items()) if factor else None

    g = torch.Generator().manual_seed(7)
    xg = torch.rand(per * world, *img, generator=g)
    if factor:
        h = per // 2
        e1g, e2g = torch.randn(h * world, z, generator=g), torch.randn(h * world, z, generator=g)
        permsg = [torch.stack([torch.randperm(h, generator=g) for _ in range(z)]) for _ in range(world)]
    else:
        epsg = torch.randn(per * world, z, generator=g)

    # ---- oracle: loss and gradients of every shard, mean over shards --------------------------------------
    leaf = O.make_leaf_params(p0)
    dleaf = O.make_leaf_params(d0) if factor else None
    o_losses, gsum = [], None
    if glob:                                           # one process, the whole batch
        recon, (mu, lv), zz = O.vae_forward(leaf, xg, epsg)
        l, _ = O.loss_btcvae(xg, recon, mu, lv, zz, n_data, 1, 6, 1, "bernoulli", 1, 0)
        l.backward()
        o_losses = [l.item()] * world
        gsum = OrderedDict((k, v.grad.clone() * world) for k, v in leaf.items())
    for r in range(0 if glob else world):
        for v in list(leaf.values()) + (list(dleaf.values()) if factor else []):
            v.grad = None
        xr = shard_batch(xg, r, world)
        if factor:
            l, _, _ = O.factor_step(leaf, dleaf, O.make_adam(leaf, 0.0), O.make_adam(dleaf, 0.0, betas=(0.5, 0.9)), xr,
                                    dict(rec_dist="bernoulli", reg_anneal=0, factor_G=6.4), step=1,
                                    eps1=shard_batch(e1g, r, world), eps2=shard_batch(e2g, r, world), perms=permsg[r])
        else:
            er = shard_batch(epsg, r, world)
            recon, (mu, lv), zz = O.vae_forward(leaf, xr, er)
            if args.loss == "btcvae":
                l, _ = O.loss_btcvae(xr, recon, mu, lv, zz, n_data, 1, 6, 1, "bernoulli", 1, 0)
            else:
                l, _ = O.loss_betaH(xr, recon, mu, lv, 4, "bernoulli", 1, 0)
            l.backward()
        o_losses.append(l.item())
        gr = OrderedDict((k, v.grad.clone()) for k, v in leaf.items())
        if factor:
            gr.update(("disc." + k, v.grad.clone()) for k, v in dleaf.items())
        gsum = gr if gsum is None else OrderedDict((k, gsum[k] + gr[k]) for k in gr)
    gmean = OrderedDict((k, v / world) for k, v in gsum.items())

    # ---- ours: gradients only, then one real step ---------------------------------------------------------
    x = shard_batch(xg, rank, world)
    inject = {}
    if factor:
        inject = dict(eps1=shard_batch(e1g, rank, world).to(dev), eps2=shard_batch(e2g, rank, world).to(dev), perms=permsg[rank])
    else:
        model.inject_noise([shard_batch(epsg, rank, world)])
    loss = tr._grads_only(x, None, **inject).item()
    lf.n_train_steps = 0
    rep = {"rank": rank, "backend": "gloo(shared cuda:0)" if shared else "nccl", "loss": loss, "oracle_loss": o_losses[rank]}
    if glob:                                           # a rank's loss is its rows' share: compare the mean over ranks
        allv = [None] * world
        dist.all_gather_object(allv, loss)
        loss = sum(allv) / world
        rep["loss_mean_over_ranks"] = loss
    rep["loss_rel"] = abs(loss - o_losses[rank]) / abs(o_losses[rank])
    named = OrderedDict(model.named_parameters())
    if factor:
        named.update(("disc." + k, p) for k, p in lf.discriminator.named_parameters())
    worst = 0.0
    for k, p in named.items():
        e = ((p.grad.detach().cpu() - gmean[k]).abs().max() / gmean[k].abs().max().clamp_min(1e-30)).item()
        worst = max(worst, e)
    rep["avg_grad_rel_err"] = worst

    # one real step with the same injected noise: Adam moments are linear/quadratic in the averaged gradient
    if not factor:
        model.inject_noise([shard_batch(epsg, rank, world)])
        tr.use_cuda_graph = False
        loss2 = tr._step(x, None).item()
        tr.use_cuda_graph = True
    else:
        loss2 = tr._grads_only(x, None, **inject).item()             # same gradients again ...
        tr._optimizer_steps()                                        # ... and the two deferred optimizer steps
    if glob:
        allv = [None] * world
        dist.all_gather_object(allv, loss2)
        loss2 = sum(allv) / world
    rep["step_loss_rel"] = abs(loss2 - o_losses[rank]) / abs(o_losses[rank])
    m_err = v_err = 0.0
    for k, p in named.items():
        is_d = k.startswith("disc.")
        st = (lf.optimizer_d if is_d else opt).state[p]
        b1, b2 = (0.5, 0.9) if is_d else (0.9, 0.999)
        gm = gmean[k]
        m_err = max(m_err, ((st["exp_avg"].cpu() - (1 - b1) * gm).abs().max() / ((1 - b1) * gm).abs().max().clamp_min(1e-30)).item())
        v_err = max(v_err, ((st["exp_avg_sq"].cpu() - (1 - b2) * gm * gm).abs().max()
                            / ((1 - b2) * gm * gm).abs().max().clamp_min(1e-30)).item())
    rep["exp_avg_rel_err"], rep["exp_avg_sq_rel_err"] = m_err, v_err

    # ---- lock-step over further steps (device noise; CUDA-graph path where the loss allows it) ---------------
    torch.manual_seed(99)
    first = last = None
    xb = x.to(dev)
    buf = tr._grad_avg.flat                            # the gradient buffer (built by the first _grads_only)
    all_reduce, n_grad_reduce = dist.all_reduce, [0]

    def counting_all_reduce(t, *a, **k):
        if t is buf:
            n_grad_reduce[0] += 1
        return all_reduce(t, *a, **k)

    def grads_in_one_buffer():
        return {p.grad.untyped_storage().data_ptr() for p in named.values()} == {buf.untyped_storage().data_ptr()}

    dist.all_reduce, counts = counting_all_reduce, []
    for it in range(args.steps):
        n_grad_reduce[0] = 0
        v = tr._step(xb, None).item()
        counts.append(n_grad_reduce[0])
        if it == 0:
            rep["grads_in_one_buffer_eager"] = grads_in_one_buffer()
        first = v if first is None else first
        last = v
    dist.all_reduce = all_reduce
    rep["grads_in_one_buffer_last"] = grads_in_one_buffer()
    rep["grad_allreduces_per_step"] = counts             # steps 1-2 eager, then replays on the graph path
    flat = torch.cat([p.detach().flatten() for p in named.values()])
    if shared:
        flat = flat.cpu()                                            # gloo has no CUDA all_gather
    gathered = [torch.empty_like(flat) for _ in range(world)]
    dist.all_gather(gathered, flat)
    rep["in_sync"] = all(torch.equal(gathered[0], t) for t in gathered)
    rep["graph_path"] = bool(tr._graphs)
    rep["global_btcvae"] = glob
    rep["loss_first"], rep["loss_last"] = first, last
    # gradients: this checks the PLUMBING (shards, averaging, deferred optimizer steps) -- an error there is O(1); the
    # arithmetic is held to 1e-4 on the same ReLU branch by tests/test_fullsize_gpu.py.  3e-3 leaves room for the
    # occasional ReLU unit that two fp32 evaluation orders round to opposite sides of zero (oracle/same_branch.py).
    ok = (rep["loss_rel"] < 1e-4 and rep["step_loss_rel"] < 1e-4 and rep["avg_grad_rel_err"] < 3e-3
          and rep["exp_avg_rel_err"] < 3e-3 and rep["exp_avg_sq_rel_err"] < 6e-3 and rep["in_sync"] and last < first
          and (glob or rep["graph_path"] or dev.type != "cuda") and counts == [1] * args.steps
          and rep["grads_in_one_buffer_eager"] and rep["grads_in_one_buffer_last"])
    rep["ok"] = bool(ok)
    reps = [None] * world
    dist.all_gather_object(reps, rep)
    if rank == 0:
        print("DDP_WORKER " + json.dumps({"ok": all(r["ok"] for r in reps), "world": world, "loss": args.loss, "ranks": reps}),
              flush=True)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
