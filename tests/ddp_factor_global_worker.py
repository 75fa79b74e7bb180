#!/usr/bin/env python
"""One rank of the global-batch FactorVAE check (FactorKLoss.global_batch, SURVEY.md 8e); launched by
tests/test_factor_global_gpu.py as

    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port P \
        tests/ddp_factor_global_worker.py

With two visible GPUs every rank takes its own device over NCCL; with one, both ranks share cuda:0 and the collectives
run over gloo.  Checked on every rank, verdict gathered on rank 0 (exit code 0/1, one "DDP_FACTOR_GLOBAL {json}" line):
  (a) injected noise and global permutations: ONE oracle process on the global batch arranged as [first halves of all
      ranks; second halves of all ranks] -- its loss == the mean over ranks of the ranks' losses (1e-4), its gradients
      == the rank-averaged gradients (3e-3 of each tensor's max, as tests/ddp_worker.py), and the Adam moments after
      the deferred optimizer steps follow from them
  (b) device permutations, ranks seeded differently: every rank's z_perm == its rows of ONE permutation of the gathered
      second halves, under the seed agreed from rank 0, bit for bit; also with more than 4096 gathered rows
  (c) further eager steps: replicas bit-identical, loss decreases, no CUDA graph
"""
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
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    shared = torch.cuda.device_count() < world
    dev = torch.device("cuda", 0 if shared else local)
    torch.cuda.set_device(dev)
    if shared:
        dist.init_process_group("gloo")
    else:
        dist.init_process_group("nccl", device_id=dev)

    import disvae
    from disvae import ops
    from disvae.models.losses import get_loss_f
    from disvae.parallel import all_gather_rows, broadcast_parameters, shard_batch
    from oracle import disvae_oracle as O

    img, z, per = (1, 64, 64), 10, 32
    h = per // 2
    lr, lr_d = 5e-4, 1e-4
    torch.manual_seed(1234 + rank)                     # different seeds per rank: the permutation key must not follow
    model = disvae.init_specific_model("Burgess", img, z).to(dev)
    broadcast_parameters(model)
    opt = torch.optim.Adam(model.parameters(), lr=lr)
    lf = get_loss_f("factor", rec_dist="bernoulli", reg_anneal=0, factor_G=6.4, latent_dim=z, lr_disc=lr_d, device=dev)
    lf.global_batch = True
    tr = disvae.Trainer(model, opt, lf, device=dev, logger=logging.getLogger("ddp"), save_dir=tempfile.mkdtemp(),
                        is_progress_bar=False)
    model.train()
    broadcast_parameters(lf.discriminator)
    p0 = OrderedDict((k, v.detach().cpu().clone()) for k, v in model.state_dict().items())
    d0 = OrderedDict((k, v.detach().cpu().clone()) for k, v in lf.discriminator.state_dict().items())

    g = torch.Generator().manual_seed(7)
    xg = torch.rand(per * world, *img, generator=g)
    e1g, e2g = torch.randn(h * world, z, generator=g), torch.randn(h * world, z, generator=g)
    perms_g = torch.stack([torch.randperm(h * world, generator=g) for _ in range(z)])

    # ---- (a) oracle: ONE process on the arranged global batch ---------------------------------------------------------
    shards = [shard_batch(xg, r, world) for r in range(world)]
    x_arr = torch.cat([s[:h] for s in shards] + [s[h:] for s in shards])
    leaf, dleaf = O.make_leaf_params(p0), O.make_leaf_params(d0)
    o_loss, _, _ = O.factor_step(leaf, dleaf, O.make_adam(leaf, 0.0), O.make_adam(dleaf, 0.0, betas=(0.5, 0.9)), x_arr,
                                 dict(rec_dist="bernoulli", reg_anneal=0, factor_G=6.4), step=1,
                                 eps1=e1g, eps2=e2g, perms=perms_g)
    o_loss = o_loss.item()
    gref = OrderedDict((k, v.grad.clone()) for k, v in leaf.items())
    gref.update(("disc." + k, v.grad.clone()) for k, v in dleaf.items())

    def mean_over_ranks(v):
        allv = [None] * world
        dist.all_gather_object(allv, v)
        return sum(allv) / world

    x = shard_batch(xg, rank, world)
    inject = dict(eps1=shard_batch(e1g, rank, world).to(dev), eps2=shard_batch(e2g, rank, world).to(dev), perms=perms_g)
    loss = mean_over_ranks(tr._grads_only(x, None, **inject).item())
    lf.n_train_steps = 0
    rep = {"rank": rank, "backend": "gloo(shared cuda:0)" if shared else "nccl", "loss_mean_over_ranks": loss,
           "oracle_loss": o_loss, "loss_rel": abs(loss - o_loss) / abs(o_loss)}
    named = OrderedDict(model.named_parameters())
    named.update(("disc." + k, p) for k, p in lf.discriminator.named_parameters())
    rep["avg_grad_rel_err"] = max(((p.grad.detach().cpu() - gref[k]).abs().max() / gref[k].abs().max().clamp_min(1e-30)).item()
                                  for k, p in named.items())

    loss2 = mean_over_ranks(tr._grads_only(x, None, **inject).item())   # same gradients again ...
    tr._optimizer_steps()                                                # ... and the two deferred optimizer steps
    rep["step_loss_rel"] = abs(loss2 - o_loss) / abs(o_loss)
    m_err = v_err = 0.0
    for k, p in named.items():
        is_d = k.startswith("disc.")
        st = (lf.optimizer_d if is_d else opt).state[p]
        b1, b2 = (0.5, 0.9) if is_d else (0.9, 0.999)
        gm = gref[k]
        m_err = max(m_err, ((st["exp_avg"].cpu() - (1 - b1) * gm).abs().max() / ((1 - b1) * gm).abs().max().clamp_min(1e-30)).item())
        v_err = max(v_err, ((st["exp_avg_sq"].cpu() - (1 - b2) * gm * gm).abs().max()
                            / ((1 - b2) * gm * gm).abs().max().clamp_min(1e-30)).item())
    rep["exp_avg_rel_err"], rep["exp_avg_sq_rel_err"] = m_err, v_err

    # ---- (b) device permutations: record what the loss permutes, then restate it ----------------------------------------
    calls = []
    real_rows = ops.permute_dims_rows

    def spy(zz, row0, nrows, perms=None, seed=0, offset_dev=None):
        off0 = offset_dev.clone()
        out = real_rows(zz, row0, nrows, perms, seed, offset_dev)
        calls.append((zz.clone(), row0, nrows, seed, off0, out.clone(), offset_dev.clone()))
        return out

    ops.permute_dims_rows = spy
    xb = x.to(dev)
    tr._step(xb, None)
    big = 2 * 2100                                                      # 2 x 2100 gathered rows: the multi-CTA sort
    tr._step(torch.rand(big, *img, generator=torch.Generator().manual_seed(11 + rank)).to(dev), None)
    ops.permute_dims_rows = real_rows
    seeds = [None] * world
    dist.all_gather_object(seeds, int(torch.initial_seed()))
    agreed = (seeds[0] ^ 0x9E3779B97F4A7C15) & 0xFFFFFFFFFFFFFFFF
    perm_ok = len(calls) == 2 and seeds[0] != seeds[1]
    for zz, row0, nrows, seed, off0, out, off1 in calls:
        B = zz.size(0)
        zsame = all_gather_rows(zz.view(1, -1))                          # the gathered batch is the same on every rank
        ref = ops.permute_dims(zz, None, seed, off0.clone())
        perm_ok = (perm_ok and seed == agreed and B == world * nrows and row0 == rank * nrows
                   and all(torch.equal(zsame[0], t) for t in zsame)
                   and torch.equal(out, ref[row0:row0 + nrows]) and off1.item() == off0.item() + B * z)
    rep["perm_calls"] = [(c[0].size(0), c[1], c[2]) for c in calls]
    rep["device_perm_ok"] = bool(perm_ok)

    # ---- (c) lock-step over further eager steps ----------------------------------------------------------------------
    torch.manual_seed(99)
    first = last = None
    for _ in range(10):
        v = tr._step(xb, None).item()
        first = v if first is None else first
        last = v
    flat = torch.cat([p.detach().flatten() for p in named.values()])
    if shared:
        flat = flat.cpu()
    gathered = [torch.empty_like(flat) for _ in range(world)]
    dist.all_gather(gathered, flat)
    rep["in_sync"] = all(torch.equal(gathered[0], t) for t in gathered)
    rep["graph_path"] = bool(tr._graphs)
    rep["loss_first"], rep["loss_last"] = first, last
    ok = (rep["loss_rel"] < 1e-4 and rep["step_loss_rel"] < 1e-4 and rep["avg_grad_rel_err"] < 3e-3
          and rep["exp_avg_rel_err"] < 3e-3 and rep["exp_avg_sq_rel_err"] < 6e-3 and rep["device_perm_ok"]
          and rep["in_sync"] and last < first and not rep["graph_path"])
    rep["ok"] = bool(ok)
    reps = [None] * world
    dist.all_gather_object(reps, rep)
    if rank == 0:
        print("DDP_FACTOR_GLOBAL " + json.dumps({"ok": all(r["ok"] for r in reps), "world": world, "ranks": reps}),
              flush=True)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
