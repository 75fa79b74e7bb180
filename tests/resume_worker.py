#!/usr/bin/env python
"""One training run of tests/test_resume_gpu.py, in a process of its own:

    python tests/resume_worker.py SPEC PHASE SAVE_DIR OUT

SPEC is JSON: {"losses": [...], "img": 32|64, "loader": "device"|"host", "every": checkpoint_every, "sweep": bool}
(DISVAE_CUDA_GRAPH=0 in the environment for the eager path).  PHASE is
  * "full":   train EPOCHS epochs with save_state=True (the uninterrupted run);
  * "first":  train SPLIT epochs with save_state=True, then exit (the stopped run);
  * "resume": build the same Trainers, load training-state-{SPLIT-1}.pt from SAVE_DIR and train EPOCHS - SPLIT more.
Under torch.distributed.run (two ranks; gloo over CUDA tensors when the box has one GPU) each rank uses SAVE_DIR/rank{r}
and its own training-state file.  OUT (OUT.rank{r} under data parallelism) receives the state every member ends in:
parameters, Adam moments and step counts (the discriminator's too), Philox counters and the loss step counter.
"""
import json
import logging
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
EPOCHS, SPLIT = 4, 2
K, B, LOADER_SEED, SEED = 6, 128, 77, 5      # 6**4 = 1296 images: 10 batches of 128 and one of 16 per epoch


def dataset(size):
    """tests/synthetic_factors.FactorRectangles rounded to bytes (what ToTensor makes of 8-bit images)."""
    from synthetic_factors import FactorRectangles
    ds = FactorRectangles(k=K, size=size)
    ds.imgs = torch.round(ds.imgs * 255) / 255
    return ds


def loader(spec, dev, world):
    from disvae.data import DeviceLoader
    ds = dataset(spec["img"])
    if spec["loader"] == "device":
        return DeviceLoader(ds, B // world, shuffle=True, seed=LOADER_SEED, device=dev)
    return torch.utils.data.DataLoader(ds, batch_size=B // world, shuffle=True)


def trainer(kind, seed, img, save_dir, dev):
    """A Trainer as main.py builds one after torch.manual_seed(seed); annealing over 30 steps (the split falls at step
    22) and a recording step every 5."""
    import disvae
    from disvae.models.losses import get_loss_f
    os.makedirs(save_dir, exist_ok=True)
    torch.manual_seed(seed)
    model = disvae.init_specific_model("Burgess", (1, img, img), 10)
    opt = torch.optim.Adam(model.parameters(), lr=5e-4 if kind != "factor" else 1e-4)
    loss_f = get_loss_f(kind, rec_dist="bernoulli", reg_anneal=30, betaH_B=4, betaB_initC=0, betaB_finC=25, betaB_G=100,
                        btcvae_A=-1, btcvae_B=6, btcvae_G=1, n_data=K ** 4, factor_G=6.4, latent_dim=10, lr_disc=1e-4,
                        device=dev)
    loss_f.record_loss_every = 5
    return disvae.Trainer(model, opt, loss_f, device=dev, logger=logging.getLogger("resume"), save_dir=save_dir,
                          is_progress_bar=False)


def result(tr):
    lf = tr.loss_f
    out = {"graphs": len(tr._graphs), "steps": lf.n_train_steps, "noise": int(tr.model._rng_offset)}
    nets = [("vae", tr.model, tr.optimizer)]
    if hasattr(lf, "discriminator"):
        nets.append(("disc", lf.discriminator, lf.optimizer_d))
        out["perm"] = int(lf._perm_offset)
    for tag, net, opt in nets:
        for name, p in net.named_parameters():
            out["%s.%s" % (tag, name)] = p.detach().cpu()
            for k in ("exp_avg", "exp_avg_sq", "step"):
                out["%s.%s.%s" % (tag, name, k)] = opt.state[p][k].detach().cpu()
    return out


def main():
    for p in (ROOT, os.path.join(ROOT, "disentangling-vae_b200"), HERE):
        sys.path.insert(0, p)
    import torch.distributed as dist
    spec, phase, save_dir, out = json.loads(sys.argv[1]), sys.argv[2], sys.argv[3], sys.argv[4]
    world = int(os.environ.get("WORLD_SIZE", "1"))
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    rank = 0
    if world > 1:
        rank = int(os.environ["RANK"])
        if torch.cuda.device_count() < world:
            dist.init_process_group("gloo")
        else:
            dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", rank)))
            torch.cuda.set_device(dev)
            dist.init_process_group("nccl", device_id=dev)
        save_dir, out = os.path.join(save_dir, "rank%d" % rank), "%s.rank%d" % (out, rank)
    from disvae.training import training_state_filename
    from disvae.utils.modelIO import load_training_state

    members = [trainer(kind, SEED + k, spec["img"], os.path.join(save_dir, "m%d_%s" % (k, kind)), dev)
               for k, kind in enumerate(spec["losses"])]
    if phase == "resume":
        for m in members:
            load_training_state(m, os.path.join(m.save_dir, training_state_filename(SPLIT - 1)))
    data = loader(spec, dev, world)
    epochs = EPOCHS if phase == "full" else SPLIT if phase == "first" else EPOCHS - SPLIT
    if spec.get("sweep"):
        from disvae.sweep import Sweep
        Sweep(members, seeds=[SEED + k for k in range(len(members))])(data, epochs, spec["every"], save_state=True)
    else:
        members[0](data, epochs, spec["every"], save_state=True)
    torch.cuda.synchronize()
    torch.save([result(m) for m in members], out)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
