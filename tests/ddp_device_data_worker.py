#!/usr/bin/env python
"""One rank of the data-parallel DeviceLoader check; launched by tests/test_device_data_gpu.py as

    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port P \
        tests/ddp_device_data_worker.py

With as many GPUs as ranks every rank takes its own device over NCCL; otherwise all ranks share cuda:0 and the
collectives run over gloo.  Checked on every rank, verdict on rank 0 (one "DDP_DEVICE_DATA {json}" line):
  * every rank holds rank 0's seed and the same epoch order, which is the numpy Philox restatement's permutation
    wrapped around to a multiple of the world size;
  * the ranks' blocks of each step, joined in rank order, are one contiguous global batch of that order, and the
    steps of an epoch cover the padded order exactly once;
  * every batch holds the images of its indices, and the device dataset's bytes digest is reported for the parent to
    compare with a single-process build.
"""
import hashlib
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


class KDataset(torch.utils.data.Dataset):
    """Images of bytes k, returned as ToTensor would (float32 k/255, CHW), with a label, like the reference's datasets."""

    def __init__(self, n, shape, seed=0):
        self.imgs = np.random.default_rng(seed).integers(0, 256, size=(n,) + tuple(shape), dtype=np.uint8)

    def __len__(self):
        return len(self.imgs)

    def __getitem__(self, i):
        return torch.from_numpy(self.imgs[i]).float().div(255), 0


N, SHAPE, B, EPOCHS = 1003, (1, 32, 32), 16, 2


def digest(data):
    return hashlib.sha256(data.cpu().numpy().tobytes()).hexdigest()


def main():
    for p in (ROOT, os.path.join(ROOT, "disentangling-vae_b200"), HERE):
        sys.path.insert(0, p)
    import torch.distributed as dist
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    shared = torch.cuda.device_count() < world
    dev = torch.device("cuda", 0 if shared else local)
    torch.cuda.set_device(dev)
    if shared:
        dist.init_process_group("gloo")
    else:
        dist.init_process_group("nccl", device_id=dev)
    from disvae import parallel
    from disvae.data import DeviceLoader, batch_windows
    from test_factor_global_gpu import host_perms

    ds = KDataset(N, SHAPE, seed=5)
    dl = DeviceLoader(ds, B, shuffle=True, seed=1000 + rank)           # rank 0's seed must win
    rep = {"world": world, "rank": rank}
    rep["seed"] = dl.seed == 1000
    rep["n_padded"] = dl.n_padded == -(-N // world) * world
    rep["len"] = len(dl) == len(batch_windows(N, B, world, rank))

    def gather(t):
        return parallel.all_gather_rows(t.reshape(1, -1))

    same, host, joined_ok, cover, images = True, True, True, True, True
    for epoch in range(EPOCHS):
        order = dl.order(epoch)
        g = gather(order)
        same &= all(torch.equal(g[0], g[r]) for r in range(world))
        perm = host_perms(N, 1, dl.seed, epoch * dl.n_padded)[0]
        expect = torch.cat([perm, perm[:dl.n_padded - N]])
        host &= torch.equal(order.cpu(), expect)
        pos, seen = 0, []
        for x, idx in dl:                                                 # epoch `epoch` of the loader
            blocks = parallel.all_gather_rows(idx.view(1, -1)).cpu()      # equal block sizes on every rank
            joined = blocks.reshape(-1)
            joined_ok &= torch.equal(joined, expect[pos:pos + joined.numel()])
            pos += joined.numel()
            seen.append(joined)
            images &= torch.equal(x, torch.stack([ds[int(i)][0] for i in idx.cpu()]).to(dev))
        cover &= pos == dl.n_padded and torch.equal(torch.cat(seen), expect)
    rep.update(same_order=bool(same), host_order=bool(host), joined=bool(joined_ok), cover=bool(cover),
               images=bool(images), digest=digest(dl.data))
    reps = [None] * world
    dist.all_gather_object(reps, rep)
    if rank == 0:
        ok = all(r[k] for r in reps for k in ("seed", "n_padded", "len", "same_order", "host_order", "joined", "cover",
                                               "images"))
        ok = ok and len({r["digest"] for r in reps}) == 1
        print("DDP_DEVICE_DATA " + json.dumps(dict(ok=bool(ok), world=world, digest=reps[0]["digest"], ranks=reps)))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
