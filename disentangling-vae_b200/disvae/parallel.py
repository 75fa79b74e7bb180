"""Data-parallel plumbing: one process per GPU, one flat fp32 gradient buffer, ONE NCCL
all-reduce per step over NVLink/NVSwitch (SURVEY.md section 8e).  The reference has no
distributed code at all; semantics are defined as "rank r computes the reference loss on its
shard, gradients are averaged over ranks, every rank applies the same optimizer step"."""
import torch
import torch.distributed as dist


def is_distributed():
    return dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1


def rank_salt():
    """Folded into the device Philox keys (reparameterisation noise, latent permutations): 0 for a single process,
    a rank-dependent odd multiplier otherwise, so replicas seeded identically draw independent streams."""
    if not is_distributed():
        return 0
    return (dist.get_rank() * 0xD1342543DE82EF95) & 0xFFFFFFFFFFFFFFFF


class GradAverage:
    """The rank average of the gradients of `params` (in order: the model's, then FactorVAE's discriminator's) through
    one flat fp32 buffer.  A call gathers every `.grad` into the buffer (a missing one as zeros), all-reduces it (sum)
    and re-points every `.grad` to its view; it returns 1/world, the scale that turns those sums into the mean."""

    def __init__(self, params):
        self.params = [p for p in params if p.requires_grad]
        p0 = self.params[0]
        self.flat = torch.zeros(sum(p.numel() for p in self.params), dtype=torch.float32, device=p0.device)
        self.views, off = [], 0
        for p in self.params:
            self.views.append(self.flat[off:off + p.numel()].view_as(p))
            off += p.numel()

    def __call__(self):
        grads = [p.grad for p in self.params]
        if all(g is not None and g.data_ptr() != v.data_ptr() for g, v in zip(grads, self.views)):
            torch.cat([g.reshape(-1) for g in grads], out=self.flat)       # one kernel
        else:                                   # some gradient missing, or already in the buffer (accumulated into it)
            for g, v in zip(grads, self.views):
                if g is None:
                    v.zero_()
                elif g.data_ptr() != v.data_ptr():
                    v.copy_(g)
        dist.all_reduce(self.flat, op=dist.ReduceOp.SUM)
        for p, v in zip(self.params, self.views):
            p.grad = v
        return 1.0 / dist.get_world_size()


def shard_batch(data, rank=None, world_size=None):
    """Contiguous, equal shard of a global batch for this rank (SURVEY.md 8e)."""
    if rank is None:
        rank = dist.get_rank() if is_distributed() else 0
    if world_size is None:
        world_size = dist.get_world_size() if is_distributed() else 1
    per = data.size(0) // world_size
    return data[rank * per:(rank + 1) * per]


class ShardSampler(torch.utils.data.Sampler):
    """Index sampler for one rank of a data-parallel job -- the role torch's DistributedSampler plays for the reference's
    DataLoader (utils/datasets.py:67-71 has `shuffle=True`, one process): every epoch ONE permutation of the dataset,
    identical on all ranks (seed + epoch), padded by wrapping around to a multiple of the world size, dealt out
    round-robin; `set_epoch` like DistributedSampler.  Without shuffling: the identity order."""

    def __init__(self, dataset_len, rank=None, world_size=None, shuffle=True, seed=0, drop_last=False):
        if rank is None:
            rank = dist.get_rank() if is_distributed() else 0
        if world_size is None:
            world_size = dist.get_world_size() if is_distributed() else 1
        self.n, self.rank, self.world, self.shuffle, self.seed, self.epoch = int(dataset_len), rank, world_size, shuffle, seed, 0
        self.per_rank = self.n // world_size if drop_last else -(-self.n // world_size)
        self.total = self.per_rank * world_size

    def set_epoch(self, epoch):
        self.epoch = int(epoch)

    def __iter__(self):
        if self.shuffle:
            g = torch.Generator().manual_seed(self.seed + self.epoch)
            order = torch.randperm(self.n, generator=g).tolist()
        else:
            order = list(range(self.n))
        if self.total > self.n:
            order += order[:self.total - self.n]
        order = order[:self.total]
        return iter(order[self.rank:self.total:self.world])

    def __len__(self):
        return self.per_rank


def broadcast_parameters(module, src=0):
    """Make every rank start from rank `src`'s parameters."""
    if not is_distributed():
        return
    for p in module.parameters():
        dist.broadcast(p.data, src=src)


# ---------------------------------------------------------------------------------------------------------
# Row collectives for the global-batch beta-TCVAE estimator (SURVEY.md 8f-1) and FactorVAE permutation: every rank
# contributes the same number of rows.  NCCL: one all_gather_into_tensor / reduce_scatter_tensor.  gloo (CPU tests;
# CUDA tensors of ranks that share one GPU in tests/ddp_worker.py) has neither for CUDA tensors nor reduce_scatter at
# all: staged through an all_gather / all_reduce on the host, same results.
# ---------------------------------------------------------------------------------------------------------
def _backend(group=None):
    return dist.get_backend(group)


def all_gather_rows(t, group=None):
    """[b, n] on every rank -> [world * b, n], rank-major (rank r's rows at [r*b, (r+1)*b))."""
    world = dist.get_world_size(group)
    t = t.contiguous()
    if _backend(group) == "nccl":
        out = torch.empty((world * t.size(0),) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
        dist.all_gather_into_tensor(out, t, group=group)
        return out
    host = t.detach().cpu()
    parts = [torch.empty_like(host) for _ in range(world)]
    dist.all_gather(parts, host, group=group)
    return torch.cat(parts, dim=0).to(t.device)


def _small_tensor(values, group=None):
    """int64 tensor for a small collective: on the current GPU for NCCL, on the host for gloo."""
    dev = torch.device("cuda", torch.cuda.current_device()) if _backend(group) == "nccl" else torch.device("cpu")
    return torch.tensor(values, dtype=torch.int64, device=dev)


def check_equal_rows(n, group=None):
    """Raise RuntimeError unless every rank passes the same row count `n` (one MAX all-reduce of (n, -n)).  The row
    collectives need equal blocks: all_gather_into_tensor with mismatched sizes hangs or mixes up rows."""
    t = _small_tensor([n, -n], group)
    dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
    hi, lo = int(t[0]), -int(t[1])
    if hi != lo:
        raise RuntimeError("data parallel: the ranks hold different numbers of rows (from %d to %d; this rank %d); "
                           "the global-batch losses need equal shards" % (lo, hi, n))


def broadcast_u64(value, src=0, group=None):
    """Rank `src`'s unsigned 64-bit integer on every rank (e.g. a Philox key all ranks must share)."""
    v = int(value) & 0xFFFFFFFFFFFFFFFF
    t = _small_tensor([v - (1 << 64) if v >= (1 << 63) else v], group)
    dist.broadcast(t, src=src, group=group)
    return int(t[0]) & 0xFFFFFFFFFFFFFFFF


def reduce_scatter_rows(t, group=None):
    """[world * b, n] partial sums on every rank -> this rank's [b, n] block of the sum over ranks."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    t = t.contiguous()
    b = t.size(0) // world
    if _backend(group) == "nccl":
        out = torch.empty((b,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
        dist.reduce_scatter_tensor(out, t, op=dist.ReduceOp.SUM, group=group)
        return out
    host = t.detach().cpu().clone()
    dist.all_reduce(host, op=dist.ReduceOp.SUM, group=group)
    return host[rank * b:(rank + 1) * b].to(t.device)
