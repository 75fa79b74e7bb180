"""Device-resident training data: the dataset is decoded once, kept on the GPU as uint8, and every epoch is shuffled
and batched there.

The reference feeds training through a `DataLoader` that calls the dataset's Python `__getitem__` once per image
(utils/datasets.py:67-71; `ToTensor` at :182,206-210), every epoch.  `DeviceLoader` runs that `__getitem__` once per
image at construction and then yields each batch with two kinds of launch: one permutation per epoch
(dv_index_permutation) and one gather + byte-to-float conversion per batch (dv_gather_u8_to_f32).

Limits:
  * every value the dataset returns must be k/255 in fp32 (what `ToTensor` makes from bytes); anything else, such as
    normalised images, raises instead of being quantised;
  * the whole dataset must fit in free device memory as uint8 (dSprites 3.0 GB, CelebA 64x64 2.5 GB); there is no
    host fallback;
  * `__getitem__` is evaluated once, so a random transform (augmentation) would be frozen at its first draw.  Such a
    dataset needs the host `DataLoader`.
"""
import torch
import torch.distributed as dist

from disvae import ops, parallel

_DECODE_ROWS = 1024      # items read through __getitem__ per host -> device copy while the dataset is materialised


# ---- epoch plan (host only) ------------------------------------------------------------------------------------------
def padded_length(n, world=1, drop_last=False):
    """Positions of one epoch's order: n wrapped around to a multiple of `world`, or, with drop_last, cut down to one
    (the rule of parallel.ShardSampler)."""
    return n // world * world if drop_last else -(-n // world) * world


def batch_windows(n, batch_size, world=1, rank=0, drop_last=False):
    """(start, size) of this rank's block of every global batch in the epoch order (padded_length positions).

    A global batch is `world * batch_size` consecutive positions; rank r takes positions [r*b, (r+1)*b) of it.  The
    last, shorter global batch (its length is a multiple of `world`) is split equally among the ranks, or dropped with
    drop_last.  With world = 1 these are the batches of a DataLoader over the same order."""
    total = padded_length(n, world, drop_last)
    g = world * batch_size
    out = [(k * g + rank * batch_size, batch_size) for k in range(total // g)]
    rest = total % g
    if rest and not drop_last:
        per = rest // world
        out.append((total - rest + rank * per, per))
    return out


def quantize_unit_bytes(x, first_index=0):
    """fp32 images whose every value is k/255 (k = 0..255) -> the uint8 k.  Raises RuntimeError naming the first
    offending item (item `first_index + i` for row i of x) otherwise: only exact ToTensor output is stored as bytes."""
    if x.dtype != torch.float32:
        raise RuntimeError("DeviceLoader: dataset item %d is %s; expected float32 images in [0, 1] (ToTensor output)"
                           % (first_index, x.dtype))
    k = torch.round(x * 255)
    bad = ((k / 255) != x) | (k < 0) | (k > 255)
    if bool(bad.any()):
        row = int(bad.flatten(1).any(1).nonzero()[0])
        v = float(x[row][bad[row]][0])
        raise RuntimeError("DeviceLoader: dataset item %d holds %r, which is not k/255 for a byte k; only ToTensor images "
                           "of uint8 data can be kept on the device as bytes (normalised or resampled images cannot)"
                           % (first_index + row, v))
    return k.to(torch.uint8)


# ---- the loader ------------------------------------------------------------------------------------------------------
class DeviceLoader:
    """DeviceLoader(dataset, batch_size, shuffle=True, drop_last=False, seed=None, device=None)

    Drop-in for the reference's training `DataLoader`: iterating yields (images fp32 [b, C, H, W], dataset indices
    int64 [b]), both on the device; `len()` is the number of batches and `.dataset` the source dataset.  Each
    `iter()` is one epoch.  shuffle=True draws a new permutation per epoch on the device, keyed by `seed` (default
    `torch.initial_seed()`) and the epoch number; shuffle=False keeps the index order.

    The dataset is read once, at construction, through its own `__getitem__` (items `(image, label)` like the
    reference's datasets; images fp32 with values k/255), and stored as one uint8 tensor on the device.  See the module
    docstring for the limits.

    Under data parallelism (disvae.parallel.is_distributed()) every rank holds the whole dataset (each decodes 1/world
    of it, the slices are all-gathered), all ranks share rank 0's seed, and step i hands rank r the block
    [r*b, (r+1)*b) of global batch i, so every rank gets equally many rows and the ranks' blocks of one step, in rank
    order, form one batch of the single-process epoch order.
    """

    def __init__(self, dataset, batch_size, shuffle=True, drop_last=False, seed=None, device=None):
        self.dataset, self.batch_size, self.shuffle, self.drop_last = dataset, int(batch_size), bool(shuffle), bool(drop_last)
        if self.batch_size < 1:
            raise ValueError("DeviceLoader: batch_size must be positive, got %d" % self.batch_size)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("DeviceLoader keeps the dataset on a CUDA device; got %s (there is no host path)" % self.device)
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        ddp = parallel.is_distributed()
        self.world = dist.get_world_size() if ddp else 1
        self.rank = dist.get_rank() if ddp else 0
        self.n = len(dataset)
        if self.n < 1:
            raise ValueError("DeviceLoader: the dataset is empty")
        seed = torch.initial_seed() if seed is None else seed
        self.seed = parallel.broadcast_u64(seed) if ddp else int(seed) & 0xFFFFFFFFFFFFFFFF
        self.data = self._materialise()
        self.n_padded = padded_length(self.n, self.world, self.drop_last)
        self.windows = batch_windows(self.n, self.batch_size, self.world, self.rank, self.drop_last)
        self.epoch = 0
        self._offset = torch.zeros(1, dtype=torch.int64, device=self.device)

    def _materialise(self):
        first = self.dataset[0][0]
        shape = tuple(first.shape)
        row_bytes = first.numel()
        if row_bytes % 16:
            raise RuntimeError("DeviceLoader: an image of %s holds %d bytes, not a multiple of 16 (the gather kernel reads "
                               "16-byte chunks)" % ("x".join(map(str, shape)), row_bytes))
        per = -(-self.n // self.world)                       # rows this rank decodes (the last rank's slice is padded)
        lo, hi = min(self.rank * per, self.n), min((self.rank + 1) * per, self.n)
        need = (self.n if self.world == 1 else (self.world + 1) * per) * row_bytes   # + the gathered copy under DP
        free, _ = torch.cuda.mem_get_info(self.device)
        if need > free:
            raise RuntimeError("DeviceLoader: the dataset needs %d bytes of device memory as uint8 (%d items of %s) but "
                               "only %d bytes are free on %s; use the host DataLoader for it"
                               % (need, self.n, "x".join(map(str, shape)), free, self.device))
        rows = torch.empty((self.n if self.world == 1 else per,) + shape, dtype=torch.uint8, device=self.device)
        for a in range(lo, hi, _DECODE_ROWS):
            b = min(a + _DECODE_ROWS, hi)
            x = torch.stack([torch.as_tensor(self.dataset[i][0]) for i in range(a, b)])
            rows[a - lo:b - lo].copy_(quantize_unit_bytes(x, a))
        if self.world == 1:
            return rows
        if hi - lo < per:
            rows[hi - lo:].zero_()                           # padding rows, cut off after the gather
        return parallel.all_gather_rows(rows)[:self.n]

    def order(self, epoch):
        """The epoch's order of dataset indices (int64, n_padded entries, on the device): the permutation (or the
        identity) of [0, n), wrapped around to n_padded, or cut short with drop_last."""
        if self.shuffle:
            self._offset.fill_(epoch * self.n_padded)         # disjoint Philox counters per epoch
            perm = ops.index_permutation(self.n, self.seed, self._offset)
        else:
            perm = torch.arange(self.n, dtype=torch.int64, device=self.device)
        if self.n_padded > self.n:
            perm = torch.cat([perm, perm[:self.n_padded - self.n]])
        return perm[:self.n_padded]

    def epoch_indices(self):
        """The dataset indices of each batch of the next epoch (CUDA int64 views of one permutation); what `iter()`
        gathers.  Advances the epoch like `iter()`."""
        order = self.order(self.epoch)
        self.epoch += 1
        for start, size in self.windows:
            yield order[start:start + size]

    def __iter__(self):
        for idx in self.epoch_indices():
            yield ops.gather_u8_to_f32(self.data, idx), idx

    def __len__(self):
        return len(self.windows)


def device_loader_for(loader, device=None):
    """The DeviceLoader that stands in for a torch DataLoader: same dataset, batch size, shuffling and drop_last."""
    return DeviceLoader(loader.dataset, loader.batch_size, shuffle=isinstance(loader.sampler, torch.utils.data.RandomSampler),
                        drop_last=loader.drop_last, device=device)
