"""What the GPU tests of the disentanglement-score kernels share: guarded device buffers, raw C-ABI calls that check
their launch count, bit comparisons, graph replays, the layouts of mu, grid values, and the synthetic codes and
datasets of the DCI and modularity tests.  Not collected by pytest; importing it needs no GPU."""
import numpy as np
import torch

DEV = torch.device("cuda", 0)
OFFB = 16                    # every operand starts 16 bytes into its allocation
GUARDB = 1024                # bytes of sentinel after it
SENT32 = 0x7FBADBAD          # NaN as fp32
SENT64 = 0x7FFBADBADBADBADB  # NaN as fp64
DV_OK, DV_ERR_BAD_SHAPE, DV_ERR_BAD_ARG, DV_ERR_WORKSPACE = 0, -1, -2, -3
LAYOUTS = ["contiguous", "q_zCx", "padded", "colmajor"]


class Buf:
    """n elements of `dtype` 16 bytes into a device allocation, sentinel words before and after them."""

    def __init__(self, n, dtype, fill=None):
        self.es = torch.empty(0, dtype=dtype).element_size()
        self.n = n
        self.raw = torch.empty(OFFB + n * self.es + GUARDB, dtype=torch.uint8, device=DEV)
        self._words().fill_(SENT32 if self.es == 4 else SENT64)
        self.body = self.raw[OFFB:OFFB + n * self.es].view(dtype)
        if fill is not None:
            if torch.is_tensor(fill):
                self.body.copy_(fill.reshape(-1))
            else:
                self.body.fill_(fill)

    def _words(self):
        return self.raw.view(torch.int32 if self.es == 4 else torch.int64)

    @property
    def ptr(self):
        return self.raw.data_ptr() + OFFB

    def intact(self):
        w, k = self._words(), OFFB // self.es
        s = SENT32 if self.es == 4 else SENT64
        return bool((w[:k] == s).all()) and bool((w[k + self.n:] == s).all())


def layout_strides(layout, N, D):
    return {"contiguous": (1, D), "q_zCx": (2, 2 * D), "padded": (3, 3 * D + 5), "colmajor": (N, 1)}[layout]


def place_mu(x, layout):
    """fp32 x [N, D] at element (n, d) = n rs + d ld of a guarded NaN-filled buffer -> (Buf, ld, rs)."""
    N, D = x.shape
    ld, rs = layout_strides(layout, N, D)
    buf = Buf((N - 1) * rs + (D - 1) * ld + 1, torch.float32, float("nan"))
    idx = torch.arange(N, device=DEV)[:, None] * rs + torch.arange(D, device=DEV)[None, :] * ld
    buf.body[idx.reshape(-1)] = x.to(DEV, torch.float32).reshape(-1)
    return buf, ld, rs


def _lib():
    from disvae import _native as N
    return N.lib(), N.stream()


def _call(launches, name, *args):
    L, _ = _lib()
    torch.cuda.synchronize()
    before = L.dv_launch_count()
    rc = getattr(L, name)(*args)
    torch.cuda.synchronize()
    assert rc == DV_OK, (name, rc)
    assert L.dv_launch_count() - before == launches, name


def _bits(t):
    t = t.contiguous()
    return t.view(torch.int32) if t.element_size() == 4 else t.view(torch.int64)


def _same(a, b, tag):
    assert torch.equal(_bits(a), _bits(b)), tag + ": differs bit for bit"


def _graph_replays(run, outs, tag):
    """Capture `run()` (one raw call on the current stream) in a CUDA graph, clear `outs`, replay, and compare the
    replay's bits with the eager ones."""
    eager = [o.body.clone() for o in outs]
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            run()
    torch.cuda.current_stream().wait_stream(s)
    for o in outs:
        o.body.view(torch.uint8).fill_(0xA5)
    g.replay()
    torch.cuda.synchronize()
    for e, o in zip(eager, outs):
        _same(e, o.body, tag + " graph replay")
        assert o.intact(), tag + " graph replay wrote past an output"


def _layout(x, layout):
    """`x` [N, D] as the kernel reads it: a contiguous copy, or the mean half of an interleaved [N, D, 2] buffer."""
    if layout == "contig":
        return x.contiguous()
    q = torch.full(x.shape + (2,), float("nan"), device=x.device)
    q[..., 0] = x
    return q.unbind(-1)[0]


def grid_values(lat_sizes):
    """int64 [prod(lat_sizes), K]: the factor values of every item of the full grid, in C order."""
    n = int(np.prod(lat_sizes))
    return torch.from_numpy(np.stack(np.unravel_index(np.arange(n), lat_sizes), 1))


# ---- the synthetic codes and datasets of the DCI and modularity tests ---------------------------------------------
def _rows(n, num, seed, where=None):
    g = torch.Generator().manual_seed(seed)
    rows = torch.randint(n, (num,), generator=g)
    return rows if where is None else where[rows % len(where)]


def _code(lat_sizes, D, seed, noise=0.3):
    """Latent d follows factor d (scaled to [0, 1)) plus noise; the latents past the factors are noise."""
    g = torch.Generator().manual_seed(seed)
    v = grid_values(lat_sizes).float()
    x = torch.randn(v.size(0), D, generator=g)
    K = min(D, len(lat_sizes))
    x[:, :K] = v[:, :K] / torch.tensor(lat_sizes[:K]).float() + noise * x[:, :K]
    return x


class _Code(torch.nn.Module):
    """An encoder whose means are a fixed linear map of the factor values the synthetic images carry."""

    def __init__(self, M):
        super().__init__()
        self.latent_dim = M.shape[1]
        self.register_buffer("M", M)

    def encoder(self, x):
        v = x.view(x.size(0), -1)[:, :self.M.shape[0]]
        return v @ self.M, torch.zeros(x.size(0), self.latent_dim, device=x.device)

    def reparameterize(self, mean, logvar):
        return mean


class _Factors(torch.utils.data.Dataset):
    """The full grid of `lat_sizes`; an item's 'image' holds its factor values (plus small noise) in its first pixels."""

    def __init__(self, lat_sizes, noise, seed):
        self.lat_sizes, self.lat_names = np.array(lat_sizes), tuple("f%d" % k for k in range(len(lat_sizes)))
        v = grid_values(lat_sizes).float() / torch.tensor(lat_sizes).float()
        g = torch.Generator().manual_seed(seed)
        self.imgs = torch.zeros(v.size(0), 1, 8, 8)
        self.imgs.view(v.size(0), -1)[:, :len(lat_sizes)] = v + noise * torch.randn(v.shape, generator=g)

    def __len__(self):
        return len(self.imgs)

    def __getitem__(self, i):
        return self.imgs[i], 0
