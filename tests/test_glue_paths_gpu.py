"""The glue kernels of the training step (csrc/dv_glue.cu) and the layout and activation kernels at the end of
csrc/dv_conv.cu, through the raw C ABI, against aten and fp64 references.

Plans, restated from the kernels (sized for the 132 SMs of an H100 SXM):
- act_bwd_kernel (dv_act_bwd): min(ceil(n / 256), 16 x 132) blocks of 256 threads, grid-stride, one element per step.
- act_bwd_chansum_kernel (dv_act_bwd_chansum): grid = min(B C, 296).  Block k walks planes p = k, k + grid, ... (p =
  b C + c); thread t takes the float4s t, t + 256, ... of a plane and adds (g.x + g.y) + (g.z + g.w) of each to its
  plane sum, which it adds to its channel's sum.  A 5-level shuffle tree per warp, the 8 warp sums in order, into
  workspace row k (32 words: 0 for channels >= C).  chansum_final32_kernel: thread (w, c) adds rows w, w + 32, ... in
  order, then thread c adds the 32 slices in order.
- channel_sum_nhwc_kernel (dv_channel_sum, nchw == 0): grid = min(ceil(rows / 8), 296); warp w of block k adds rows
  8k + w, 8(k + grid) + w, ... of its lane's channel, the 8 warps in order into row k (32 words, 0 past C).
  channel_sum_nchw_kernel: grid = min(B, 296); for each channel thread t adds elements t, t + 256, ... of images k,
  k + grid, ...; shuffle tree, 8 warps, into words 0 .. C-1 of row k (the others untouched).  Both end in
  channel_sum_final_kernel, the same two stages as chansum_final32_kernel.
- flat_transpose_kernel: min(ceil(n / 256), 8 x 132) blocks of 256 threads, grid-stride: at C = 32, S = 16 one stride
  is 528 images.
- u8_to_f32_kernel: min(max(ceil((n / 16) / 256), 1), 8 x 132) blocks: the 16-byte chunks grid-stride, then the tail
  bytes past the last whole chunk.  gather_u8_to_f32_kernel: min(ceil(nrows row_bytes / 16 / 256), 8 x 132) blocks, one
  16-byte chunk per thread step, the source offset idx[row] * row_bytes in 64 bits.
- the combination, beta-VAE_B and record kernels: one block, thread 0 computes, the whole block writes the log row.

Bounds: g, the transposes, the byte conversions, the coefficients and the loss gradients must be bit-identical to aten
or to the host value.  A channel sum is held to |got - sum(g64)| <= (tau + e) sum|g64| + 2^-148 per element, with g64
the fp64 gradient, e the per-element rounding of g (3 u for sigmoid's subtraction and two products, 1 u for the leaky
product, 0 otherwise) and tau = u times the longest chain of fp32 additions an element passes through in the plan
above.  The combined loss is held to (max(na, nb) + 1) u sum|c v|: one FMA chain per vector, then one add.  The CPU
section shows each bound has teeth at case shapes: a dropped or doubled plane, row, image or block partial, the old
sigmoid association, a swapped coefficient or dropped term, and a log row at the wrong ring index all fail it.  At
2^20 NHWC rows a single row is 2^-20 of its channel: no rounding bound of a 443-long chain can see it, and the dropped
block partial is the fault checked there.

The one intended difference from aten: ReLU at y = NaN gives 0 (every ReLU mask of the library is [y > 0]) where
threshold_backward passes dy; those elements are checked for +0 and left out of the aten comparison.

Outputs, workspaces and rings sit 16 bytes into NaN-filled buffers between sentinel words; inputs start 16 bytes into
theirs.  Every raw call is counted with dv_launch_count() and runs twice, bit for bit.  Each GPU case prints its
worst error as a fraction of its bound (pytest -s)."""
import ctypes
import math

import numpy as np
import pytest
import torch

from disvae.models.losses import linear_annealing

U = 2.0 ** -24              # fp32 unit roundoff
TINY = 2.0 ** -149          # smallest fp32 subnormal
SM_COUNT = 132              # kNumSMs in csrc/dv_common.cuh
CS_BLOCKS = 296             # kCsBlocks: channel-sum partial rows
ACT_GRID_CAP = 16 * SM_COUNT
COPY_GRID_CAP = 8 * SM_COUNT
THREADS = 256
GUARD = 1024                # words of sentinel after each output
SENTINEL = 0x7FBADBAD       # a NaN bit pattern no kernel writes
NAN_FILL = 0x7FC00000       # torch's NaN: the fill of every output body
OFF = 4                     # floats: every operand starts 16 bytes into its allocation
DV_OK, DV_ERR_BAD_SHAPE, DV_ERR_BAD_ARG = 0, -1, -2
ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_LEAKY = 0, 1, 2, 3
INT_MAX = 2 ** 31 - 1
WS_FLOATS = CS_BLOCKS * 32

ACTS = [("sigmoid", ACT_SIGMOID, 0.0), ("relu", ACT_RELU, 0.0), ("leaky0.2", ACT_LEAKY, 0.2),
        ("leaky0.01", ACT_LEAKY, 0.01), ("leaky0", ACT_LEAKY, 0.0), ("none", ACT_NONE, 0.0)]
ELEM_ULPS = {ACT_SIGMOID: 3, ACT_LEAKY: 1, ACT_RELU: 0, ACT_NONE: 0}


def _cdiv(a, b):
    return -(-a // b)


# ---------------------------------------------------------------------------------------------------------------------
# plans and rounding chains
# ---------------------------------------------------------------------------------------------------------------------
def act_grid(n):
    return min(max(_cdiv(n, THREADS), 1), ACT_GRID_CAP)


def chansum_grid(B, C):
    return min(B * C, CS_BLOCKS)


def nhwc_grid(rows):
    return min(max(_cdiv(rows, 8), 1), CS_BLOCKS)


def nchw_grid(B):
    return min(B, CS_BLOCKS)


def final_depth(grid):
    """channel_sum_final_kernel / chansum_final32_kernel: every 32nd partial row in order, then the 32 slices."""
    return _cdiv(grid, 32) + 32


def tau_act_chansum(B, C, hw):
    """The float4's pair tree (2), the thread's float4s of a plane, its planes of the block, the shuffle tree (5), the
    8 warps, the final stage."""
    grid = chansum_grid(B, C)
    return U * (2 + _cdiv(hw // 4, THREADS) + _cdiv(B * C, grid) + 5 + 8 + final_depth(grid))


def tau_nhwc(rows):
    """A warp's rows in order, the 8 warps, the final stage."""
    grid = nhwc_grid(rows)
    return U * (_cdiv(rows, 8 * grid) + 8 + final_depth(grid))


def tau_nchw(B, hw):
    """A thread's elements of each of its block's images in order, the shuffle tree, the 8 warps, the final stage."""
    grid = nchw_grid(B)
    return U * (_cdiv(B, grid) * _cdiv(hw, THREADS) + 5 + 8 + final_depth(grid))


def tau_combine(na, nb):
    return U * (max(na, nb) + 1)


def log_row(s, every, cap):
    """Ring row of a recording step (losses.py's rule s % every == 1), None when step s does not record."""
    return (s - 1) // every % cap if s % every == 1 else None


# ---------------------------------------------------------------------------------------------------------------------
# references
# ---------------------------------------------------------------------------------------------------------------------
def aten_act_bwd(dy, y, act, slope):
    """What autograd computes from the activation's output y."""
    if act == ACT_SIGMOID:
        return torch.ops.aten.sigmoid_backward(dy, y)
    if act == ACT_RELU:
        return torch.ops.aten.threshold_backward(dy, y, 0)
    if act == ACT_LEAKY:
        return torch.ops.aten.leaky_relu_backward(dy, y, slope, True)
    return dy.clone()


def fp64_act_bwd(dy, y, act, slope):
    d, v = dy.double(), y.double()
    if act == ACT_SIGMOID:
        return d * (1 - v) * v
    if act == ACT_RELU:
        return torch.where(v > 0, d, torch.zeros_like(d))
    if act == ACT_LEAKY:
        return torch.where(v > 0, d, d * float(np.float32(slope)))
    return d


def old_sigmoid_bwd(dy, y):
    """The association the kernels had before: dy * ((1 - y) * y)."""
    return dy * ((1 - y) * y)


def sum_ratio(got, ref, mag, tau, n):
    """|got - ref| / (tau mag + n 2^-148) per entry; NaN or inf in got counts as infinite, a zero bound must be met
    exactly."""
    got = got.double().to(ref.device)
    err = (got - ref).abs()
    r = torch.where(err == 0, 0.0, err / (tau * mag + n * 2 * TINY))
    return torch.where(torch.isfinite(got), r, math.inf)


def check_sums(got, ref, mag, tau, n, tag):
    r = sum_ratio(got, ref, mag, tau, n)
    worst = r.max().item()
    assert worst <= 1, "%s: sums %s, fp64 %s, sum|x| %s: %.2f x the bound" % (
        tag, got.tolist(), ref.tolist(), mag.tolist(), worst)
    return worst


def combine_ref(vals, coefs):
    """fp64 sum c v and sum |c v| of the fp32 values and coefficients."""
    p = [float(c) * float(v) for c, v in zip(coefs, vals)]
    return math.fsum(p), math.fsum(abs(x) for x in p)


def combine_ratio(got, vals, coefs, na, nb):
    ref, mag = combine_ref(vals, coefs)
    err = abs(float(got) - ref)
    return 0.0 if err == 0 else err / (tau_combine(na, nb) * mag)


def host_coefs(base, mask, init, fin, s, steps_anneal, is_train):
    """The coefficients the host path forms: np.float32(linear_annealing(...) * base) where the mask bit is set."""
    A = linear_annealing(init, fin, s, steps_anneal) if is_train else fin
    return np.array([A * b if (mask >> k) & 1 else b for k, b in enumerate(base)], dtype=np.float32)


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
Y_EDGES_SIGMOID = torch.cat([torch.tensor([0.0, -0.0, 1.0, 1e-40, TINY, 1 - 2.0 ** -24, 0.5]),
                             torch.sigmoid(torch.tensor([30.0, -30.0]))])
Y_EDGES_OTHER = torch.tensor([0.0, -0.0, 1e-40, -1e-40, TINY, -TINY, 1.0, -1.0, math.inf, -math.inf])
DY_ALL = torch.tensor([0.0, -0.0, 1.0, -1.0, 1e30, -1e30, 3e38, -3e38, 1e-40, -1e-40, math.inf, -math.inf, math.nan,
                       12345.678, -12345.677, 0.3])


def act_inputs(n, act, seed, regime="biased"):
    """(dy, y) fp32 CPU.  y = sigmoid(3 randn) for sigmoid, randn otherwise, every 61st element an edge value (exact
    0, -0, 1, subnormals, sigmoid(+-30), +-inf for the others).  dy regimes: 'biased' randn + 0.5 (a dropped plane
    moves the sum by about its share), 'zero-mean' randn (sums that cancel), 'large' randn * 1e30; every 37th dy is
    +0 or -0."""
    g = torch.Generator().manual_seed(seed)
    y = torch.sigmoid(3 * torch.randn(n, generator=g)) if act == ACT_SIGMOID else torch.randn(n, generator=g)
    dy = torch.randn(n, generator=g)
    if regime == "biased":
        dy += 0.5
    elif regime == "large":
        dy *= 1e30
    ye = Y_EDGES_SIGMOID if act == ACT_SIGMOID else Y_EDGES_OTHER
    i = torch.arange(0, n, 61)
    y[i] = ye[torch.arange(len(i)) % len(ye)]
    j = torch.arange(min(5, n - 1), n, 37)
    dy[j] = torch.tensor([0.0, -0.0])[torch.arange(len(j)) % 2]
    return dy, y


def edge_cross():
    """Every edge y (NaN included) against every edge dy, padded with zeros to a multiple of 4."""
    ys = torch.cat([Y_EDGES_SIGMOID, Y_EDGES_OTHER, torch.tensor([math.nan])])
    y = ys.repeat_interleave(len(DY_ALL))
    dy = DY_ALL.repeat(len(ys))
    pad = (-len(y)) % 4
    return torch.cat([dy, torch.zeros(pad)]), torch.cat([y, torch.full((pad,), 0.5)])


def combo_inputs(na, nb, seed):
    """a [na + 3] (the producing node's whole output: only the first na are weighted), b [nb]: alternating signs of
    magnitudes 1 to 100, so the sums cancel; base doubles most of which fp32 cannot hold.  Every term is then far
    above the loss bound, so a dropped one shows."""
    rng = np.random.default_rng(seed)

    def vals(k):
        m = 10.0 ** rng.uniform(0, 2, k)
        return (m * np.where(np.arange(k) % 2, -1.0, 1.0)).astype(np.float32)
    base = rng.choice([1.0, 6.4, 0.37, 4.0, 2.5, 0.1, 1 / 3], na + nb)
    return vals(na + 3), vals(nb), [float(x) for x in base]


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the references and bounds have teeth
# ---------------------------------------------------------------------------------------------------------------------
def test_aten_sigmoid_backward_is_the_left_to_right_product():
    """aten's sigmoid_backward rounds as (dy * (1 - y)) * y; the old association differs from it in many elements,
    so the bit comparison rejects it."""
    dy, y = act_inputs(1 << 20, ACT_SIGMOID, 1)
    y = torch.sigmoid(3 * torch.randn(1 << 20, generator=torch.Generator().manual_seed(2)))
    ref = aten_act_bwd(dy, y, ACT_SIGMOID, 0.0)
    assert torch.equal(((dy * (1 - y)) * y).view(torch.int32), ref.view(torch.int32))
    assert (old_sigmoid_bwd(dy, y).view(torch.int32) != ref.view(torch.int32)).sum().item() > 1000


CHANSUM_TEETH = [(1, 1, 4096), (2048, 1, 4), (99, 3, 1024), (74, 4, 12), (149, 2, 4100), (97, 3, 4096)]


@pytest.mark.parametrize("act,code,slope", ACTS, ids=[a[0] for a in ACTS])
@pytest.mark.parametrize("B,C,hw", CHANSUM_TEETH, ids=["%dx%dx%d" % c for c in CHANSUM_TEETH])
def test_chansum_bound_catches_dropped_planes_and_partials(B, C, hw, act, code, slope):
    """The fp32 aten gradient summed in fp32 passes; with one plane dropped or doubled, or one block's partial (its
    planes k, k + grid, ...) dropped, some channel breaks the bound."""
    dy, y = act_inputs(B * C * hw, code, B + C + hw)
    g32 = aten_act_bwd(dy, y, code, slope).view(B, C, hw)
    g64 = fp64_act_bwd(dy, y, code, slope).view(B, C, hw)
    ref, mag = g64.sum((0, 2)), g64.abs().sum((0, 2))
    tau = tau_act_chansum(B, C, hw) + ELEM_ULPS[code] * U
    n = B * hw
    check_sums(g32.sum((0, 2)), ref, mag, tau, n, "fp32 sums of the aten gradient")
    planes = g32.reshape(B * C, hw).double()
    chan = torch.arange(B * C) % C

    def sums(w):
        return torch.stack([(planes[chan == c] * w[chan == c, None]).sum() for c in range(C)])

    def caught(w):
        return sum_ratio(sums(w), ref, mag, tau, n).max().item() > 1
    grid = chansum_grid(B, C)
    # near the start, the middle and the end, the plane with the largest |sum| (a plane that sums to about 0, as a
    # 4-pixel ReLU plane may, cannot be told from a dropped one by any sum)
    psum = planes.sum(1).abs()
    P = B * C
    for lo in {0, max(P // 2 - 4, 0), max(P - 8, 0)}:
        p = lo + int(psum[lo:lo + 8].argmax())
        w = torch.ones(B * C, dtype=torch.float64)
        w[p] = 0
        assert caught(w), ("dropped plane", p)
        w[p] = 2
        assert caught(w), ("doubled plane", p)
    for k in {0, grid - 1}:
        w = torch.ones(B * C, dtype=torch.float64)
        w[k::grid] = 0
        assert caught(w), ("dropped block partial", k)


NHWC_TEETH = [(1, 1), (7, 5), (8, 32), (2367, 3), (2368, 17), (2369, 32), (1 << 20, 4)]


@pytest.mark.parametrize("rows,C", NHWC_TEETH, ids=["%dx%d" % c for c in NHWC_TEETH])
def test_nhwc_channel_sum_bound_catches_dropped_rows_and_partials(rows, C):
    x = channel_sum_input(rows * C, rows + C).view(rows, C)
    ref, mag = x.double().sum(0), x.double().abs().sum(0)
    tau = tau_nhwc(rows)
    check_sums(x.sum(0), ref, mag, tau, rows, "fp32 sums")
    grid = nhwc_grid(rows)
    if 1 < rows < 1 << 20:          # at 2^20 rows one row is below the bound of a 443-long chain (module docstring)
        drop = x.double().clone()
        drop[-1] = 0
        assert sum_ratio(drop.sum(0), ref, mag, tau, rows).max().item() > 1, "dropped row"
        drop[-1] = 2 * x[-1].double()
        assert sum_ratio(drop.sum(0), ref, mag, tau, rows).max().item() > 1, "doubled row"
    for k in {0, grid - 1}:
        rows_of_block = torch.arange(rows).div(8, rounding_mode="floor") % grid == k
        drop = x.double().clone()
        drop[rows_of_block] = 0
        if grid > 1:
            assert sum_ratio(drop.sum(0), ref, mag, tau, rows).max().item() > 1, ("dropped block partial", k)


NCHW_TEETH = [(1, 255), (295, 1), (296, 257), (297, 256), (1000, 4096)]


@pytest.mark.parametrize("B,hw", NCHW_TEETH, ids=["%dx%d" % c for c in NCHW_TEETH])
def test_nchw_channel_sum_bound_catches_dropped_images_and_partials(B, hw):
    C = 3
    x = channel_sum_input(B * C * hw, B + hw).view(B, C, hw)
    ref, mag = x.double().sum((0, 2)), x.double().abs().sum((0, 2))
    tau = tau_nchw(B, hw)
    check_sums(x.sum((0, 2)), ref, mag, tau, B * hw, "fp32 sums")
    grid = nchw_grid(B)
    for b in {0, B - 1}:
        drop = x.double().clone()
        drop[b] = 0
        if B > 1:
            assert sum_ratio(drop.sum((0, 2)), ref, mag, tau, B * hw).max().item() > 1, ("dropped image", b)
        drop[b] = 2 * x[b].double()
        assert sum_ratio(drop.sum((0, 2)), ref, mag, tau, B * hw).max().item() > 1, ("doubled image", b)
    if grid > 1:
        drop = x.double().clone()
        drop[grid - 1::grid] = 0
        assert sum_ratio(drop.sum((0, 2)), ref, mag, tau, B * hw).max().item() > 1, "dropped block partial"


@pytest.mark.parametrize("na,nb", [(1, 0), (2, 3), (8, 8), (3, 1), (8, 0), (1, 8)])
def test_combination_bound_catches_swapped_coefficients_and_dropped_terms(na, nb):
    """An fp32 left-to-right evaluation passes; a coefficient swapped with its neighbour, or one term left out, breaks
    (max(na, nb) + 1) u sum |c v|."""
    a, b, base = combo_inputs(na, nb, 7 * na + nb)
    c = np.array(base, dtype=np.float32)
    vals = list(a[:na]) + list(b)
    s = np.float32(0)
    for i in range(na):
        s = np.float32(s + c[i] * a[i])
    t = np.float32(0)
    for j in range(nb):
        t = np.float32(t + c[na + j] * b[j])
    assert combine_ratio(np.float32(s + t), vals, c, na, nb) <= 1
    for k in range(na + nb):
        wrong = list(vals)
        wrong[k] = 0.0
        assert combine_ratio(combine_ref(wrong, c)[0], vals, c, na, nb) > 1, ("dropped term", k)
        if k + 1 < na + nb and c[k] != c[k + 1]:
            sw = c.copy()
            sw[k], sw[k + 1] = c[k + 1], c[k]
            assert combine_ratio(combine_ref(vals, sw)[0], vals, c, na, nb) > 1, ("swapped coefficients", k)


def ring_after(steps, every, cap, rule=None):
    """The ring [cap] a log leaves after the recording calls of `steps`, each writing its step number; rule(s) -> row
    or None stands in for log_row."""
    ring = [math.nan] * cap
    for s in steps:
        r = log_row(s, every, cap) if rule is None else rule(s)
        if r is not None:
            ring[r] = float(s)
    return ring


def test_log_ring_catches_a_wrong_row_or_step():
    """The ring the step sequence of the GPU test must leave differs from what a kernel writing the row s % cap, the
    next row, or recording with the counter before its advance would leave; with every = 1 nothing records (s % 1 is
    never 1: the host rule of losses.py never records then)."""
    for cap, every in [(3, 2), (3, 50), (1, 2), (1, 50)]:
        steps = log_steps(every)
        good = ring_after(steps, every, cap)
        assert not all(map(math.isnan, good))
        wrong = [lambda s: log_row(s - 1, every, cap)]                     # the counter before the advance
        if cap > 1:
            wrong += [lambda s: s % cap if s % every == 1 else None,
                      lambda s: ((s - 1) // every + 1) % cap if s % every == 1 else None]
        for rule in wrong:
            assert ring_after(steps, every, cap, rule) != good
    assert all(map(math.isnan, ring_after(log_steps(1), 1, 3)))
    assert log_row(2 ** 31 + 1, 2, 3) == 2 ** 30 % 3 and log_row(2 ** 31 + 2, 2, 3) is None


def log_steps(every):
    """Step values that record and that do not, including the wrap-around of a 3-row ring and counters past 2^31."""
    out = [1, 2, 3, every, every + 1, every + 2, 2 * every + 1, 3 * every + 1, 4 * every + 1]
    for base in (2 ** 31, 2 ** 32 + 5):
        k = base // every * every + 1
        out += [k, k + 1, k + every]
    return list(dict.fromkeys(s for s in out if s >= 1))


def channel_sum_input(n, seed):
    """randn + 0.5: a dropped row, image or partial moves a channel's sum by about its share of sum |x|."""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, generator=g) + 0.5


# ---------------------------------------------------------------------------------------------------------------------
# device buffers and raw calls
# ---------------------------------------------------------------------------------------------------------------------
def _bits(t):
    return t.contiguous().view(torch.int32)


def _input(t):
    """Device copy of fp32 `t` 16 bytes into a NaN-filled allocation, with GUARD NaN after it."""
    t = t.reshape(-1)
    buf = torch.full((OFF + t.numel() + GUARD,), float("nan"), device="cuda")
    buf[OFF:OFF + t.numel()] = t.to("cuda")
    return buf


def _output(n):
    """n NaN words 16 bytes into an allocation, sentinel words before and after."""
    buf = torch.full((OFF + n + GUARD,), float("nan"), device="cuda")
    _bits(buf)[:OFF] = SENTINEL
    _bits(buf)[OFF + n:] = SENTINEL
    return buf


def _addr(buf, shift=0):
    return None if buf is None else buf.data_ptr() + 4 * OFF + shift


def _intact(buf, n):
    b = _bits(buf)
    return bool((b[:OFF] == SENTINEL).all()) and bool((b[OFF + n:] == SENTINEL).all())


def _body(buf, n):
    return buf[OFF:OFF + n]


def _u8_input(src):
    """Device copy of uint8 `src` 16 bytes into an 0xA5-filled allocation, GUARD bytes after it."""
    n = src.numel()
    buf = torch.full((16 + n + GUARD,), 0xA5, dtype=torch.uint8, device="cuda")
    buf[16:16 + n] = src.reshape(-1).to("cuda")
    return buf, buf.data_ptr() + 16


def _counter(value):
    """An int64 device step counter 16 bytes into a sentinel-filled allocation -> (buffer, address)."""
    buf = torch.full((2 + 1 + 8,), -0x5A5A5A5A5A5A5A5A, dtype=torch.int64, device="cuda")
    buf[2] = value
    return buf, buf.data_ptr() + 16


def _counter_intact(buf):
    return bool((buf[:2] == -0x5A5A5A5A5A5A5A5A).all()) and bool((buf[3:] == -0x5A5A5A5A5A5A5A5A).all())


def _native():
    from disvae import _native as N
    return N


def _launch(n_kernels, name, *args):
    """One raw call that must succeed and launch `n_kernels` kernels."""
    N = _native()
    before = N.lib().dv_launch_count()
    rc = getattr(N.lib(), name)(*args)
    assert rc == DV_OK, (name, rc)
    assert N.lib().dv_launch_count() - before == n_kernels, name
    torch.cuda.synchronize()


def _stream():
    return _native().stream()


def _same_bits(a, b, tag):
    assert torch.equal(_bits(a), _bits(b)), tag + ": the repeat differs"


# ---------------------------------------------------------------------------------------------------------------------
# dv_act_bwd_chansum and dv_act_bwd
# ---------------------------------------------------------------------------------------------------------------------
def run_act_chansum(dyb, yb, B, C, hw, act, slope):
    """Two raw calls on fresh guarded outputs -> (g, chansum, workspace) of the first, asserted equal to the second."""
    n = B * C * hw
    outs = []
    for _ in range(2):
        g, cs, ws = _output(n), _output(C), _output(WS_FLOATS)
        _launch(2, "dv_act_bwd_chansum", _addr(dyb), _addr(yb), _addr(g), B, C, hw, act, slope, _addr(cs), _addr(ws),
                _stream())
        assert _intact(g, n) and _intact(cs, C) and _intact(ws, WS_FLOATS), "dv_act_bwd_chansum wrote past a buffer"
        outs.append((_body(g, n), _body(cs, C), _body(ws, WS_FLOATS)))
    for x, y_, tag in zip(outs[0], outs[1], ("g", "chansum", "workspace")):
        _same_bits(x, y_, tag)
    return outs[0]


def run_act_bwd(dyb, yb, n, act, slope):
    outs = []
    for _ in range(2):
        g = _output(n)
        _launch(1, "dv_act_bwd", _addr(dyb), _addr(yb), _addr(g), n, act, slope, _stream())
        assert _intact(g, n), "dv_act_bwd wrote past its output"
        outs.append(_body(g, n))
    _same_bits(outs[0], outs[1], "g")
    return outs[0]


def check_grid_rows(ws, grid, C, nchw_words=False):
    """The first `grid` partial rows written (words past C: 0, or untouched on the NCHW path), the others untouched."""
    rows = _bits(ws).view(CS_BLOCKS, 32)
    vals = ws.view(CS_BLOCKS, 32)
    assert torch.isfinite(vals[:grid, :C]).all(), "a partial row of the grid is missing"
    if nchw_words:
        assert (rows[:grid, C:] == NAN_FILL).all()
    else:
        assert (rows[:grid, C:] == 0).all()
    assert (rows[grid:] == NAN_FILL).all(), "partial rows past the grid were written"


def _act_chansum_shapes():
    out = []
    for C in (1, 2, 3, 4):
        Bs = {1} | {b for b in range(1, 300) if 295 <= b * C <= 297} | {294 // C, _cdiv(298, C)}
        for hw in (4, 12, 1024, 4096, 4100):
            out += [(B, C, hw) for B in sorted(Bs)]
    return out


ACT_CHANSUM_SHAPES = _act_chansum_shapes()
LARGE_CHANSUM_SHAPES = [(97, 1, 4096), (97, 3, 4096), (2048, 1, 4096), (2048, 3, 4096)]


def check_act_chansum_case(B, C, hw, regime="biased", acts=ACTS):
    n = B * C * hw
    worst = 0.0
    for name, act, slope in acts:
        dy, y = act_inputs(n, act, B * 31 + C * 7 + hw, regime)
        dyb, yb = _input(dy), _input(y)
        dy_d, y_d = _body(dyb, n), _body(yb, n)
        g, cs, ws = run_act_chansum(dyb, yb, B, C, hw, act, slope)
        want = aten_act_bwd(dy_d, y_d, act, slope)
        assert torch.equal(_bits(g), _bits(want)), "%s: g differs from aten in %d elements" % (
            name, int((_bits(g) != _bits(want)).sum()))
        g1 = run_act_bwd(dyb, yb, n, act, slope)
        assert torch.equal(_bits(g1), _bits(g)), name + ": dv_act_bwd differs from dv_act_bwd_chansum"
        g64 = fp64_act_bwd(dy_d, y_d, act, slope).view(B, C, hw)
        tau = tau_act_chansum(B, C, hw) + ELEM_ULPS[act] * U
        worst = max(worst, check_sums(cs, g64.sum((0, 2)), g64.abs().sum((0, 2)), tau, B * hw,
                                      "%s B=%d C=%d hw=%d" % (name, B, C, hw)))
        check_grid_rows(ws, chansum_grid(B, C), C)
    print("act_bwd_chansum B=%d C=%d hw=%d %s grid %d: worst sum err %.3f of the bound"
          % (B, C, hw, regime, chansum_grid(B, C), worst))


@pytest.mark.gpu
@pytest.mark.parametrize("B,C,hw", ACT_CHANSUM_SHAPES, ids=["%dx%dx%d" % c for c in ACT_CHANSUM_SHAPES])
def test_act_bwd_chansum_shapes(B, C, hw):
    """Every activation code: g bit for bit against aten (and dv_act_bwd), the channel sums against fp64, the grid in
    the workspace rows, at plane counts around the 296-block cap."""
    check_act_chansum_case(B, C, hw)


@pytest.mark.gpu
@pytest.mark.parametrize("B,C,hw", LARGE_CHANSUM_SHAPES, ids=["%dx%dx%d" % c for c in LARGE_CHANSUM_SHAPES])
def test_act_bwd_chansum_training_shapes(B, C, hw):
    check_act_chansum_case(B, C, hw)


REGIME_SHAPES = [(99, 3, 1024), (2048, 1, 4096), (1, 4, 4100)]


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["zero-mean", "large"])
@pytest.mark.parametrize("B,C,hw", REGIME_SHAPES, ids=["%dx%dx%d" % c for c in REGIME_SHAPES])
def test_act_bwd_chansum_cancelling_and_large_inputs(B, C, hw, regime):
    check_act_chansum_case(B, C, hw, regime)


@pytest.mark.gpu
@pytest.mark.parametrize("act,code,slope", ACTS, ids=[a[0] for a in ACTS])
def test_act_bwd_input_edges(act, code, slope):
    """Every edge y (0, -0, 1, subnormals, sigmoid(+-30), +-inf, NaN) against every edge dy (+-0, +-1e30, +-3e38,
    subnormals, +-inf, NaN): g bit for bit against aten through both entry points, except ReLU at y = NaN, which must
    be +0."""
    dy, y = edge_cross()
    n = dy.numel()
    dyb, yb = _input(dy), _input(y)
    dy_d, y_d = _body(dyb, n), _body(yb, n)
    want = aten_act_bwd(dy_d, y_d, code, slope)
    cpu = aten_act_bwd(dy, y, code, slope)
    diff = (_bits(want.cpu()) != _bits(cpu)) & ~(torch.isnan(cpu) & torch.isnan(want.cpu()))
    print("%s: CUDA aten differs from CPU aten in %d of %d edge elements (NaN payloads aside)"
          % (act, int(diff.sum()), n))
    keep = ~torch.isnan(y_d) if code == ACT_RELU else torch.ones_like(y_d, dtype=torch.bool)
    g1 = run_act_bwd(dyb, yb, n, code, slope)
    g2, _, _ = run_act_chansum(dyb, yb, 1, 1, n, code, slope)
    for g, tag in ((g1, "dv_act_bwd"), (g2, "dv_act_bwd_chansum")):
        bad = (_bits(g) != _bits(want)) & keep
        assert not bad.any(), "%s %s: %d elements differ from aten, e.g. dy %r y %r: %r vs %r" % (
            tag, act, int(bad.sum()), dy_d[bad][0].item(), y_d[bad][0].item(), g[bad][0].item(), want[bad][0].item())
        if code == ACT_RELU:
            assert (_bits(g)[~keep] == 0).all(), tag + ": ReLU at y = NaN is not +0"


ACT_N = [1, 255, 256, 257, 4096, ACT_GRID_CAP * THREADS - 1, ACT_GRID_CAP * THREADS, ACT_GRID_CAP * THREADS + 1,
         2 * ACT_GRID_CAP * THREADS + 5, 2 ** 24 + 3]


@pytest.mark.gpu
@pytest.mark.parametrize("n", ACT_N)
def test_act_bwd_grid_stride(n):
    """n across the 16 x 132-block grid-stride boundary: every activation bit for bit against aten."""
    for name, act, slope in ACTS:
        dy, y = act_inputs(n, act, n % 1000 + act)
        dyb, yb = _input(dy), _input(y)
        g = run_act_bwd(dyb, yb, n, act, slope)
        assert torch.equal(_bits(g), _bits(aten_act_bwd(_body(dyb, n), _body(yb, n), act, slope))), (name, n)
    print("act_bwd n=%d grid %d: bit-identical to aten" % (n, act_grid(n)))


@pytest.mark.gpu
@pytest.mark.parametrize("C", [3, 4])
def test_chansum_nan_poisons_only_its_channel(C):
    B, hw = 300, 1024
    for name, act, slope in ACTS:
        dy, y = act_inputs(B * C * hw, act, 5 + act)
        dy.view(B, C, hw)[B // 2, 1, 77] = math.nan
        y.view(B, C, hw)[B // 2, 1, 77] = 0.5       # where every activation passes dy on
        g, cs, ws = run_act_chansum(_input(dy), _input(y), B, C, hw, act, slope)
        assert torch.isnan(cs[1]) and torch.isfinite(cs[torch.arange(C) != 1]).all(), (name, cs.tolist())


# ---------------------------------------------------------------------------------------------------------------------
# dv_flat_transpose
# ---------------------------------------------------------------------------------------------------------------------
def run_transpose(src_b, B, C, S, to_nhwc):
    n = B * C * S
    outs = []
    for _ in range(2):
        dst = _output(n)
        _launch(1, "dv_flat_transpose", _addr(src_b), _addr(dst), B, C, S, to_nhwc, _stream())
        assert _intact(dst, n), "dv_flat_transpose wrote past its output"
        outs.append(_body(dst, n))
    _same_bits(outs[0], outs[1], "transpose")
    return outs[0]


def random_words(n, seed):
    """fp32 words of every kind: random bit patterns (NaN payloads, infinities, subnormals, -0) as int32."""
    g = torch.Generator().manual_seed(seed)
    w = torch.randint(-2 ** 31, 2 ** 31, (n,), generator=g, dtype=torch.int64).to(torch.int32)
    special = torch.tensor([0, -2 ** 31, 1, 0x7F800001, -0x00400001, 0x007FFFFF], dtype=torch.int32)
    w[:min(n, 6)] = special[:min(n, 6)]
    return w


TRANSPOSE_CASES = ([(B, 32, 16) for B in (1, 527, 528, 529, 1055, 1056, 1057, 4096, 65536)]
                   + [(1, 1, 1), (3, 3, 7), (5, 512, 1), (4, 1, 512), (1000, 7, 13), (2, 2048, 300)])


@pytest.mark.gpu
@pytest.mark.parametrize("B,C,S", TRANSPOSE_CASES, ids=["%dx%dx%d" % c for c in TRANSPOSE_CASES])
def test_flat_transpose_is_permute(B, C, S):
    """Both directions and the round trip equal permute as int32 words."""
    n = B * C * S
    words = random_words(n, B + C + S).to("cuda")
    src = _input(words.view(torch.float32))
    nhwc = run_transpose(src, B, C, S, 1)
    assert torch.equal(_bits(nhwc).view(B, S, C), words.view(B, C, S).permute(0, 2, 1)), "to NHWC"
    nchw = run_transpose(src, B, S, C, 0)           # src read as [B][C'=S][S'=C] rows in the other direction
    assert torch.equal(_bits(nchw).view(B, S, C), words.view(B, C, S).permute(0, 2, 1)), "to NCHW of the swapped shape"
    back = run_transpose(_input(nhwc), B, C, S, 0)
    assert torch.equal(_bits(back), words), "round trip"
    print("flat_transpose B=%d C=%d S=%d grid %d: permute bit for bit" % (B, C, S, min(_cdiv(n, THREADS), COPY_GRID_CAP)))


# ---------------------------------------------------------------------------------------------------------------------
# dv_channel_sum
# ---------------------------------------------------------------------------------------------------------------------
def run_channel_sum(xb, rows, C, nchw, hw):
    outs = []
    for _ in range(2):
        out, ws = _output(C), _output(WS_FLOATS)
        _launch(2, "dv_channel_sum", _addr(xb), _addr(out), rows, C, nchw, hw, _addr(ws), _stream())
        assert _intact(out, C) and _intact(ws, WS_FLOATS), "dv_channel_sum wrote past a buffer"
        outs.append((_body(out, C), _body(ws, WS_FLOATS)))
    _same_bits(outs[0][0], outs[1][0], "sums")
    _same_bits(outs[0][1], outs[1][1], "partials")
    return outs[0]


NHWC_ROWS = [1, 7, 8, 2367, 2368, 2369, 1 << 20]


@pytest.mark.gpu
@pytest.mark.parametrize("rows", NHWC_ROWS)
def test_channel_sum_nhwc(rows):
    worst = 0.0
    for C in range(1, 33):
        x = channel_sum_input(rows * C, rows * 40 + C)
        xb = _input(x)
        out, ws = run_channel_sum(xb, rows, C, 0, 0)
        xd = _body(xb, rows * C).view(rows, C).double()
        worst = max(worst, check_sums(out, xd.sum(0), xd.abs().sum(0), tau_nhwc(rows), rows, "C=%d" % C))
        check_grid_rows(ws, nhwc_grid(rows), C)
    print("channel_sum NHWC rows=%d C=1..32 grid %d: worst err %.3f of the bound" % (rows, nhwc_grid(rows), worst))


@pytest.mark.gpu
@pytest.mark.parametrize("hw", [1, 255, 256, 257, 4096])
@pytest.mark.parametrize("B", [1, 295, 296, 297, 1000])
def test_channel_sum_nchw(B, hw):
    worst = 0.0
    for C in (1, 3, 32):
        x = channel_sum_input(B * C * hw, B + hw + C)
        xb = _input(x)
        out, ws = run_channel_sum(xb, B, C, 1, hw)
        xd = _body(xb, B * C * hw).view(B, C, hw).double()
        worst = max(worst, check_sums(out, xd.sum((0, 2)), xd.abs().sum((0, 2)), tau_nchw(B, hw), B * hw, "C=%d" % C))
        check_grid_rows(ws, nchw_grid(B), C, nchw_words=True)
    print("channel_sum NCHW B=%d hw=%d grid %d: worst err %.3f of the bound" % (B, hw, nchw_grid(B), worst))


# ---------------------------------------------------------------------------------------------------------------------
# dv_u8_to_f32 and dv_gather_u8_to_f32
# ---------------------------------------------------------------------------------------------------------------------
def u8_data(n, seed):
    g = torch.Generator().manual_seed(seed)
    u = torch.randint(0, 256, (n,), generator=g, dtype=torch.int64).to(torch.uint8)
    if n >= 256:
        u[:256] = torch.randperm(256, generator=g).to(torch.uint8)
    return u


U8_STRIDE = COPY_GRID_CAP * THREADS          # 16-byte chunks one pass of the body loop covers
U8_N = list(range(1, 18)) + [31, 32, 33, 256 * 16] + [16 * U8_STRIDE + k for k in (-1, 0, 1, 15)]


@pytest.mark.gpu
@pytest.mark.parametrize("n", U8_N)
def test_u8_to_f32_grid_cap_and_tail(n):
    """Bit-identical to `src.float().div(255)` on the GPU and on the CPU, across the grid cap of the 16-byte body loop
    into the tail."""
    u = u8_data(n, n)
    buf, src = _u8_input(u)
    outs = []
    for _ in range(2):
        dst = _output(n)
        _launch(1, "dv_u8_to_f32", src, _addr(dst), n, _stream())
        assert _intact(dst, n), "dv_u8_to_f32 wrote past its output"
        outs.append(_body(dst, n))
    _same_bits(outs[0], outs[1], "u8_to_f32")
    assert torch.equal(_bits(outs[0]), _bits(true_div255(buf[16:16 + n]))), "CUDA true division"
    assert torch.equal(_bits(outs[0].cpu()), _bits(u.float().div(255))), "CPU div(255)"


def true_div255(u):
    """uint8 -> float / 255 by true division on u's device.  ToTensor's `img.float().div(255)` runs on the CPU, where
    that is what div does; on CUDA, Tensor.div by a Python scalar multiplies by the fp32 reciprocal of 255, which
    differs in the last bit for 126 of the 256 byte values, so the divisor here is a tensor."""
    x = u.float()
    return x / torch.full_like(x, 255.0)


def test_cuda_scalar_division_is_not_totensor_rounding():
    """The CPU facts true_div255 rests on: division by a tensor of 255s is div(255) bit for bit, and multiplying by
    the reciprocal (what CUDA's scalar div does) is not."""
    u = torch.arange(256, dtype=torch.uint8)
    assert torch.equal(_bits(true_div255(u)), _bits(u.float().div(255)))
    assert (_bits(u.float() * (1 / torch.tensor(255.0))) != _bits(u.float().div(255))).sum().item() == 126


@pytest.mark.gpu
def test_u8_to_f32_every_byte_value():
    u = torch.arange(256, dtype=torch.uint8).repeat(64)
    buf, src = _u8_input(u)
    dst = _output(u.numel())
    _launch(1, "dv_u8_to_f32", src, _addr(dst), u.numel(), _stream())
    assert torch.equal(_bits(_body(dst, u.numel()).cpu()), _bits(u.float().div(255)))


def run_gather(src_addr, idx, row_bytes):
    nrows = idx.numel()
    n = nrows * row_bytes
    ib = torch.full((2 + nrows + 64,), -1, dtype=torch.int64, device="cuda")
    ib[2:2 + nrows] = idx.to("cuda")
    outs = []
    for _ in range(2):
        dst = _output(n)
        _launch(1, "dv_gather_u8_to_f32", src_addr, ib.data_ptr() + 16, nrows, row_bytes, _addr(dst), _stream())
        assert _intact(dst, n), "dv_gather_u8_to_f32 wrote past its output"
        outs.append(_body(dst, n))
    _same_bits(outs[0], outs[1], "gather")
    return outs[0].view(nrows, row_bytes)


GATHER_CASES = [(16, 1), (16, U8_STRIDE + 1), (1024, 7), (3072, 64), (4096, 1055), (4096, 1056), (4096, 1057),
                (12288, 33)]


@pytest.mark.gpu
@pytest.mark.parametrize("row_bytes,nrows", GATHER_CASES, ids=["%dx%d" % c for c in GATHER_CASES])
def test_gather_u8_to_f32(row_bytes, nrows):
    N_ROWS = 2000
    data = u8_data(N_ROWS * row_bytes, row_bytes + nrows)
    buf, src = _u8_input(data)
    g = torch.Generator().manual_seed(nrows)
    idx = torch.randint(0, N_ROWS, (nrows,), generator=g)
    idx[: min(nrows, 3)] = torch.tensor([N_ROWS - 1, 0, N_ROWS - 1])[: min(nrows, 3)]
    got = run_gather(src, idx, row_bytes)
    ds = buf[16:16 + data.numel()].view(N_ROWS, row_bytes)
    assert torch.equal(_bits(got), _bits(true_div255(ds[idx.to("cuda")])))
    assert torch.equal(_bits(got.cpu()), _bits(data.view(N_ROWS, row_bytes)[idx].float().div(255)))


@pytest.mark.gpu
def test_gather_u8_to_f32_past_2gib():
    """Rows on both sides of byte 2^31 of a 2.1 GB dataset, and its last row, with repeats: the 64-bit source offset."""
    row_bytes = 4096
    R = 2 ** 31 // row_bytes + 64
    if torch.cuda.mem_get_info()[0] < 4 * 2 ** 30:
        pytest.skip("needs 4 GiB of free device memory")
    buf = torch.empty(16 + R * row_bytes + GUARD, dtype=torch.uint8, device="cuda")
    buf.random_(0, 256, generator=torch.Generator(device="cuda").manual_seed(1))
    mid = 2 ** 31 // row_bytes
    idx = torch.tensor([mid - 1, mid, mid + 1, R - 1, 0, mid, R - 1, mid - 2, mid + 63, mid - 1, 1, R - 1])
    got = run_gather(buf.data_ptr() + 16, idx, row_bytes)
    ds = buf[16:16 + R * row_bytes].view(R, row_bytes)
    assert torch.equal(_bits(got), _bits(true_div255(ds[idx.to("cuda")])))
    assert torch.equal(_bits(got.cpu()), _bits(ds[idx.to("cuda")].cpu().float().div(255)))
    print("gather past 2^31 bytes: %d rows bit for bit" % idx.numel())
    del buf, ds


# ---------------------------------------------------------------------------------------------------------------------
# loss combinations
# ---------------------------------------------------------------------------------------------------------------------
# (is_train, steps_anneal, counter before the call; None: a NULL counter)
SCHEDULES = [(0, 0, None), (0, 7, None), (0, 7, 5), (1, 0, 4), (1, 7, 0), (1, 7, 5), (1, 7, 6), (1, 7, 7),
             (1, 7, 1000), (1, 2 ** 31 + 7, 2 ** 31 + 4), (1, 2 ** 31 + 7, 2 ** 31 + 6), (1, 2 ** 31 + 7, 2 ** 31 + 9),
             (1, 2 ** 31 - 1, 2 ** 32 + 3)]
SHORT_SCHEDULES = [SCHEDULES[i] for i in (0, 3, 5, 10)]
UPSTREAM = [1.7, -2.5, 3e-3, -0.0]


def _floats(values):
    return (ctypes.c_float * max(len(values), 1))(*[float(v) for v in values])


class Combination:
    """Guarded device copies of one (a, b) and the raw calls of both combination pairs on them."""

    def __init__(self, na, nb, seed):
        self.na, self.nb = na, nb
        self.na_total = na + 3
        a, b, self.base = combo_inputs(na, nb, seed)
        self.a_host, self.b_host = a, b
        self.a = _input(torch.from_numpy(a))
        self.b = _input(torch.from_numpy(b)) if nb else None

    def sched_fwd(self, mask, init, fin, steps_anneal, is_train, pre, log=None):
        """-> (loss, coefs, counter after) of two calls from the same counter, asserted equal."""
        k = self.na + self.nb
        base = (ctypes.c_double * k)(*self.base)
        outs = []
        for _ in range(2):
            loss, coefs = _output(1), _output(k)
            cnt, caddr = _counter(pre) if pre is not None else (None, None)
            _launch(1, "dv_loss_combine_sched_fwd", _addr(self.a), self.na, _addr(self.b), self.nb, base, mask,
                    float(init), float(fin), steps_anneal, is_train, caddr, _addr(loss), _addr(coefs), log, _stream())
            assert _intact(loss, 1) and _intact(coefs, k), "scheduled forward wrote past its outputs"
            assert cnt is None or _counter_intact(cnt)
            outs.append((_body(loss, 1), _body(coefs, k), None if cnt is None else int(cnt[2])))
        _same_bits(outs[0][0], outs[1][0], "loss")
        _same_bits(outs[0][1], outs[1][1], "coefs")
        return outs[0]

    def sched_bwd(self, g, coefs):
        gb = _input(torch.tensor([g]))
        cb = _input(coefs.cpu())
        return self._bwd(lambda ga, gbo: _launch(1, "dv_loss_combine_sched_bwd", _addr(gb), _addr(cb), self.na,
                                                 self.na_total, self.nb, _addr(ga), _addr(gbo), _stream()))

    def host_fwd(self, coefs):
        c = coefs.cpu().numpy()
        outs = []
        for _ in range(2):
            loss = _output(1)
            _launch(1, "dv_loss_combine_fwd", _addr(self.a), _floats(c[:self.na]), self.na, _addr(self.b),
                    _floats(c[self.na:]) if self.nb else None, self.nb, _addr(loss), _stream())
            assert _intact(loss, 1)
            outs.append(_body(loss, 1))
        _same_bits(outs[0], outs[1], "host loss")
        return outs[0]

    def host_bwd(self, g, coefs):
        c = coefs.cpu().numpy()
        gb = _input(torch.tensor([g]))
        return self._bwd(lambda ga, gbo: _launch(1, "dv_loss_combine_bwd", _addr(gb), _floats(c[:self.na]), self.na,
                                                 self.na_total, _floats(c[self.na:]) if self.nb else None, self.nb,
                                                 _addr(ga), _addr(gbo), _stream()))

    def _bwd(self, call):
        outs = []
        for _ in range(2):
            ga, gbo = _output(self.na_total), _output(max(self.nb, 1))
            call(ga, gbo)
            assert _intact(ga, self.na_total) and _intact(gbo, max(self.nb, 1)), "backward wrote past its outputs"
            if not self.nb:
                assert _bits(_body(gbo, 1)).item() == NAN_FILL, "g_b written with nb = 0"
            outs.append((_body(ga, self.na_total), _body(gbo, self.nb)))
        _same_bits(outs[0][0], outs[1][0], "g_a")
        _same_bits(outs[0][1], outs[1][1], "g_b")
        return outs[0]


def check_combination(cmb, mask, schedule, g, init, fin):
    is_train, steps_anneal, pre = schedule
    na, nb = cmb.na, cmb.nb
    loss, coefs, after = cmb.sched_fwd(mask, init, fin, steps_anneal, is_train, pre)
    s = pre + 1 if is_train else 0
    if pre is not None:
        assert after == (pre + 1 if is_train else pre), "counter %s -> %s with is_train %d" % (pre, after, is_train)
    want = host_coefs(cmb.base, mask, init, fin, s, steps_anneal, is_train)
    got = coefs.cpu().numpy()
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (schedule, mask, got, want)
    vals = list(cmb.a_host[:na]) + list(cmb.b_host)
    r = combine_ratio(loss.item(), vals, got, na, nb)
    assert r <= 1, ("loss", schedule, mask, r)
    ga, gb = cmb.sched_bwd(g, coefs)
    c32 = torch.from_numpy(want)
    assert torch.equal(_bits(ga[:na].cpu()), _bits(torch.tensor([g], dtype=torch.float32) * c32[:na])), "g_a"
    assert (_bits(ga[na:]) == 0).all(), "g_a past na is not +0"
    assert torch.equal(_bits(gb.cpu()), _bits(torch.tensor([g], dtype=torch.float32) * c32[na:])), "g_b"
    # the host-coefficient pair with the same coefficients gives the same bits
    assert torch.equal(_bits(cmb.host_fwd(coefs)), _bits(loss)), "host-coefficient loss"
    ha, hb = cmb.host_bwd(g, coefs)
    assert torch.equal(_bits(ha), _bits(ga)) and torch.equal(_bits(hb), _bits(gb)), "host-coefficient gradients"
    return r


@pytest.mark.gpu
@pytest.mark.parametrize("na", range(1, 9))
def test_loss_combination(na):
    """Every nb in 0..8 and masks none, all and mixed, on every schedule: the coefficients equal the host values bit for
    bit, the loss is within its bound of fp64, the gradients are fp32(g c) with +0 past na, the host-coefficient pair
    gives the same bits, and the counter advances only on training steps."""
    worst = 0.0
    for nb in range(0, 9):
        k = na + nb
        cmb = Combination(na, nb, 100 * na + nb)
        init, fin = (0.0, 1.0) if k % 2 == 0 else (0.25, 3.0)
        rng = np.random.default_rng(k)
        masks = [(1 << k) - 1, 0, int(rng.integers(0, 1 << k))]
        for m, mask in enumerate(masks):
            for i, sched in enumerate(SCHEDULES if m == 0 else SHORT_SCHEDULES):
                worst = max(worst, check_combination(cmb, mask, sched, UPSTREAM[(i + m) % len(UPSTREAM)], init, fin))
    print("loss combination na=%d nb=0..8: worst loss err %.3f of the bound" % (na, worst))


# ---------------------------------------------------------------------------------------------------------------------
# beta-VAE_B backward
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", [2, 3, 12])
def test_betab_backward(n):
    """g_rec_kl = (0 + g, 0 + (g gamma) sgn(kl - C), +0 ...): +0 at kl == C for g of either sign, never -0."""
    C, gm = np.float32(12.5), np.float32(100.0)
    for kl in (C, C + np.float32(1.5), C - np.float32(0.75), np.nextafter(C, np.float32(0))):
        for g in (1.5, -1.5, 0.0, -0.0, 1e36):
            rec_kl = torch.tensor([123.0, float(kl)] + [7.0] * (n - 2))
            rb, cb, gb = _input(rec_kl), _input(torch.tensor([float(C), float(gm)])), _input(torch.tensor([g]))
            outs = []
            for _ in range(2):
                out = _output(n)
                _launch(1, "dv_betab_loss_bwd", _addr(gb), _addr(rb), _addr(cb), n, _addr(out), _stream())
                assert _intact(out, n)
                outs.append(_body(out, n).cpu())
            _same_bits(outs[0], outs[1], "betab backward")
            got = outs[0]
            g32 = torch.tensor([g], dtype=torch.float32)
            d = torch.tensor([float(kl)]) - torch.tensor([float(C)])
            want = torch.cat([0 + g32, 0 + (g32 * float(gm)) * torch.sign(d), torch.zeros(n - 2)])
            assert torch.equal(_bits(got), _bits(want)), (kl, g, got.tolist(), want.tolist())
            if kl == C:
                assert _bits(got)[1].item() == 0, "g_kl at kl == C is not +0"
            assert (_bits(got)[2:] == 0).all()


# ---------------------------------------------------------------------------------------------------------------------
# the device loss log
# ---------------------------------------------------------------------------------------------------------------------
SRC_LENS = [2, 0, 5, 1, 7, 3, 0, 4]


def make_log(ring_addr, cap, every, srcs):
    """srcs: list of (device address or None, length)."""
    N = _native()
    L = N.LossLog()
    L.ring, L.cap, L.every, L.nsrc = ring_addr, cap, every, len(srcs)
    L.ncols = sum(n for _, n in srcs)
    for k, (p, n) in enumerate(srcs):
        L.src[k], L.len[k] = p, n
    return L


def log_configs(entry):
    """(nsrc, position of the NULL self-source or None)."""
    if entry == "record":
        return [(1, None), (3, None), (8, None)]
    return [(1, 0)] + [(3, j) for j in range(3)] + [(8, j) for j in range(8)]


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["sched", "betab", "record"])
@pytest.mark.parametrize("every", [1, 2, 50])
@pytest.mark.parametrize("cap", [1, 3])
def test_loss_log(cap, every, entry):
    """Every call of a step sequence: a recording step writes its row (s - 1) // every % cap, bit for bit the sources
    (the NULL source: the loss the same launch computed), rows not due keep their NaN or earlier contents, and a call
    with is_train = 0 records nothing and leaves the counter alone."""
    pool_host = torch.arange(1, 65, dtype=torch.float32) * 1.25 - 17
    pool = _input(pool_host)
    a_host = torch.tensor([3.5, -1.25, 0.5, 9.0])
    a = _input(a_host)
    rows_written = 0
    for nsrc, null_at in log_configs(entry):
        srcs, off = [], 0
        for k in range(nsrc):
            if k == null_at:
                srcs.append((None, 1))
            else:
                n = SRC_LENS[k]
                srcs.append((_addr(pool, 4 * off), n))
                off += n + 1
        ncols = sum(n for _, n in srcs)
        if ncols == 0:
            srcs[-1] = (srcs[-1][0], 1)
            ncols = 1
        ring = _output(cap * ncols)
        log = make_log(_addr(ring), cap, every, srcs)
        want = torch.full((cap, ncols), float("nan"))
        for s in log_steps(every):
            for is_train in (1, 0):
                if entry == "record" and not is_train:
                    continue
                cnt, caddr = _counter(s - 1 if entry != "record" else s)
                before = _native().lib().dv_launch_count()
                loss = _output(1)
                if entry == "sched":
                    base = (ctypes.c_double * 2)(1.0, 0.37)
                    coefs = _output(2)
                    rc = _native().lib().dv_loss_combine_sched_fwd(_addr(a), 2, None, 0, base, 2, 0.0, 1.0, 7,
                                                                   is_train, caddr, _addr(loss), _addr(coefs),
                                                                   ctypes.byref(log), _stream())
                elif entry == "betab":
                    consts = _output(2)
                    rc = _native().lib().dv_betab_loss_fwd(_addr(a), 100.0, 0.0, 25.0, 7, is_train, caddr,
                                                           _addr(loss), _addr(consts), ctypes.byref(log), _stream())
                else:
                    rc = _native().lib().dv_loss_record(caddr, ctypes.byref(log), _stream())
                assert rc == DV_OK and _native().lib().dv_launch_count() - before == 1
                torch.cuda.synchronize()
                assert _counter_intact(cnt)
                if entry != "record":
                    assert int(cnt[2]) == (s if is_train else s - 1), "counter"
                row = log_row(s, every, cap) if is_train else None
                if row is not None:
                    vals = []
                    for p, n in srcs:
                        if p is None:
                            vals.append(_body(loss, 1).cpu())
                        else:
                            o = (p - _addr(pool)) // 4
                            vals.append(pool_host[o:o + n])
                    want[row] = torch.cat(vals)
                    rows_written += 1
                assert _intact(ring, cap * ncols), "the log wrote past its ring"
                got = _body(ring, cap * ncols).view(cap, ncols).cpu()
                assert torch.equal(_bits(got), _bits(want)), (entry, s, is_train, row, got, want)
    assert rows_written > 0 or every == 1
    print("loss log %s cap=%d every=%d: %d recording calls, every ring bit as expected" % (entry, cap, every,
                                                                                       rows_written))


# ---------------------------------------------------------------------------------------------------------------------
# the Python wrappers call the same kernels
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_ops_wrappers_are_the_raw_calls():
    """disvae.ops' channel_sum, flat_transpose, act_bwd, act_bwd_chansum, u8_to_f32, gather_u8_to_f32 and
    LossCombineFn (a vector, a 0-dim and no second operand) give the raw calls' bits."""
    from disvae import ops
    B, C, hw = 37, 3, 4096
    dy, y = act_inputs(B * C * hw, ACT_SIGMOID, 3)
    dyb, yb = _input(dy), _input(y)
    g_raw, cs_raw, _ = run_act_chansum(dyb, yb, B, C, hw, ACT_SIGMOID, 0.0)
    g, cs = ops.act_bwd_chansum(dy.view(B, C, 64, 64).cuda(), y.view(B, C, 64, 64).cuda(), ACT_SIGMOID)
    assert torch.equal(_bits(g).view(-1), _bits(g_raw)) and torch.equal(_bits(cs), _bits(cs_raw))
    assert torch.equal(_bits(ops.act_bwd(dy.cuda(), y.cuda(), ACT_SIGMOID)), _bits(g_raw))
    x = channel_sum_input(1000 * 32, 1)
    out, _ = run_channel_sum(_input(x), 1000, 32, 0, 0)
    assert torch.equal(_bits(ops.channel_sum(x.cuda(), 1000, 32, 0, 0)), _bits(out))
    out, _ = run_channel_sum(_input(dy), B, C, 1, hw)
    assert torch.equal(_bits(ops.channel_sum(dy.cuda(), B, C, 1, hw)), _bits(out))
    t = random_words(9 * 512, 9).view(torch.float32)
    nhwc = ops.flat_transpose(t.view(9, 512).cuda(), 9, to_nhwc=True)
    assert torch.equal(_bits(nhwc).view(9, 16, 32), _bits(t).view(9, 32, 16).permute(0, 2, 1).cuda())
    assert torch.equal(_bits(ops.flat_transpose(nhwc, 9, to_nhwc=False)), _bits(t).view(9, 512).cuda())
    for n in (3, 16, 12345 * 16 + 7, 1 << 20):
        u = u8_data(n, n)
        assert torch.equal(_bits(ops.u8_to_f32(u.cuda()).cpu()), _bits(u.float().div(255)))
    data = u8_data(50 * 4096, 5).view(50, 4096).cuda()
    idx = torch.tensor([49, 0, 3, 3, 17], device="cuda")
    assert torch.equal(_bits(ops.gather_u8_to_f32(data, idx)), _bits(true_div255(data[idx])))
    # LossCombineFn: the fused loss output (12 entries, two weighted) with a vector, a 0-dim tensor and no second
    # operand; gradients in the operands' shapes, zeros past the weighted entries
    a = torch.randn(12, generator=torch.Generator().manual_seed(1)).cuda()
    for b, ca, cb in ((torch.tensor([0.5, -2.0, 3.0]).cuda(), [1.0, 0.37], [1.0, 6.0, 0.25]),
                      (torch.tensor(0.8).cuda(), [1.0, 1.0], [6.4]), (None, [1.0, 4.0], None)):
        ad = a.clone().requires_grad_(True)
        bd = b.clone().requires_grad_(True) if b is not None else None
        loss = ops.LossCombineFn.apply(ad, bd, ca, cb)
        c = np.array(ca + (cb or []), dtype=np.float32)
        vals = a[:2].tolist() + ([] if b is None else b.reshape(-1).tolist())
        assert loss.shape == () and combine_ratio(loss.item(), vals, c, 2, len(cb or [])) <= 1
        (loss * 1.7).backward()
        g17 = torch.tensor([1.7], dtype=torch.float32)
        assert torch.equal(_bits(ad.grad[:2].cpu()), _bits(g17 * torch.from_numpy(c[:2])))
        assert (_bits(ad.grad[2:]) == 0).all()
        if b is not None:
            assert bd.grad.shape == b.shape
            assert torch.equal(_bits(bd.grad.reshape(-1).cpu()), _bits(g17 * torch.from_numpy(c[2:])))


# ---------------------------------------------------------------------------------------------------------------------
# refusals: status code, nothing launched, outputs untouched
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_refusals_launch_nothing():
    """Every refusal of every glue entry point, and the layout and activation refusals of dv_conv.cu: NULL pointers,
    bad counts, masks and logs, shapes whose indices would overflow int, unknown activation codes and misaligned
    operands come back as status codes with no kernel launched and every output untouched."""
    N = _native()
    L, S = N.lib(), _stream()
    inp = _input(torch.ones(1 << 16))
    a = _addr(inp)
    outs = [_output(1 << 16) for _ in range(4)]
    o, o2, o3, ws = (_addr(t) for t in outs)
    cnt, step = _counter(5)
    ring = _output(64)
    ib = torch.zeros(64, dtype=torch.int64, device="cuda")
    idx = ib.data_ptr() + 16

    def refused(status, fn, *args):
        before = L.dv_launch_count()
        rc = getattr(L, fn)(*args)
        torch.cuda.synchronize()
        assert rc == status, "%s%s returned %d, expected %d" % (fn, args, rc, status)
        assert L.dv_launch_count() == before, fn + ": launched a kernel"
        for t in outs + [ring]:
            assert (_bits(t)[OFF:-GUARD] == NAN_FILL).all() and _intact(t, t.numel() - OFF - GUARD), fn + " wrote"
        assert int(cnt[2]) == 5 and _counter_intact(cnt), fn + " moved the counter"

    # dv_act_bwd_chansum (dy, y, g, B, C, hw, act, slope, chansum, workspace)
    def chansum(status, B=4, C=3, hw=64, act=ACT_SIGMOID, **p):
        q = dict(dict(dy=a, y=a, g=o, cs=o2, ws=ws), **p)
        refused(status, "dv_act_bwd_chansum", q["dy"], q["y"], q["g"], B, C, hw, act, 0.0, q["cs"], q["ws"], S)
    for k in ("dy", "y", "g", "cs", "ws"):
        chansum(DV_ERR_BAD_ARG, **{k: None})
    for shape in (dict(B=0), dict(B=-1), dict(C=0), dict(C=5), dict(hw=0), dict(hw=2), dict(hw=6), dict(hw=4098),
                  dict(B=2 ** 30, C=2), dict(B=INT_MAX, C=4), dict(B=INT_MAX // 3 + 1, C=3)):
        chansum(DV_ERR_BAD_SHAPE, **shape)
    for act in (-1, 4, 99):
        chansum(DV_ERR_BAD_ARG, act=act)
    for off in (4, 8, 12):
        for k, base in (("dy", a), ("y", a), ("g", o)):
            chansum(DV_ERR_BAD_ARG, **{k: base + off})
    for off in (1, 2, 3):
        chansum(DV_ERR_BAD_ARG, cs=o2 + off)
        chansum(DV_ERR_BAD_ARG, ws=ws + off)
    # dv_act_bwd (dy, y, g, n, act, slope)
    for i in range(3):
        args = [a, a, o]
        args[i] = None
        refused(DV_ERR_BAD_ARG, "dv_act_bwd", *args, 64, ACT_SIGMOID, 0.0, S)
    for n in (0, -1):
        refused(DV_ERR_BAD_SHAPE, "dv_act_bwd", a, a, o, n, ACT_SIGMOID, 0.0, S)
    for act in (-1, 4, 99):
        refused(DV_ERR_BAD_ARG, "dv_act_bwd", a, a, o, 64, act, 0.0, S)
    # dv_flat_transpose (src, dst, B, C, S, to_nhwc)
    refused(DV_ERR_BAD_ARG, "dv_flat_transpose", None, o, 2, 32, 16, 1, S)
    refused(DV_ERR_BAD_ARG, "dv_flat_transpose", a, None, 2, 32, 16, 1, S)
    for B_, C_, S_ in ((0, 32, 16), (2, 0, 16), (2, 32, 0), (-1, 32, 16), (1, 65536, 32768), (1, INT_MAX, 2),
                       (1, 2, INT_MAX)):
        refused(DV_ERR_BAD_SHAPE, "dv_flat_transpose", a, o, B_, C_, S_, 1, S)
    # dv_channel_sum (x, out, rows, C, nchw, hw, workspace)
    for i in (0, 1, 6):
        args = [a, o2, 64, 3, 0, 0, ws]
        args[i] = None
        refused(DV_ERR_BAD_ARG, "dv_channel_sum", *args, S)
    for rows, C_, nchw, hw in ((0, 3, 0, 0), (-1, 3, 0, 0), (64, 0, 0, 0), (64, 33, 0, 0), (4, 3, 1, 0),
                               (4, 3, 1, -1), (2 ** 31, 1, 1, 1), (2 ** 40, 1, 1, 1)):
        refused(DV_ERR_BAD_SHAPE, "dv_channel_sum", a, o2, rows, C_, nchw, hw, ws, S)
    # dv_u8_to_f32 (src, dst, n)
    refused(DV_ERR_BAD_ARG, "dv_u8_to_f32", None, o, 64, S)
    refused(DV_ERR_BAD_ARG, "dv_u8_to_f32", a, None, 64, S)
    for n in (0, -1):
        refused(DV_ERR_BAD_SHAPE, "dv_u8_to_f32", a, o, n, S)
    for off in range(1, 16):
        refused(DV_ERR_BAD_ARG, "dv_u8_to_f32", a + off, o, 64, S)
    for off in (4, 8, 12):
        refused(DV_ERR_BAD_ARG, "dv_u8_to_f32", a, o + off, 64, S)
    # dv_gather_u8_to_f32 (src, idx, nrows, row_bytes, dst)
    for i in (0, 1, 4):
        args = [a, idx, 4, 64, o]
        args[i] = None
        refused(DV_ERR_BAD_ARG, "dv_gather_u8_to_f32", *args, S)
    for nrows, rb in ((0, 64), (-1, 64), (4, 0), (4, 8), (4, 24), (4, -16)):
        refused(DV_ERR_BAD_SHAPE, "dv_gather_u8_to_f32", a, idx, nrows, rb, o, S)
    for off in range(1, 16):
        refused(DV_ERR_BAD_ARG, "dv_gather_u8_to_f32", a + off, idx, 4, 64, o, S)
    for off in (4, 8, 12):
        refused(DV_ERR_BAD_ARG, "dv_gather_u8_to_f32", a, idx, 4, 64, o + off, S)
    refused(DV_ERR_BAD_ARG, "dv_gather_u8_to_f32", a, idx + 4, 4, 64, o, S)
    # dv_loss_combine_fwd / _bwd (host coefficients)
    c8 = _floats([1.0] * 9)

    def combine_fwd(status, na=2, nb=3, **p):
        q = dict(dict(a=a, ca=c8, b=a, cb=c8, loss=o), **p)
        refused(status, "dv_loss_combine_fwd", q["a"], q["ca"], na, q["b"], q["cb"], nb, q["loss"], S)
    for k in ("a", "ca", "loss", "b", "cb"):
        combine_fwd(DV_ERR_BAD_ARG, **{k: None})
    for na, nb in ((0, 3), (9, 3), (-1, 3), (2, -1), (2, 9)):
        combine_fwd(DV_ERR_BAD_ARG, na=na, nb=nb)

    def combine_bwd(status, na=2, na_total=5, nb=3, **p):
        q = dict(dict(g=a, ca=c8, cb=c8, ga=o, gb=o2), **p)
        refused(status, "dv_loss_combine_bwd", q["g"], q["ca"], na, na_total, q["cb"], nb, q["ga"], q["gb"], S)
    for k in ("g", "ca", "ga", "cb"):
        combine_bwd(DV_ERR_BAD_ARG, **{k: None})
    for na, na_total, nb in ((0, 5, 3), (9, 12, 3), (2, 1, 3), (2, 5, -1), (2, 5, 9)):
        combine_bwd(DV_ERR_BAD_ARG, na=na, na_total=na_total, nb=nb)
    # the log checks shared by the forward entry points and dv_loss_record
    bad_logs = [(DV_ERR_BAD_ARG, make_log(None, 2, 1, [(a, 3)])),
                (DV_ERR_BAD_ARG, make_log(_addr(ring), 0, 1, [(a, 3)])),
                (DV_ERR_BAD_ARG, make_log(_addr(ring), -1, 1, [(a, 3)])),
                (DV_ERR_BAD_ARG, make_log(_addr(ring), 2, 0, [(a, 3)])),
                (DV_ERR_BAD_ARG, make_log(_addr(ring), 2, -3, [(a, 3)])),
                (DV_ERR_BAD_ARG, make_log(_addr(ring), 2, 1, [])),
                (DV_ERR_BAD_ARG, make_log(_addr(ring), 2, 1, [(None, 2)])),
                (DV_ERR_BAD_ARG, make_log(_addr(ring), 2, 1, [(a, 3), (None, 0)])),
                (DV_ERR_BAD_ARG, make_log(_addr(ring), 2, 1, [(a, -1), (a, 4)]))]
    nine = make_log(_addr(ring), 2, 1, [(a, 1)] * 8)
    nine.nsrc = 9
    bad_logs.append((DV_ERR_BAD_ARG, nine))
    for ncols in (2, 4, 0):
        L_ = make_log(_addr(ring), 2, 1, [(a, 3)])
        L_.ncols = ncols
        bad_logs.append((DV_ERR_BAD_SHAPE, L_))
    base = (ctypes.c_double * 16)(*([1.0] * 16))

    def sched_fwd(status, na=2, nb=3, mask=1, steps_anneal=7, is_train=1, log=None, **p):
        q = dict(dict(a=a, b=a, base=base, step=step, loss=o, coefs=o2), **p)
        refused(status, "dv_loss_combine_sched_fwd", q["a"], na, q["b"], nb, q["base"], mask, 0.0, 1.0, steps_anneal,
                is_train, q["step"], q["loss"], q["coefs"], None if log is None else ctypes.byref(log), S)
    for k in ("a", "b", "base", "loss", "coefs"):
        sched_fwd(DV_ERR_BAD_ARG, **{k: None})
    sched_fwd(DV_ERR_BAD_ARG, step=None)                           # is_train without a step counter
    for na, nb in ((0, 3), (9, 3), (2, -1), (2, 9)):
        sched_fwd(DV_ERR_BAD_ARG, na=na, nb=nb)
    for na, nb in ((2, 3), (8, 8), (1, 0)):
        for mask in (1 << (na + nb), 0xFFFFFFFF, (1 << 31)):
            sched_fwd(DV_ERR_BAD_ARG, na=na, nb=nb, mask=mask)
    for sa in (-1, -2 ** 40):
        sched_fwd(DV_ERR_BAD_ARG, steps_anneal=sa)
        refused(DV_ERR_BAD_ARG, "dv_betab_loss_fwd", a, 100.0, 0.0, 25.0, sa, 1, step, o, o2, None, S)
    for status, log in bad_logs:
        sched_fwd(status, log=log)
        refused(status, "dv_betab_loss_fwd", a, 100.0, 0.0, 25.0, 7, 1, step, o, o2, ctypes.byref(log), S)
        refused(status, "dv_loss_record", step, ctypes.byref(log), S)
    # dv_loss_combine_sched_bwd (g, coefs, na, na_total, nb, g_a, g_b)
    for i in (0, 1, 5):
        args = [a, a, 2, 5, 3, o, o2]
        args[i] = None
        refused(DV_ERR_BAD_ARG, "dv_loss_combine_sched_bwd", *args, S)
    for na, na_total, nb in ((0, 5, 3), (9, 12, 3), (2, 1, 3), (2, 5, -1), (2, 5, 9)):
        refused(DV_ERR_BAD_ARG, "dv_loss_combine_sched_bwd", a, a, na, na_total, nb, o, o2, S)
    # dv_betab_loss_fwd / _bwd
    for i in (0, 7, 8):
        args = [a, 100.0, 0.0, 25.0, 7, 1, step, o, o2, None]
        args[i] = None
        refused(DV_ERR_BAD_ARG, "dv_betab_loss_fwd", *args, S)
    refused(DV_ERR_BAD_ARG, "dv_betab_loss_fwd", a, 100.0, 0.0, 25.0, 7, 1, None, o, o2, None, S)
    for i in (0, 1, 2, 4):
        args = [a, a, a, 4, o]
        args[i] = None
        refused(DV_ERR_BAD_ARG, "dv_betab_loss_bwd", *args, S)
    for n in (1, 0, -1):
        refused(DV_ERR_BAD_ARG, "dv_betab_loss_bwd", a, a, a, n, o, S)
    # dv_loss_record: a NULL counter or log, and a NULL source even of length 1 (it has no loss of its own)
    refused(DV_ERR_BAD_ARG, "dv_loss_record", None, ctypes.byref(make_log(_addr(ring), 2, 1, [(a, 3)])), S)
    refused(DV_ERR_BAD_ARG, "dv_loss_record", step, None, S)
    refused(DV_ERR_BAD_ARG, "dv_loss_record", step, ctypes.byref(make_log(_addr(ring), 2, 1, [(a, 3), (None, 1)])), S)
