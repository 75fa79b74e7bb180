"""The convolutions (csrc/dv_conv.cu, csrc/dv_conv_tc.cu, csrc/dv_conv_img.cu) on every path they can take, against fp64
references, through the raw C ABI.

Every Burgess layer links lo[B, H, W, 32] (NHWC) and hi[B, 2H, 2W, CH] through w[32][CH][4][4] (4x4, stride 2, pad 1).
CH = 32 (lo 4, 8, 16, hi NHWC) runs on the wgmma 3xTF32 kernels, CH in {1, 3} (lo 16, 32, hi NCHW) on the exact-fp32
CUDA-core kernels; the weight gradient of both ends in the split-K reduction `conv_wgrad_reduce_kernel`, the channel
sums of `dv_conv_down` in `channel_sum_final_kernel`.  The tile, grid and split plans of every kernel are restated
below; each case asserts the workspace query against them and counts the kernels each call launches.

Every element of every output is checked against `|got - ref| <= tau * sum|terms| + EPI * |ref|`: fp64 value and the
fp64 magnitude of what the kernel adds up, with tau derived per path from the longest rounding chain of its code
(written beside each plan).  Where the earlier tests held a whole tensor to WHOLE_TOL of its largest |ref| that check
stays too.  Outputs, bit words, workspaces and reductions sit in NaN-filled buffers between sentinel words, inputs are
followed by NaN, every operand starts 16 bytes into its allocation, and every call runs twice and must repeat bit for
bit.

The bound is first shown to have teeth on the CPU; everything else needs an H100 (pytest -m gpu).  Each GPU case
prints its worst error as a fraction of the bound (pytest -s shows them)."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

U = 2.0 ** -24          # fp32 unit roundoff (round to nearest)
# 3xTF32: a = ah + al and w = wh + wl, each hi the nearest tf32 (error <= 2^-11 |a|) and each lo the nearest tf32 of the
# residual (error <= 2^-22 |a|).  ah.wh + ah.wl + al.wh leaves out al.wl and carries the two lo roundings: <= 3 * 2^-22
# of |a w| per product.  Every product is exact in the fp32 accumulator; a tensor-core k8 step adds 8 of them to it and
# is charged 2 u (its adder may truncate), an fp32 add or FMA 1 u, each relative to the |terms| summed so far.
RHO = 12 * U
EPI = 2.0 ** -21        # the epilogue's own roundings relative to |ref| (sigmoid's exp and division)
WHOLE_TOL = 4e-6        # max |got - ref| over an output tensor relative to its max |ref|, as the earlier tests held
WHOLE_TOL_SUMS = {32: 4e-6, 1: 1e-5, 3: 1e-5}   # ... and over dw, dbias and channel sums (image layers: 1M-pixel sums)
SM_COUNT = 132          # kNumSMs in csrc/dv_common.cuh: the plans are sized for an H100 SXM
IMG_GRID = 2 * SM_COUNT
CS_BLOCKS = 296         # kCsBlocks: channel-sum partials (also caps the image down kernel's grid with colsum_out)
HALO_STAGE_BYTES = 26 * 1024
GUARD = 1024            # words of sentinel after each output and workspace
SENTINEL = 0x7FBADBAD   # a NaN bit pattern no kernel writes
OFF = 4                 # floats: every operand starts 16 bytes into its allocation
DV_OK, DV_ERR_BAD_SHAPE, DV_ERR_BAD_ARG, DV_ERR_WORKSPACE = 0, -1, -2, -3     # include/disvae_b200.h
ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_LEAKY = 0, 1, 2, 3


def _cdiv(a, b):
    return -(-a // b)


# ---------------------------------------------------------------------------------------------------------------------
# plans and rounding chains, restated from the kernels' host code
# ---------------------------------------------------------------------------------------------------------------------
def tc_down_plan(B, H):
    """conv_down32_tc: 128 lo pixels per tile = 128 / W image rows; TR rows of TB images; persistent grid."""
    W = H
    rpt = 128 // W
    TR = min(rpt, H)
    tiles = _cdiv(B * H * W, 128)
    return dict(TR=TR, TB=rpt // TR, tiles=tiles, grid=min(tiles, SM_COUNT))


def halo_up_plan(B, H):
    """conv_up_halo: whole small images per tile (TB > 1, as many as the 26 KB stage holds) or 128 / W rows of one."""
    W = H
    rpt = 128 // W
    if rpt >= H:
        TR, TB = H, max(rpt // H, 1)
        while TB > 1 and TB * (H + 2) * W * 128 > HALO_STAGE_BYTES:
            TB -= 1
        tiles_per_img, tiles = 1, _cdiv(B, TB)
    else:
        TR, TB, tiles_per_img = rpt, 1, _cdiv(H, rpt)
        tiles = B * tiles_per_img
    return dict(TR=TR, TB=TB, tiles_per_img=tiles_per_img, tiles=tiles, grid=min(tiles, SM_COUNT))


def img_down_plan(B, H):
    """img::conv_down: 16 lo rows per tile, grid min(tiles, 2 x 132) (and <= CS_BLOCKS with channel sums)."""
    tiles = B * (H // 16)
    return dict(tiles=tiles, grid=min(tiles, IMG_GRID, CS_BLOCKS))


def up_tile_rows(W):
    return (128 // (W // 2)) * 2            # up_tile_rows<W>: 16 (W = 32), 32 (W = 16)


def img_up_plan(B, H):
    TR = up_tile_rows(H)
    tiles = B * _cdiv(H, TR)
    return dict(TR=TR, tiles=tiles, grid=min(tiles, IMG_GRID))


def wgrad_plan(B, H, CH):
    """-> (S, tiles, tiles per CTA): tc wgrad_splits spreads 128-pixel tiles over at most 132 CTAs with no empty CTA;
    img::wgrad_splits runs min(16-row tiles, 264 (CH = 1) or 132 (CH = 3)) persistent CTAs."""
    if CH == 32:
        tiles = _cdiv(B * H * H, 128)
        grid = min(tiles, SM_COUNT)
        per = _cdiv(tiles, grid)
        return _cdiv(tiles, per), tiles, per
    tiles = B * (H // 16)
    S = min(tiles, (2 if CH == 1 else 1) * SM_COUNT)
    return S, tiles, _cdiv(tiles, S)


def wgrad_ws_bytes(B, H, CH):
    return wgrad_plan(B, H, CH)[0] * (16 * CH + 1) * 32 * 4


def packed_floats(CH):
    return 2 * 16 * 64 * 32 if CH == 32 else 2 * 32 * CH * 16


def max_batch(H):
    """The largest B with B * 4 * H * W * 32 < 2^31 (int pixel indices)."""
    return (2 ** 31 - 1) // (4 * H * H * 32)


# Rounding chains (tau: error relative to sum|terms|).
def tau_down(CH):
    if CH == 32:
        # per tap 4 k8 slices into acc (2u each), 16 taps folded into the fp32 total (1u each), total + corr, + bias;
        # corr (<= 2^-10 of the terms) accumulates 128 k8 steps
        return RHO + 2 * U * 4 + U * 16 + 2 * U + 2 * U * 128 / 1024
    return (16 * CH + 1) * U               # 16 CH sequential FMAs, + bias


def tau_up(CH):
    if CH == 32:
        # per output phase 4 (shift, tap) products of 4 k8 slices each, 4 folds, total + corr, + bias; corr: 32 steps
        return RHO + 2 * U * 4 + U * 4 + 2 * U + 2 * U * 32 / 1024
    return (128 + 1) * U                   # 8 channel chunks x 4 taps x 4 FMAs in one chain, + bias


def tau_wgrad(B, H, CH):
    """-> (tau of dw, tau of dbias_lo)."""
    S, tiles, per = wgrad_plan(B, H, CH)
    reduce = _cdiv(S, 8) + 3               # conv_wgrad_reduce_kernel: every 8th split in sequence, then a 3-level tree
    if CH == 32:
        # 16 k8 slices over a tile's 128 pixels, acc + corr, one add per tile into the CTA's total; the bias gradient
        # is exact fp32: 16 rows of a tile per warp in sequence over the CTA's tiles, then the 8 warps
        return RHO + 2 * U * 16 + 2 * U * 32 / 1024 + U * (1 + per + reduce), U * (16 * per + 8 + reduce)
    # a stream owns every output and walks W pixels of each of its CTA's tiles, then the 16 streams in sequence
    t = U * (H * _cdiv(tiles, S) + 16 + reduce)
    return t, t


def tau_colsum(B, H, CH):
    """Channel sums of the stored output: per thread over its pixels of every tile, 3 shuffle levels, 8 warps, then
    channel_sum_final_kernel (every 32nd partial in sequence, then the 32 slices)."""
    if CH == 32:
        p = tc_down_plan(B, H)
        per_thread = 2 * _cdiv(p["tiles"], p["grid"])          # MMA rows g and g + 8 of every tile
    else:
        p = img_down_plan(B, H)
        per_thread = (H // 4) * _cdiv(p["tiles"], p["grid"])   # PXG = 16 W / 64 pixels of every tile
    return U * (per_thread + 3 + 8 + _cdiv(p["grid"], 32) + 32)


# ---------------------------------------------------------------------------------------------------------------------
# cases: (B, H of lo, CH); each runs down, up and wgrad
# ---------------------------------------------------------------------------------------------------------------------
def _network_cases():
    out = []
    for B in (64, 256, 512, 1024):
        for S in (32, 64):                  # image size: the image layer at lo S / 2, the 32-channel layers below it
            for C in (1, 3):
                out.append((B, S // 2, C))
                H = S // 4
                while H >= 4:
                    out.append((B, H, 32))
                    H //= 2
    return list(dict.fromkeys(out))


NETWORK_CASES = _network_cases()
# tile counts on both sides of one and two CTA waves: tc lo 8 (two images per tile) 1, 131, 132, 133, 264, 265 tiles
# (wgrad S = 67 at 133, 89 at 265); image kernels 263, 264, 265 tiles at lo 16 and 264, 266 at lo 32
TILE_CASES = ([(B, 8, 32) for B in (1, 261, 264, 265, 528, 529)]
              + [(B, 16, CH) for CH in (1, 3) for B in (263, 264, 265)]
              + [(B, 32, CH) for CH in (1, 3) for B in (132, 133)])
# partial multi-image tiles: lo 4 (TB = 8) with B % 8 in {1, 7}, lo 8 (TB = 2) with odd B, and B = 1 everywhere
PARTIAL_CASES = [(1, 4, 32), (9, 4, 32), (15, 4, 32), (3, 8, 32), (33, 8, 32), (1, 16, 32), (1, 16, 1), (1, 16, 3),
                 (1, 32, 1), (1, 32, 3)]
# every shape the earlier per-kernel, wgmma and full-size convolution tests checked
LEGACY_CASES = [(3, 16, 1), (2, 32, 3), (5, 16, 32), (4, 8, 32), (7, 4, 32), (3, 4, 32), (2, 32, 1), (1, 16, 3),
                (170, 16, 32), (301, 8, 32), (1201, 4, 32), (40, 32, 1), (40, 32, 3), (100, 32, 1), (330, 32, 1),
                (300, 16, 3), (64, 16, 32), (33, 32, 3),
                (5, 32, 1), (333, 32, 1), (150, 32, 3), (77, 16, 1), (200, 16, 3),
                (16, 16, 32), (9, 8, 32), (40, 4, 32), (200, 16, 32), (330, 16, 32), (700, 8, 32),
                (4, 16, 3), (4, 8, 32),
                (37, 4, 32), (33, 8, 32), (170, 16, 32), (600, 16, 32), (96, 8, 32), (64, 8, 32)]
LEGACY_CASES += [(B, H, 32) for B in (1024, 512, 256) for H in (16, 8, 4)]
LEGACY_CASES += [(1024, 32, 1), (1024, 16, 32), (1024, 8, 32), (1024, 4, 32), (512, 32, 3), (256, 32, 3),
                 (512, 16, 32), (256, 16, 32)]
LEGACY_RUN = [c for c in dict.fromkeys(LEGACY_CASES) if c not in NETWORK_CASES + TILE_CASES + PARTIAL_CASES]
# the input regimes on one case of each path: tc lo 4 (TB = 8, partial), lo 8 (TB = 2, partial), lo 16 (TB = 1);
# image kernels CH = 3 at lo 16 and CH = 1 at lo 32
REGIME_CASES = [(9, 4, 32), (33, 8, 32), (20, 16, 32), (7, 16, 3), (5, 32, 1)]
REGIMES = ("randn", "spread", "dead", "cancel", "contrast")
# the largest batches the shape guard accepts, as a periodic batch of P distinct images
LARGEST_CASES = [(max_batch(16), 16, 32), (max_batch(32), 32, 3)]
PERIOD = 7

# epilogues the training nodes use (ops.EncoderFn, ops.DecoderFn): (name, bias, act, mask, mask words, bits out, colsum)
DOWN_EPILOGUES = [("bias+relu+bits", True, ACT_RELU, False, False, True, False),
                  ("mask", False, ACT_NONE, True, False, False, False),
                  ("mask+words", False, ACT_NONE, True, True, False, False),
                  ("mask+words+colsum", False, ACT_NONE, True, True, False, True)]
UP_EPILOGUES = {32: [("bias+relu+bits", True, ACT_RELU, False, False, True),
                     ("mask", False, ACT_NONE, True, False, False),
                     ("mask+words", False, ACT_NONE, True, True, False)],
                1: [("bias+sigmoid", True, ACT_SIGMOID, False, False, False),
                    ("bias", True, ACT_NONE, False, False, False),
                    ("plain", False, ACT_NONE, False, False, False)]}
UP_EPILOGUES[3] = UP_EPILOGUES[1]


def _id(c):
    return "B%d-lo%d-ch%d" % tuple(c[:3])


def path_tags(B, H, CH):
    """The regimes a case exercises (see test_case_lists_cover_every_regime)."""
    if CH == 32:
        d, u = tc_down_plan(B, H), halo_up_plan(B, H)
        S, tiles, _ = wgrad_plan(B, H, CH)
        tags = {"tc.down.tiles=%d" % d["tiles"], "tc.wgrad.S=%d" % S, "tc.up.TB=%d" % u["TB"]}
        if d["TB"] > 1 and B % d["TB"]:
            tags.add("tc.partial-multi-image")
        if B * H * H % 128:
            tags.add("tc.partial-tile")
        return tags
    return {"img.down.tiles=%d" % img_down_plan(B, H)["tiles"], "img.ch%d.lo%d" % (CH, H),
            "img.wgrad.S=%d.ch%d" % (wgrad_plan(B, H, CH)[0], CH)}


# ---------------------------------------------------------------------------------------------------------------------
# inputs and fp64 references
# ---------------------------------------------------------------------------------------------------------------------
def _spread(shape, g):
    """Magnitudes 10^U(-4, 4), random signs: both ends of the hi/lo split."""
    mag = torch.pow(10.0, torch.rand(shape, generator=g, dtype=torch.float64) * 8 - 4)
    sign = torch.where(torch.rand(shape, generator=g) < 0.5, -1.0, 1.0).double()
    return (mag * sign).float()


def _alt(n):
    return 1.0 - 2.0 * (torch.arange(n) % 2).float()


def make_mask(shape, g):
    """Post-activation stand-in: exact 0.0 and -0.0 every few elements, negatives, positives."""
    m = torch.randn(shape, generator=g)
    flat = m.view(-1)
    idx = torch.arange(flat.numel())
    flat[idx % 5 == 2] = 0.0
    flat[idx % 5 == 4] = -0.0
    return m


def make_inputs(B, H, CH, regime, seed=0):
    """Logical NCHW fp32 tensors: hi [B, CH, 2H, 2H], lo [B, 32, H, H], w [32, CH, 4, 4], b32 [32], bch [CH]."""
    g = torch.Generator().manual_seed(seed + B * 1000003 + H * 1009 + CH)
    hi = torch.randn(B, CH, 2 * H, 2 * H, generator=g)
    lo = torch.randn(B, 32, H, H, generator=g)
    w = torch.randn(32, CH, 4, 4, generator=g) / math.sqrt(16 * CH)
    b32, bch = torch.randn(32, generator=g), torch.randn(CH, generator=g)
    if regime == "spread":
        hi, lo, w = _spread(hi.shape, g), _spread(lo.shape, g), _spread(w.shape, g)
        b32, bch = _spread((32,), g), _spread((CH,), g)
    elif regime == "dead":                  # whole pixels exactly 0 (every channel), as behind a ReLU
        hi.view(B, CH, -1)[:, :, torch.arange(4 * H * H) % 5 == 1] = 0.0
        lo.view(B, 32, -1)[:, :, torch.arange(H * H) % 3 == 1] = 0.0
    elif regime == "cancel":                # 10^3 +- 1, signs alternating along every reduction
        hi = 1000.0 + torch.randn(hi.shape, generator=g)
        lo = (1000.0 + torch.randn(lo.shape, generator=g)) * _alt(H).view(1, 1, 1, H)
        w = ((1000.0 + torch.randn(w.shape, generator=g)) * _alt(32).view(32, 1, 1, 1) * _alt(CH).view(1, CH, 1, 1)
             * _alt(4).view(1, 1, 1, 4))
    elif regime == "contrast":              # neighbouring images 1e8 apart
        s = torch.where(torch.arange(B) % 2 == 0, 1e4, 1e-4).float()
        hi, lo = hi * s.view(B, 1, 1, 1), lo * s.view(B, 1, 1, 1)
    else:
        assert regime == "randn", regime
    return dict(hi=hi, lo=lo, w=w, b32=b32, bch=bch)


def nhwc(t):
    return t.permute(0, 2, 3, 1)


def hi_layout(t, CH):
    """Logical NCHW hi -> the kernel's layout (NHWC for CH = 32)."""
    return nhwc(t) if CH == 32 else t


def ref_act(pre, act):
    if act == ACT_RELU:
        return torch.relu(pre)
    if act == ACT_SIGMOID:
        return torch.sigmoid(pre)
    return pre


class Reference:
    """fp64 results of one case in the kernels' layouts (down: lo NHWC; up: hi layout; dw [32][CH][4][4]) and the
    sums of |terms| that bound their errors."""

    def __init__(self, inp, CH, dev="cpu"):
        hi, lo, w = (inp[k].to(dev).double() for k in ("hi", "lo", "w"))
        self.CH = CH
        self.down = nhwc(F.conv2d(hi, w, stride=2, padding=1))
        self.down_t = nhwc(F.conv2d(hi.abs(), w.abs(), stride=2, padding=1))
        self.up = hi_layout(F.conv_transpose2d(lo, w, stride=2, padding=1), CH)
        self.up_t = hi_layout(F.conv_transpose2d(lo.abs(), w.abs(), stride=2, padding=1), CH)
        self.b32, self.bch = inp["b32"].to(dev).double(), inp["bch"].to(dev).double()
        self._hi, self._lo = hi, lo

    def down_out(self, bias, act, mask):
        pre, terms = self.down, self.down_t
        if bias:
            pre, terms = pre + self.b32, terms + self.b32.abs()
        out = ref_act(pre, act)
        if mask is not None:
            keep = (mask.to(out.device) > 0).double()
            out, terms = out * keep, terms * keep
        return out, terms

    def up_out(self, bias, act, mask):
        pre, terms = self.up, self.up_t
        if bias:
            b = self.bch.view(1, -1, 1, 1) if self.CH != 32 else self.bch
            pre, terms = pre + b, terms + b.abs()
        out = ref_act(pre, act)
        if mask is not None:
            keep = (mask.to(out.device) > 0).double()
            out, terms = out * keep, terms * keep
        return out, terms

    def wgrad(self, lo=None):
        """dw, |dw| terms, db, |db| terms for lo (default: the case's lo), hi = the case's hi."""
        lo = self._lo if lo is None else lo.to(self._lo.device).double()
        shape = (32, self.CH, 4, 4)
        dw = torch.nn.grad.conv2d_weight(self._hi, shape, lo, stride=2, padding=1)
        dw_t = torch.nn.grad.conv2d_weight(self._hi.abs(), shape, lo.abs(), stride=2, padding=1)
        return dw, dw_t, lo.sum((0, 2, 3)), lo.abs().sum((0, 2, 3))


def bound_ratio(got, ref, terms, tau):
    """Per element |got - ref| / (tau * terms + EPI * |ref|), fp64 on ref's device; NaN in `got` counts as infinite,
    and an element whose bound is 0 must be exact."""
    got = got.to(ref.device).double()
    err = (got - ref).abs()
    lim = tau * terms + EPI * ref.abs()
    r = torch.where(err == 0, 0.0, err / lim)
    return torch.where(torch.isnan(got), math.inf, r)


def check(got, ref, terms, tau, tag, whole=None):
    """Asserts the element-wise bound (and the whole-tensor one when `whole` is a tolerance);
    -> worst |got - ref| / (tau * terms + EPI |ref|)."""
    got = got.reshape(ref.shape)
    assert torch.isfinite(ref).all(), tag
    r = bound_ratio(got, ref, terms, tau)
    worst = r.max().item()
    if worst > 1:
        i = int(r.argmax())
        at = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), r.shape))
        raise AssertionError("%s: element %s got %r, fp64 %r, |terms| %.3e: %.2f x the bound"
                             % (tag, at, got.reshape(-1)[i].item(), ref.reshape(-1)[i].item(),
                                terms.reshape(-1)[i].item(), worst))
    if whole is not None and ref.numel() >= 32:
        e = ((got.to(ref.device).double() - ref).abs().max() / ref.abs().max().clamp_min(1e-300)).item()
        assert e <= whole, "%s: max err %.3e of max |ref| > %.1e" % (tag, e, whole)
    return worst


def words(t):
    """[t > 0] of a [..., 32] tensor as one int32 word per pixel (bit c = channel c)."""
    w = ((t > 0).to(torch.int64) << torch.arange(32, device=t.device)).sum(-1)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


def _tf32(t):
    """fp32 -> nearest tf32, ties away from zero (tf32_round in csrc/dv_ptx.cuh)."""
    bits = t.float().contiguous().view(torch.int32)
    return ((bits + 0x1000) & ~0x1FFF).view(torch.float32)


def packed_ref(w, CH):
    """The packed layout conv_pack_multi_kernel writes, restated: CH in {1, 3}: [tap * CH + c][cl] twice; CH = 32: the
    down section [tap][32 hi | 32 lo rows of cl][c], then the up section [tap][32 hi | 32 lo rows of c][cl]."""
    wt = w.float().reshape(32, CH, 16)
    if CH != 32:
        sec = wt.permute(2, 1, 0).reshape(-1)
        return torch.cat([sec, sec])
    hi = _tf32(wt)
    lo = _tf32(wt - hi)
    down = torch.cat([hi.permute(2, 0, 1), lo.permute(2, 0, 1)], 1)
    up = torch.cat([hi.permute(2, 1, 0), lo.permute(2, 1, 0)], 1)
    return torch.cat([down.reshape(-1), up.reshape(-1)])


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the bound has teeth
# ---------------------------------------------------------------------------------------------------------------------
def _caught(wrong, ref, terms, tau):
    return bound_ratio(wrong, ref, terms, tau).max().item() > 1


TEETH_CASES = [(3, 4, 32), (3, 8, 32), (2, 16, 32), (2, 16, 3), (2, 32, 1)]


@pytest.mark.parametrize("B,H,CH", TEETH_CASES, ids=[_id(c) for c in TEETH_CASES])
def test_bound_catches_wrong_convolutions(B, H, CH):
    """fp32 CPU simulations of the faults a kernel can have, at case shapes: each breaks the bound somewhere, while the
    exact result rounded to fp32 and an fp32 CPU convolution pass."""
    inp = make_inputs(B, H, CH, "randn")
    ref = Reference(inp, CH)
    hi, lo, w = inp["hi"], inp["lo"], inp["w"]
    td, tu = tau_down(CH), tau_up(CH)
    down, down_t = ref.down_out(True, ACT_NONE, None)
    up, up_t = ref.up_out(True, ACT_NONE, None)
    check(down.float(), down, down_t, td, "fp32 rounding of down")
    check(up.float(), up, up_t, tu, "fp32 rounding of up")
    check(nhwc(F.conv2d(hi, w, inp["b32"], stride=2, padding=1)), down, down_t, td, "fp32 down")
    check(hi_layout(F.conv_transpose2d(lo, w, inp["bch"], stride=2, padding=1), CH), up, up_t, tu, "fp32 up")

    # a dropped border tap: the left padding column read as the image's first column
    hp = F.pad(hi, (1, 1, 1, 1))
    hp[..., 0] = hp[..., 1]
    wrong = nhwc(F.conv2d(hp, w, inp["b32"], stride=2))
    assert _caught(wrong, down, down_t, td)
    # a halo row from the neighbouring image: the row above each image (but the first) is the last row of the one
    # before it, as a multi-image tile would read it without the image boundary
    hp = F.pad(hi, (1, 1, 1, 1))
    hp[1:, :, 0, 1:-1] = hi[:-1, :, -1]
    assert _caught(nhwc(F.conv2d(hp, w, inp["b32"], stride=2)), down, down_t, td)
    ext = torch.cat([torch.zeros_like(lo[:, :, :1]), lo], 2)
    ext[1:, :, 0] = lo[:-1, :, -1]
    wrong = hi_layout(F.conv_transpose2d(ext, w, inp["bch"], stride=2, padding=1)[:, :, 2:], CH)
    assert _caught(wrong, up, up_t, tu)
    # a dropped last partial tile (down: the last 128 pixels, or the tail past the last whole tile)
    total = B * H * H
    tail = total % 128 or min(128, total)
    wrong = down.reshape(-1, 32).clone()
    wrong[total - tail:] = 0
    assert _caught(wrong.view(down.shape), down, down_t, td)
    # single-pass TF32: the operands rounded to tf32, products and sums exact
    if CH == 32:
        single = nhwc(F.conv2d(_tf32(hi).double(), _tf32(w).double(), inp["b32"].double(), stride=2, padding=1))
        assert _caught(single, down, down_t, td)
        single = nhwc(F.conv_transpose2d(_tf32(lo).double(), _tf32(w).double(), inp["bch"].double(), stride=2,
                                         padding=1))
        assert _caught(single, up, up_t, tu)
    # a missing bias on one channel
    wrong = down.clone()
    wrong[..., 5] -= inp["b32"][5].double()
    assert _caught(wrong, down, down_t, td)
    wrong = up.clone()
    if CH == 32:
        wrong[..., 2] -= inp["bch"][2].double()
    else:
        wrong[:, CH - 1] -= inp["bch"][CH - 1].double()
    assert _caught(wrong, up, up_t, tu)


def test_bound_catches_a_mask_taken_at_zero():
    """Where the mask is exactly 0.0 or -0.0 the output is exactly 0; `mask >= 0` keeps the value there."""
    B, H, CH = 3, 8, 32
    inp = make_inputs(B, H, CH, "randn")
    ref = Reference(inp, CH)
    mask = make_mask((B, H, H, 32), torch.Generator().manual_seed(1))
    assert (mask == 0).any() and (torch.signbit(mask) & (mask == 0)).any() and (mask < 0).any()
    want, terms = ref.down_out(False, ACT_NONE, mask)
    wrong = ref.down * (mask >= 0).double()
    assert _caught(wrong, want, terms, tau_down(CH))


# (B, H, CH): small (64 to 4096 pixels per reduction) and medium (16K to 64K) pixel counts of both weight-gradient paths
WGRAD_TEETH_CASES = [(1, 8, 32), (16, 16, 32), (64, 16, 32), (2, 32, 3), (16, 32, 1)]


@pytest.mark.parametrize("B,H,CH", WGRAD_TEETH_CASES, ids=[_id(c) for c in WGRAD_TEETH_CASES])
def test_bound_catches_wrong_weight_gradients(B, H, CH):
    """A dropped last tile (dw and dbias), a dropped border tap, and on the tensor cores single-pass TF32, break the
    weight-gradient bound.  The bound grows with the chain of partial sums while a random per-product error averages
    out against sum|terms|: single-pass TF32 is caught at these pixel counts (up to 64K per reduction), not at a
    million pixels, where the element-wise bound is carried by the other checks."""
    inp = make_inputs(B, H, CH, "randn")
    ref = Reference(inp, CH)
    hi, lo = inp["hi"].double(), inp["lo"].double()
    dw, dw_t, db, db_t = ref.wgrad()
    t_dw, t_db = tau_wgrad(B, H, CH)
    check(dw.float(), dw, dw_t, t_dw, "fp32 rounding of dw")
    check(torch.nn.grad.conv2d_weight(inp["hi"], dw.shape, inp["lo"], stride=2, padding=1), dw, dw_t, t_dw, "fp32 dw")
    # the last tile: 128 pixels (tc), 16 lo rows of the last image (img)
    if CH == 32:
        flat = nhwc(lo).reshape(-1, 32).clone()
        n = flat.shape[0]
        flat[n - (n % 128 or min(128, n)):] = 0
        lo_cut = flat.view(B, H, H, 32).permute(0, 3, 1, 2)
    else:
        lo_cut = lo.clone()
        lo_cut[-1, :, -16:] = 0
    dw_cut = torch.nn.grad.conv2d_weight(hi, dw.shape, lo_cut, stride=2, padding=1)
    assert _caught(dw_cut, dw, dw_t, t_dw)
    assert _caught(lo_cut.sum((0, 2, 3)), db, db_t, t_db)
    # a dropped border tap: the top padding row read as the image's first row
    hp = F.pad(hi, (1, 1, 1, 1))
    hp[:, :, 0] = hp[:, :, 1]
    dw_pad = torch.nn.grad.conv2d_weight(hp, dw.shape, lo, stride=2, padding=0)
    assert _caught(dw_pad, dw, dw_t, t_dw)
    if CH == 32:
        single = torch.nn.grad.conv2d_weight(_tf32(inp["hi"]).double(), dw.shape, _tf32(inp["lo"]).double(),
                                             stride=2, padding=1)
        assert _caught(single, dw, dw_t, t_dw)


def test_bound_catches_a_wrong_channel_sum():
    """The channel sums with one image's outputs left out, or with one channel's bias missing, break their bound."""
    B, H, CH = 33, 8, 32
    inp = make_inputs(B, H, CH, "randn")
    ref = Reference(inp, CH)
    mask = make_mask((B, H, H, 32), torch.Generator().manual_seed(2))
    out, terms = ref.down_out(False, ACT_NONE, mask)
    cs, cs_t = out.sum((0, 1, 2)), terms.sum((0, 1, 2))
    tau = tau_down(CH) + tau_colsum(B, H, CH)
    check(cs.float(), cs, cs_t, tau, "fp32 rounding of the channel sums")
    assert _caught(out[:-1].sum((0, 1, 2)), cs, cs_t, tau)


def test_case_lists_cover_every_regime():
    """Every network geometry, both sides of one and two CTA waves on every kernel, partial multi-image tiles, every
    earlier shape and the largest batches are in the lists, with the plans their comments name."""
    for B in (64, 256, 512, 1024):
        for c in [(B, 16, 1), (B, 16, 3), (B, 32, 1), (B, 32, 3), (B, 16, 32), (B, 8, 32), (B, 4, 32)]:
            assert c in NETWORK_CASES, c
    run = NETWORK_CASES + TILE_CASES + PARTIAL_CASES + LEGACY_RUN + REGIME_CASES
    assert set(LEGACY_CASES) <= set(run)
    seen = set()
    for c in run:
        seen |= path_tags(*c)
    for t in (1, 131, 132, 133, 264, 265):
        assert "tc.down.tiles=%d" % t in seen, t
    assert {"tc.wgrad.S=67", "tc.wgrad.S=89", "tc.wgrad.S=132", "tc.partial-multi-image", "tc.partial-tile",
            "tc.up.TB=8", "tc.up.TB=2", "tc.up.TB=1"} <= seen
    for t in (263, 264, 265, 266):
        assert "img.down.tiles=%d" % t in seen, t
    for CH in (1, 3):
        for H in (16, 32):
            assert "img.ch%d.lo%d" % (CH, H) in seen
    assert {"img.wgrad.S=264.ch1", "img.wgrad.S=132.ch3", "img.wgrad.S=1.ch1", "img.wgrad.S=1.ch3"} <= seen
    # the plans the comments name
    assert [tc_down_plan(B, 8)["tiles"] for B in (1, 261, 264, 265, 528, 529)] == [1, 131, 132, 133, 264, 265]
    assert wgrad_plan(265, 8, 32)[0] == 67 and wgrad_plan(529, 8, 32)[0] == 89
    assert (tc_down_plan(9, 4)["TB"], tc_down_plan(9, 8)["TB"], tc_down_plan(9, 16)["TB"]) == (8, 2, 1)
    assert (halo_up_plan(9, 4)["TB"], halo_up_plan(9, 8)["TB"], halo_up_plan(9, 16)["TB"]) == (8, 2, 1)
    assert halo_up_plan(9, 16)["tiles_per_img"] == 2 and halo_up_plan(9, 4)["tiles"] == 2
    assert (up_tile_rows(32), up_tile_rows(16)) == (16, 32)
    assert {B % 8 for B, H, CH in PARTIAL_CASES if H == 4} >= {1, 7}
    assert any(H == 8 and B % 2 for B, H, CH in PARTIAL_CASES)
    assert LARGEST_CASES == [(65535, 16, 32), (16383, 32, 3)]


def test_workspace_queries_match_the_restated_plans():
    """dv_conv_wgrad_workspace_bytes and dv_conv_packed_floats give what the plans restate for every case (the
    queries run on the host); one image past the largest batch, and shapes outside the layers, query 0."""
    from disvae import _native as N
    L = N.lib()
    for B, H, CH in NETWORK_CASES + TILE_CASES + PARTIAL_CASES + LEGACY_RUN + REGIME_CASES + LARGEST_CASES:
        assert L.dv_conv_wgrad_workspace_bytes(B, H, H, CH) == wgrad_ws_bytes(B, H, CH), (B, H, CH)
    for B, H, CH in LARGEST_CASES:
        assert L.dv_conv_wgrad_workspace_bytes(B + 1, H, H, CH) == 0
    for B, H, W, CH in [(2, 8, 8, 3), (2, 64, 64, 1), (2, 32, 32, 32), (2, 8, 16, 32), (2, 32, 16, 3), (0, 8, 8, 32),
                        (2, 8, 8, 2)]:
        assert L.dv_conv_wgrad_workspace_bytes(B, H, W, CH) == 0
    for CH in (1, 3, 32):
        assert L.dv_conv_packed_floats(CH) == packed_floats(CH)


# ---------------------------------------------------------------------------------------------------------------------
# device buffers
# ---------------------------------------------------------------------------------------------------------------------
def _bits(t):
    return t.contiguous().view(torch.int32)


def _input(t):
    """Device copy of `t` (fp32 or int32 words) 16 bytes into a NaN-filled allocation, with GUARD NaN after it."""
    t = t.reshape(-1)
    if t.dtype == torch.int32:
        t = t.view(torch.float32)
    n = t.numel()
    buf = torch.full((OFF + n + GUARD,), float("nan"), device="cuda")
    buf[OFF:OFF + n] = t.to("cuda", non_blocking=False)
    return buf


def _output(n, fill=float("nan")):
    """n words of `fill` 16 bytes into an allocation, sentinel words before and after."""
    buf = torch.full((OFF + n + GUARD,), fill, device="cuda")
    _bits(buf)[:OFF] = SENTINEL
    _bits(buf)[OFF + n:] = SENTINEL
    return buf


def _addr(buf, shift=0):
    return None if buf is None else buf.data_ptr() + 4 * OFF + shift


def _intact(buf, n):
    b = _bits(buf)
    return bool((b[:OFF] == SENTINEL).all()) and bool((b[OFF + n:] == SENTINEL).all())


def _body(buf, n, shape=None):
    t = buf[OFF:OFF + n]
    return t if shape is None else t.view(shape)


def _native():
    from disvae import _native as N
    return N


# ---------------------------------------------------------------------------------------------------------------------
# one layer through every entry point
# ---------------------------------------------------------------------------------------------------------------------
class ConvCase:
    def __init__(self, B, H, CH, regime="randn", seed=0):
        self.B, self.H, self.CH, self.regime = B, H, CH, regime
        self.nchw = int(CH != 32)
        self.cpu = make_inputs(B, H, CH, regime, seed)
        self.ref = Reference(self.cpu, CH, "cuda")
        g = torch.Generator().manual_seed(seed + 77)
        self.mask_lo = make_mask((B, H, H, 32), g)
        self.mask_hi = make_mask((B, 2 * H, 2 * H, 32), g) if CH == 32 else None
        self.n_lo, self.n_hi = B * H * H * 32, B * CH * 4 * H * H
        self.dev = dict(hi=_input(hi_layout(self.cpu["hi"], CH).contiguous()),
                        lo=_input(nhwc(self.cpu["lo"]).contiguous()), w=_input(self.cpu["w"]),
                        b32=_input(self.cpu["b32"]), bch=_input(self.cpu["bch"]), mask_lo=_input(self.mask_lo),
                        words_lo=_input(words(self.mask_lo)))
        if CH == 32:
            self.dev.update(mask_hi=_input(self.mask_hi), words_hi=_input(words(self.mask_hi)))
        self.whole = regime != "cancel"
        self.L, self.st = _native().lib(), _native().stream()
        self.tag = "%s %s" % (_id((B, H, CH)), regime)

    def p(self, name):
        return _addr(self.dev[name])

    def _launch(self, fn, *args, launches):
        before = self.L.dv_launch_count()
        rc = fn(*args)
        assert rc == DV_OK, "%s: %s returned %d" % (self.tag, fn.__name__, rc)
        torch.cuda.synchronize()
        got = self.L.dv_launch_count() - before
        assert got == launches, "%s: %s launched %d kernels, expected %d" % (self.tag, fn.__name__, got, launches)

    def pack(self):
        """dv_conv_pack_multi of this w alone -> guarded packed buffer, checked against the restated layout."""
        pf = packed_floats(self.CH)
        pk = _output(pf)
        self._launch(self.L.dv_conv_pack_multi, 1, (ctypes.c_void_p * 1)(self.p("w")),
                     (ctypes.c_void_p * 1)(_addr(pk)), (ctypes.c_int * 1)(self.CH), self.st, launches=1)
        assert _intact(pk, pf), self.tag + ": pack wrote outside its buffer"
        assert torch.equal(_bits(_body(pk, pf)), _bits(packed_ref(self.cpu["w"], self.CH).cuda())), \
            self.tag + ": packed layout differs from the restatement"
        return pk

    def down(self, pk):
        B, H, CH = self.B, self.H, self.CH
        n_out, n_px = self.n_lo, B * H * H
        tau = tau_down(CH)
        worst, results = 0.0, {}
        cs_ws_n = self.L.dv_channel_sum_workspace_bytes() // 4
        for name, bias, act, masked, use_words, bits, colsum in DOWN_EPILOGUES:
            tag = "%s down %s" % (self.tag, name)
            runs = []
            for rep in range(2):
                out, bo = _output(n_out), _output(n_px) if bits else None
                cs, ws = (_output(32), _output(cs_ws_n)) if colsum else (None, None)
                self._launch(self.L.dv_conv_down, self.p("hi"), _addr(pk), self.p("b32") if bias else None,
                             self.p("mask_lo") if masked else None, _addr(out), B, H, H, CH, self.nchw, act,
                             _addr(cs), _addr(ws), self.p("words_lo") if use_words else None, _addr(bo), self.st,
                             launches=2 if colsum else 1)
                assert _intact(out, n_out), tag + ": wrote past the output"
                assert bo is None or _intact(bo, n_px), tag + ": wrote past the bit words"
                assert cs is None or (_intact(cs, 32) and _intact(ws, cs_ws_n)), tag + ": wrote past the channel sums"
                runs.append([_body(out, n_out, (B, H, H, 32)).clone(), None if bo is None else _body(bo, n_px).clone(),
                             None if cs is None else _body(cs, 32).clone()])
            for a, b in zip(runs[0], runs[1]):
                assert a is None or torch.equal(_bits(a), _bits(b)), tag + ": not deterministic"
            got, bo, cs = runs[0]
            results[name] = got
            if bo is not None:
                assert torch.equal(_bits(bo), words(got).view(-1)), tag + ": relu_bits_out is not [out > 0]"
            ref, terms = self.ref.down_out(bias, act, self.mask_lo if masked else None)
            worst = max(worst, check(got, ref, terms, tau, tag, WHOLE_TOL if self.whole else None))
            if cs is not None:
                cref, cterms = ref.sum((0, 1, 2)), terms.sum((0, 1, 2))
                worst = max(worst, check(cs, cref, cterms, tau + tau_colsum(B, H, CH), tag + " colsum",
                                         WHOLE_TOL_SUMS[CH] if self.whole else None))
        for name in ("mask+words", "mask+words+colsum"):
            assert torch.equal(_bits(results[name]), _bits(results["mask"])), \
                "%s down: %s differs from the float mask" % (self.tag, name)
        return worst

    def up(self, pk):
        B, H, CH = self.B, self.H, self.CH
        n_out, n_px = self.n_hi, B * 4 * H * H
        shape = (B, 2 * H, 2 * H, 32) if CH == 32 else (B, CH, 2 * H, 2 * H)
        tau = tau_up(CH)
        worst, results = 0.0, {}
        for name, bias, act, masked, use_words, bits in UP_EPILOGUES[CH]:
            tag = "%s up %s" % (self.tag, name)
            runs = []
            for rep in range(2):
                out, bo = _output(n_out), _output(n_px) if bits else None
                self._launch(self.L.dv_conv_up, self.p("lo"), _addr(pk), self.p("bch") if bias else None,
                             self.p("mask_hi") if masked else None, _addr(out), B, H, H, CH, self.nchw, act,
                             self.p("words_hi") if use_words else None, _addr(bo), self.st, launches=1)
                assert _intact(out, n_out), tag + ": wrote past the output"
                assert bo is None or _intact(bo, n_px), tag + ": wrote past the bit words"
                runs.append([_body(out, n_out, shape).clone(), None if bo is None else _body(bo, n_px).clone()])
            for a, b in zip(runs[0], runs[1]):
                assert a is None or torch.equal(_bits(a), _bits(b)), tag + ": not deterministic"
            got, bo = runs[0]
            results[name] = got
            if bo is not None:
                assert torch.equal(_bits(bo), words(got).view(-1)), tag + ": relu_bits_out is not [out > 0]"
            ref, terms = self.ref.up_out(bias, act, self.mask_hi if masked else None)
            whole = WHOLE_TOL if self.whole and act != ACT_SIGMOID else None
            worst = max(worst, check(got, ref, terms, tau, tag, whole))
        if CH == 32:
            assert torch.equal(_bits(results["mask+words"]), _bits(results["mask"])), \
                self.tag + " up: the mask words differ from the float mask"
        return worst

    def wgrad(self):
        """Both roles: the encoder's (lo = output gradient, hi = the layer's input) with and without dbias_lo, and the
        decoder's (lo = the ConvTranspose2d input, a ReLU output; hi = its output gradient)."""
        B, H, CH = self.B, self.H, self.CH
        S = wgrad_plan(B, H, CH)[0]
        nbytes = self.L.dv_conv_wgrad_workspace_bytes(B, H, H, CH)
        assert nbytes == wgrad_ws_bytes(B, H, CH), "%s: workspace %d, plan %d" % (self.tag, nbytes, wgrad_ws_bytes(B, H, CH))
        t_dw, t_db = tau_wgrad(B, H, CH)
        n_dw = 32 * CH * 16
        lo_dec = torch.relu(self.cpu["lo"])
        roles = {"enc": self.dev["lo"], "dec": _input(nhwc(lo_dec).contiguous())}
        worst = 0.0
        for role, lo_buf in roles.items():
            dw_ref, dw_t, db_ref, db_t = self.ref.wgrad(None if role == "enc" else lo_dec)
            runs = {}
            for with_db in (True, False):
                tag = "%s wgrad[S=%d] %s dbias %d" % (self.tag, S, role, with_db)
                for rep in range(2):
                    dw, db, ws = _output(n_dw), _output(32) if with_db else None, _output(nbytes // 4)
                    self._launch(self.L.dv_conv_wgrad, _addr(lo_buf), self.p("hi"), _addr(dw), _addr(db), _addr(ws),
                                 nbytes, B, H, H, CH, self.nchw, self.st, launches=2)
                    assert _intact(dw, n_dw) and _intact(ws, nbytes // 4), tag + ": wrote out of bounds"
                    assert db is None or _intact(db, 32), tag + ": wrote past dbias"
                    runs[with_db, rep] = (_body(dw, n_dw, (32, CH, 4, 4)).clone(),
                                          None if db is None else _body(db, 32).clone())
            tag = "%s wgrad[S=%d] %s" % (self.tag, S, role)
            for key, (dw, db) in runs.items():
                assert torch.equal(_bits(dw), _bits(runs[True, 0][0])), "%s: dw differs (dbias %d, run %d)" % ((tag,) + key)
            assert torch.equal(_bits(runs[True, 1][1]), _bits(runs[True, 0][1])), tag + ": dbias not deterministic"
            whole = WHOLE_TOL_SUMS[CH] if self.whole else None
            worst = max(worst, check(runs[True, 0][0], dw_ref, dw_t, t_dw, tag + " dw", whole))
            worst = max(worst, check(runs[True, 0][1], db_ref, db_t, t_db, tag + " dbias", whole))
        return worst

    def run(self):
        pk = self.pack()
        e_d, e_u, e_w = self.down(pk), self.up(pk), self.wgrad()
        path = "tc" if self.CH == 32 else "img"
        print("%s: down[%s] %.3f, up[%s] %.3f, wgrad[%s S=%d] %.3f of the bound"
              % (self.tag, path, e_d, path, e_u, path, wgrad_plan(self.B, self.H, self.CH)[0], e_w))


@pytest.mark.gpu
def test_gpu_fp64_reference_matches_the_cpu_one():
    """The fp64 references are computed on the GPU; on small shapes of every geometry they agree with the CPU ones to
    fp64 rounding."""
    for B, H, CH in [(3, 4, 32), (2, 8, 32), (2, 16, 32), (2, 16, 3), (2, 32, 1)]:
        inp = make_inputs(B, H, CH, "spread")
        c, g = Reference(inp, CH, "cpu"), Reference(inp, CH, "cuda")
        pairs = [(c.down, g.down, c.down_t), (c.up, g.up, c.up_t)]
        cw, gw = c.wgrad(), g.wgrad()
        pairs += [(cw[0], gw[0], cw[1]), (cw[2], gw[2], cw[3])]
        for a, b, t in pairs:
            assert ((b.cpu() - a).abs() <= 1e-12 * t).all(), (B, H, CH)


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,CH", NETWORK_CASES, ids=[_id(c) for c in NETWORK_CASES])
def test_network_layers(B, H, CH):
    """Every conv layer of the encoder and decoder on 32x32 and 64x64 images with 1 or 3 channels, B in
    {64, 256, 512, 1024}."""
    ConvCase(B, H, CH).run()


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,CH", TILE_CASES + PARTIAL_CASES, ids=[_id(c) for c in TILE_CASES + PARTIAL_CASES])
def test_tile_waves_and_partial_tiles(B, H, CH):
    ConvCase(B, H, CH).run()


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,CH", LEGACY_RUN, ids=[_id(c) for c in LEGACY_RUN])
def test_earlier_conv_shapes(B, H, CH):
    ConvCase(B, H, CH).run()


@pytest.mark.gpu
@pytest.mark.parametrize("regime", REGIMES[1:])
@pytest.mark.parametrize("B,H,CH", REGIME_CASES, ids=[_id(c) for c in REGIME_CASES])
def test_input_regimes(B, H, CH, regime):
    """Magnitudes over 10^+-4, dead pixels, 10^3 +- 1 with alternating signs, and neighbouring images 1e8 apart (a
    halo or padding row leaking across an image or tile edge breaks the bound of the small image)."""
    ConvCase(B, H, CH, regime).run()


@pytest.mark.gpu
def test_pack_multi_equals_per_layer_packs():
    """One table of 11 layers (> 8: two launches) writes the buffers dv_conv_pack_weights writes, layer by layer."""
    L, st = _native().lib(), _native().stream()
    chans = [1, 32, 32, 32, 3, 32, 32, 32, 32, 3, 1]
    g = torch.Generator().manual_seed(9)
    ws = [_input(torch.randn(32, ch, 4, 4, generator=g)) for ch in chans]
    packs = [_output(packed_floats(ch)) for ch in chans]
    n = len(chans)
    arr_p = ctypes.c_void_p * n
    before = L.dv_launch_count()
    rc = L.dv_conv_pack_multi(n, arr_p(*[_addr(w) for w in ws]), arr_p(*[_addr(p) for p in packs]),
                              (ctypes.c_int * n)(*chans), st)
    torch.cuda.synchronize()
    assert rc == DV_OK and L.dv_launch_count() - before == _cdiv(n, 8)
    for w, pk, ch in zip(ws, packs, chans):
        pf = packed_floats(ch)
        single = _output(pf)
        before = L.dv_launch_count()
        assert L.dv_conv_pack_weights(_addr(w), _addr(single), ch, st) == DV_OK
        torch.cuda.synchronize()
        assert L.dv_launch_count() - before == 1
        assert _intact(pk, pf) and _intact(single, pf), ch
        assert torch.equal(_bits(_body(pk, pf)), _bits(_body(single, pf))), ch
        assert torch.equal(_bits(_body(pk, pf)), _bits(packed_ref(_body(w, 32 * ch * 16).cpu(), ch).cuda())), ch


@pytest.mark.gpu
def test_weight_gradient_beside_up_on_two_streams():
    """The Trainer runs dv_conv_wgrad on a side stream beside the main stream's dv_conv_up: run concurrently, both
    give the bits they give one after the other."""
    L = _native().lib()
    c = ConvCase(512, 8, 32)
    pk = c.pack()
    nbytes = L.dv_conv_wgrad_workspace_bytes(512, 8, 8, 32)

    def run(st_w, st_u):
        dw, db, ws, out = _output(32 * 32 * 16), _output(32), _output(nbytes // 4), _output(c.n_hi)
        torch.cuda.synchronize()
        assert L.dv_conv_wgrad(c.p("lo"), c.p("hi"), _addr(dw), _addr(db), _addr(ws), nbytes, 512, 8, 8, 32, 0,
                               st_w) == DV_OK
        assert L.dv_conv_up(c.p("lo"), _addr(pk), c.p("bch"), c.p("mask_hi"), _addr(out), 512, 8, 8, 32, 0, ACT_NONE,
                            c.p("words_hi"), None, st_u) == DV_OK
        torch.cuda.synchronize()
        return [_body(t, n).clone() for t, n in ((dw, 32 * 32 * 16), (db, 32), (out, c.n_hi))]

    main = _native().stream()
    alone = run(main, main)
    both = run(torch.cuda.Stream().cuda_stream, main)
    for a, b in zip(alone, both):
        assert torch.equal(_bits(a), _bits(b))


# ---------------------------------------------------------------------------------------------------------------------
# the largest accepted batches, as periodic batches (image b = image b mod P)
# ---------------------------------------------------------------------------------------------------------------------
def _periodic_input(base, B):
    """Guarded device buffer holding B images, image b = base[b % P] (base: [P, ...] in the kernel's layout)."""
    P = base.shape[0]
    per = base[0].numel()
    buf = torch.full((OFF + B * per + GUARD,), float("nan"), device="cuda")
    body = buf[OFF:OFF + B * per].view(B, per)
    src = base.reshape(P, per).cuda()
    step = P * max(1, (1 << 24) // (P * per))
    for s in range(0, B, step):
        e = min(B, s + step)
        body[s:e] = src[torch.arange(s, e, device="cuda") % P]
    return buf


def _digest(t):
    """Order-sensitive integer digest of a tensor's bits (two runs repeat bit for bit iff the digests agree, barring a
    collision)."""
    flat, total, step = _bits(t).reshape(-1), 0, 1 << 26
    for s in range(0, flat.numel(), step):
        b = flat[s:s + step].to(torch.int64)
        total += int((b * ((torch.arange(s, s + b.numel(), device=b.device) % 1021) + 1)).sum())
    return total


def _check_periodic(got, ref, terms, tau, B, tag, whole):
    """got [B, ...] against ref[b % P] image by image, in chunks."""
    P = ref.shape[0]
    worst, err_max = 0.0, 0.0
    step = 2048
    for s in range(0, B, step):
        idx = torch.arange(s, min(B, s + step), device="cuda") % P
        g, r, t = got[s:s + step], ref[idx], terms[idx]
        rat = bound_ratio(g, r, t, tau)
        w = rat.max().item()
        assert w <= 1, "%s: images %d..: %.2f x the bound" % (tag, s, w)
        worst = max(worst, w)
        err_max = max(err_max, (g.double() - r).abs().max().item())
    if whole is not None:
        e = err_max / ref.abs().max().item()
        assert e <= whole, "%s: max err %.3e of max |ref| > %.1e" % (tag, e, whole)
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,CH", LARGEST_CASES, ids=[_id(c) for c in LARGEST_CASES])
def test_largest_accepted_batch(B, H, CH):
    """At the largest B the int pixel-index guard accepts (lo 16 / CH 32: 65535 images, lo 32 / CH 3: 16383), down
    (bias, ReLU, bit words), up (bias, ReLU and bit words; bias and sigmoid on the image layer) and wgrad with dbias
    against fp64, every output image against its period representative and dw / dbias against the representatives
    weighted by their multiplicities.  One image more is refused."""
    P = PERIOD
    nchw = int(CH != 32)
    n_lo, n_hi, n_px_lo, n_px_hi = B * H * H * 32, B * CH * 4 * H * H, B * H * H, B * 4 * H * H
    need = 4 * (2 * n_lo + 2 * n_hi + n_px_lo + n_px_hi) + (2 << 30)
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip("needs %.1f GB of free device memory, %.1f GB free" % (need / 2 ** 30, free / 2 ** 30))
    L, st = _native().lib(), _native().stream()
    inp = make_inputs(P, H, CH, "randn", seed=5)
    ref = Reference(inp, CH, "cuda")
    hi = _periodic_input(hi_layout(inp["hi"], CH).contiguous(), B)
    lo = _periodic_input(nhwc(inp["lo"]).contiguous(), B)
    w, b32, bch = _input(inp["w"]), _input(inp["b32"]), _input(inp["bch"])
    pk = _output(packed_floats(CH))
    assert L.dv_conv_pack_weights(_addr(w), _addr(pk), CH, st) == DV_OK
    report = []

    # down: bias + ReLU + bit words
    out, bo = _output(n_lo), _output(n_px_lo)
    digests = []
    for rep in range(2):
        assert L.dv_conv_down(_addr(hi), _addr(pk), _addr(b32), None, _addr(out), B, H, H, CH, nchw, ACT_RELU, None,
                              None, None, _addr(bo), st) == DV_OK
        torch.cuda.synchronize()
        digests.append((_digest(_body(out, n_lo)), _digest(_body(bo, n_px_lo))))
    assert digests[0] == digests[1] and _intact(out, n_lo) and _intact(bo, n_px_lo)
    want, terms = ref.down_out(True, ACT_RELU, None)
    got = _body(out, n_lo, (B, H, H, 32))
    report.append(("down", _check_periodic(got, want, terms, tau_down(CH), B, "down", WHOLE_TOL)))
    for s in range(0, B, 4096):
        assert torch.equal(_bits(_body(bo, n_px_lo, (B, H, H))[s:s + 4096]), words(got[s:s + 4096])), s
    del out, bo, got

    # up: bias + ReLU + bit words (CH = 32), bias + sigmoid (image layer)
    n_bits = n_px_hi if CH == 32 else 0
    out, bo = _output(n_hi), _output(n_bits) if n_bits else None
    act = ACT_RELU if CH == 32 else ACT_SIGMOID
    digests = []
    for rep in range(2):
        assert L.dv_conv_up(_addr(lo), _addr(pk), _addr(bch), None, _addr(out), B, H, H, CH, nchw, act, None,
                            _addr(bo), st) == DV_OK
        torch.cuda.synchronize()
        digests.append(_digest(_body(out, n_hi)))
    assert digests[0] == digests[1] and _intact(out, n_hi) and (bo is None or _intact(bo, n_bits))
    want, terms = ref.up_out(True, act, None)
    got = _body(out, n_hi, (B,) + tuple(want.shape[1:]))
    report.append(("up", _check_periodic(got, want, terms, tau_up(CH), B, "up",
                                         WHOLE_TOL if act != ACT_SIGMOID else None)))
    if bo is not None:
        for s in range(0, B, 2048):
            assert torch.equal(_bits(_body(bo, n_bits, (B, 2 * H, 2 * H))[s:s + 2048]), words(got[s:s + 2048])), s
    del out, bo, got

    # wgrad with dbias: the representatives weighted by their multiplicities (exact in fp64)
    nbytes = L.dv_conv_wgrad_workspace_bytes(B, H, H, CH)
    assert nbytes == wgrad_ws_bytes(B, H, CH)
    mult = torch.tensor([B // P + (r < B % P) for r in range(P)], dtype=torch.float64, device="cuda")
    dw_ref, dw_t, db_ref, db_t = ref.wgrad(ref._lo * mult.view(P, 1, 1, 1))
    runs = []
    for rep in range(2):
        dw, db, ws = _output(32 * CH * 16), _output(32), _output(nbytes // 4)
        assert L.dv_conv_wgrad(_addr(lo), _addr(hi), _addr(dw), _addr(db), _addr(ws), nbytes, B, H, H, CH, nchw,
                               st) == DV_OK
        torch.cuda.synchronize()
        assert _intact(dw, 32 * CH * 16) and _intact(db, 32) and _intact(ws, nbytes // 4)
        runs.append((_body(dw, 32 * CH * 16, (32, CH, 4, 4)).clone(), _body(db, 32).clone()))
    assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(runs[0], runs[1]))
    t_dw, t_db = tau_wgrad(B, H, CH)
    report.append(("wgrad dw", check(runs[0][0], dw_ref, dw_t, t_dw, "wgrad dw")))
    report.append(("wgrad dbias", check(runs[0][1], db_ref, db_t, t_db, "wgrad dbias")))

    # one image more is refused before any launch
    before = L.dv_launch_count()
    assert L.dv_conv_down(_addr(hi), _addr(pk), None, None, _addr(pk), B + 1, H, H, CH, nchw, ACT_NONE, None, None,
                          None, None, st) == DV_ERR_BAD_SHAPE
    assert L.dv_conv_up(_addr(lo), _addr(pk), None, None, _addr(pk), B + 1, H, H, CH, nchw, ACT_NONE, None, None,
                        st) == DV_ERR_BAD_SHAPE
    assert L.dv_conv_wgrad(_addr(lo), _addr(hi), _addr(pk), None, _addr(pk), 1 << 40, B + 1, H, H, CH, nchw,
                           st) == DV_ERR_BAD_SHAPE
    assert L.dv_launch_count() == before and L.dv_conv_wgrad_workspace_bytes(B + 1, H, H, CH) == 0
    print("%s largest batch (period %d): %s of the bound"
          % (_id((B, H, CH)), P, ", ".join("%s %.3f" % kv for kv in report)))


# ---------------------------------------------------------------------------------------------------------------------
# refusals: status code, nothing launched, outputs untouched
# ---------------------------------------------------------------------------------------------------------------------
class Refusals:
    """Buffers for one geometry and the raw calls on them.  With no argument changed each call is a valid one; every
    test changes one thing and `expect` asserts the status, that no kernel ran and that every output and workspace
    still holds its fill."""
    FILL = 7.0

    def __init__(self, B, H, CH):
        self.B, self.H, self.CH = B, H, CH
        inp = make_inputs(B, H, CH, "randn")
        g = torch.Generator().manual_seed(3)
        m_lo, m_hi = make_mask((B, H, H, 32), g), make_mask((B, 2 * H, 2 * H, 32), g)
        self.inp = dict(hi=_input(hi_layout(inp["hi"], CH).contiguous()), lo=_input(nhwc(inp["lo"]).contiguous()),
                        wp=_input(packed_ref(inp["w"], CH)), b32=_input(inp["b32"]), bch=_input(inp["bch"]),
                        mask_lo=_input(m_lo), mask_hi=_input(m_hi), words_lo=_input(words(m_lo)),
                        words_hi=_input(words(m_hi)))
        self.L, self.st = _native().lib(), _native().stream()
        self.ws_bytes = self.L.dv_conv_wgrad_workspace_bytes(B, H, H, CH)
        self.sizes = dict(lo_out=B * H * H * 32, hi_out=B * CH * 4 * H * H, bits_lo=B * H * H, bits_hi=B * 4 * H * H,
                          cs=32, cs_ws=self.L.dv_channel_sum_workspace_bytes() // 4, dw=32 * CH * 16, db=32,
                          ws=self.ws_bytes // 4)
        self.out = {k: _output(n, self.FILL) for k, n in self.sizes.items()}

    def p(self, name, shift=0):
        return _addr(self.inp[name] if name in self.inp else self.out[name], shift)

    def expect(self, status, fn, *args):
        before = self.L.dv_launch_count()
        rc = fn(*args)
        torch.cuda.synchronize()
        assert rc == status, "%s%s returned %d, expected %d" % (fn.__name__, args[5:12], rc, status)
        assert self.L.dv_launch_count() == before, fn.__name__ + ": launched a kernel"
        for k, n in self.sizes.items():
            assert (_body(self.out[k], n) == self.FILL).all() and _intact(self.out[k], n), fn.__name__ + " wrote " + k

    def _ptrs(self, names, given, shift):
        """given[k]: 0 or absent -> the default buffer, None -> NULL, a name -> that buffer."""
        out = []
        for k, default in names:
            v = given.get(k, 0)
            out.append(None if v is None else self.p(default if isinstance(v, int) else v, shift.get(k, 0)))
        return out

    def down(self, status, shift=None, B=None, H=None, W=None, CH=None, nchw=None, act=ACT_NONE, **given):
        """hi, wp, bias, mask, lo, colsum, ws, mask_bits, bits_out = 0: the buffer; None: NULL.  shift = {name: bytes}
        moves a pointer off its alignment."""
        ch = self.CH if CH is None else CH
        names = [("hi", "hi"), ("wp", "wp"), ("bias", "b32"), ("mask", "mask_lo"), ("lo", "lo_out")]
        tail = [("colsum", "cs"), ("ws", "cs_ws"), ("mask_bits", "words_lo"), ("bits_out", "bits_lo")]
        sh = shift or {}
        p = self._ptrs(names, given, sh)
        q = self._ptrs(tail, given, sh)
        self.expect(status, self.L.dv_conv_down, *p, self.B if B is None else B, self.H if H is None else H,
                    (self.H if H is None else H) if W is None else W, ch, int(ch != 32) if nchw is None else nchw, act,
                    *q, self.st)

    def up(self, status, shift=None, B=None, H=None, W=None, CH=None, nchw=None, act=None, **given):
        ch = self.CH if CH is None else CH
        if ch != 32:                        # the image layer has no mask epilogue
            given = dict(dict(mask=None, mask_bits=None, bits_out=None), **given)
        names = [("lo", "lo"), ("wp", "wp"), ("bias", "bch"), ("mask", "mask_hi"), ("hi", "hi_out")]
        tail = [("mask_bits", "words_hi"), ("bits_out", "bits_hi")]
        sh = shift or {}
        p = self._ptrs(names, given, sh)
        q = self._ptrs(tail, given, sh)
        a = (ACT_RELU if ch == 32 else ACT_SIGMOID) if act is None else act
        self.expect(status, self.L.dv_conv_up, *p, self.B if B is None else B, self.H if H is None else H,
                    (self.H if H is None else H) if W is None else W, ch, int(ch != 32) if nchw is None else nchw, a,
                    *q, self.st)

    def wgrad(self, status, shift=None, B=None, H=None, W=None, CH=None, nchw=None, ws_bytes=None, **given):
        ch = self.CH if CH is None else CH
        names = [("lo", "lo"), ("hi", "hi"), ("dw", "dw"), ("db", "db"), ("ws", "ws")]
        p = self._ptrs(names, given, shift or {})
        self.expect(status, self.L.dv_conv_wgrad, *p, self.ws_bytes if ws_bytes is None else ws_bytes,
                    self.B if B is None else B, self.H if H is None else H,
                    (self.H if H is None else H) if W is None else W, ch, int(ch != 32) if nchw is None else nchw,
                    self.st)


REFUSAL_SHAPES = [(9, 4, 32), (2, 16, 32), (2, 16, 3), (2, 32, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,CH", REFUSAL_SHAPES, ids=[_id(c) for c in REFUSAL_SHAPES])
def test_refusals_null_shape_act_workspace(B, H, CH):
    r = Refusals(B, H, CH)
    for null in ("hi", "wp", "lo"):
        r.down(DV_ERR_BAD_ARG, **{null: None})
    for null in ("lo", "wp", "hi"):
        r.up(DV_ERR_BAD_ARG, **{null: None})
    for null in ("lo", "hi", "dw", "ws"):
        r.wgrad(DV_ERR_BAD_ARG, **{null: None})
    # hi_nchw must match CH
    r.down(DV_ERR_BAD_SHAPE, nchw=1 - int(CH != 32))
    r.up(DV_ERR_BAD_SHAPE, nchw=1 - int(CH != 32))
    r.wgrad(DV_ERR_BAD_SHAPE, nchw=1 - int(CH != 32))
    # activations: NONE / RELU on down, NONE / RELU / SIGMOID on up, SIGMOID only after the image layer
    for act in (ACT_SIGMOID, ACT_LEAKY, -1, 99):
        r.down(DV_ERR_BAD_ARG, act=act)
    for act in (ACT_LEAKY, -1, 99) + ((ACT_SIGMOID,) if CH == 32 else ()):
        r.up(DV_ERR_BAD_ARG, act=act)
    # mask words without the float mask
    r.down(DV_ERR_BAD_ARG, mask=None)
    if CH == 32:
        r.up(DV_ERR_BAD_ARG, mask=None)
    else:                                   # no mask epilogue on the image layer
        r.up(DV_ERR_BAD_ARG, mask="mask_hi")
        r.up(DV_ERR_BAD_ARG, bits_out="bits_hi")
    r.down(DV_ERR_WORKSPACE, ws=None)        # colsum without its workspace
    r.wgrad(DV_ERR_WORKSPACE, ws_bytes=r.ws_bytes - 1)
    # shapes outside the Burgess layers (those of the earlier refusal test), non-square, B <= 0, one image too many
    for b, h, w, ch in [(2, 8, 8, 3), (2, 64, 64, 1), (2, 32, 32, 32), (2, 8, 16, 32), (2, 32, 16, 3),
                        (0, H, H, CH), (-1, H, H, CH), (max_batch(H) + 1, H, H, CH), (2, H, H, 2)]:
        dims = dict(B=b, H=h, W=w, CH=ch, nchw=int(ch != 32))
        r.down(DV_ERR_BAD_SHAPE, **dims)
        r.up(DV_ERR_BAD_SHAPE, act=ACT_NONE, mask=None, mask_bits=None, bits_out=None, **dims)
        r.wgrad(DV_ERR_BAD_SHAPE, **dims)


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,CH", REFUSAL_SHAPES, ids=[_id(c) for c in REFUSAL_SHAPES])
def test_refusals_misaligned_operands(B, H, CH):
    """Activations, masks, w_packed and workspaces need 16 bytes; bias, dw, dbias, colsum_out and the bit words 4.  A
    pointer off by less is refused with DV_ERR_BAD_ARG before anything runs (on the tensor-core path such a call used
    to fail in the TMA descriptor encoding with DV_ERR_CUDA; the image kernels would have launched on it)."""
    r = Refusals(B, H, CH)
    for off in (4, 8, 12):
        for k in ("hi", "wp", "mask", "lo", "ws"):
            r.down(DV_ERR_BAD_ARG, shift={k: off})
        for k in ("lo", "wp", "hi") + (("mask",) if CH == 32 else ()):
            r.up(DV_ERR_BAD_ARG, shift={k: off})
        for k in ("lo", "hi", "ws"):
            r.wgrad(DV_ERR_BAD_ARG, shift={k: off})
    for off in (1, 2, 3):
        for k in ("bias", "colsum", "mask_bits", "bits_out"):
            r.down(DV_ERR_BAD_ARG, shift={k: off})
        for k in ("bias",) + (("mask_bits", "bits_out") if CH == 32 else ()):
            r.up(DV_ERR_BAD_ARG, shift={k: off})
        for k in ("dw", "db"):
            r.wgrad(DV_ERR_BAD_ARG, shift={k: off})
