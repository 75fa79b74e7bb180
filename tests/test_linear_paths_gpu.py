"""The fully connected layers (csrc/dv_linear.cu, csrc/dv_linear_tc.cu) on every path they can take, against fp64
references, through the raw C ABI.

The shape picks the kernel.  The forward and the input gradient run on the tensor cores (3xTF32 mma.sync, operands
fed by TMA, weights packed into hi/lo planes first) when their reduction length R (K forward, N input gradient) is a
multiple of 4 and at least 32, and on the CUDA cores (FFMA) otherwise.  The weight gradient runs on the tensor cores
when N % 4 == 0, K % 4 == 0, K >= 32 and M >= 32, and on the CUDA cores otherwise; each of its two kernels splits the
batch (split-K) by its own plan (`plan` below restates both).  Each case reads its path and split count back from the
workspace queries, asserts them against that restatement, and counts the kernels each call launches.

Every element of every output is checked against `|got - ref| <= TAU * sum|terms| + EPI * |ref|`, the fp64 value and
the magnitude of what the kernel adds up; the whole tensor also stays within WHOLE_TOL of its largest |ref|.  Outputs
and workspaces sit in NaN-filled buffers between sentinel words, inputs are followed by NaN (an over-read poisons the
result), every operand starts 16 bytes into its allocation, and every call runs twice and must repeat bit for bit.

The bound is first shown to have teeth on the CPU; everything else needs an H100 (pytest -m gpu).  Each GPU case
prints its worst error as a fraction of the bound (pytest -s shows them)."""
import ctypes
import math

import pytest
import torch

# 3xTF32 splits each fp32 operand into a tf32 hi part and a tf32 residual: the dropped lo*lo product and the rounding of
# the residual leave ~2^-22 of each product.  The products are exact in the fp32 accumulators, which round once per
# addition: within a 32-wide K block, then once per block (tensor cores), or once per FMA along a split and once per
# split in the reduction (CUDA cores).  Summed over the longest chain here (R = 1000: 32 + 32 additions; the CUDA-core
# chains are shorter) that is at most ~64 u = 2^-18 of sum|terms|.  Rounding errors do not all align: over every case
# here the worst measured on an H100 (SXM, 700 W) is about 0.2 of 2^-18, so the bound is 2^-19 (worst 0.42 of it).
# Without the correction terms (single-pass TF32) the error is ~2^-12 per product and breaks it
# (test_bound_catches_dropped_terms).
TAU = 2.0 ** -19
EPI = 2.0 ** -21       # the epilogue's own roundings (bias add, LeakyReLU slope, sigmoid), relative to |ref|
WHOLE_TOL = 4e-6       # max |got - ref| over the tensor, relative to max |ref|: not applied to the cancelling regime,
WHOLE_MIN = 64         # below 64 elements (max |ref| can itself be a cancelled sum) or after a sigmoid (it maps
                       # arguments of any scale into (0, 1); max |ref| says nothing about the error they carry)
SM_COUNT = 132         # kNumSMs in csrc/dv_common.cuh: the split plans are sized for an H100 SXM
GUARD = 1024           # floats of sentinel after each output and workspace
SENTINEL = 0x7FBADBAD  # a NaN bit pattern no kernel writes
OFF = 4                # floats: every operand starts 16 bytes into its allocation
DV_OK, DV_ERR_BAD_SHAPE, DV_ERR_BAD_ARG, DV_ERR_WORKSPACE = 0, -1, -2, -3     # include/disvae_b200.h
ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_LEAKY = 0, 1, 2, 3

FWD_EPILOGUES = [(ACT_NONE, 0.0), (ACT_RELU, 0.0), (ACT_LEAKY, 0.2), (ACT_LEAKY, 0.01), (ACT_SIGMOID, 0.0)]
DGRAD_MASKS = [(ACT_NONE, 0.0, False), (ACT_RELU, 0.0, False), (ACT_RELU, 0.0, True), (ACT_LEAKY, 0.2, True),
               (ACT_LEAKY, 0.01, True)]      # (act, slope, mask given); no mask: act must not matter


def _cdiv(a, b):
    return -(-a // b)


# ---------------------------------------------------------------------------------------------------------------------
# dispatch and split plans, restated
# ---------------------------------------------------------------------------------------------------------------------
def nt_path(R):
    """Forward (R = K) and input gradient (R = N): nt_ok in dv_linear_tc.cu."""
    return "tc" if R % 4 == 0 and R >= 32 else "cc"


def wgrad_path(M, N, K):
    """wgrad_ok in dv_linear_tc.cu."""
    return "tc" if N % 4 == 0 and K % 4 == 0 and K >= 32 and M >= 32 else "cc"


def plan(M, N, K):
    """-> (path, S, rows per split, rows of the last split) of the weight gradient: wgrad_plan (128-row tiles spread
    over about one wave of CTAs, no empty split) on the tensor cores, wgrad_splits (about two waves, at least 64 rows
    per split, at most 32 splits; split length rounded up to 16 rows, so the last split may be empty) otherwise."""
    if wgrad_path(M, N, K) == "tc":
        m_tiles = _cdiv(M, 128)
        want = max(min(_cdiv(SM_COUNT, _cdiv(N, 32) * _cdiv(K, 64)), m_tiles), 1)
        per = _cdiv(m_tiles, want)
        S = _cdiv(m_tiles, per)
        return "tc", S, per * 128, M - (S - 1) * per * 128
    tiles = _cdiv(K, 64) * _cdiv(N, 64)
    S = 1 if tiles >= 120 else max(min(_cdiv(2 * SM_COUNT, tiles), _cdiv(M, 64), 32), 1)
    per = _cdiv(_cdiv(M, S), 16) * 16
    return "cc", S, per, M - (S - 1) * per


def packed_floats(N, K):
    r4 = lambda v: (v + 3) & ~3
    return 2 * N * r4(K) + 2 * K * r4(N)


def wgrad_ws_floats(M, N, K):
    path, S, _, _ = plan(M, N, K)
    if S == 1:
        return 0
    return S * N * K + (S * N if path == "tc" else 0)


def regime_of(M, N, K):
    """The regime names a case is listed under (see test_case_lists_cover_every_path_and_split_regime)."""
    path, S, per, last = plan(M, N, K)
    tags = {"fwd." + nt_path(K), "dgrad." + nt_path(N), "wgrad.%s.S=1" % path if S == 1 else "wgrad.%s.S>1" % path}
    if S > 1 and last < per:
        tags.add("wgrad.%s.short-last" % path)
    if path == "cc" and S == 32:
        tags.add("wgrad.cc.cap32")
    if path == "cc" and last <= 0:
        tags.add("wgrad.cc.empty-last")
    return tags


# ---------------------------------------------------------------------------------------------------------------------
# cases: (M, N, K) of a layer; each runs the forward, the input gradient and the weight gradient
# ---------------------------------------------------------------------------------------------------------------------
def _network_cases():
    out = []
    for z in (10, 16, 32, 64):
        for B in (64, 256, 512, 1024):
            out += [(B, 256, 512), (B, 256, 256), (B, 2 * z, 256),      # encoder (encoders.py:81-86)
                    (B, 256, z), (B, 256, 256), (B, 512, 256)]           # decoder (decoders.py:71-73)
        for M in (128, 512, 1024):
            out += [(M, 1000, z), (M, 1000, 1000), (M, 2, 1000)]         # FactorVAE discriminator (discriminator.py)
    return list(dict.fromkeys(out))


NETWORK_CASES = _network_cases()
# R on both sides of the tensor-core condition, as the forward's K and the input gradient's N at once
BOUNDARY_CASES = [(130, R, R) for R in (28, 30, 31, 32, 33, 36, 64, 68)]
# the weight gradient's condition: M, K and N around 32 / multiples of 4
WGRAD_BOUNDARY_CASES = [(M, N, K) for M in (31, 32, 33) for K in (28, 32, 36) for N in (2, 4, 6, 20)]
# 128-row tiles x 64-column output tiles x the K tail of a 32-wide block, as the forward (M, Nout, R) and as the input
# gradient (M, R, Nout)
TAIL_CASES = list(dict.fromkeys([c for M in (1, 127, 128, 129, 257) for n_out in (1, 2, 63, 64, 65, 1000)
                                 for R in (36, 1000) for c in ((M, n_out, R), (M, R, n_out))]))
# weight-gradient split plans: (M, N, K, path, S, rows per split, rows of the last split)
SPLIT_CASES = [
    (64, 256, 10, "cc", 1, 64, 64),            # S = 1: a single 64-row split
    (1024, 256, 10, "cc", 16, 64, 64),         # S > 1, equal splits
    (1000, 256, 10, "cc", 16, 64, 40),         # last split shorter
    (1024, 256, 510, "cc", 9, 128, 0),         # split length rounded up to 16 rows: the last split is empty
    (4096, 2, 10, "cc", 32, 128, 128),         # capped at 32 splits
    (3000, 2, 10, "cc", 32, 96, 24),           # capped, last split shorter
    (1024, 1000, 1000, "tc", 1, 1024, 1024),   # S = 1: enough CTAs without splitting
    (64, 256, 256, "tc", 1, 128, 64),          # S = 1: one partial tile
    (1024, 20, 256, "tc", 8, 128, 128),        # S > 1, one 128-row tile per split
    (1024, 256, 512, "tc", 3, 384, 256),       # three tiles per split, the last has two
    (1000, 256, 512, "tc", 3, 384, 232),       # ... and ends in a partial tile
    (3000, 4, 64, "tc", 24, 128, 56),          # 24 one-tile splits, the last partial
]
# every shape the earlier per-kernel and full-size tests checked
LEGACY_CASES = [(64, 256, 512), (7, 20, 256), (130, 256, 10), (33, 1000, 1000), (256, 2, 1000), (5, 128, 64),
                (1, 512, 256), (1024, 256, 512), (1000, 20, 256), (513, 256, 10),
                (1024, 256, 512), (256, 1000, 1000), (300, 1000, 12), (77, 512, 256),
                (130, 256, 512), (130, 256, 256), (130, 20, 256), (130, 256, 10), (130, 1000, 1000), (130, 2, 1000),
                (130, 1000, 10),
                (1024, 256, 256), (1024, 20, 256), (1024, 256, 10), (1024, 512, 256), (512, 256, 512),
                (512, 512, 256), (256, 128, 256), (256, 256, 64), (256, 1000, 10)]
# the input regimes on one case of each path and split kind
REGIME_CASES = [(257, 1000, 36), (257, 36, 1000), (257, 65, 33), (257, 33, 65), (1000, 256, 10), (1000, 256, 512),
                (3000, 2, 10), (33, 20, 36)]
REGIMES = ("randn", "spread", "dead", "cancel")


def _id(c):
    return "%dx%dx%d" % tuple(c[:3])


# ---------------------------------------------------------------------------------------------------------------------
# inputs and fp64 references
# ---------------------------------------------------------------------------------------------------------------------
def _spread(shape, g):
    """Magnitudes 10^U(-4, 4), random signs: both ends of the hi/lo split."""
    mag = torch.pow(10.0, torch.rand(shape, generator=g, dtype=torch.float64) * 8 - 4)
    sign = torch.where(torch.rand(shape, generator=g) < 0.5, -1.0, 1.0).double()
    return (mag * sign).float()


def make_inputs(M, N, K, regime, seed=0):
    """x [M, K], w [N, K], b [N], g [M, N] (the output gradient) and mask [M, K] (the previous layer's output: exact
    0.0 and -0.0 every few elements, negatives, positives), all fp32."""
    g_ = torch.Generator().manual_seed(seed + M * 1000003 + N * 1009 + K)
    x = torch.randn(M, K, generator=g_)
    w = torch.randn(N, K, generator=g_) / math.sqrt(K)
    b = torch.randn(N, generator=g_)
    g = torch.randn(M, N, generator=g_)
    if regime == "spread":
        x, w, b, g = _spread((M, K), g_), _spread((N, K), g_), _spread((N,), g_), _spread((M, N), g_)
    elif regime == "dead":                 # rows of g and columns of x behind dead ReLUs
        g[torch.arange(M) % 5 == 1] = 0.0
        x[:, torch.arange(K) % 7 == 3] = 0.0
    elif regime == "cancel":               # 10^3 +- 1 with alternating signs along every reduction
        alt = lambda n: 1.0 - 2.0 * (torch.arange(n) % 2).float()
        x = 1000.0 + torch.randn(M, K, generator=g_)
        w = (1000.0 + torch.randn(N, K, generator=g_)) * alt(N).unsqueeze(1) * alt(K).unsqueeze(0)
        g = (1000.0 + torch.randn(M, N, generator=g_)) * alt(M).unsqueeze(1)
    else:
        assert regime == "randn", regime
    mask = torch.randn(M, K, generator=g_)
    flat = mask.view(-1)
    idx = torch.arange(flat.numel())
    flat[idx % 5 == 2] = 0.0
    flat[idx % 5 == 4] = -0.0
    return x, w, b, g, mask


def ref_act(pre, act, slope):
    if act == ACT_RELU:
        return torch.relu(pre)
    if act == ACT_LEAKY:
        return torch.where(pre > 0, pre, pre * slope)
    if act == ACT_SIGMOID:
        return torch.sigmoid(pre)
    return pre


def ref_mask_factor(mask, act, slope):
    """act'(y) taken from the fp32 post-activation y: 1 where y > 0; 0 (ReLU) or slope (LeakyReLU) at 0, -0.0 and
    below."""
    if act == ACT_RELU:
        return (mask > 0).double()
    if act == ACT_LEAKY:
        return torch.where(mask > 0, 1.0, float(slope)).double()
    return torch.ones(mask.shape, dtype=torch.float64)


class Reference:
    """fp64 products of one case's inputs and the sums of |terms| that bound their errors."""

    def __init__(self, x, w, b, g):
        x, w, b, g = x.double(), w.double(), b.double(), g.double()
        self.pre, self.pre_terms = x @ w.t(), x.abs() @ w.abs().t()                  # forward, before the bias
        self.b = b
        self.dx, self.dx_terms = g @ w, g.abs() @ w.abs()                          # input gradient, before the mask
        self.dw, self.dw_terms = g.t() @ x, g.abs().t() @ x.abs()                  # weight gradient
        self.db, self.db_terms = g.sum(0), g.abs().sum(0)

    def fwd(self, act, slope, bias):
        pre = self.pre + self.b if bias else self.pre
        terms = self.pre_terms + self.b.abs() if bias else self.pre_terms
        return ref_act(pre, act, slope), terms

    def dgrad(self, mask, act, slope):
        if mask is None:
            return self.dx, self.dx_terms
        f = ref_mask_factor(mask, act, slope)
        return self.dx * f, self.dx_terms * f


def bound_ratio(got, ref, terms):
    """Per element |got - ref| / (TAU * terms + EPI * |ref|), fp64; NaN in `got` counts as infinite, and an element
    whose bound is 0 must be exact."""
    got = got.double().cpu()
    err = (got - ref).abs()
    lim = TAU * terms + EPI * ref.abs()
    r = torch.where(err == 0, 0.0, err / lim)
    return torch.where(torch.isnan(got), math.inf, r)


def check(got, ref, terms, tag, whole=True):
    """Asserts the element-wise bound (and the whole-tensor one); -> worst |got - ref| / (TAU * terms + EPI |ref|)."""
    assert tuple(got.shape) == tuple(ref.shape), (tag, got.shape, ref.shape)
    assert torch.isfinite(ref).all(), tag
    r = bound_ratio(got, ref, terms)
    worst = r.max().item()
    if worst > 1:
        i = int(r.argmax())
        at = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), r.shape))
        raise AssertionError("%s: element %s got %r, fp64 %r, |terms| %.3e: %.2f x the bound"
                             % (tag, at, got.reshape(-1)[i].item(), ref.reshape(-1)[i].item(),
                                terms.reshape(-1)[i].item(), worst))
    if whole and ref.numel() >= WHOLE_MIN:
        e = ((got.double().cpu() - ref).abs().max() / ref.abs().max().clamp_min(1e-300)).item()
        assert e <= WHOLE_TOL, "%s: max err %.3e of max |ref| > %.1e" % (tag, e, WHOLE_TOL)
    return worst


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the bound has teeth
# ---------------------------------------------------------------------------------------------------------------------
def _tf32(t):
    """fp32 -> tf32 (10 explicit mantissa bits), round to nearest: what a single-pass TF32 GEMM multiplies."""
    bits = t.float().contiguous().view(torch.int32)
    return ((bits + 0x1000) & ~0x1FFF).view(torch.float32)


def test_bound_catches_dropped_terms():
    """At K-tail shapes an fp64 result missing one reduction term (the last K of the last 32-wide block), missing the
    last 128-row tile of the weight gradient, or computed from tf32-rounded operands (3xTF32 without its correction
    terms) breaks the bound somewhere, while the exact fp64 result and its fp32 rounding pass."""
    for M, N, K in [(129, 65, 36), (257, 64, 1000), (257, 1000, 36)]:
        x, w, b, g, _ = make_inputs(M, N, K, "randn")
        ref = Reference(x, w, b, g)
        y, terms = ref.fwd(ACT_NONE, 0.0, True)
        check(y.float(), y, terms, "fp32 rounding of the forward")
        check(ref.dw.float(), ref.dw, ref.dw_terms, "fp32 rounding of the weight gradient")
        x64, w64, g64 = x.double(), w.double(), g.double()
        drop_k = y - x64[:, -1:] * w64[:, -1].unsqueeze(0)
        assert bound_ratio(drop_k, y, terms).max() > 1, (M, N, K)
        drop_n = ref.dx - g64[:, -1:] * w64[-1].unsqueeze(0)
        assert bound_ratio(drop_n, ref.dx, ref.dx_terms).max() > 1, (M, N, K)
        tail = (M - 1) // 128 * 128
        drop_tile = ref.dw - g64[tail:].t() @ x64[tail:]
        assert bound_ratio(drop_tile, ref.dw, ref.dw_terms).max() > 1, (M, N, K)
        drop_bias = ref.db - g64[tail:].sum(0)
        assert bound_ratio(drop_bias, ref.db, ref.db_terms).max() > 1, (M, N, K)
        single = _tf32(x).double() @ _tf32(w).double().t() + b.double()
        assert bound_ratio(single, y, terms).max() > 1, (M, N, K)
        single_w = _tf32(g).double().t() @ _tf32(x).double()
        assert bound_ratio(single_w, ref.dw, ref.dw_terms).max() > 1, (M, N, K)


def test_bound_catches_a_mask_taken_at_zero():
    """dx where the mask is exactly 0 or -0.0 is 0 (ReLU) or slope times the product (LeakyReLU); the value of y >= 0
    in their place breaks the bound."""
    M, N, K = 129, 36, 65
    x, w, b, g, mask = make_inputs(M, N, K, "randn")
    ref = Reference(x, w, b, g)
    zero = mask == 0
    assert zero.any() and (zero & torch.signbit(mask)).any() and (mask < 0).any()
    for act, slope in [(ACT_RELU, 0.0), (ACT_LEAKY, 0.2)]:
        want, terms = ref.dgrad(mask, act, slope)
        wrong = torch.where(zero, ref.dx, want)
        assert bound_ratio(wrong, want, terms).max() > 1, act


def test_case_lists_cover_every_path_and_split_regime():
    """Every path of every operation and every weight-gradient split regime is run by at least one case, and the
    split cases' plans are the ones their comments name."""
    for M, N, K, path, S, per, last in SPLIT_CASES:
        assert plan(M, N, K) == (path, S, per, last), (M, N, K, plan(M, N, K))
    seen = set()
    for c in NETWORK_CASES + BOUNDARY_CASES + WGRAD_BOUNDARY_CASES + TAIL_CASES + LEGACY_CASES + REGIME_CASES:
        seen |= regime_of(*c[:3])
    for c in SPLIT_CASES:
        seen |= regime_of(*c[:3])
    want = {"fwd.cc", "fwd.tc", "dgrad.cc", "dgrad.tc", "wgrad.cc.S=1", "wgrad.cc.S>1", "wgrad.cc.short-last",
            "wgrad.cc.cap32", "wgrad.cc.empty-last", "wgrad.tc.S=1", "wgrad.tc.S>1", "wgrad.tc.short-last"}
    assert want <= seen, want - seen
    # the layers of the networks land on both sides of both conditions
    net = set()
    for c in NETWORK_CASES:
        net |= regime_of(*c)
    assert {"fwd.cc", "fwd.tc", "dgrad.cc", "dgrad.tc", "wgrad.cc.S>1", "wgrad.tc.S=1", "wgrad.tc.S>1"} <= net


def test_workspace_queries_match_the_restated_plans():
    """The library's workspace queries give the path and split count `plan` restates, for every case here (the
    queries run on the host)."""
    from disvae import _native as N
    L = N.lib()
    cases = NETWORK_CASES + BOUNDARY_CASES + WGRAD_BOUNDARY_CASES + TAIL_CASES + LEGACY_CASES + REGIME_CASES
    for M, Nn, K in cases + [c[:3] for c in SPLIT_CASES]:
        assert L.dv_linear_fwd_workspace_bytes(M, Nn, K) == (4 * packed_floats(Nn, K) if nt_path(K) == "tc" else 0)
        assert L.dv_linear_dgrad_workspace_bytes(M, Nn, K) == (4 * packed_floats(Nn, K) if nt_path(Nn) == "tc" else 0)
        assert L.dv_linear_wgrad_workspace_bytes(M, Nn, K) == 4 * wgrad_ws_floats(M, Nn, K), (M, Nn, K)
        assert L.dv_linear_packed_floats(Nn, K) == packed_floats(Nn, K)
    for q in (L.dv_linear_fwd_workspace_bytes, L.dv_linear_dgrad_workspace_bytes, L.dv_linear_wgrad_workspace_bytes):
        assert q(0, 64, 64) == 0 and q(64, -1, 64) == 0 and q(64, 64, 0) == 0
    assert L.dv_linear_packed_floats(0, 4) == 0 and L.dv_linear_packed_floats(4, -4) == 0


# ---------------------------------------------------------------------------------------------------------------------
# device buffers
# ---------------------------------------------------------------------------------------------------------------------
def _bits(t):
    return t.contiguous().view(torch.int32)


def _input(t):
    """Device copy of `t` starting 16 bytes into a NaN-filled allocation, with GUARD NaN after it."""
    n = t.numel()
    buf = torch.full((OFF + n + GUARD,), float("nan"), device="cuda")
    buf[OFF:OFF + n] = t.reshape(-1).cuda()
    return buf


def _output(n, fill=float("nan")):
    """n floats of `fill` 16 bytes into an allocation, sentinel words before and after."""
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
    t = buf[OFF:OFF + n].clone()
    return t if shape is None else t.view(shape)


def _native():
    from disvae import _native as N
    return N


# ---------------------------------------------------------------------------------------------------------------------
# one layer through every entry point
# ---------------------------------------------------------------------------------------------------------------------
class Layer:
    def __init__(self, M, N, K, regime="randn", seed=0):
        self.M, self.N, self.K = M, N, K
        self.regime = regime
        self.cpu = dict(zip("x w b g mask".split(), make_inputs(M, N, K, regime, seed)))
        self.dev = {k: _input(v) for k, v in self.cpu.items()}
        self.ref = Reference(self.cpu["x"], self.cpu["w"], self.cpu["b"], self.cpu["g"])
        self.whole = regime != "cancel"
        self.L, self.st = _native().lib(), _native().stream()
        self.tag = "%s %s" % (_id((M, N, K)), regime)

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
        """dv_linear_pack_multi of this w alone -> guarded planes (one launch)."""
        pf = packed_floats(self.N, self.K)
        pk = _output(pf)
        self._launch(self.L.dv_linear_pack_multi, 1, (ctypes.c_void_p * 1)(self.p("w")),
                     (ctypes.c_void_p * 1)(_addr(pk)), (ctypes.c_int * 1)(self.N), (ctypes.c_int * 1)(self.K),
                     self.st, launches=1)
        assert _intact(pk, pf), self.tag + ": pack wrote outside its planes"
        return pk

    def fwd(self, pk):
        M, N, K = self.M, self.N, self.K
        path = nt_path(K)
        nbytes = self.L.dv_linear_fwd_workspace_bytes(M, N, K)
        assert nbytes == (4 * packed_floats(N, K) if path == "tc" else 0), self.tag
        worst = 0.0
        for act, slope in FWD_EPILOGUES:
            for bias in (False, True):
                tag = "%s fwd[%s] act %d slope %g bias %d" % (self.tag, path, act, slope, bias)
                runs = []
                for rep in range(2):
                    y, ws = _output(M * N), _output(nbytes // 4)
                    wsp = _addr(ws) if nbytes or rep == 0 else None       # NULL is allowed when the query is 0
                    self._launch(self.L.dv_linear_fwd, self.p("x"), self.p("w"), self.p("b") if bias else None,
                                 _addr(y), M, N, K, act, slope, wsp, self.st, launches=2 if path == "tc" else 1)
                    assert _intact(y, M * N) and _intact(ws, nbytes // 4), tag + ": wrote out of bounds"
                    runs.append(_body(y, M * N, (M, N)))
                    if nbytes and pk is not None:
                        assert torch.equal(_bits(_body(ws, nbytes // 4)), _bits(_body(pk, nbytes // 4))), \
                            tag + ": the per-call pack differs from dv_linear_pack_multi"
                assert torch.equal(_bits(runs[0]), _bits(runs[1])), tag + ": not deterministic"
                yp = _output(M * N)
                self._launch(self.L.dv_linear_fwd_packed, self.p("x"), self.p("w"), _addr(pk),
                             self.p("b") if bias else None, _addr(yp), M, N, K, act, slope, self.st, launches=1)
                assert _intact(yp, M * N) and torch.equal(_bits(_body(yp, M * N, (M, N))), _bits(runs[0])), \
                    tag + ": dv_linear_fwd_packed differs"
                ref, terms = self.ref.fwd(act, slope, bias)
                worst = max(worst, check(runs[0], ref, terms, tag, self.whole and act != ACT_SIGMOID))
        return worst

    def dgrad(self, pk):
        M, N, K = self.M, self.N, self.K
        path = nt_path(N)
        nbytes = self.L.dv_linear_dgrad_workspace_bytes(M, N, K)
        assert nbytes == (4 * packed_floats(N, K) if path == "tc" else 0), self.tag
        worst = 0.0
        for act, slope, masked in DGRAD_MASKS:
            tag = "%s dgrad[%s] act %d slope %g mask %d" % (self.tag, path, act, slope, masked)
            mp = self.p("mask") if masked else None
            runs = []
            for rep in range(2):
                dx, ws = _output(M * K), _output(nbytes // 4)
                wsp = _addr(ws) if nbytes or rep == 0 else None
                self._launch(self.L.dv_linear_dgrad, self.p("g"), self.p("w"), mp, _addr(dx), M, N, K, act, slope,
                             wsp, self.st, launches=2 if path == "tc" else 1)
                assert _intact(dx, M * K) and _intact(ws, nbytes // 4), tag + ": wrote out of bounds"
                runs.append(_body(dx, M * K, (M, K)))
                if nbytes and pk is not None:
                    assert torch.equal(_bits(_body(ws, nbytes // 4)), _bits(_body(pk, nbytes // 4))), \
                        tag + ": the per-call pack differs from dv_linear_pack_multi"
            assert torch.equal(_bits(runs[0]), _bits(runs[1])), tag + ": not deterministic"
            dxp = _output(M * K)
            self._launch(self.L.dv_linear_dgrad_packed, self.p("g"), self.p("w"), _addr(pk), mp, _addr(dxp), M, N, K,
                         act, slope, self.st, launches=1)
            assert _intact(dxp, M * K) and torch.equal(_bits(_body(dxp, M * K, (M, K))), _bits(runs[0])), \
                tag + ": dv_linear_dgrad_packed differs"
            ref, terms = self.ref.dgrad(self.cpu["mask"] if masked else None, act, slope)
            worst = max(worst, check(runs[0], ref, terms, tag, self.whole))
        return worst

    def wgrad(self, expect=None):
        M, N, K = self.M, self.N, self.K
        path, S, per, last = plan(M, N, K)
        if expect is not None:
            assert (path, S, per, last) == expect, (self.tag, (path, S, per, last), expect)
        nbytes = self.L.dv_linear_wgrad_workspace_bytes(M, N, K)
        # the split count, read back from the query: S x [N, K] partials (+ S x [N] bias partials on the tensor cores)
        per_split = N * K + (N if path == "tc" else 0)
        assert nbytes % (4 * per_split) == 0, self.tag
        S_read = max(nbytes // (4 * per_split), 1)
        assert S_read == S and (nbytes == 0) == (S == 1), "%s: query says %d splits, plan %d" % (self.tag, S_read, S)
        tag = "%s wgrad[%s S=%d]" % (self.tag, path, S)
        runs = {}
        for bias in (True, False):
            for rep in range(2):
                dw, db, ws = _output(N * K), _output(N) if bias else None, _output(nbytes // 4)
                wsp = _addr(ws) if nbytes or rep == 0 else None
                launches = 1 + (S > 1) * (1 + bias) if path == "tc" else 1 + (S > 1) + bias
                self._launch(self.L.dv_linear_wgrad, self.p("g"), self.p("x"), _addr(dw), _addr(db), M, N, K, wsp,
                             self.st, launches=launches)
                assert _intact(dw, N * K) and _intact(ws, nbytes // 4), tag + ": wrote out of bounds"
                assert db is None or _intact(db, N), tag + ": wrote past dbias"
                runs[bias, rep] = (_body(dw, N * K, (N, K)), None if db is None else _body(db, N))
        for key, (dw, db) in runs.items():
            assert torch.equal(_bits(dw), _bits(runs[True, 0][0])), "%s: dw differs (dbias %d, run %d)" % ((tag,) + key)
        assert torch.equal(_bits(runs[True, 1][1]), _bits(runs[True, 0][1])), tag + ": dbias not deterministic"
        w_dw = check(runs[True, 0][0], self.ref.dw, self.ref.dw_terms, tag + " dw", self.whole)
        w_db = check(runs[True, 0][1], self.ref.db, self.ref.db_terms, tag + " dbias", self.whole)
        return max(w_dw, w_db)

    def run(self, expect=None):
        pk = self.pack()
        e_f, e_d, e_w = self.fwd(pk), self.dgrad(pk), self.wgrad(expect)
        path, S, _, _ = plan(self.M, self.N, self.K)
        print("%s: fwd[%s] %.3f, dgrad[%s] %.3f, wgrad[%s S=%d] %.3f of the bound"
              % (self.tag, nt_path(self.K), e_f, nt_path(self.N), e_d, path, S, e_w))


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", NETWORK_CASES, ids=[_id(c) for c in NETWORK_CASES])
def test_network_layers(M, N, K):
    """Every layer of the encoder, decoder and FactorVAE discriminator at z in {10, 16, 32, 64}, B in
    {64, 256, 512, 1024} and discriminator batches of 128, 512 and 1024."""
    Layer(M, N, K).run()


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", BOUNDARY_CASES + WGRAD_BOUNDARY_CASES,
                         ids=[_id(c) for c in BOUNDARY_CASES + WGRAD_BOUNDARY_CASES])
def test_dispatch_boundaries(M, N, K):
    Layer(M, N, K).run()


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", TAIL_CASES, ids=[_id(c) for c in TAIL_CASES])
def test_tile_tails(M, N, K):
    Layer(M, N, K).run()


@pytest.mark.gpu
@pytest.mark.parametrize("case", SPLIT_CASES, ids=[_id(c) for c in SPLIT_CASES])
def test_weight_gradient_split_plans(case):
    Layer(*case[:3]).run(expect=case[3:])


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", list(dict.fromkeys(LEGACY_CASES)), ids=[_id(c) for c in dict.fromkeys(LEGACY_CASES)])
def test_earlier_linear_shapes(M, N, K):
    Layer(M, N, K).run()


@pytest.mark.gpu
@pytest.mark.parametrize("regime", REGIMES[1:])
@pytest.mark.parametrize("M,N,K", REGIME_CASES, ids=[_id(c) for c in REGIME_CASES])
def test_input_regimes(M, N, K, regime):
    """Magnitudes over 10^+-4, dead rows of g and columns of x (those outputs must be exactly 0), and 10^3 +- 1 with
    alternating signs, whose cancellation leaves outputs far below the terms they add up."""
    Layer(M, N, K, regime).run()


@pytest.mark.gpu
def test_pack_multi_splits_long_tables():
    """One table with every weight matrix of the encoder, decoder and discriminator (12 > 8: two launches) writes the
    planes the per-call pack writes, and the packed forward and input gradient on them equal the per-call ones."""
    z, M = 10, 129
    shapes = [(256, 512), (256, 256), (2 * z, 256), (256, z), (256, 256), (512, 256),
              (1000, z), (1000, 1000), (1000, 1000), (1000, 1000), (1000, 1000), (2, 1000)]
    N = _native()
    L, st = N.lib(), N.stream()
    layers = [Layer(M, n, k, seed=i) for i, (n, k) in enumerate(shapes)]
    packs = [_output(packed_floats(n, k)) for n, k in shapes]
    n = len(shapes)
    arr_p, arr_i = ctypes.c_void_p * n, ctypes.c_int * n
    before = L.dv_launch_count()
    rc = L.dv_linear_pack_multi(n, arr_p(*[lay.p("w") for lay in layers]), arr_p(*[_addr(p) for p in packs]),
                                arr_i(*[s[0] for s in shapes]), arr_i(*[s[1] for s in shapes]), st)
    torch.cuda.synchronize()
    assert rc == DV_OK and L.dv_launch_count() - before == 2
    for lay, pk, (nn, k) in zip(layers, packs, shapes):
        pf = packed_floats(nn, k)
        assert _intact(pk, pf), (nn, k)
        single = lay.pack()
        assert torch.equal(_bits(_body(pk, pf)), _bits(_body(single, pf))), (nn, k)
        lay.fwd(pk)
        lay.dgrad(pk)


# ---------------------------------------------------------------------------------------------------------------------
# refusals: status code, nothing launched, outputs untouched
# ---------------------------------------------------------------------------------------------------------------------
class Refusals:
    """Buffers for one (M, N, K) and the raw calls on them; `expect` runs a call and asserts its status, that no kernel
    ran and that every output and workspace still holds its fill."""
    FILL = 7.0

    def __init__(self, M, N, K):
        self.M, self.N, self.K = M, N, K
        x, w, b, g, mask = make_inputs(M, N, K, "randn")
        self.inp = {k: _input(v) for k, v in dict(x=x, w=w, b=b, g=g, mask=mask).items()}
        pf = packed_floats(N, K)
        self.sizes = dict(y=M * N, dx=M * K, dw=N * K, db=N, ws=pf + N * K * 33, pk=pf)
        self.out = {k: _output(n, self.FILL) for k, n in self.sizes.items()}
        self.L, self.st = _native().lib(), _native().stream()

    def p(self, name, shift=0):
        return _addr(self.inp[name] if name in self.inp else self.out[name], shift)

    def _dims(self, M, N, K):
        return (self.M if M is None else M, self.N if N is None else N, self.K if K is None else K)

    def expect(self, status, fn, *args):
        before = self.L.dv_launch_count()
        rc = fn(*args)
        torch.cuda.synchronize()
        assert rc == status, "%s%s returned %d, expected %d" % (fn.__name__, args[4:], rc, status)
        assert self.L.dv_launch_count() == before, fn.__name__ + ": launched a kernel"
        for k, n in self.sizes.items():
            assert (_body(self.out[k], n) == self.FILL).all() and _intact(self.out[k], n), fn.__name__ + " wrote " + k

    def fwd(self, status, x=0, w=0, b=0, y=0, ws=0, M=None, N=None, K=None, act=ACT_RELU, shift=None):
        """x, w, ... = 0: the buffer; None: NULL.  shift = {name: bytes} moves a pointer off its 16-byte alignment."""
        sh = shift or {}
        ptrs = [None if v is None else self.p(k, sh.get(k, 0)) for k, v in dict(x=x, w=w, b=b, y=y).items()]
        self.expect(status, self.L.dv_linear_fwd, *ptrs, *self._dims(M, N, K), act, 0.2,
                    None if ws is None else self.p("ws", sh.get("ws", 0)), self.st)

    def fwd_packed(self, status, x=0, w=0, pk=0, b=0, y=0, M=None, N=None, K=None, act=ACT_RELU, shift=None):
        sh = shift or {}
        ptrs = [None if v is None else self.p(k, sh.get(k, 0)) for k, v in dict(x=x, w=w, pk=pk, b=b, y=y).items()]
        self.expect(status, self.L.dv_linear_fwd_packed, *ptrs, *self._dims(M, N, K), act, 0.2,
                    self.st)

    def dgrad(self, status, g=0, w=0, mask=0, dx=0, ws=0, M=None, N=None, K=None, act=ACT_LEAKY, shift=None):
        sh = shift or {}
        ptrs = [None if v is None else self.p(k, sh.get(k, 0)) for k, v in dict(g=g, w=w, mask=mask, dx=dx).items()]
        self.expect(status, self.L.dv_linear_dgrad, *ptrs, *self._dims(M, N, K), act, 0.2,
                    None if ws is None else self.p("ws", sh.get("ws", 0)), self.st)

    def dgrad_packed(self, status, g=0, w=0, pk=0, mask=0, dx=0, M=None, N=None, K=None, act=ACT_LEAKY, shift=None):
        sh = shift or {}
        ptrs = [None if v is None else self.p(k, sh.get(k, 0))
                for k, v in dict(g=g, w=w, pk=pk, mask=mask, dx=dx).items()]
        self.expect(status, self.L.dv_linear_dgrad_packed, *ptrs, *self._dims(M, N, K), act, 0.2,
                    self.st)

    def wgrad(self, status, g=0, x=0, dw=0, db=0, ws=0, M=None, N=None, K=None, shift=None):
        sh = shift or {}
        ptrs = [None if v is None else self.p(k, sh.get(k, 0)) for k, v in dict(g=g, x=x, dw=dw, db=db).items()]
        self.expect(status, self.L.dv_linear_wgrad, *ptrs, *self._dims(M, N, K),
                    None if ws is None else self.p("ws", sh.get("ws", 0)), self.st)


TC_SHAPE = (1024, 64, 64)     # every operation on the tensor cores, the weight gradient with S = 2
CC_SHAPE = (1024, 30, 30)     # every operation on the CUDA cores, the weight gradient with S = 16


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [TC_SHAPE, CC_SHAPE], ids=["tc", "cc"])
def test_refusals_null_shape_act_workspace(shape):
    M, N, K = shape
    assert nt_path(K) == nt_path(N) == plan(M, N, K)[0] == ("tc" if shape == TC_SHAPE else "cc")
    assert plan(M, N, K)[1] > 1
    r = Refusals(M, N, K)
    tc = shape == TC_SHAPE
    for null in ("x", "w", "y"):
        r.fwd(DV_ERR_BAD_ARG, **{null: None})
        r.fwd_packed(DV_ERR_BAD_ARG, **{null: None})
    for null in ("g", "w", "dx"):
        r.dgrad(DV_ERR_BAD_ARG, **{null: None})
        r.dgrad_packed(DV_ERR_BAD_ARG, **{null: None})
    for null in ("g", "x", "dw"):
        r.wgrad(DV_ERR_BAD_ARG, **{null: None})
    for dims in (dict(M=0), dict(M=-1), dict(N=0), dict(N=-4), dict(K=0), dict(K=-32)):
        for call in (r.fwd, r.fwd_packed, r.dgrad, r.dgrad_packed, r.wgrad):
            call(DV_ERR_BAD_SHAPE, **dims)
    for act in (-1, 4, 99):
        r.fwd(DV_ERR_BAD_ARG, act=act)
        r.fwd_packed(DV_ERR_BAD_ARG, act=act)
    if tc:
        r.fwd(DV_ERR_WORKSPACE, ws=None)
        r.fwd_packed(DV_ERR_WORKSPACE, pk=None)
        r.dgrad(DV_ERR_WORKSPACE, ws=None)
        r.dgrad_packed(DV_ERR_WORKSPACE, pk=None)
    r.wgrad(DV_ERR_WORKSPACE, ws=None)                          # S > 1 on both paths



@pytest.mark.gpu
@pytest.mark.parametrize("shape", [TC_SHAPE, CC_SHAPE], ids=["tc", "cc"])
def test_dgrad_refuses_an_act_outside_none_relu_leaky(shape):
    """The input gradient's act names the activation whose derivative masks it: SIGMOID or an unknown value is refused
    with or without a mask (a mask with such an act used to be ignored, returning DV_OK and an unmasked gradient)."""
    r = Refusals(*shape)
    for act in (ACT_SIGMOID, -1, 4, 99):
        for mask in (0, None):
            r.dgrad(DV_ERR_BAD_ARG, act=act, mask=mask)
            r.dgrad_packed(DV_ERR_BAD_ARG, act=act, mask=mask)


@pytest.mark.gpu
def test_tensor_core_path_refuses_misaligned_tma_operands():
    """The tensor-core GEMMs read x (forward), g (input gradient), g and x (weight gradient) and the packed planes
    through TMA, which needs 16-byte aligned addresses: 4-, 8- and 12-byte offsets are refused before anything runs
    (before, the pack kernel ran and the call failed afterwards with DV_ERR_CUDA).  The CUDA-core shapes take any
    4-byte aligned operand and give the same bits as from aligned ones."""
    r = Refusals(*TC_SHAPE)
    for off in (4, 8, 12):
        r.fwd(DV_ERR_BAD_ARG, shift=dict(x=off))
        r.fwd(DV_ERR_BAD_ARG, shift=dict(ws=off))
        r.fwd_packed(DV_ERR_BAD_ARG, shift=dict(x=off))
        r.fwd_packed(DV_ERR_BAD_ARG, shift=dict(pk=off))
        r.dgrad(DV_ERR_BAD_ARG, shift=dict(g=off))
        r.dgrad(DV_ERR_BAD_ARG, shift=dict(ws=off))
        r.dgrad_packed(DV_ERR_BAD_ARG, shift=dict(g=off))
        r.dgrad_packed(DV_ERR_BAD_ARG, shift=dict(pk=off))
        r.wgrad(DV_ERR_BAD_ARG, shift=dict(g=off))
        r.wgrad(DV_ERR_BAD_ARG, shift=dict(x=off))

    M, N, K = CC_SHAPE
    L, st = _native().lib(), _native().stream()
    x, w, b, g, mask = make_inputs(M, N, K, "randn")
    ref = Reference(x, w, b, g)
    nbytes = L.dv_linear_wgrad_workspace_bytes(M, N, K)
    for off in (0, 4, 8, 12):
        sh = off // 4
        xs, ws_, bs, gs, ms = [torch.full((t.numel() + 8,), float("nan"), device="cuda") for t in (x, w, b, g, mask)]
        for buf, t in zip((xs, ws_, bs, gs, ms), (x, w, b, g, mask)):
            buf[sh:sh + t.numel()] = t.reshape(-1).cuda()
        y, dx, dw, db, wk = (torch.full((n + 4,), float("nan"), device="cuda")
                             for n in (M * N, M * K, N * K, N, nbytes // 4))
        a = lambda t: t.data_ptr() + off
        assert L.dv_linear_fwd(a(xs), a(ws_), a(bs), a(y), M, N, K, ACT_LEAKY, 0.2, None, st) == DV_OK
        assert L.dv_linear_dgrad(a(gs), a(ws_), a(ms), a(dx), M, N, K, ACT_LEAKY, 0.2, None, st) == DV_OK
        assert L.dv_linear_wgrad(a(gs), a(xs), a(dw), a(db), M, N, K, a(wk), st) == DV_OK
        torch.cuda.synchronize()
        got = [t[sh:sh + n].clone() for t, n in ((y, M * N), (dx, M * K), (dw, N * K), (db, N))]
        if off == 0:
            first = got
            check(got[0].view(M, N), *ref.fwd(ACT_LEAKY, 0.2, True), "fwd from 4-byte aligned operands")
            check(got[1].view(M, K), *ref.dgrad(mask, ACT_LEAKY, 0.2), "dgrad from 4-byte aligned operands")
            check(got[2].view(N, K), ref.dw, ref.dw_terms, "wgrad from 4-byte aligned operands")
        else:
            for a_, b_ in zip(got, first):
                assert torch.equal(_bits(a_), _bits(b_)), off


@pytest.mark.gpu
def test_pack_multi_refuses_bad_tables():
    """n < 1, NULL arrays, and a NULL pointer, a size <= 0 or a misaligned plane buffer anywhere in the table (also
    past the first 8 entries, which go to a second launch) are refused before any launch."""
    L, st = _native().lib(), _native().stream()
    n = 11
    shapes = [(64, 64)] * n
    ws = [_input(torch.randn(nn, k)) for nn, k in shapes]
    pf = packed_floats(64, 64)
    packs = [_output(pf, 7.0) for _ in shapes]
    arr_p, arr_i = ctypes.c_void_p * n, ctypes.c_int * n

    def call(status, count=n, w=None, pk=None, N=None, K=None, arrays=(True, True, True, True)):
        wl = [_addr(t) for t in ws] if w is None else w
        pl = [_addr(t) for t in packs] if pk is None else pk
        Nl = [s[0] for s in shapes] if N is None else N
        Kl = [s[1] for s in shapes] if K is None else K
        args = [arr_p(*wl), arr_p(*pl), arr_i(*Nl), arr_i(*Kl)]
        args = [a if keep else None for a, keep in zip(args, arrays)]
        before = L.dv_launch_count()
        rc = L.dv_linear_pack_multi(count, *args, st)
        torch.cuda.synchronize()
        assert rc == status, (rc, status)
        if status != DV_OK:
            assert L.dv_launch_count() == before
            for p in packs:
                assert (_body(p, pf) == 7.0).all() and _intact(p, pf)

    for count in (0, -1):
        call(DV_ERR_BAD_ARG, count=count)
    for i in range(4):
        call(DV_ERR_BAD_ARG, arrays=[j != i for j in range(4)])
    for i in (0, 9):
        swap = lambda lst, v: lst[:i] + [v] + lst[i + 1:]
        call(DV_ERR_BAD_ARG, w=swap([_addr(t) for t in ws], None))
        call(DV_ERR_BAD_ARG, pk=swap([_addr(t) for t in packs], None))
        call(DV_ERR_BAD_ARG, N=swap([64] * n, 0))
        call(DV_ERR_BAD_ARG, N=swap([64] * n, -64))
        call(DV_ERR_BAD_ARG, K=swap([64] * n, 0))
        for off in (4, 8, 12):
            call(DV_ERR_BAD_ARG, pk=swap([_addr(t) for t in packs], _addr(packs[i], off)))
    before = L.dv_launch_count()
    call(DV_OK)
    assert L.dv_launch_count() - before == 2


# ---------------------------------------------------------------------------------------------------------------------
# the discriminator node (ops.MlpFn) against fp64 autograd on the kernel's branch
# ---------------------------------------------------------------------------------------------------------------------
MLP_TOL = 5e-6        # outputs and gradients, max error relative to the largest |ref| of the tensor (of the layer);
                      # measured on an H100 (SXM, 700 W): 9e-7 at worst
FLIP_TOL = 1e-3       # a LeakyReLU whose sign differs from fp64: |pre-activation| relative to the layer's mean |pre|


def _run_mlp(x, params, g_out, slope):
    from disvae import ops
    xd = x.cuda().requires_grad_(True)
    pd = [p.detach().cuda().requires_grad_(True) for p in params]
    trace = ops.start_trace()
    try:
        out = ops.MlpFn.apply(xd, slope, *pd)
    finally:
        ops.stop_trace()
    out.backward(g_out.cuda())
    torch.cuda.synchronize()
    return out.detach().cpu(), xd.grad.cpu(), [None if p.grad is None else p.grad.cpu() for p in pd], \
        [t.detach().cpu() for _, t in trace]


@pytest.mark.gpu
@pytest.mark.parametrize("z", [10, 64])
def test_discriminator_node_matches_fp64_on_its_branch(z, monkeypatch):
    """The six-layer FactorVAE discriminator (z -> 1000 x5 -> 2, LeakyReLU 0.2) at M = 512: the logits, every hidden
    activation, dx and every parameter gradient against fp64 autograd of the same layers, with the LeakyReLU branch
    taken from the kernel's own activations; every unit whose branch differs from the fp64 sign must be ambiguous.
    The input-gradient-only backward and the single-stream backward give the same bits."""
    from disvae import ops
    from disvae.models.discriminator import Discriminator
    torch.manual_seed(100 + z)
    disc = Discriminator(latent_dim=z)
    slope = disc.neg_slope
    layers = (disc.lin1, disc.lin2, disc.lin3, disc.lin4, disc.lin5, disc.lin6)
    params = [t.detach().clone() for lay in layers for t in (lay.weight, lay.bias)]
    M = 512
    x = torch.randn(M, z)
    g_out = torch.randn(M, 2)
    out, dx, grads, acts = _run_mlp(x, params, g_out, slope)
    assert len(acts) == 5

    x64 = x.double().requires_grad_(True)
    p64 = [p.double().requires_grad_(True) for p in params]
    h, flips, hidden = x64, 0, []
    for i in range(6):
        pre = h @ p64[2 * i].t() + p64[2 * i + 1]
        if i == 5:
            h = pre
            break
        on = acts[i] > 0
        dis = on != (pre.detach() > 0)
        if dis.any():
            flips += int(dis.sum())
            rel = (pre.detach()[dis].abs().max() / pre.detach().abs().mean()).item()
            assert rel <= FLIP_TOL, "layer %d: a unit took the other branch at |pre| = %.2e of the mean" % (i + 1, rel)
        h = torch.where(on, pre, pre * slope)
        hidden.append(h.detach())
    h.backward(g_out.double())

    def err(a, b, scale=None):
        return ((a.double() - b).abs().max() / (b.abs().max() if scale is None else scale)).item()

    e = {"logits": err(out, h.detach()), "dx": err(dx, x64.grad)}
    for i in range(5):
        e["h%d" % (i + 1)] = err(acts[i], hidden[i])
    for i in range(6):
        scale = max(p64[2 * i].grad.abs().max().item(), p64[2 * i + 1].grad.abs().max().item())
        e["lin%d.weight" % (i + 1)] = err(grads[2 * i], p64[2 * i].grad, scale)
        e["lin%d.bias" % (i + 1)] = err(grads[2 * i + 1], p64[2 * i + 1].grad, scale)
    worst = max(e, key=e.get)
    print("discriminator z=%d M=%d: %d LeakyReLU units off the fp64 branch; worst %s %.2e"
          % (z, M, flips, worst, e[worst]))
    assert e[worst] <= MLP_TOL, "%s: %.2e > %.1e" % (worst, e[worst], MLP_TOL)

    with ops.mlp_input_grad_only():
        out_i, dx_i, grads_i, _ = _run_mlp(x, params, g_out, slope)
    assert all(gr is None for gr in grads_i)
    assert torch.equal(_bits(out_i), _bits(out)) and torch.equal(_bits(dx_i), _bits(dx))

    monkeypatch.setenv("DISVAE_SIDE_STREAM", "0")
    out_s, dx_s, grads_s, _ = _run_mlp(x, params, g_out, slope)
    assert torch.equal(_bits(out_s), _bits(out)) and torch.equal(_bits(dx_s), _bits(dx))
    for a, b in zip(grads_s, grads):
        assert torch.equal(_bits(a), _bits(b))
