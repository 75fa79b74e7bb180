"""The DIP-VAE covariance penalty (csrc/dv_dip.cu: dv_dip_fwd, dv_dip_bwd, dv_dip_workspace_bytes) on every path it can
take, against fp64, through the raw C ABI.

Plan, restated from the kernels (sized for the 132 SMs of an H100 SXM):
- tps = ceil(D / 32) tiles per side, ntiles = tps^2 tiles of 32 x 32 entries of C.  The batch is split into
  want = clamp(min(264 // ntiles, ceil(B / 64)), 1) parts, each rounded up to chunk = 32 ceil(ceil(B / want) / 32)
  rows; nchunks = ceil(B / chunk), the last chunk holds B - (nchunks - 1) chunk rows.
- Workspace, in floats, every piece rounded up to a multiple of 4: counters [ntiles + 1], m1 [D], r [D], v [D],
  C [D][D], chunk partials [nchunks][ntiles][32 x 32], tile (od, dd) [ntiles][2].
- dip_mean_kernel: one CTA of 256 threads per column.  Thread t adds rows t, t + 256, ... in order, a 5-level shuffle
  tree per warp, then the 8 warp sums: m1 = mu_0 + sum(mu - mu_0) / B, then the same for r = sum(mu - m1) / B, and
  v = sum(exp(logvar)) / B (DIP-II).  It also zeroes the ntiles + 1 counters.
- dip_cov_kernel: grid (ntiles, nchunks).  Thread (ty, tx) of a CTA keeps the 4 entries (i0 + ty, j0 + tx + 8q) of its
  tile, one FMA per row of its chunk on c = (mu - m1) - r (0 past column D), and writes them as the chunk's partial.
  The last CTA of a tile (counter cnt[tile] ends at nchunks) adds the chunks in order, divides by B, adds v on the
  diagonal (DIP-II), writes C, and takes the tile's (od, dd): the thread's 4 entries, the CTA tree.  The last tile
  (cnt[ntiles] ends at ntiles) adds the tiles' (od, dd): thread k adds tiles k, k + 256, ..., then the CTA tree.
- dip_bwd_kernel: grid (tps, ceil(B / 32)), one CTA per 32 rows x 32 columns of g_mu: D FMAs of c_bj G_ji in order of
  j, times 2 / B.  g_logvar = (2 g_dd (C_ii - 1)) exp(logvar) / B.

Bounds.  Each element is held to |got - ref| <= tau sum|terms| plus the error it inherits, with the fp64 reference
taken from the same fp32 inputs and tau = u times the longest rounding chain of the plan:
- centring: a_bd = 3 u |c_bd| + tau_mean mean_b |c_bd|, tau_mean = u (ceil(B / 256) + 5 + 3 + 3): the thread's chain,
  the shuffle tree, the 8 warps, the subtraction, the division and u |r| (r is the residual of a mean already accurate
  to the batch's spread).  Neither the column's offset nor row 0 appears in it: the centred batch must not depend on
  where the data sits or which row comes first.
- C_ij: u (rows + nchunks + 1) sum_b |c_bi c_bj| / B (the chunk's FMAs, the chunk adds, the division) plus
  sum_b (a_bi |c_bj| + |c_bi| a_bj + a_bi a_bj) / B; DIP-II adds tau_v mean exp(logvar_i) + u |C_ii| on the diagonal,
  tau_v = u (ceil(B / 256) + 8 + 1 + 4) (the chain, the trees, the division, expf's 2 ulp).
- od, dd: u (5 + 8 + ceil(ntiles / 256) + 8) sum C_ij^2 (the thread's 4 entries, the CTA tree, the tiles' chain, the
  CTA tree) plus what C's bound carries into each square; dd one u more for C_ii - 1.
- g_mu: (2 / B) [u (D + 3) sum_j |c_bj G_ji| + sum_j a_bj (|G_ji| + dG_ji) + sum_j |c_bj| dG_ji] with
  dG = 2 |g| bound(C) + 2 u |G| (the D FMAs, 2 / B and its product; C's error carried into G).
- g_logvar: (8 u |G_ii| + 2 |g_dd| bound(C_ii)) exp(logvar) / B.
The whole-tensor checks of the earlier tests (1e-5 of max |ref|) stay as well, where they ran.  The CPU section runs
an fp32 simulation of the plan: it passes every bound, and a dropped or doubled chunk partial, a dropped tile of
(od, dd), a ragged last tile read past column D, DIP-II without v, g_logvar without its 1 / B and the row-0 centring
the kernel had before (which rounds every row at the scale of an outlier in row 0) each break one.

Buffers.  Every operand starts 16 bytes into a NaN-filled allocation with sentinel words after it; strided inputs have
NaN in every unused slot; the workspace starts as 0xFF bytes (counters 0xFFFFFFFF, partials NaN).  Every call runs
twice on the same workspace and must repeat bit for bit, and must equal a call on a zeroed workspace.  Each GPU case
prints its worst error as a fraction of its bound (pytest -s)."""
import math

import numpy as np
import pytest
import torch

U = 2.0 ** -24              # fp32 unit roundoff
TINY = 2.0 ** -149          # smallest fp32 subnormal
SM_COUNT = 132              # kNumSMs in csrc/dv_common.cuh
TILE, THREADS = 32, 256
TARGET_CTAS = 2 * SM_COUNT  # kDipTargetCtas
MIN_CHUNK = 64              # kDipMinChunk
MAX_B = 65535 * TILE        # kDipMaxB: the backward's grid y is ceil(B / 32)
DIP_I, DIP_II = 1, 2
GUARD = 1024                # words of sentinel after each output
SENTINEL = 0x7FBADBAD       # a NaN bit pattern no kernel writes
OFF = 4                     # floats: every operand starts 16 bytes into its allocation
DV_OK, DV_ERR_BAD_SHAPE, DV_ERR_BAD_ARG = 0, -1, -2
WHOLE_TOL = 1e-5            # the earlier tests' whole-tensor tolerance, at their shapes, regimes and g_terms:
OLD_SHAPES = {(1, 10), (2, 10), (33, 7), (64, 10), (1000, 10), (1024, 10), (256, 64), (2048, 64), (1024, 1),
              (512, 1024)}
OLD_REGIMES = {"normal", "offset", "collapsed", "collinear", "wide_logvar"}
G_TERMS = [(0.7, 1.3), (0.0, 1.0), (1.0, 0.0), (-0.3, -1.7)]


def _cdiv(a, b):
    return -(-a // b)


def _round4(n):
    return (n + 3) & ~3


# ---------------------------------------------------------------------------------------------------------------------
# plan and rounding chains
# ---------------------------------------------------------------------------------------------------------------------
def dip_plan(B, D):
    tps = _cdiv(D, TILE)
    ntiles = tps * tps
    want = max(min(TARGET_CTAS // ntiles, _cdiv(B, MIN_CHUNK)), 1)
    chunk = _cdiv(_cdiv(B, want), TILE) * TILE
    nchunks = _cdiv(B, chunk)
    p = dict(tps=tps, ntiles=ntiles, chunk=chunk, nchunks=nchunks, last=B - (nchunks - 1) * chunk)
    p["m"] = _round4(ntiles + 1)
    p["r"] = p["m"] + _round4(D)
    p["v"] = p["r"] + _round4(D)
    p["c"] = p["v"] + _round4(D)
    p["part"] = p["c"] + _round4(D * D)
    p["red"] = p["part"] + nchunks * ntiles * TILE * TILE
    p["total"] = p["red"] + _round4(2 * ntiles)
    return p


def tau_mean(B):
    return U * (_cdiv(B, THREADS) + 5 + 3 + 3)


def tau_v(B):
    return U * (_cdiv(B, THREADS) + 8 + 1 + 4)


def tau_cov(B, p):
    return U * (min(p["chunk"], B) + p["nchunks"] + 1)


def tau_od(p):
    return U * (5 + 8 + _cdiv(p["ntiles"], THREADS) + 8)


# ---------------------------------------------------------------------------------------------------------------------
# fp64 reference and bounds (device-agnostic: the GPU cases run them on the device, the CPU section on the host)
# ---------------------------------------------------------------------------------------------------------------------
class Ref:
    def __init__(self, mu, lv, dip_type):
        B, D = mu.shape
        self.B, self.D, self.dip_type, self.p = B, D, dip_type, dip_plan(B, D)
        m = mu.double()
        self.mean = m.mean(0)
        c = m - self.mean
        ac = c.abs()
        self.c, self.ac = c, ac
        self.mac = ac.mean(0)                                             # mean_b |c_bd|
        a = 3 * U * ac + tau_mean(B) * self.mac                           # centring allowance
        self.a = a
        C = c.t() @ c / B
        Cb = tau_cov(B, self.p) * (ac.t() @ ac) / B + (a.t() @ ac + ac.t() @ a + a.t() @ a) / B + 2 * TINY * B
        self.e = lv.double().exp()
        if dip_type == DIP_II:
            self.vref = self.e.mean(0)
            self.vb = tau_v(B) * self.vref
            C = C + torch.diag(self.vref)
            Cb = Cb + torch.diag(self.vb + U * C.diagonal().abs())
        self.C, self.Cb = C, Cb
        eye = torch.eye(D, dtype=torch.bool, device=C.device)
        off = ~eye
        d = C.diagonal() - 1
        db = Cb.diagonal()
        self.od = (C[off] ** 2).sum().item()
        self.dd = (d ** 2).sum().item()
        self.od_b = tau_od(self.p) * self.od + (2 * C.abs() * Cb + Cb ** 2)[off].sum().item() + 2 * TINY
        self.dd_b = (tau_od(self.p) + U) * self.dd + (2 * d.abs() * db + db ** 2).sum().item() + 2 * TINY
        self.eye = eye

    def grads(self, g_terms):
        """(g_mu, bound, g_logvar, bound) in fp64 for the upstream gradient g_terms = (g_od, g_dd)."""
        g_od, g_dd = (float(np.float32(g)) for g in g_terms)
        B, D, C, Cb = self.B, self.D, self.C, self.Cb
        G = torch.where(self.eye, 2 * g_dd * (C - 1), 2 * g_od * C)
        dG = torch.where(self.eye, 2 * abs(g_dd) * Cb, 2 * abs(g_od) * Cb) + 2 * U * G.abs()
        aG = G.abs()
        g_mu = (2.0 / B) * (self.c @ G)
        b_mu = (2.0 / B) * (U * (D + 3) * (self.ac @ aG) + self.a @ (aG + dG) + self.ac @ dG) + 2 * TINY * D
        if self.dip_type == DIP_II:
            Gd, dGd = G.diagonal(), dG.diagonal()
            g_lv = Gd * self.e / B
            b_lv = (8 * U * Gd.abs() + dGd) * self.e / B + 2 * TINY
        else:
            g_lv = torch.zeros_like(g_mu)
            b_lv = torch.zeros_like(g_mu)
        return g_mu, b_mu, g_lv, b_lv


def ratio(got, ref, bound):
    """|got - ref| / bound per entry; 0 where they are equal, infinite where got is not finite."""
    got = got.double().to(ref.device) if torch.is_tensor(got) else torch.tensor(float(got), dtype=torch.float64)
    ref = ref if torch.is_tensor(ref) else torch.tensor(float(ref), dtype=torch.float64)
    bound = bound if torch.is_tensor(bound) else torch.tensor(float(bound), dtype=torch.float64)
    got, ref, bound = got.to(ref.device), ref, bound.to(ref.device)
    err = (got - ref).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    return torch.where(torch.isfinite(got), r, torch.full_like(r, math.inf))


def worst(ref, terms, C, grads):
    """Worst ratio to the bound of each output: terms (od, dd), C [D, D], grads {g_terms: (g_mu, g_logvar)}."""
    w = dict(od=ratio(terms[0], torch.tensor(ref.od), ref.od_b).item(),
             dd=ratio(terms[1], torch.tensor(ref.dd), ref.dd_b).item(),
             C=ratio(C, ref.C, ref.Cb).max().item(), g_mu=0.0, g_lv=0.0)
    for gt, (g_mu, g_lv) in grads.items():
        r_mu, b_mu, r_lv, b_lv = ref.grads(gt)
        w["g_mu"] = max(w["g_mu"], ratio(g_mu, r_mu, b_mu).max().item())
        w["g_lv"] = max(w["g_lv"], ratio(g_lv, r_lv, b_lv).max().item())
    return w


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
REGIMES = ["normal", "offset", "collapsed", "collinear", "inactive", "wide_logvar", "big", "small",
           "outlier1e2_row0", "outlier1e4_row0", "outlier1e2_late", "outlier1e4_late"]


def make_inputs(B, D, regime, seed):
    """(mu, logvar) fp32 [B, D] on the host.  normal: randn; offset: 100 + 0.01 randn; collapsed: column D // 2 all
    3.25; collinear: every column the first plus 1e-3 randn; inactive: a trained model's unused dimensions, 0.5 +
    1e-4 randn; wide_logvar: logvar uniform in [-20, 10]; big / small: randn times 1e4 / 1e-4; outlier*: randn with
    row 0 (row_0) or row 2B / 3 (late) moved 1e2 or 1e4 standard deviations off."""
    g = torch.Generator().manual_seed(seed)
    mu = torch.randn(B, D, generator=g)
    lv = 0.5 * torch.randn(B, D, generator=g)
    if regime == "offset":
        mu = 100 + 0.01 * torch.randn(B, D, generator=g)
    elif regime == "collapsed":
        mu[:, D // 2] = 3.25
    elif regime == "collinear":
        mu[:, 1:] = mu[:, :1] + 1e-3 * torch.randn(B, D - 1, generator=g)
    elif regime == "inactive":
        mu = 0.5 + 1e-4 * torch.randn(B, D, generator=g)
    elif regime == "wide_logvar":
        lv = torch.rand(B, D, generator=g) * 30 - 20
    elif regime == "big":
        mu = mu * 1e4
    elif regime == "small":
        mu = mu * 1e-4
    elif regime.startswith("outlier"):
        row = 0 if regime.endswith("row0") else 2 * B // 3
        mu[row] += 1e2 if "1e2" in regime else 1e4
    return mu, lv


# ---------------------------------------------------------------------------------------------------------------------
# fp32 simulation of the plan (CPU), with the faults the bounds must catch
# ---------------------------------------------------------------------------------------------------------------------
F32, F64 = np.float32, np.float64


def _block_sum(t):
    """t [256, n] fp32 per thread -> [n]: the 5-level shuffle tree of each warp, then the 8 warp sums (warp 0's tree
    over 8 values and 24 zeros)."""
    w = t.reshape(8, 32, -1)
    for h in (16, 8, 4, 2, 1):
        w = w[:, :h] + w[:, h:2 * h]
    w = w[:, 0]
    for h in (4, 2, 1):
        w = w[:h] + w[h:2 * h]
    return w[0]


def _col_sum(x):
    """dip_mean_kernel's sum of each column of x [B, D] fp32: thread t adds rows t, t + 256, ... in order."""
    B, D = x.shape
    xp = np.zeros((_cdiv(B, THREADS) * THREADS, D), F32)
    xp[:B] = x
    t = np.zeros((THREADS, D), F32)
    for blk in xp.reshape(-1, THREADS, D):
        t = t + blk
    return _block_sum(t)


def _fma(acc, a, b):
    return (acc.astype(F64) + a.astype(F64) * b.astype(F64)).astype(F32)


def simulate(mu, lv, dip_type, g_list, centring="accurate", fault=None):
    """fp32 run of the restated plan -> (terms (od, dd), C [D, D], {g_terms: (g_mu, g_logvar)}), numpy.
    fault: None | 'drop_chunk0' | 'drop_chunk_last' | 'double_chunk' | 'drop_tile' | 'ragged_cov' | 'ragged_bwd' |
    'no_v' | 'g_logvar_no_div'.  centring: 'accurate' (m1 and r) | 'row0' (the earlier c = (mu - mu_0) - r)."""
    mu, lv = mu.numpy().astype(F32), lv.numpy().astype(F32)
    B, D = mu.shape
    p = dip_plan(B, D)
    s = mu[0]
    if centring == "row0":
        r = _col_sum(mu - s) / F32(B)
        cen = (mu - s) - r
    else:
        m1 = s + _col_sum(mu - s) / F32(B)
        r = _col_sum(mu - m1) / F32(B)
        cen = (mu - m1) - r
    v = _col_sum(np.exp(lv)) / F32(B) if dip_type == DIP_II else np.zeros(D, F32)
    Dp = p["tps"] * TILE
    # column D + k of row b past the last column: what a contiguous [B, D] layout holds there (the next row's values)
    flat = cen.reshape(-1)
    garbage = flat[(np.arange(B)[:, None] * D + D + np.arange(Dp - D)[None, :]) % flat.size]

    def padded(ragged):
        X = np.zeros((p["nchunks"] * p["chunk"], Dp), F32)
        X[:B, :D] = cen
        if ragged:
            X[:B, D:] = garbage
        return X
    # (1) chunk partials, (2) chunk sums in order
    Xc = padded(fault == "ragged_cov").reshape(p["nchunks"], p["chunk"], Dp)
    part = np.zeros((p["nchunks"], Dp, Dp), F32)
    for k in range(p["chunk"]):
        part = _fma(part, Xc[:, k, :, None], Xc[:, k, None, :])
    if fault == "drop_chunk0":
        part[0] = 0
    elif fault == "drop_chunk_last":
        part[-1] = 0
    elif fault == "double_chunk":
        part[p["nchunks"] // 2] *= 2
    acc = np.zeros((Dp, Dp), F32)
    for q in range(p["nchunks"]):
        acc = acc + part[q]
    C = acc / F32(B)
    if dip_type == DIP_II and fault != "no_v":
        C[np.arange(D), np.arange(D)] += v
    # (3) od, dd: per tile the thread's 4 entries, the CTA tree; then the tiles' chain and the CTA tree
    lim = Dp if fault == "ragged_cov" else D
    I, J = np.meshgrid(np.arange(Dp), np.arange(Dp), indexing="ij")
    inside = (I < lim) & (J < lim)
    od_e = np.where(inside & (I != J), C * C, F32(0)).astype(F32)
    dd_e = np.where(inside & (I == J), (C - F32(1)) * (C - F32(1)), F32(0)).astype(F32)
    tps, ntiles = p["tps"], p["ntiles"]

    def tiles(e):
        t = e.reshape(tps, TILE, tps, 4, 8).transpose(0, 2, 1, 4, 3).reshape(ntiles, THREADS, 4)
        o = np.zeros((ntiles, THREADS), F32)
        for q in range(4):
            o = o + t[:, :, q]
        red = _block_sum(o.T)
        if fault == "drop_tile":
            red[-1] = 0
        k = np.zeros(_cdiv(ntiles, THREADS) * THREADS, F32)
        k[:ntiles] = red
        acc_t = np.zeros(THREADS, F32)
        for blk in k.reshape(-1, THREADS):
            acc_t = acc_t + blk
        return _block_sum(acc_t[:, None])[0]
    terms = (tiles(od_e), tiles(dd_e))
    # backward
    grads = {}
    Xb = padded(fault == "ragged_bwd")[:B]
    Cb = C.copy()
    if fault == "ragged_bwd":             # C past column D as the covariance kernel would form it from those reads
        Cg = (Xb.astype(F64).T @ Xb.astype(F64) / B).astype(F32)
        Cb[D:, :] = Cg[D:, :]
        Cb[:, D:] = Cg[:, D:]
    else:
        Cb[D:, :] = 0
        Cb[:, D:] = 0
    for gt in g_list:
        god2, gdd2 = F32(2) * F32(gt[0]), F32(2) * F32(gt[1])
        G = np.where(I == J, gdd2 * (Cb - F32(1)), god2 * Cb).astype(F32)
        if fault != "ragged_bwd":
            G[D:, :] = 0
            G[:, D:] = 0
        a = np.zeros((B, Dp), F32)
        for j in range(Dp):
            a = _fma(a, Xb[:, j, None], G[j, None, :])
        g_mu = a[:, :D] * (F32(2) / F32(B))
        if dip_type == DIP_II:
            gii = gdd2 * (C[np.arange(D), np.arange(D)] - F32(1))
            g_lv = gii * np.exp(lv)
            if fault != "g_logvar_no_div":
                g_lv = g_lv / F32(B)
        else:
            g_lv = np.zeros((B, D), F32)
        grads[gt] = (torch.from_numpy(g_mu), torch.from_numpy(g_lv.astype(F32)))
    return (float(terms[0]), float(terms[1])), torch.from_numpy(C[:D, :D].copy()), grads


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the plan restatement, and the bounds have teeth
# ---------------------------------------------------------------------------------------------------------------------
# (B, D): (tps, ntiles, chunk, nchunks, rows of the last chunk), worked out by hand from dip_plan in csrc/dv_dip.cu
PLAN_TABLE = {
    (1, 1): (1, 1, 32, 1, 1), (1, 10): (1, 1, 32, 1, 1), (2, 10): (1, 1, 32, 1, 2), (33, 7): (1, 1, 64, 1, 33),
    (64, 10): (1, 1, 64, 1, 64), (65, 10): (1, 1, 64, 2, 1), (1000, 10): (1, 1, 64, 16, 40),
    (1024, 1): (1, 1, 64, 16, 64), (1024, 10): (1, 1, 64, 16, 64), (2048, 10): (1, 1, 64, 32, 64),
    (256, 64): (2, 4, 64, 4, 64), (2048, 64): (2, 4, 64, 32, 64), (1024, 33): (2, 4, 64, 16, 64),
    (777, 65): (3, 9, 64, 13, 9), (4096, 100): (4, 16, 256, 16, 256), (512, 1024): (32, 1024, 512, 1, 512),
    (4096, 1024): (32, 1024, 4096, 1, 4096), (1024, 1000): (32, 1024, 1024, 1, 1024),
    (MAX_B, 10): (1, 1, 7968, 264, 1536),
}
SHAPES = list(PLAN_TABLE)


@pytest.mark.parametrize("B,D", SHAPES, ids=["%dx%d" % s for s in SHAPES])
def test_plan_restatement(B, D):
    p = dip_plan(B, D)
    assert (p["tps"], p["ntiles"], p["chunk"], p["nchunks"], p["last"]) == PLAN_TABLE[(B, D)]
    assert 1 <= p["last"] <= p["chunk"] and p["chunk"] % TILE == 0
    assert _cdiv(B, TILE) <= 65535                       # the backward's grid y
    offs = [p[k] for k in ("m", "r", "v", "c", "part", "red", "total")]
    assert all(o % 4 == 0 for o in offs) and offs == sorted(offs)


def test_workspace_bytes_match_the_plan():
    """The library's workspace query against the restated layout (a host function: no device needed)."""
    from disvae import _native as N
    L = N.lib()
    for B, D in SHAPES + [(3, 31), (129, 32), (MAX_B, 1024), (1, 1024), (7000, 513)]:
        assert L.dv_dip_workspace_bytes(B, D) == 4 * dip_plan(B, D)["total"], (B, D)
    for B, D in ((0, 10), (-1, 10), (10, 0), (10, 1025), (MAX_B + 1, 10), (2 ** 31 - 1, 1)):
        assert L.dv_dip_workspace_bytes(B, D) == 0, (B, D)


TEETH = [(33, 7, "normal"), (65, 10, "normal"), (1000, 10, "normal"), (1024, 10, "offset"), (256, 64, "normal"),
         (1024, 33, "normal"), (777, 65, "collinear"), (1024, 10, "outlier1e4_row0"), (2048, 64, "outlier1e4_row0"),
         (1024, 10, "outlier1e2_row0")]
FAULTS = ["drop_chunk0", "drop_chunk_last", "double_chunk", "drop_tile", "ragged_cov", "ragged_bwd", "no_v",
          "g_logvar_no_div"]


def _sim_worst(mu, lv, dip_type, ref, **kw):
    terms, C, grads = simulate(mu, lv, dip_type, G_TERMS[:1], **kw)
    return worst(ref, terms, C, grads)


@pytest.mark.parametrize("B,D,regime", TEETH, ids=["%dx%d-%s" % t for t in TEETH])
def test_bounds_catch_faults_of_the_plan(B, D, regime):
    """The fp32 simulation of the plan passes every bound; each fault a kernel could have breaks one of them."""
    mu, lv = make_inputs(B, D, regime, seed=B * 31 + D)
    p = dip_plan(B, D)
    for dip_type in (DIP_I, DIP_II):
        ref = Ref(mu, lv, dip_type)
        w = _sim_worst(mu, lv, dip_type, ref)
        assert max(w.values()) <= 1, ("the plan itself", dip_type, w)
        for fault in FAULTS:
            if fault in ("drop_chunk_last", "double_chunk") and p["nchunks"] == 1:
                continue
            if fault == "drop_tile" and p["ntiles"] == 1:
                continue
            if fault.startswith("ragged") and D % TILE == 0:
                continue
            if fault in ("no_v", "g_logvar_no_div") and dip_type == DIP_I:
                continue
            w = _sim_worst(mu, lv, dip_type, ref, fault=fault)
            assert max(w.values()) > 1, (fault, dip_type, w)
        if "row0" in regime:
            w = _sim_worst(mu, lv, dip_type, ref, centring="row0")
            assert w["g_mu"] > 1, ("row-0 centring", dip_type, w)
            # the outlier moved to a later row: the row-0 centring passes there, the bound is not the difference
            late = make_inputs(B, D, regime.replace("row0", "late"), seed=B * 31 + D)
            assert max(_sim_worst(*late, dip_type, Ref(*late, dip_type), centring="row0").values()) <= 1


def test_permuted_batch_stays_within_bound_cpu():
    """The simulation of a batch with its outlier first and of the same rows in another order both pass."""
    mu, lv = make_inputs(1024, 10, "outlier1e4_row0", seed=3)
    perm = torch.randperm(1024, generator=torch.Generator().manual_seed(4))
    for m, l in ((mu, lv), (mu[perm], lv[perm])):
        assert max(_sim_worst(m, l, DIP_II, Ref(m, l, DIP_II)).values()) <= 1


# ---------------------------------------------------------------------------------------------------------------------
# device buffers and raw calls
# ---------------------------------------------------------------------------------------------------------------------
LAYOUTS = ["interleaved", "contiguous", "padded", "colmajor"]


def layout_strides(layout, B, D):
    """(ld, row_stride, mu and logvar share one allocation at offsets 0 and 1)."""
    return {"interleaved": (2, 2 * D, True), "contiguous": (1, D, False), "padded": (3, 3 * D + 5, True),
            "colmajor": (B, 1, False)}[layout]


def _bits(t):
    return t.contiguous().view(torch.int32)


def _place(ts, ld, rs):
    """Device allocation holding the [B, D] tensors ts at offsets 0, 1, ... of element (b, d) = b rs + d ld, 16 bytes
    in, NaN in every other word and GUARD NaN after -> (buffer, element offsets)."""
    B, D = ts[0].shape
    idx = (torch.arange(B, device="cuda")[:, None] * rs + torch.arange(D, device="cuda")[None, :] * ld)
    n = (B - 1) * rs + (D - 1) * ld + len(ts)
    buf = torch.full((OFF + n + GUARD,), float("nan"), device="cuda")
    for k, t in enumerate(ts):
        buf[OFF + k + idx] = t.to("cuda")
    return buf


def _output(n, fill=float("nan")):
    buf = torch.full((OFF + n + GUARD,), fill, device="cuda")
    _bits(buf)[:OFF] = SENTINEL
    _bits(buf)[OFF + n:] = SENTINEL
    return buf


def _workspace(n, byte):
    buf = _output(n)
    buf.view(torch.uint8)[4 * OFF:4 * (OFF + n)] = byte
    return buf


def _addr(buf, shift=0):
    return None if buf is None else buf.data_ptr() + 4 * OFF + 4 * shift


def _intact(buf, n):
    b = _bits(buf)
    return bool((b[:OFF] == SENTINEL).all()) and bool((b[OFF + n:] == SENTINEL).all())


def _body(buf, n):
    return buf[OFF:OFF + n]


def _lib():
    from disvae import _native as N
    return N.lib(), N.stream()


def _launch(n_kernels, name, *args):
    L, _ = _lib()
    before = L.dv_launch_count()
    rc = getattr(L, name)(*args)
    assert rc == DV_OK, (name, rc)
    assert L.dv_launch_count() - before == n_kernels, name
    torch.cuda.synchronize()


def _same(a, b, tag):
    assert torch.equal(_bits(a), _bits(b)), tag + ": differs bit for bit"


class Case:
    """One (mu, logvar, layout, dip type) on guarded device buffers."""

    def __init__(self, mu, lv, dip_type, layout):
        self.B, self.D = B, D = mu.shape
        self.dip_type, self.p = dip_type, dip_plan(B, D)
        self.ld, self.rs, shared = layout_strides(layout, B, D)
        if shared:
            self.buf_mu = _place([mu, lv], self.ld, self.rs)
            self.mu_ptr, self.lv_ptr = _addr(self.buf_mu), _addr(self.buf_mu, 1)
            self.bufs = [self.buf_mu]
        else:
            b_mu, b_lv = _place([mu], self.ld, self.rs), _place([lv], self.ld, self.rs)
            self.mu_ptr, self.lv_ptr = _addr(b_mu), _addr(b_lv)
            self.bufs = [b_mu, b_lv]
        self.ws_n = self.p["total"]
        assert _lib()[0].dv_dip_workspace_bytes(B, D) == 4 * self.ws_n

    def fwd(self, ws):
        terms = _output(2)
        _launch(2, "dv_dip_fwd", self.mu_ptr, self.lv_ptr, self.ld, self.rs, self.B, self.D, self.dip_type,
                _addr(terms), _addr(ws), _lib()[1])
        assert _intact(terms, 2) and _intact(ws, self.ws_n), "dv_dip_fwd wrote past a buffer"
        return _body(terms, 2).clone()

    def bwd(self, ws, g_terms, want_mu=True, want_lv=True):
        n = self.B * self.D
        gt = _place([torch.tensor([g_terms], dtype=torch.float32)], 1, 2)
        g_mu = _output(n) if want_mu else None
        g_lv = _output(n) if want_lv else None
        _launch(1 if (want_mu or want_lv) else 0, "dv_dip_bwd", self.mu_ptr, self.lv_ptr, self.ld, self.rs, self.B,
                self.D, self.dip_type, _addr(gt), _addr(g_mu), _addr(g_lv), _addr(ws), _lib()[1])
        for g in (g_mu, g_lv):
            assert g is None or _intact(g, n), "dv_dip_bwd wrote past an output"
        return tuple(None if g is None else _body(g, n).view(self.B, self.D) for g in (g_mu, g_lv))

    def ws_parts(self, ws):
        """The words of the workspace a forward writes: counters, m1, r, v, C, partials, tile (od, dd)."""
        p, D, body = self.p, self.D, _body(ws, self.ws_n)
        return [body[:p["ntiles"] + 1], body[p["m"]:p["m"] + D], body[p["r"]:p["r"] + D], body[p["v"]:p["v"] + D],
                body[p["c"]:p["c"] + D * D], body[p["part"]:p["red"]], body[p["red"]:p["red"] + 2 * p["ntiles"]]]


def run_case(mu, lv, dip_type, layout, tag, g_list=G_TERMS, outputs=True, whole=False):
    """Every check of one case; returns the worst ratios to the bounds.  whole: also the earlier tests' whole-tensor
    checks (with g_terms = (0.7, 1.3); elsewhere a G_ii = 2 g_dd (C_ii - 1) that cancels can put the largest relative
    error on the largest gradient, which the per-element bound allows)."""
    B, D = mu.shape
    case = Case(mu, lv, dip_type, layout)
    p = case.p
    ws = _workspace(case.ws_n, 0xFF)
    terms = case.fwd(ws)
    first = [x.clone() for x in case.ws_parts(ws)]
    _same(terms, case.fwd(ws), tag + " terms on a reused workspace")
    for a, b in zip(first, case.ws_parts(ws)):
        _same(a, b, tag + " workspace on a reused workspace")
    cnt, m1, r, v, C, _, _ = case.ws_parts(ws)
    cnt = _bits(cnt)
    assert (cnt[:p["ntiles"]] == p["nchunks"]).all() and cnt[p["ntiles"]].item() == p["ntiles"], (tag, cnt)
    C = C.view(D, D)
    assert torch.equal(_bits(C), _bits(C.t())), tag + ": C is not exactly symmetric"
    ws0 = _workspace(case.ws_n, 0)
    _same(terms, case.fwd(ws0), tag + " terms on a zeroed workspace")
    for a, b in zip(case.ws_parts(ws), case.ws_parts(ws0)):
        _same(a, b, tag + " workspace on a zeroed workspace")

    ref = Ref(mu.cuda(), lv.cuda(), dip_type)
    grads = {}
    for gt in g_list:
        g_mu, g_lv = case.bwd(ws, gt)
        again = case.bwd(ws, gt)
        zeroed = case.bwd(ws0, gt)
        for x, y, what in zip((g_mu, g_lv) * 2, again + zeroed, ["repeat"] * 2 + ["zeroed workspace"] * 2):
            _same(x, y, "%s g_terms %s: %s" % (tag, gt, what))
        if outputs:
            _same(case.bwd(ws, gt, want_lv=False)[0], g_mu, tag + ": g_mu alone")
            _same(case.bwd(ws, gt, want_mu=False)[1], g_lv, tag + ": g_logvar alone")
        if dip_type == DIP_I:
            assert not _bits(g_lv).any(), tag + ": DIP-I writes +0 to g_logvar"
        if B == 1:
            assert not g_mu.any(), tag + ": the covariance of one row is 0"
        grads[gt] = (g_mu, g_lv)
        if not (whole and gt == G_TERMS[0]):
            continue
        r_mu, _, r_lv, _ = ref.grads(gt)
        for got, want, what in ((g_mu, r_mu, "g_mu"), (g_lv, r_lv, "g_logvar")):
            err = (got.double() - want).abs().max().item()
            assert err <= WHOLE_TOL * want.abs().max().item(), "%s %s: whole-tensor %.3e" % (tag, what, err)
    if outputs:
        case.bwd(ws, g_list[0], want_mu=False, want_lv=False)
    for got, want, what in ((terms[0], ref.od, "od"), (terms[1], ref.dd, "dd")):
        assert not whole or abs(got.item() - want) <= WHOLE_TOL * max(abs(want), 1.0), "%s %s: whole" % (tag, what)

    w = worst(ref, terms.cpu(), C, grads)
    # m1 + r is the mean the batch was centred on, v the mean of exp(logvar)
    rd = r.double().abs()
    w["r"] = ratio(m1.double() + r.double(), ref.mean,
                   tau_mean(B) * (ref.mac + rd) + 2 * U * rd + 2 * TINY).max().item()
    if dip_type == DIP_II:
        w["v"] = ratio(v, ref.vref, ref.vb + 2 * TINY).max().item()
    else:
        assert not _bits(v).any(), tag + ": DIP-I writes v = 0"
    print("%s: worst |err| / bound %s" % (tag, " ".join("%s %.3f" % kv for kv in w.items())))
    assert max(w.values()) <= 1, (tag, w)
    return w


# ---------------------------------------------------------------------------------------------------------------------
# GPU cases
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("dip_type", [DIP_I, DIP_II], ids=["I", "II"])
@pytest.mark.parametrize("B,D", SHAPES, ids=["%dx%d" % s for s in SHAPES])
def test_shapes_and_layouts(B, D, dip_type, layout):
    mu, lv = make_inputs(B, D, "normal", seed=B * 7919 + D)
    run_case(mu, lv, dip_type, layout, "dip%s %dx%d %s" % ("I" * dip_type, B, D, layout), whole=(B, D) in OLD_SHAPES)


REGIME_SHAPES = [(1, 10), (2, 10), (33, 7), (64, 10), (1000, 10), (1024, 10), (2048, 10), (256, 64), (2048, 64),
                 (1024, 1), (1024, 33), (777, 65), (512, 1024)]


@pytest.mark.gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("dip_type", [DIP_I, DIP_II], ids=["I", "II"])
@pytest.mark.parametrize("B,D", REGIME_SHAPES, ids=["%dx%d" % s for s in REGIME_SHAPES])
def test_regimes(B, D, dip_type, regime):
    """Every input regime on the encoder's interleaved layout, then the same rows in a seeded random order."""
    if regime == "wide_logvar" and dip_type == DIP_I:
        pytest.skip("DIP-VAE-I does not read logvar")
    if regime == "collinear" and D < 2:
        pytest.skip("one column")
    if regime.endswith("late") and B < 3:
        pytest.skip("no later row")
    mu, lv = make_inputs(B, D, regime, seed=B * 7919 + D + len(regime))
    tag = "dip%s %dx%d %s" % ("I" * dip_type, B, D, regime)
    whole = (B, D) in OLD_SHAPES and regime in OLD_REGIMES
    run_case(mu, lv, dip_type, "interleaved", tag, whole=whole)
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(B + D))
    run_case(mu[perm], lv[perm], dip_type, "interleaved", tag + " permuted", outputs=False, whole=whole)


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["outlier1e2_row0", "outlier1e4_row0"])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_outlier_row0_on_every_layout(layout, regime):
    """A first row 1e2 or 1e4 standard deviations off, at the c2 and z64 training shapes, on every layout."""
    for B, D in ((1024, 10), (256, 64)):
        mu, lv = make_inputs(B, D, regime, seed=B + D)
        run_case(mu, lv, DIP_II, layout, "dipII %dx%d %s %s" % (B, D, layout, regime), g_list=G_TERMS[:1])


@pytest.mark.gpu
def test_refusals_launch_nothing():
    """Bad shapes, strides and types, and NULL or misaligned pointers, come back as status codes with no launch."""
    L, S = _lib()
    buf = torch.zeros(1 << 16, device="cuda")
    a = buf.data_ptr()
    terms = torch.full((2,), 7.0, device="cuda")
    B, D = 8, 4

    def refused(rc_want, fn, *args):
        before = L.dv_launch_count()
        rc = getattr(L, fn)(*args)
        torch.cuda.synchronize()
        assert rc == rc_want and L.dv_launch_count() == before, (fn, args, rc)

    def fwd(mu=a, lv=a, ld=2, rs=None, B_=B, D_=D, t=1, out=terms.data_ptr(), ws=a):
        return (mu, lv, ld, 2 * D_ if rs is None else rs, B_, D_, t, out, ws, S)

    def bwd(mu=a, lv=a, ld=2, rs=None, B_=B, D_=D, t=2, g=a, gm=a, gl=a, ws=a):
        return (mu, lv, ld, 2 * D_ if rs is None else rs, B_, D_, t, g, gm, gl, ws, S)

    for shape in (dict(B_=0), dict(B_=-1), dict(D_=0), dict(D_=1025), dict(t=0), dict(t=3), dict(ld=0), dict(ld=-1),
                  dict(rs=0), dict(rs=-8), dict(B_=MAX_B + 1), dict(B_=2 ** 31 - 1)):
        refused(DV_ERR_BAD_SHAPE, "dv_dip_fwd", *fwd(**shape))
        refused(DV_ERR_BAD_SHAPE, "dv_dip_bwd", *bwd(**shape))
    for bad in (dict(mu=None), dict(lv=None), dict(out=None), dict(ws=None), dict(mu=a + 2), dict(lv=a + 1),
                dict(out=terms.data_ptr() + 2), dict(ws=a + 4)):
        refused(DV_ERR_BAD_ARG, "dv_dip_fwd", *fwd(**bad))
    for bad in (dict(mu=None), dict(lv=None), dict(g=None), dict(ws=None), dict(g=a + 2), dict(gm=a + 2),
                dict(gl=a + 3), dict(ws=a + 8)):
        refused(DV_ERR_BAD_ARG, "dv_dip_bwd", *bwd(**bad))
    refused(0, "dv_dip_bwd", *bwd(gm=None, gl=None))           # nothing asked for: nothing launched
    assert torch.equal(terms, torch.full((2,), 7.0, device="cuda"))
    for b, d in ((0, 10), (10, 0), (10, 1025), (MAX_B + 1, 10)):
        assert L.dv_dip_workspace_bytes(b, d) == 0
    assert L.dv_dip_workspace_bytes(1, 1) > 0 and L.dv_dip_workspace_bytes(2048, 1024) % 16 == 0
