"""The disentanglement-score kernels (csrc/dv_factor_score.cu: dv_group_variance; csrc/dv_sap.cu: dv_sap_score_matrix;
csrc/dv_beta_vae_score.cu: dv_pair_abs_diff_mean, dv_logistic_fit) on every path they can take, against fp64, through
the raw C ABI.  The earlier tests of these kernels at the shapes a user meets (through the Python wrappers) and their
refusal tests stay in test_{factor,sap,beta_vae}_score_gpu.py, beside each score's known-answer and Evaluator tests;
this file adds the paths those do not reach.

Plans, restated from the kernels (sized for the 132 SMs of an H100 SXM):
- dv_group_variance: 256 threads a CTA, `dt` dim lanes (a power of two, the smallest >= min(D, 32)) times
  lanes = 256 / dt row lanes; dt halves while V * ceil(D / dt) < 264 = 2 x 132.  Votes: grid (V, 1), the CTA walks
  every dim; var only: grid (V, ceil(D / dt)), the last slice ragged when dt does not divide D.  Row lane j adds rows
  j, j + lanes, ... in order; a fixed tree adds the lanes.
- dv_sap_score_matrix: one CTA of 16 warps per (latent, factor); warp w solves problems w, w + 16, ... of the factor's
  nc = clamp(n_classes[k], 0, class_stride) classes (nc problems above two, one for two, none below); the training
  column and labels sit in 5 * num_train + 6208 bytes of dynamic shared memory (170 KB at num_train = 32768).
- dv_logistic_fit: one CTA of 512 threads, nc = clamp(*n_classes, 1, K), R = nc above two, 1 for two, 0 for one, and
  O = R (D + 1) parameters.  A sum over the training rows is cut into S = 1 (O >= 512), min(512 / O, n) segments;
  the training mean likewise with D for O.  Workspace, in doubles: mean [D], ten vectors of K (D + 1), P / Q / U
  [n][K], part [2 max(512, K (D + 1))].

Bound of dv_group_variance.  Per element, with fp64 taken from the same fp32 inputs, e_l = x_l - s (s the group's
first row, as the kernel centres), r = mean_l e_l and c_l = e_l - r:
  |var - var64| <= [tau sum c_l^2 + sum_l (2 |c_l| a_l + a_l^2)] / (L - 1),
  tau = u (ceil(L / lanes) + log2(lanes) + 4),  a_l = u (|e_l| + |c_l|) + tau sum_l |e_l| / L + u |r|:
the lane's chain, the lane tree, the division and the squares; a_l is the centring allowance, from the rounding of e_l
and of r.  Since s is a row of the group, |s - mean| <= sqrt(L sum c^2), so the row-0 shift costs at most about
2 u sqrt(L) sum c^2 there: the kernel keeps its one shift rather than a second centring pass.  The CPU section runs an
fp32 simulation of the plan: it passes the bound, and a dropped or doubled lane partial, a row added twice, a division
by L, a one-pass E[x^2] - E[x]^2 and a missing r each break it.

Votes are checked exactly: the expected vote is the argmin of the fp32 ratio var / global_var, divided by numpy from
the kernel's own var_out (IEEE division: the library is built without fast math), over the dims with global_var >=
min_var and a ratio that is not NaN, lowest d on a tie.

Buffers.  Every operand starts 16 bytes into its allocation with sentinel words before and after it (a NaN pattern for
floating-point data); a strided mu has NaN in every gap; the logistic-fit workspace starts as 0xFF bytes and is exactly
the queried size.  Every call runs twice and must repeat bit for bit, checks its launch count, and leaves every
sentinel intact; one captured CUDA graph per entry point must replay to the eager bits.  Each GPU case prints its
worst error as a fraction of its bound (pytest -s).
"""
import math
import time

import numpy as np
import pytest
import torch

import beta_vae_reference as BR
import sap_reference as SR
from score_kernels import DEV, DV_ERR_WORKSPACE, LAYOUTS, Buf, _bits, _call, _graph_replays, _lib, _same, place_mu

U = 2.0 ** -24               # fp32 unit roundoff
TINY = 2.0 ** -149
SM_COUNT = 132               # kNumSMs in csrc/dv_common.cuh
FS_THREADS, WARP = 256, 32   # kFsThreads, kWarp
SAP_WARPS = 16               # kSapThreads / kWarp
SAP_MAX_TRAIN = 32768
FIT_THREADS = 512            # kFitThreads
MIN_VAR = 0.05               # FACTOR_SCORE_MIN_VAR
SAP_COEF_RTOL, SAP_KKT_TOL, SAP_MARGIN = 1e-7, 1e-8, 1e-7      # as test_sap_score_gpu.py
FIT_COEF_RTOL, FIT_KKT_TOL, FIT_MARGIN = 1e-7, 1e-8, 1e-7      # as test_beta_vae_score_gpu.py


def _cdiv(a, b):
    return -(-a // b)


# ---------------------------------------------------------------------------------------------------------------------
# plans
# ---------------------------------------------------------------------------------------------------------------------
def fs_plan(D, V, votes):
    """(dt, lanes, slices) of dv_group_variance."""
    dt = 1
    while dt < D and dt < WARP:
        dt <<= 1
    while dt > 1 and V * _cdiv(D, dt) < 2 * SM_COUNT:
        dt >>= 1
    return dt, FS_THREADS // dt, 1 if votes else _cdiv(D, dt)


def fs_tau(L, lanes):
    return U * (_cdiv(L, lanes) + int(math.log2(lanes)) + 4)


def segments(O, n):
    """colsum's segment count S."""
    return 1 if O >= FIT_THREADS else min(FIT_THREADS // O, n)


def fit_workspace_doubles(n, D, K):
    OK = K * (D + 1)
    return D + 10 * OK + 3 * n * K + 2 * max(FIT_THREADS, OK)


def sap_smem_bytes(n):
    return 256 * 8 + 256 * 16 + SAP_WARPS * 4 + 5 * n


# ---------------------------------------------------------------------------------------------------------------------
# dv_group_variance: fp64 reference and bound, and the fp32 simulation of the plan
# ---------------------------------------------------------------------------------------------------------------------
def gv_reference(x, rows, lanes):
    """(var64 [V, D], bound [V, D]) in fp64 for fp32 x [N, D] and rows [V, L] (torch, any device), in group chunks."""
    V, L = rows.shape
    D = x.shape[1]
    tau = fs_tau(L, lanes)
    x64 = x.double()
    out, bnd = [], []
    step = max(1, (1 << 24) // (L * D))
    for g0 in range(0, V, step):
        xs = x64[rows[g0:g0 + step]]                           # [v, L, D]
        e = xs - xs[:, :1]
        r = e.mean(1, keepdim=True)
        c = e - r
        s2 = (c * c).sum(1)
        a = U * (e.abs() + c.abs()) + tau * e.abs().mean(1, keepdim=True) + U * r.abs()
        out.append(s2 / (L - 1))
        bnd.append((tau * s2 + (2 * c.abs() * a + a * a).sum(1)) / (L - 1) + 2 * TINY)
    return torch.cat(out), torch.cat(bnd)


F32, F64 = np.float32, np.float64


def _fma32(acc, a, b):
    return (acc.astype(F64) + a.astype(F64) * b.astype(F64)).astype(F32)


def gv_simulate(x, rows, lanes, fault=None):
    """fp32 run of the restated plan -> var [V, D].  fault: None | 'drop_lane' | 'double_lane' | 'row_twice' |
    'div_L' | 'one_pass' | 'no_r'."""
    x = np.asarray(x, F32)
    V, L = rows.shape
    xs = x[rows]                                               # [V, L, D]
    s = xs[:, :1]
    if fault == "row_twice":
        xs = np.concatenate([xs, xs[:, 1:2]], 1)
    Lp = _cdiv(xs.shape[1], lanes) * lanes
    on = np.zeros((V, Lp, 1), bool)
    on[:, :xs.shape[1]] = True
    xp = np.zeros((V, Lp, x.shape[1]), F32)
    xp[:, :xs.shape[1]] = xs

    def tree(part):                                            # part [V, lanes, D]
        if fault == "drop_lane":                               # lane 1: every group has a row 1
            part[:, 1] = 0
        elif fault == "double_lane":
            part[:, 1] *= 2
        h = lanes // 2
        while h:
            part = part[:, :h] + part[:, h:2 * h]
            h //= 2
        return part[:, 0]
    if fault == "one_pass":
        acc = np.zeros((V, lanes, x.shape[1]), F32)
        acc2 = np.zeros_like(acc)
        for blk in range(Lp // lanes):
            v = xp[:, blk * lanes:(blk + 1) * lanes]
            acc = acc + v
            acc2 = _fma32(acc2, v, v)
        sm, sq = tree(acc), tree(acc2)
        return (sq - sm * sm / F32(L)) / F32(L - 1)
    acc = np.zeros((V, lanes, x.shape[1]), F32)
    for blk in range(Lp // lanes):
        sl = slice(blk * lanes, (blk + 1) * lanes)
        acc = acc + np.where(on[:, sl], xp[:, sl] - s, F32(0))
    r = tree(acc) / F32(L)
    if fault == "no_r":
        r = np.zeros_like(r)
    acc = np.zeros((V, lanes, x.shape[1]), F32)
    for blk in range(Lp // lanes):
        sl = slice(blk * lanes, (blk + 1) * lanes)
        c = np.where(on[:, sl], (xp[:, sl] - s) - r[:, None], F32(0))
        acc = _fma32(acc, c, c)
    return tree(acc) / F32(L if fault == "div_L" else L - 1)


def expected_votes(var32, gv32, min_var):
    """Exact votes from the kernel's own fp32 variances: argmin of the IEEE fp32 ratio over the dims with gv >=
    min_var and a ratio that is not NaN, the lowest d on a tie; -1 if none qualifies."""
    var32, gv32 = np.asarray(var32, F32), np.asarray(gv32, F32)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = var32 / gv32[None, :]
    ok = (gv32 >= F32(min_var))[None, :] & ~np.isnan(q)
    qm = np.where(ok, q, np.inf)
    best = qm.min(1, keepdims=True)
    hit = ok & (q == best)
    return np.where(ok.any(1), hit.argmax(1), -1)


def argmin_simulate(q, qualify, rule="fixed"):
    """The kernel's argmin over one group's ratios q [D] (fp32) of dims `qualify` [D] (global_var >= min_var): each
    of the 256 threads scans d = t, t + 256, ..., an xor butterfly per warp, then thread 0 over the 8 warp results.
    rule: 'fixed' (NaN ratios do not qualify) | 'old' (they do) | 'high_tie' (the highest d wins a tie)."""
    def better(ob, oi, best, bi):
        if oi < 0:
            return False
        if bi < 0 or ob < best:
            return True
        return ob == best and (oi > bi if rule == "high_tie" else oi < bi)
    st = []
    for t in range(FS_THREADS):
        best, bi = F32(0), -1
        for d in range(t, len(q), FS_THREADS):
            if not qualify[d] or (rule != "old" and np.isnan(q[d])):
                continue
            if bi < 0 or q[d] < best or (rule == "high_tie" and q[d] == best):
                best, bi = q[d], d
        st.append((best, bi))
    for o in (16, 8, 4, 2, 1):
        st = [st[t ^ o] if better(*st[t ^ o], *st[t]) else st[t] for t in range(FS_THREADS)]
    best, bi = st[0]
    for w in range(1, FS_THREADS // WARP):
        if better(*st[WARP * w], best, bi):
            best, bi = st[WARP * w]
    return bi


# ---------------------------------------------------------------------------------------------------------------------
# checks of the SAP and logistic fits (shared by the GPU cases and the CPU section)
# ---------------------------------------------------------------------------------------------------------------------
def sap_fit_ok(z, want, x, s, c):
    """(w, b) z [P, 2] of problems x, s, c [P, n] against the fp64 solve `want` [P, 2]: coefficient and KKT."""
    err = np.abs(z - want).max(1)
    ref = np.maximum(np.abs(want).max(1), 1e-300)
    g, scale = SR.gradient(z, x, s, c)
    return bool((err <= SAP_COEF_RTOL * ref).all() and (np.abs(g).max(1) <= SAP_KKT_TOL * scale).all())


def fit_ok(W, b, x, y, nc):
    """(W, b) of the logistic fit on x, y against the fp64 solve: coefficient, KKT and sum b = 0 (nc > 2)."""
    wW, wb, _ = BR.fit(x, y, nc)
    ref = max(np.abs(wW).max(), np.abs(wb).max(), 1e-300)
    err = max(np.abs(W - wW).max(), np.abs(b - wb).max())
    _, gr, sc = BR.objective(x, y, nc, W, b)
    ok = err <= FIT_COEF_RTOL * ref and np.abs(gr).max() <= FIT_KKT_TOL * sc.max()
    return bool(ok and (nc <= 2 or abs(b.sum()) <= 1e-12 * ref))


def _minimise(f, z0):
    from scipy.optimize import minimize
    r = minimize(f, z0, method="BFGS", options=dict(gtol=1e-12, maxiter=10000))
    return minimize(f, r.x, method="Nelder-Mead", options=dict(xatol=1e-13, fatol=1e-16, maxiter=20000)).x


def _report(tag, **w):
    print("%s: worst |err| / bound %s" % (tag, " ".join("%s %.3f" % kv for kv in w.items())))


# ---------------------------------------------------------------------------------------------------------------------
# dv_group_variance runs
# ---------------------------------------------------------------------------------------------------------------------
class GvCase:
    """mu placed in one layout, rows and global_var on guarded buffers."""

    def __init__(self, x, rows, layout, gv=None):
        self.N, self.D = x.shape
        self.V, self.L = rows.shape
        self.mu, self.ld, self.rs = place_mu(x, layout)
        self.rows = Buf(self.V * self.L, torch.int64, rows.to(DEV))
        self.gv = None if gv is None else Buf(self.D, torch.float32, torch.as_tensor(gv, dtype=torch.float32).to(DEV))

    def run(self, var=True, votes=False, min_var=MIN_VAR):
        V, D = self.V, self.D
        vo = Buf(V * D, torch.float32, float("nan")) if var else None
        ao = Buf(V, torch.int32, -7) if votes else None
        args = (self.mu.ptr, self.ld, self.rs, self.N, D, self.rows.ptr, V, self.L,
                self.gv.ptr if votes else None, float(min_var), vo.ptr if var else None, ao.ptr if votes else None)
        _call(1, "dv_group_variance", *args, _lib()[1])
        outs = [o for o in (vo, ao) if o is not None]
        first = [o.body.clone() for o in outs]
        _call(1, "dv_group_variance", *args, _lib()[1])
        for f, o in zip(first, outs):
            _same(f, o.body, "dv_group_variance repeat")
            assert o.intact(), "dv_group_variance wrote past an output"
        for b in (self.mu, self.rows) + ((self.gv,) if self.gv is not None else ()):
            assert b.intact()
        self.last = (args, outs)
        return (vo.body.view(V, D).clone() if var else None), (ao.body.clone() if votes else None)

    def graph(self):
        args, outs = self.last
        _graph_replays(lambda: _lib()[0].dv_group_variance(*args, torch.cuda.current_stream().cuda_stream), outs,
                       "dv_group_variance")


def gv_inputs(N, D, V, L, regime, seed):
    """(x fp32 [N, D], rows int64 [V, L]) of one regime: normal; far (100 + 0.01 randn); constant (every third column
    3.25); duplicate (odd columns copy column 0); outlier_row0 (each group's first row 1e3 off in every column)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, D, generator=g, dtype=torch.float64)
    if regime == "far":
        x = 100 + 0.01 * x
    elif regime == "constant":
        x[:, ::3] = 3.25
    elif regime == "duplicate":
        x[:, 1::2] = x[:, :1]
    rows = torch.randint(N, (V, L), generator=g)
    if regime == "outlier_row0":
        out = torch.randint(N, (1,), generator=g).item()
        x[out] += 1e3
        rows[:, 0] = out
    return x.float(), rows


def gv_check(x, rows, layouts, tag, gv=None):
    """Every layout, every output choice: the bound, bit-equality across layouts and outputs, exact votes."""
    V, L = rows.shape
    D = x.shape[1]
    dt, lanes, _ = fs_plan(D, V, False)
    assert fs_plan(D, V, True)[:2] == (dt, lanes)
    want, bound = gv_reference(x.to(DEV), rows.to(DEV), lanes)
    if gv is None:
        gv = np.where(np.arange(D) % 5 == 4, 0.01, 0.5 + np.arange(D) % 7 / 7).astype(F32)   # some dims inactive
    first = None
    for layout in layouts:
        case = GvCase(x, rows, layout, gv)
        var, _ = case.run(var=True)
        var2, votes = case.run(var=True, votes=True)
        _, votes1 = case.run(var=False, votes=True)
        _same(var, var2, "%s %s: var alone vs with votes" % (tag, layout))
        _same(votes, votes1, "%s %s: votes alone vs with var" % (tag, layout))
        if first is None:
            first = (var, votes)
            r = (var.double() - want).abs()
            r = torch.where(r == 0, r, r / bound)
            w = r.max().item()
            _report("%s dt %d" % (tag, dt), var=w)
            assert w <= 1, (tag, layout, w)
            exp = expected_votes(var.cpu().numpy(), gv, MIN_VAR)
            assert np.array_equal(votes.cpu().numpy(), exp), (tag, layout)
        else:
            _same(first[0], var, "%s %s: var vs %s" % (tag, layout, layouts[0]))
            _same(first[1], votes, "%s %s: votes vs %s" % (tag, layout, layouts[0]))
    return case


# (N, D, V, L): every D of the plan's dim-lane choices, V on both sides of the 264-CTA threshold, L across lane counts
GV_SHAPES = [(600, 1, 1, 10000), (600, 2, 1, 2), (600, 3, 263, 3), (600, 31, 264, 255), (600, 32, 263, 256),
             (600, 32, 264, 257), (600, 33, 132, 64), (600, 100, 1, 10000), (600, 255, 2, 256), (600, 256, 15000, 2),
             (600, 257, 3, 255), (600, 1000, 1, 3), (600, 1024, 1, 10000), (600, 1024, 264, 64),
             (3000, 10, 15000, 64), (3000, 1, 15000, 2), (600, 17, 16, 257), (600, 23, 50, 100),
             (600, 30, 100, 40)]
GV_REGIMES = ["normal", "far", "constant", "duplicate", "outlier_row0"]
GV_REGIME_SHAPES = [(2000, 10, 264, 64), (600, 257, 3, 255), (3000, 1, 1, 10000)]


# ---------------------------------------------------------------------------------------------------------------------
# CPU: plans, bounds with teeth, the argmin restatement, fit checks with teeth
# ---------------------------------------------------------------------------------------------------------------------
# (D, V, votes): (dt, lanes, slices), worked out by hand from fs_plan in csrc/dv_factor_score.cu
FS_PLAN_TABLE = {
    (1, 1, False): (1, 256, 1), (3, 263, False): (2, 128, 2), (31, 264, False): (32, 8, 1),
    (32, 263, False): (16, 16, 2), (32, 264, False): (32, 8, 1), (32, 264, True): (32, 8, 1),
    (33, 132, False): (32, 8, 2), (100, 1, False): (1, 256, 100), (257, 3, False): (2, 128, 129),
    (257, 3, True): (2, 128, 1), (1024, 264, False): (32, 8, 32), (17, 16, False): (1, 256, 17), (23, 50, False): (4, 64, 6), (30, 100, False): (8, 32, 4),
    (255, 2, False): (1, 256, 255), (10, 15000, True): (16, 16, 1), (2, 1, False): (1, 256, 2),
}


def test_fs_plan_restatement():
    for (D, V, votes), want in FS_PLAN_TABLE.items():
        assert fs_plan(D, V, votes) == want, (D, V, votes)


def _gv_shapes_branches():
    seen = set()
    for N, D, V, L in GV_SHAPES:
        dt, lanes, slices = fs_plan(D, V, False)
        seen.add(("dt", dt))
        seen.add(("threshold", V * _cdiv(D, 32) >= 2 * SM_COUNT))
        if slices > 1 and D % dt:
            seen.add("ragged slice")
        if slices > 1:
            seen.add("several slices")
        seen.add(("L vs lanes", L % lanes == 0, L > lanes))
    return seen


def test_gpu_cases_hit_every_plan_branch():
    seen = _gv_shapes_branches()
    for dt in (1, 2, 4, 8, 16, 32):
        assert ("dt", dt) in seen, dt
    assert {("threshold", True), ("threshold", False), "ragged slice", "several slices"} <= seen
    assert {("L vs lanes", a, b) for a in (True, False) for b in (True, False)} - {("L vs lanes", True, False)} <= seen
    branches = {"one": False, "ratio": False, "n": False}
    for c in FIT_CASES:
        nc = min(max(c["ncv"], 1), c["K"])
        if nc < 2:
            continue
        O = (nc if nc > 2 else 1) * (c["D"] + 1)
        S = segments(O, c["n"])
        branches["one" if O >= FIT_THREADS else ("n" if S == c["n"] else "ratio")] = True
    assert all(branches.values()), branches
    ncv = {c["ncv"] for c in FIT_CASES}
    assert 0 in ncv and any(c["ncv"] > c["K"] for c in FIT_CASES)
    assert any(c["ncv"] < c["K"] and c["ncv"] >= 2 for c in FIT_CASES)                 # NaN rows of coef
    assert any(c["eval"] == 0 for c in FIT_CASES)
    assert {c["D"] for c in FIT_CASES if c["K"] == 4 and c["ncv"] == 4} >= {126, 127, 128}
    # SAP: one warp per problem and warps taking several, num_train at the shared-memory limit, clamped class counts
    nps = [max(c["nc"]) for c in SAP_CASES]
    assert any(n <= SAP_WARPS for n in nps) and any(n > SAP_WARPS for n in nps)
    assert any(c["n_train"] == SAP_MAX_TRAIN for c in SAP_CASES) and sap_smem_bytes(SAP_MAX_TRAIN) > 48 * 1024 * 3
    assert sap_smem_bytes(8589) > 48 * 1024 >= sap_smem_bytes(8588)
    assert any(c["n_train"] == 8589 for c in SAP_CASES)
    assert any(0 in c["ncv"] for c in SAP_CASES)
    assert any(v > c["cs"] for c in SAP_CASES for v in c["ncv"])
    assert any(c["cs"] > max(c["nc"]) for c in SAP_CASES)


@pytest.mark.parametrize("N,D,V,L,regime", [(500, 3, 6, 257, "normal"), (500, 33, 4, 300, "normal"),
                                            (500, 2, 3, 2000, "far"), (500, 3, 5, 255, "outlier_row0"),
                                            (500, 1, 2, 10000, "normal")])
def test_group_variance_bound_catches_faults(N, D, V, L, regime):
    """The fp32 simulation of the plan passes the bound; each fault breaks it."""
    x, rows = gv_inputs(N, D, V, L, regime, seed=N + D + L)
    rows = rows.numpy()
    lanes = fs_plan(D, V, False)[1]
    want, bound = gv_reference(x, torch.from_numpy(rows), lanes)

    def worst(var):
        err = (torch.from_numpy(np.asarray(var, F32)).double() - want).abs()
        return torch.where(err == 0, err, err / bound).max().item()
    assert worst(gv_simulate(x.numpy(), rows, lanes)) <= 1
    faults = ["drop_lane", "double_lane", "row_twice", "div_L", "no_r"] + (["one_pass"] if regime == "far" else [])
    for fault in faults:
        assert worst(gv_simulate(x.numpy(), rows, lanes, fault)) > 1, fault


def test_argmin_restatement():
    """The kernel's reduction: a NaN ratio met on the way loses the minimum under the old rule, not under the fixed
    one; the exact check catches '>' for '>=' at min_var and a highest-index tie rule."""
    q = np.ones(64, F32)
    q[17] = F32(0.01)
    q[1] = F32(np.nan)
    qual = np.ones(64, bool)
    assert argmin_simulate(q, qual, "old") == 0
    assert argmin_simulate(q, qual) == 17
    var = q[None, :]
    assert expected_votes(var, np.ones(64, F32), MIN_VAR)[0] == 17
    rng = np.random.default_rng(0)
    for D in (64, 257, 1024):
        for p in [0, 1, 2, 4, 8, 16, 31, 32, 255, 256, D - 1]:
            if p >= D:
                continue
            q = rng.uniform(1, 2, D).astype(F32)
            q[p] = F32(0.5)
            for nan_at in [None, p ^ 1, p ^ 16, (p + 32) % D, 0]:
                qq = q.copy()
                if nan_at is not None and nan_at != p and nan_at < D:
                    qq[nan_at] = F32(np.nan)
                got = argmin_simulate(qq, np.ones(D, bool))
                assert got == expected_votes(qq[None, :], np.ones(D, F32), 0.0)[0] == p, (D, p, nan_at)
    # global_var exactly min_var: '>' for '>=' votes elsewhere
    gv = np.ones(8, F32)
    gv[3] = F32(MIN_VAR)
    var = np.full((1, 8), 1.0, F32)
    var[0, 3] = F32(0.001)
    exp = expected_votes(var, gv, MIN_VAR)[0]
    assert exp == 3 and argmin_simulate(var[0] / gv, gv > F32(MIN_VAR)) != exp
    # exact ties: the lowest index
    q = np.ones(300, F32)
    q[[5, 37, 261]] = F32(0.25)
    assert expected_votes(q[None, :] * 1, np.ones(300, F32), 0)[0] == argmin_simulate(q, np.ones(300, bool)) == 5
    assert argmin_simulate(q, np.ones(300, bool), "high_tie") != 5


def _sap_problem(seed, C, n=60):
    rng = np.random.default_rng(seed)
    y = rng.integers(0, 3, n)
    x = np.round(rng.standard_normal(n) * 4) / 4 + 0.6 * y          # repeated x values under different labels
    s, c, pos = SR.problems(y, 3, C, n)
    P = len(pos)
    return np.tile(x, (P, 1)), s, c, y


@pytest.mark.parametrize("C", [0.01, 100.0])
def test_sap_checks_reject_nearby_objectives(C):
    """The fp64 minimisers of objectives near LinearSVC's fail the coefficient / KKT check; its own passes."""
    x, s, c, y = _sap_problem(1, C)
    want, steps = SR.solve(x, s, c)
    assert (steps >= 0).all() and sap_fit_ok(want, want, x, s, c)

    def variant(kind, p):
        xi, si, ci = x[p], s[p], c[p]
        if kind == "unbalanced":
            ci = np.full_like(ci, C)

        def f(z):
            m = np.maximum(0, 1 - si * (z[0] * xi + z[1]))
            loss = (ci * (m if kind == "hinge" else m * m)).sum()
            reg = {"unpenalised_b": 0.5 * z[0] ** 2, "c_on_reg": 0.5 * C * (z @ z)}.get(kind, 0.5 * (z @ z))
            return reg + (loss / C if kind == "c_on_reg" else loss)
        return _minimise(f, want[p].copy())
    for kind in ("unpenalised_b", "unbalanced", "c_on_reg", "hinge"):
        z = np.stack([variant(kind, p) for p in range(x.shape[0])])
        assert not sap_fit_ok(z, want, x, s, c), kind


def test_fit_checks_reject_nearby_objectives():
    rng = np.random.default_rng(2)
    n, D, nc = 300, 3, 3
    y = rng.integers(0, nc, n)
    x = 0.5 * np.abs(rng.standard_normal((n, D)))
    x[np.arange(n), y] += 0.4
    W, b, steps = BR.fit(x, y, nc)
    assert steps >= 0 and fit_ok(W, b, x, y, nc)
    xa = np.c_[x, np.ones(n)]

    def f(theta, kind):
        th = theta.reshape(nc, D + 1)
        z = xa @ th.T
        m = z.max(1)
        loss = (m + np.log(np.exp(z - m[:, None]).sum(1)) - z[np.arange(n), y]).sum()
        reg = 0.5 * (th[:, :D] ** 2).sum()
        if kind == "penalised_b":
            reg += 0.5 * (th[:, D] ** 2).sum()
        if kind == "mean_loss":
            loss /= n
        return reg + loss
    start = np.c_[W, b].ravel()
    for kind in ("penalised_b", "mean_loss"):
        th = _minimise(lambda t: f(t, kind), start.copy()).reshape(nc, D + 1)
        assert not fit_ok(th[:, :D], th[:, D], x, y, nc), kind
    assert not fit_ok(W, b + 0.3, x, y, nc), "no sum b = 0 projection"


def test_fit_workspace_query_matches_the_layout():
    """The library's workspace query (a host function: no device needed) against the restated layout."""
    from disvae import _native
    L = _native.lib()
    for n, D, K in ((1, 1, 1), (2, 2, 2), (7, 2, 3), (1000, 126, 4), (1000, 127, 4), (1000, 128, 4), (1500, 128, 32),
                    (10000, 10, 5), (3, 1, 32)):
        assert L.dv_logistic_fit_workspace_bytes(n, D, K) == 8 * fit_workspace_doubles(n, D, K), (n, D, K)
    for n, D, K in ((0, 1, 1), (1, 0, 1), (1, 129, 1), (1, 1, 0), (1, 1, 33)):
        assert L.dv_logistic_fit_workspace_bytes(n, D, K) == 0


class _OnDevice(torch.Tensor):
    """A host tensor that reports itself as a CUDA tensor, so that each case below breaks one clause only."""

    @property
    def is_cuda(self):
        return True


def test_group_variance_wrapper_refusals(monkeypatch):
    """`group_variance` refuses a malformed output or global variance before any kernel call: each case breaks one of
    dtype, contiguity, shape and device; well-formed tensors reach the kernel call."""
    from disvae import evaluate
    monkeypatch.setattr(evaluate.N, "require_cuda_f32", lambda *t: None)
    monkeypatch.setattr(evaluate.N, "ptr", lambda t: None if t is None else 0)
    monkeypatch.setattr(evaluate.N, "stream", lambda: None)
    calls = []
    monkeypatch.setattr(evaluate.N, "call", lambda *a, **k: calls.append(a[0]))

    def dev(t):
        return t.as_subclass(_OnDevice)
    mu = dev(torch.zeros(50, 6))
    rows = torch.zeros(4, 8, dtype=torch.int64)
    good = dict(var_out=dev(torch.zeros(4, 6)), argmin_out=dev(torch.zeros(4, dtype=torch.int32)),
                global_var=dev(torch.ones(6)))
    evaluate.group_variance(mu, rows, **good)
    assert calls == ["dv_group_variance"]
    bad = [("var_out", dev(torch.zeros(4, 6, dtype=torch.float64))), ("var_out", dev(torch.zeros(6, 4)).t()),
           ("var_out", dev(torch.zeros(4, 5))), ("var_out", dev(torch.zeros(24))), ("var_out", torch.zeros(4, 6)),
           ("argmin_out", dev(torch.zeros(4, dtype=torch.int64))),
           ("argmin_out", dev(torch.zeros(8, dtype=torch.int32))[::2]),
           ("argmin_out", dev(torch.zeros(5, dtype=torch.int32))), ("argmin_out", dev(torch.zeros(4, 1).int())),
           ("argmin_out", torch.zeros(4, dtype=torch.int32)),
           ("global_var", dev(torch.ones(6).double())), ("global_var", dev(torch.ones(12))[::2]),
           ("global_var", dev(torch.ones(1, 6))), ("global_var", torch.ones(6))]
    for name, t in bad:
        g = good[name]
        broken = [t.dtype != g.dtype, not t.is_contiguous(), tuple(t.shape) != tuple(g.shape), not t.is_cuda]
        assert sum(broken) == 1, (name, broken)
        with pytest.raises(ValueError, match="group_variance: %s must be a contiguous CUDA" % name):
            evaluate.group_variance(mu, rows, **dict(good, **{name: t}))
    assert calls == ["dv_group_variance"]


# ---------------------------------------------------------------------------------------------------------------------
# GPU: dv_group_variance
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("N,D,V,L", GV_SHAPES, ids=["N%d-D%d-V%d-L%d" % s for s in GV_SHAPES])
def test_group_variance_shapes_and_layouts(N, D, V, L):
    x, rows = gv_inputs(N, D, V, L, "normal", seed=N * 7 + D * 3 + V + L)
    gv_check(x, rows, LAYOUTS, "gv N%d D%d V%d L%d" % (N, D, V, L))


@pytest.mark.gpu
@pytest.mark.parametrize("regime", GV_REGIMES)
@pytest.mark.parametrize("N,D,V,L", GV_REGIME_SHAPES, ids=["N%d-D%d-V%d-L%d" % s for s in GV_REGIME_SHAPES])
def test_group_variance_regimes(N, D, V, L, regime):
    """Every regime on the q_zCx and column-major layouts, then with every group's rows permuted."""
    x, rows = gv_inputs(N, D, V, L, regime, seed=N + D + V + L + len(regime))
    tag = "gv N%d D%d V%d L%d %s" % (N, D, V, L, regime)
    case = gv_check(x, rows, ["q_zCx", "colmajor"], tag)
    var = case.run()[0]
    if regime == "constant":
        assert not _bits(var[:, ::3]).any(), tag + ": a constant column has variance +0"
    if regime == "duplicate" and D > 1:
        for j in range(1, D, 2):
            _same(var[:, 0], var[:, j], tag + ": duplicate columns")
    g = torch.Generator().manual_seed(V + L)
    perm = torch.stack([torch.randperm(L, generator=g) for _ in range(V)])
    gv_check(x, torch.gather(rows, 1, perm), ["q_zCx"], tag + " permuted")


def _vote_inputs(D, mins, nans, ties, L=40, seed=0):
    """x and rows with one group per entry of `mins` (own rows): the group's column mins[g] has 1e-2 the spread of
    the others, column nans[g] (if not None) holds a NaN, and ties[g] (if not None) is a copy of column mins[g]."""
    V = len(mins)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(V * L, D, generator=g)
    for k, (m, q, t) in enumerate(zip(mins, nans, ties)):
        sl = slice(k * L, (k + 1) * L)
        x[sl, m] *= 1e-2
        if t is not None:
            x[sl, t] = x[sl, m]
        if q is not None:
            x[k * L + 3, q] = float("nan")
    return x, torch.arange(V * L).view(V, L)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [64, 257, 1024])
def test_votes_at_every_butterfly_distance(D):
    """The minimum at each butterfly distance and in each warp, alone, beside a NaN variance at its partners, and
    exactly tied with a copy in another thread, warp or pass of the same thread."""
    pos = [p for p in (0, 1, 2, 4, 8, 16, 17, 31, 32, 64, 128, 255, 256, 511, 1023) if p < D]
    mins, nans, ties = [], [], []
    for p in pos:
        for q in (None, p ^ 1, p ^ 2, p ^ 16, (p + 32) % D, (p + 256) % D, 0, 1):
            if q is not None and (q >= D or q == p):
                continue
            mins.append(p), nans.append(q), ties.append(None)
        for t in (p ^ 1, p ^ 4, p ^ 16, p + 32, p + 256, p + 512, p - 1):
            if 0 <= t < D and t != p:
                mins.append(p), nans.append(None), ties.append(t)
    x, rows = _vote_inputs(D, mins, nans, ties, seed=D)
    gv = np.ones(D, F32)
    case = GvCase(x, rows, "q_zCx", gv)
    var, votes = case.run(var=True, votes=True)
    votes = votes.cpu().numpy()
    var = var.cpu().numpy()
    assert np.array_equal(votes, expected_votes(var, gv, MIN_VAR))
    for k, (m, q, t) in enumerate(zip(mins, nans, ties)):
        if q is not None:
            assert np.isnan(var[k, q]), (k, q)
        want = m if t is None else min(m, t)
        assert votes[k] == want, (D, m, q, t, votes[k])
    _report("votes D%d" % D, groups=len(mins))
    case.graph()


@pytest.mark.gpu
def test_nan_variance_does_not_take_the_vote():
    """64 dims, ratio about 0.01 at d = 17, a NaN variance at d = 1: the vote is 17."""
    x, rows = _vote_inputs(64, [17, 17, 5], [1, None, 3], [None, None, None], seed=5)
    x[:, 17] /= 1e-2
    gv = np.ones(64, F32)
    gv[17] = 100.0
    var, votes = GvCase(x, rows, "contiguous", gv).run(var=True, votes=True)
    assert votes.tolist() == [17, 17, 5], votes.tolist()
    assert np.isnan(var[0, 1].item()) and np.array_equal(votes.cpu().numpy(), expected_votes(var.cpu().numpy(), gv,
                                                                                             MIN_VAR))


@pytest.mark.gpu
def test_votes_at_the_global_variance_edges():
    """global_var exactly min_var, one ulp below, NaN, +inf, and 0 with min_var = 0 (var / 0 is +inf or NaN)."""
    D = 12
    x, rows = _vote_inputs(D, list(range(D)) * 2, [None] * D + [5] * D, [None] * (2 * D), seed=7)
    x[:, 9] = 1.5                                               # a constant column: var 0
    below = np.nextafter(F32(MIN_VAR), F32(0))
    configs = []
    for k, edge in enumerate([F32(MIN_VAR), below, F32(np.nan), F32(np.inf)]):
        gv = np.ones(D, F32)
        gv[k] = edge
        configs.append((gv, MIN_VAR))
    gv = np.ones(D, F32)
    gv[[0, 9]] = 0
    configs += [(gv, 0.0), (np.zeros(D, F32), 0.0), (np.full(D, below, F32), MIN_VAR)]
    for gv, mv in configs:
        case = GvCase(x, rows, "padded", gv)
        var, votes = case.run(var=True, votes=True, min_var=mv)
        want = expected_votes(var.cpu().numpy(), gv, mv)
        assert np.array_equal(votes.cpu().numpy(), want), (gv, mv, votes.tolist(), want.tolist())
    assert (want == -1).all()


@pytest.mark.gpu
def test_group_variance_graph_replay():
    x, rows = gv_inputs(2000, 33, 300, 64, "normal", seed=3)
    case = GvCase(x, rows, "q_zCx", np.ones(33, F32))
    case.run(var=True, votes=True)
    case.graph()
    case.run(var=True)
    case.graph()


@pytest.mark.gpu
def test_group_variance_wrapper_checks():
    from disvae.evaluate import group_variance
    mu = torch.randn(50, 6, device=DEV)
    rows = torch.randint(50, (4, 8), device=DEV)
    ok = dict(var_out=torch.empty(4, 6, device=DEV), argmin_out=torch.empty(4, dtype=torch.int32, device=DEV),
              global_var=torch.ones(6, device=DEV))
    group_variance(mu, rows, **ok)
    for name, bad in (("var_out", torch.empty(6, 4, device=DEV).t()), ("var_out", torch.empty(4, 6)),
                      ("var_out", torch.empty(4, 5, device=DEV)), ("argmin_out", torch.empty(5, dtype=torch.int32,
                                                                                              device=DEV)),
                      ("argmin_out", torch.empty(4, dtype=torch.int64, device=DEV)),
                      ("argmin_out", torch.empty(8, dtype=torch.int32, device=DEV)[::2]),
                      ("global_var", torch.ones(6, device=DEV, dtype=torch.float64)),
                      ("global_var", torch.ones(7, device=DEV))):
        with pytest.raises(ValueError, match=name):
            group_variance(mu, rows, **dict(ok, **{name: bad}))


# ---------------------------------------------------------------------------------------------------------------------
# GPU: dv_sap_score_matrix
# ---------------------------------------------------------------------------------------------------------------------
def _sap_case(name, D=3, nc=(3,), ncv=None, cs=None, n_train=400, n_test=700, C=0.01, data="overlap", neg_test=False,
              N=None, seed=0):
    return dict(name=name, D=D, nc=list(nc), ncv=list(nc if ncv is None else ncv), cs=max(nc) if cs is None else cs,
                n_train=n_train, n_test=n_test, C=C, data=data, neg_test=neg_test, N=N, seed=seed)


SAP_CASES = [
    _sap_case("nc0_clamped", nc=(1, 2), ncv=(0, 2), cs=4),
    _sap_case("nc1_2_3", nc=(1, 2, 3)),
    _sap_case("nc16", nc=(16,), n_train=800),
    _sap_case("nc17", nc=(17, 2), n_train=800),
    _sap_case("nc256", D=2, nc=(256,), n_train=2000, n_test=513),
    _sap_case("stride_gt_nc", nc=(3, 2), cs=9),
    _sap_case("ncv_gt_stride", nc=(4, 4), ncv=(4, 7), cs=4),
    _sap_case("ntrain1", nc=(1,), n_train=1, n_test=511),
    _sap_case("ntrain2", nc=(2,), n_train=2, n_test=512),
    _sap_case("ntrain33", nc=(3, 2), n_train=33, n_test=1023),
    _sap_case("ntrain8589", D=2, nc=(3,), n_train=8589, n_test=1024),
    _sap_case("ntrain32768", D=2, nc=(3, 2), n_train=SAP_MAX_TRAIN, n_test=1025),
    _sap_case("test_minus1", nc=(4, 3), neg_test=True),
    _sap_case("many_ctas", D=1024, nc=(2, 3, 2, 4, 2, 3), n_train=200, n_test=300, N=200),
] + [_sap_case("C%g_%s" % (C, data), nc=(2, 3), C=C, data=data) for C in (1e-4, 0.01, 1.0, 100.0)
     for data in ("separable", "overlap")]


def _sap_inputs(c):
    """(x fp32 [N, D], train_rows, test_rows, train_cls [K, n], test_cls [K, m], n_classes (device values) [K],
    counts [K, cs]) for one case: every class of factor k present in the training rows."""
    rng = np.random.default_rng(c["seed"] + len(c["name"]))
    K, D, n, m = len(c["nc"]), c["D"], c["n_train"], c["n_test"]
    N = c["N"] or max(n, 64)
    train_rows = rng.integers(0, N, n)
    test_rows = rng.integers(0, N, m)
    train_cls = np.zeros((K, n), np.int32)
    test_cls = np.zeros((K, m), np.int32)
    for k, nc in enumerate(c["nc"]):
        y = rng.integers(0, nc, n)
        y[:min(nc, n)] = np.arange(min(nc, n))
        train_cls[k] = y
        test_cls[k] = rng.integers(-1 if c["neg_test"] else 0, nc, m)
    x = rng.standard_normal((N, D))
    if c["data"] == "overlap":
        x = np.round(x * 4) / 4                             # repeated values under different labels
    # the first min(D, K) latents carry factor k's labels of the training rows (last write wins on a repeated row)
    for k in range(min(D, K)):
        spread = 0.05 if c["data"] == "separable" else 1.0
        x[train_rows, k] = train_cls[k] + spread * rng.standard_normal(n)
    x = x.astype(F32)
    counts = np.zeros((K, c["cs"]), np.int32)
    for k in range(K):
        counts[k, :c["nc"][k]] = np.bincount(train_cls[k], minlength=c["nc"][k])[:c["nc"][k]]
    return x, train_rows, test_rows, train_cls, test_cls, np.array(c["ncv"], np.int32), counts


def _sap_run(c, x, layout, inputs):
    train_rows, test_rows, train_cls, test_cls, ncv, counts = inputs
    N, D = x.shape
    K, cs = counts.shape
    mu, ld, rs = place_mu(torch.from_numpy(x), layout)
    ins = [Buf(a.size, torch.int64 if a.dtype == np.int64 else torch.int32, torch.from_numpy(np.ascontiguousarray(a))
               .to(DEV)) for a in (train_rows, test_rows, train_cls, test_cls, ncv, counts)]
    score = Buf(D * K, torch.float32, float("nan"))
    coef = Buf(D * K * cs * 2, torch.float64, 7.0)
    iters = Buf(D * K * cs, torch.int32, -7)
    args = (mu.ptr, ld, rs, N, D, ins[0].ptr, len(train_rows), ins[1].ptr, len(test_rows), ins[2].ptr, ins[3].ptr,
            ins[4].ptr, ins[5].ptr, K, cs, float(c["C"]), score.ptr, coef.ptr, iters.ptr)
    outs = [score, coef, iters]
    _call(1, "dv_sap_score_matrix", *args, _lib()[1])
    first = [o.body.clone() for o in outs]
    _call(1, "dv_sap_score_matrix", *args, _lib()[1])
    for f, o in zip(first, outs):
        _same(f, o.body, c["name"] + " repeat")
        assert o.intact(), c["name"] + ": wrote past an output"
    assert all(b.intact() for b in ins + [mu])
    return [o.body.clone() for o in outs], args, outs + ins + [mu]         # the inputs stay alive for a graph


def _sap_check(c, x, inputs, got):
    """The kernel's outputs against the fp64 solve: (w, b), KKT, convergence, NaN / 0 beyond a factor's problems, and
    the score within the test rows near a tie.  Returns the worst coefficient error over its tolerance."""
    train_rows, test_rows, train_cls, test_cls, ncv, counts = inputs
    N, D = x.shape
    K, cs = counts.shape
    score, coef, iters = got
    score = score.view(D, K).cpu().numpy()
    coef = coef.view(D, K, cs, 2).cpu().numpy()
    iters = iters.view(D, K, cs).cpu().numpy()
    nc_eff = np.clip(ncv, 0, cs)
    w_score, w_coef, w_steps, gap = SR.score_matrix(x, train_rows, test_rows, train_cls, test_cls,
                                                    np.maximum(nc_eff, 1), counts, c["C"])
    fitted = ~np.isnan(w_coef[..., 0])
    assert np.array_equal(fitted, ~np.isnan(coef[..., 0])), c["name"]
    assert (w_steps[fitted] >= 0).all() and (iters[fitted] >= 0).all(), c["name"] + ": a fit did not converge"
    assert (iters[~fitted] == 0).all() and np.isnan(coef[~fitted]).all()
    worst = 0.0
    if fitted.any():
        err = np.abs(coef - w_coef).max(-1)[fitted]
        ref = np.maximum(np.abs(w_coef).max(-1)[fitted], 1e-300)
        worst = float((err / ref).max() / SAP_COEF_RTOL)
    x_train = x[train_rows].astype(F64)
    for k in range(K):
        s, cc, pos = SR.problems(train_cls[k].astype(np.int64), max(int(nc_eff[k]), 1), c["C"], len(train_rows))
        if pos:
            z = coef[:, k, :len(pos)].reshape(-1, 2)
            xx = np.repeat(x_train.T, len(pos), axis=0)
            ss, cw = np.tile(s, (D, 1)), np.tile(cc, (D, 1))
            assert sap_fit_ok(z, w_coef[:, k, :len(pos)].reshape(-1, 2), xx, ss, cw), (c["name"], k)
    x_test = x[test_rows].astype(F64)
    for d in range(D):
        for k in range(K):
            lines = w_coef[d, k][fitted[d, k]]
            scale = 1 + (np.abs(SR.decisions(lines, x_test[:, d])).max() if len(lines) else 0)
            loose = int((gap[d, k] <= SAP_MARGIN * scale).sum())
            assert abs(float(score[d, k]) - float(w_score[d, k])) <= loose / len(test_rows) + 1e-7, (c["name"], d, k)
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("case", SAP_CASES, ids=[c["name"] for c in SAP_CASES])
def test_sap_paths(case):
    t0 = time.time()
    x, *inputs = _sap_inputs(case)
    first = None
    for layout in LAYOUTS:
        got, args, outs = _sap_run(case, x, layout, inputs)
        if first is None:
            first = got
            w = _sap_check(case, x, inputs, got)
            _report("sap %s" % case["name"], coef=w)
            assert w <= 1
        else:
            for a, b in zip(first, got):
                _same(a, b, "%s %s vs %s" % (case["name"], layout, LAYOUTS[0]))
    if case["name"] == "nc17":
        _graph_replays(lambda: _lib()[0].dv_sap_score_matrix(*args, torch.cuda.current_stream().cuda_stream),
                       outs[:3], "dv_sap_score_matrix")
    print("  %.1f s" % (time.time() - t0))


# ---------------------------------------------------------------------------------------------------------------------
# GPU: dv_pair_abs_diff_mean
# ---------------------------------------------------------------------------------------------------------------------
PAIR_CASES = [(300, 7, 36, 1), (300, 10, 26, 2), (300, 1, 257, 64), (300, 128, 5, 1000), (300, 3, 85, 1000),
              (2000, 64, 4, 64)]


@pytest.mark.gpu
@pytest.mark.parametrize("N,D,V,L", PAIR_CASES, ids=["N%d-D%d-V%d-L%d" % s for s in PAIR_CASES])
def test_pair_abs_diff_mean_paths(N, D, V, L):
    """Bit for bit against the in-order fp64 sum (NaN-equal), V * D across block boundaries, every layout, and
    rows_a == rows_b giving exactly 0."""
    g = torch.Generator().manual_seed(N + D + V + L)
    x = torch.randn(N, D, generator=g)
    x[:, ::3] = 100 + 0.01 * x[:, ::3]
    x[5, 0] = float("nan")
    a = torch.randint(N, (V, L), generator=g)
    b = torch.randint(N, (V, L), generator=g)
    b[0] = a[0]
    want = BR.features(x.numpy(), a.numpy(), b.numpy())
    first = None
    for layout in LAYOUTS:
        mu, ld, rs = place_mu(x, layout)
        ra, rb = Buf(V * L, torch.int64, a.to(DEV)), Buf(V * L, torch.int64, b.to(DEV))
        out = Buf(V * D, torch.float64, 7.0)
        args = (mu.ptr, ld, rs, N, D, ra.ptr, rb.ptr, V, L, out.ptr)
        for rep in range(2):
            _call(1, "dv_pair_abs_diff_mean", *args, _lib()[1])
            assert out.intact() and mu.intact() and ra.intact() and rb.intact()
            got = out.body.view(V, D).clone()
            if first is None:
                first = got
                assert np.array_equal(got.cpu().numpy(), want, equal_nan=True)
                assert not _bits(got[0][~torch.isnan(got[0])]).any()
            _same(first, got, "pair %s rep %d" % (layout, rep))
    _graph_replays(lambda: _lib()[0].dv_pair_abs_diff_mean(*args, torch.cuda.current_stream().cuda_stream), [out],
                   "dv_pair_abs_diff_mean")
    _report("pair N%d D%d V%d L%d" % (N, D, V, L), exact=0.0)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: dv_logistic_fit
# ---------------------------------------------------------------------------------------------------------------------
def _fit_case(name, D=4, nc=3, K=None, ncv=None, n=400, eval=200, data="normal"):
    return dict(name=name, D=D, nc=nc, K=nc if K is None else K, ncv=nc if ncv is None else ncv, n=n, eval=eval,
                data=data)


FIT_CASES = [
    _fit_case("ncv0", nc=1, K=4, ncv=0), _fit_case("ncv1", nc=1, K=4, ncv=1), _fit_case("ncv2", nc=2, K=4, ncv=2),
    _fit_case("ncv3", nc=3, K=4, ncv=3), _fit_case("ncvK", nc=4), _fit_case("ncv_gt_K", nc=4, ncv=9),
    _fit_case("eval0", nc=3, eval=0),
    _fit_case("n2", D=2, nc=2, n=2), _fit_case("n3", D=2, nc=3, n=3), _fit_case("n7", D=2, nc=3, n=7),
    _fit_case("O508", D=126, nc=4, n=600), _fit_case("O512", D=127, nc=4, n=600), _fit_case("O516", D=128, nc=4, n=600),
    _fit_case("D128_K32", D=128, nc=32, n=1500, eval=100),
    _fit_case("zero_features", nc=3, data="zero"), _fit_case("collinear", D=6, nc=3, data="collinear"),
    _fit_case("far", nc=4, data="far"), _fit_case("single_row_class", nc=4, data="single_row"),
    _fit_case("large_margins", nc=3, data="margins"),
    _fit_case("segments_ratio", D=20, nc=2, n=3000),
]


def _fit_inputs(c):
    rng = np.random.default_rng(len(c["name"]) * 7 + c["D"])
    n, D, nc = c["n"], c["D"], c["nc"]
    y = rng.integers(0, nc, n)
    y[:min(nc, n)] = np.arange(min(nc, n))
    if c["data"] == "single_row":
        y[y == nc - 1] = 0
        y[n // 2] = nc - 1
    rows = n + c["eval"]
    x = 0.5 * np.abs(rng.standard_normal((rows, D)))
    ye = np.r_[y, rng.integers(0, nc, c["eval"])]
    x[np.arange(rows), ye % D] += 0.3
    if c["data"] == "zero":
        x[:] = 0
    elif c["data"] == "collinear":
        x[:, 3:] = 2 * x[:, :3]
        x[:, 1] = x[:, 0]
    elif c["data"] == "far":
        x = 100 + 0.01 * x
    elif c["data"] == "margins":
        x[np.arange(rows), ye % D] += 3.0
        x *= 5
    return x, y


@pytest.mark.gpu
@pytest.mark.parametrize("case", FIT_CASES, ids=[c["name"] for c in FIT_CASES])
def test_logistic_fit_paths(case):
    L, S = _lib()
    x, y = _fit_inputs(case)
    n, D, K, rows = case["n"], case["D"], case["K"], case["n"] + case["eval"]
    nc = min(max(case["ncv"], 1), K)
    nbytes = L.dv_logistic_fit_workspace_bytes(n, D, K)
    assert nbytes == 8 * fit_workspace_doubles(n, D, K)
    xb = Buf(rows * D, torch.float64, torch.from_numpy(x).to(DEV))
    lab = Buf(n, torch.int32, torch.from_numpy(y.astype(np.int32)).to(DEV))
    ncb = Buf(1, torch.int32, case["ncv"])
    ws = Buf(nbytes // 8, torch.float64)
    ws.body.view(torch.uint8).fill_(0xFF)
    coef, pred, it = Buf(K * (D + 1), torch.float64, 7.0), Buf(rows, torch.int32, -7), Buf(1, torch.int32, -7)
    args = (xb.ptr, D, n, case["eval"], lab.ptr, ncb.ptr, K, coef.ptr, pred.ptr, it.ptr)
    torch.cuda.synchronize()
    before = L.dv_launch_count()
    assert L.dv_logistic_fit(*args, ws.ptr, nbytes - 1, S) == DV_ERR_WORKSPACE
    assert L.dv_launch_count() == before
    first = None
    for rep in range(2):
        _call(1, "dv_logistic_fit", *args, ws.ptr, nbytes, S)
        for b in (coef, pred, it, ws, xb, lab, ncb):
            assert b.intact(), case["name"] + ": wrote past a buffer"
        got = [coef.body.clone(), pred.body.clone(), it.body.clone()]
        if first is None:
            first = got
        for a, b in zip(first, got):
            _same(a, b, case["name"] + " repeat")
    W = coef.body.view(K, D + 1).cpu().numpy()
    p = pred.body.cpu().numpy()
    iters = int(it.body.item())
    R = nc if nc > 2 else nc - 1
    assert np.isnan(W[R:]).all() and not np.isnan(W[:R]).any(), case["name"]
    if R == 0:
        assert iters == 0 and (p == 0).all()
        _report("fit %s" % case["name"], coef=0.0)
        return
    assert iters >= 0, case["name"] + ": the fit did not converge"
    Wt, b = W[:R, :-1], W[:R, -1]
    assert fit_ok(Wt, b, x[:n], y, nc), case["name"]
    wW, wb, _ = BR.fit(x[:n], y, nc)
    ref = max(np.abs(wW).max(), np.abs(wb).max(), 1e-300)
    worst = max(np.abs(Wt - wW).max(), np.abs(b - wb).max()) / ref / FIT_COEF_RTOL
    want, gap = BR.predict(wW, wb, nc, x)
    loose = gap <= FIT_MARGIN * (1 + np.abs(BR.decisions(wW, wb, x)).max(1))
    assert np.array_equal(p[~loose], want[~loose]), case["name"]
    if case["data"] == "zero":
        assert (Wt == 0).all()
    _report("fit %s S %d" % (case["name"], segments(R * (D + 1), n)), coef=worst)
    if case["name"] == "ncvK":
        _graph_replays(lambda: L.dv_logistic_fit(*args, ws.ptr, nbytes, torch.cuda.current_stream().cuda_stream),
                       [coef, pred, it], "dv_logistic_fit")
