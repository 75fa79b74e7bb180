"""The beta-TCVAE estimator (csrc/dv_btcvae.cu) on every path it can take, against a chunked fp64 reference.

dv_btcvae_fwd runs one of two forward paths: the single-launch cluster kernel (D <= 16, whole batch, up to B = 4096 at
D = 10 and 2048 at other D) or the three-launch tiled kernels (everything else: D > 16, larger batches, every row
window), with four tiled instantiations and two column-tile widths.  dv_btcvae_bwd dispatches to eight instantiations.
Each case below asserts which forward path it ran (from dv_launch_count) and checks the row statistics, the three
terms and the gradients against `ref_rowstats` / `ref_grads`, which evaluate the selected rows against all B columns in
fp64, a few rows at a time, so that batches far beyond what the oracle's B x B x D tensor allows can be checked.
Outlier rows (samples tens of sigma away from every posterior) run on every forward path.

The two references are first checked against the oracle (oracle/disvae_oracle.py) on the CPU; everything else needs
an H100 (pytest -m gpu)."""
import math

import pytest
import torch

from oracle import disvae_oracle as O

RTOL = 1e-4          # gradients: the suite's fp32 tolerance
STAT_TOL = 2e-5      # row statistics and terms, relative to the scale of the statistic
CHUNK_ELEMS = 1 << 22
GUARD = 4096         # floats of sentinel after the workspace
SENTINEL = 0x7FBADBAD  # a NaN bit pattern no kernel writes


# ---------------------------------------------------------------------------------------------------------------------
# fp64 reference, a few rows at a time
# ---------------------------------------------------------------------------------------------------------------------
def _log_weights(B, n_data):
    """log W[i, j] for the three distinct weights (1/N, strat, 1/M), built like O.log_importance_weight_matrix:
    fp32 weights, fp32 log."""
    m = B - 1
    strat = (n_data - m) / (n_data * m)
    w = torch.empty(3, 64, dtype=torch.float32)
    w[0], w[1], w[2] = 1.0 / n_data, strat, 1.0 / m
    return w.log()[:, 0].double()


def _weight_rows(rows, B, lw):
    """[len(rows), B] log-weights of the given rows: 1/N in column 0, strat in column 1 and at (B-2, 0), 1/M elsewhere."""
    w = lw[2].expand(len(rows), B).clone()
    w[:, 0] = lw[0]
    w[:, 1] = lw[1]
    w[rows == B - 2, 0] = lw[1]
    return w


def _chunk(B, D, chunk):
    return chunk if chunk is not None else max(1, CHUNK_ELEMS // (B * D))


def _rowstats_of(zr, rows, mu, lv, n_data, is_mss):
    """(log_pz, log_qz, log_prod_qzi, log_q_zCx, P[n, D]) of rows `rows` (whose z is `zr`) against all columns."""
    B, D = mu.shape
    log_q_zcx = O.log_density_gaussian(zr, mu[rows], lv[rows]).sum(1)
    log_pz = O.log_density_gaussian(zr, torch.zeros_like(zr), torch.zeros_like(zr)).sum(1)
    mat = O.log_density_gaussian(zr.unsqueeze(1), mu.unsqueeze(0), lv.unsqueeze(0))     # [n, B, D]
    if is_mss:
        mat = mat + _weight_rows(rows, B, _log_weights(B, n_data)).unsqueeze(2)
    log_qz = torch.logsumexp(mat.sum(2), dim=1)
    P = torch.logsumexp(mat, dim=1)
    return log_pz, log_qz, P.sum(1), log_q_zcx, P


def ref_rowstats(z, mu, lv, n_data, is_mss, rows, chunk=None):
    """fp64 row statistics of `rows` (a 1-D index tensor): (log_pz, log_qz, log_prod_qzi, log_q_zCx, P[len(rows), D])."""
    z, mu, lv = z.double(), mu.double(), lv.double()
    rows = torch.as_tensor(rows, dtype=torch.long)
    c = _chunk(*mu.shape, chunk)
    outs = [_rowstats_of(z[rows[a:a + c]], rows[a:a + c], mu, lv, n_data, is_mss) for a in range(0, len(rows), c)]
    return tuple(torch.cat(t) for t in zip(*outs))


def ref_grads(z, mu, lv, n_data, is_mss, row0, nrows, coef, chunk=None):
    """Gradient of coef . (mi, tc, dw), each the mean over rows [row0, row0 + nrows), in fp64:
    (g_z [nrows, D] of the window's rows, g_mu [B, D], g_lv [B, D] over every column)."""
    z = z.detach().double()
    mu = mu.detach().double().clone().requires_grad_(True)
    lv = lv.detach().double().clone().requires_grad_(True)
    g_z = torch.empty(nrows, z.shape[1], dtype=torch.float64)
    c = _chunk(*mu.shape, chunk)
    for a in range(row0, row0 + nrows, c):
        rows = torch.arange(a, min(a + c, row0 + nrows))
        zr = z[rows].clone().requires_grad_(True)
        lpz, lqz, lprod, lqc, _ = _rowstats_of(zr, rows, mu, lv, n_data, is_mss)
        loss = (coef[0] * (lqc - lqz).sum() + coef[1] * (lqz - lprod).sum() + coef[2] * (lprod - lpz).sum()) / nrows
        loss.backward()
        g_z[a - row0:a - row0 + len(rows)] = zr.grad
    return g_z, mu.grad, lv.grad


# ---------------------------------------------------------------------------------------------------------------------
# CPU self-checks of the reference against the oracle
# ---------------------------------------------------------------------------------------------------------------------
def _inputs(B, D, seed, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    mu = torch.randn(B, D, generator=g)
    lv = torch.randn(B, D, generator=g) * 0.5 - 1
    z = mu + torch.exp(0.5 * lv) * torch.randn(B, D, generator=g)
    return z.to(dtype), mu.to(dtype), lv.to(dtype)


def _close64(a, b, what):
    err = ((a - b).abs().max() / b.abs().max().clamp_min(1e-300)).item()
    assert err <= 1e-12, "%s: %.3e" % (what, err)


@pytest.mark.parametrize("B", [2, 3, 7, 64, 257])
@pytest.mark.parametrize("mss", [True, False])
def test_reference_rowstats_match_the_oracle(B, mss):
    D, n_data = 5, 1000
    z, mu, lv = _inputs(B, D, B, torch.float64)
    ref = O.btcvae_log_densities(z, mu, lv, n_data, mss)
    rows = torch.arange(B)
    got = ref_rowstats(z, mu, lv, n_data, mss, rows, chunk=3)
    for a, b, name in zip(got, ref, ["log_pz", "log_qz", "log_prod_qzi", "log_q_zCx"]):
        _close64(a, b, name)
    assert got[4].shape == (B, D)
    sub = torch.tensor([B - 1, 0, B // 2])
    for a, b in zip(ref_rowstats(z, mu, lv, n_data, mss, sub), got):
        _close64(a, b[sub], "row subset")


@pytest.mark.parametrize("B", [2, 3, 7, 64, 257])
@pytest.mark.parametrize("mss", [True, False])
def test_reference_gradients_match_autograd_through_the_oracle(B, mss):
    D, n_data, coef = 4, 5000, (1.0, 6.0, -2.5)
    z, mu, lv = _inputs(B, D, 7 * B, torch.float64)
    windows = [(0, B)] + ([(1, B - 2), (B // 2, B - B // 2)] if B > 2 else [(1, 1)])
    for row0, nrows in windows:
        zo, muo, lvo = [t.clone().requires_grad_(True) for t in (z, mu, lv)]
        if (row0, nrows) == (0, B):
            mi, tc, dw = O.btcvae_terms(zo, muo, lvo, n_data, mss)
        else:
            lpz, lqz, lprod, lqc = [t[row0:row0 + nrows] for t in O.btcvae_log_densities(zo, muo, lvo, n_data, mss)]
            mi, tc, dw = (lqc - lqz).mean(), (lqz - lprod).mean(), (lprod - lpz).mean()
        (coef[0] * mi + coef[1] * tc + coef[2] * dw).backward()
        g_z, g_mu, g_lv = ref_grads(z, mu, lv, n_data, mss, row0, nrows, coef, chunk=2)
        _close64(g_z, zo.grad[row0:row0 + nrows], "g_z %s" % ((row0, nrows),))
        _close64(g_mu, muo.grad, "g_mu %s" % ((row0, nrows),))
        _close64(g_lv, lvo.grad, "g_lv %s" % ((row0, nrows),))


# ---------------------------------------------------------------------------------------------------------------------
# the kernels
# ---------------------------------------------------------------------------------------------------------------------
CLUSTER, TILED = 1, 3        # kernel launches of one forward call on each path
N_DATA = 202599
COEF = (1.0, 6.0, -2.5)
FULL_GRAD_ELEMS = 2e8        # above this many (row, column, dim) triples the gradient is checked on one row window


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def _assert_rel(a, b, tol, what):
    assert torch.isfinite(a).all(), "%s: not finite" % what
    e = _rel(a, b)
    assert e <= tol, "%s: rel err %.3e > %.1e" % (what, e, tol)


def _bits(t):
    return t.contiguous().view(torch.int32)


class Kernel:
    """Device copies of (z, mu, logvar) in either the [B, D] layout or the encoder's interleaved one (ld = 2,
    row stride 2D), and the C-ABI calls on them with workspaces sized exactly by dv_btcvae_workspace_bytes."""

    def __init__(self, z, mu, lv, interleaved):
        from disvae import _native as N
        self.N, self.B, self.D = N, *z.shape
        self.z = z.cuda()
        if interleaved:
            self.ml = torch.stack([mu, lv], dim=-1).reshape(self.B, 2 * self.D).cuda()
            self.mu_p, self.lv_p = self.ml.data_ptr(), self.ml.data_ptr() + 4
            self.ld, self.rs = 2, 2 * self.D
        else:
            self.mu, self.lv = mu.cuda(), lv.cuda()
            self.mu_p, self.lv_p = self.mu.data_ptr(), self.lv.data_ptr()
            self.ld, self.rs = 1, self.D
        self.ws_floats = N.lib().dv_btcvae_workspace_bytes(self.B, self.D) // 4

    def workspace(self):
        """Header zero, body NaN (the forward must write whatever the backward reads), then a sentinel guard."""
        ws = torch.full((self.ws_floats + GUARD,), float("nan"), device="cuda")
        ws[:16] = 0
        _bits(ws)[self.ws_floats:] = SENTINEL
        return ws

    def guard_intact(self, ws):
        return bool((_bits(ws)[self.ws_floats:] == SENTINEL).all())

    def forward(self, row0, nrows, mss, ws):
        """-> (rowstats [4 + D, B] with NaN outside the window, terms [3], kernel launches)."""
        N, B, D = self.N, self.B, self.D
        rowstats = torch.full((4 + D, B), float("nan"), device="cuda")
        terms = torch.full((3,), float("nan"), device="cuda")
        before = N.lib().dv_launch_count()
        if (row0, nrows) == (0, B):
            N.call("dv_btcvae_fwd", N.ptr(self.z), self.mu_p, self.lv_p, self.ld, self.rs, B, D, N_DATA, int(mss),
                   N.ptr(rowstats), N.ptr(terms), N.ptr(ws), N.stream())
        else:
            N.call("dv_btcvae_fwd_rows", N.ptr(self.z), self.mu_p, self.lv_p, self.ld, self.rs, B, D, row0, nrows,
                   N_DATA, int(mss), N.ptr(rowstats), N.ptr(terms), N.ptr(ws), N.stream())
        launches = N.lib().dv_launch_count() - before
        torch.cuda.synchronize()
        return rowstats, terms, launches

    def backward(self, row0, nrows, mss, rowstats, ws):
        N, B, D = self.N, self.B, self.D
        g_terms = torch.tensor(COEF, device="cuda")
        g_z = torch.full((nrows, D), float("nan"), device="cuda")
        g_mu = torch.full((B, D), float("nan"), device="cuda")
        g_lv = torch.full((B, D), float("nan"), device="cuda")
        N.call("dv_btcvae_bwd_rows", B, D, row0, nrows, N_DATA, int(mss), N.ptr(rowstats), N.ptr(ws), N.ptr(g_terms),
               N.ptr(g_z), N.ptr(g_mu), N.ptr(g_lv), N.stream())
        torch.cuda.synchronize()
        return g_z, g_mu, g_lv


def _check_rows(B, row0, nrows):
    """Every row of the window up to B = 4097; above that 512 rows: both ends of the batch and of the window, the
    MSS row B-2, and a fixed random sample."""
    if B <= 4097:
        return torch.arange(row0, row0 + nrows), True
    fixed = {0, 1, B - 2, B - 1, row0, row0 + 1, row0 + nrows - 2, row0 + nrows - 1}
    fixed = sorted(r for r in fixed if row0 <= r < row0 + nrows)
    g = torch.Generator().manual_seed(B + row0)
    extra = (row0 + torch.randperm(nrows, generator=g)).tolist()
    rows = fixed + [r for r in extra if r not in fixed][:512 - len(fixed)]
    return torch.tensor(sorted(rows)), False


def _grad_window(B, D, row0, nrows):
    """The rows whose backward is checked: the whole forward window when the reference can afford it, else its last
    256 rows (which hold the MSS row B-2 whenever the window ends the batch)."""
    if nrows * B * D <= FULL_GRAD_ELEMS:
        return row0, nrows
    return row0 + nrows - 256, 256


def run_case(z, mu, lv, windows, mss, path, interleaved=False):
    """Forward every window (twice, for bit-exactness) on the expected path, check its row statistics and terms, then
    check the backward of each window (or of its last 256 rows) against ref_grads; the workspace guard must survive."""
    B, D = z.shape
    k = Kernel(z, mu, lv, interleaved)
    for row0, nrows in windows:
        tag = "B=%d D=%d mss=%d window=(%d,%d)" % (B, D, mss, row0, nrows)
        ws = k.workspace()
        rowstats, terms, launches = k.forward(row0, nrows, mss, ws)
        assert launches == path, "%s: %d launches, expected the %s path" % (
            tag, launches, "cluster" if path == CLUSTER else "tiled")
        assert k.guard_intact(ws), "%s: forward wrote past dv_btcvae_workspace_bytes" % tag
        rs2, terms2, _ = k.forward(row0, nrows, mss, k.workspace())
        assert torch.equal(_bits(rs2), _bits(rowstats)) and torch.equal(_bits(terms2), _bits(terms)), tag + ": forward not deterministic"
        outside = torch.ones(B, dtype=torch.bool)
        outside[row0:row0 + nrows] = False
        untouched = torch.cat([rowstats[1:3], rowstats[4:]])[:, outside.cuda()]
        assert torch.isnan(untouched).all(), tag + ": rows outside the window written"

        rows, every_row = _check_rows(B, row0, nrows)
        ref = ref_rowstats(z, mu, lv, N_DATA, mss, rows)
        got = rowstats[:, rows.cuda()].cpu()
        names = ["log_pz", "log_qz", "log_prod_qzi", "log_q_zCx"]
        for s in range(4):
            _assert_rel(got[s], ref[s], STAT_TOL, "%s %s" % (tag, names[s]))
        _assert_rel(got[4:], ref[4].t(), STAT_TOL, tag + " P")
        t = terms.cpu().double()
        assert torch.isfinite(t).all(), tag + ": terms not finite"
        if every_row:
            lpz, lqz, lprod, lqc = ref[:4]
            want = torch.stack([(lqc - lqz).mean(), (lqz - lprod).mean(), (lprod - lpz).mean()])
            scale = max(r.abs().max().item() for r in ref[:4])
            tol = STAT_TOL
        else:                                    # the kernel's own means of its row statistics
            own = rowstats[:4, row0:row0 + nrows].double().cpu()
            lpz, lqz, lprod, lqc = own
            want = torch.stack([(lqc - lqz).mean(), (lqz - lprod).mean(), (lprod - lpz).mean()])
            scale = own.abs().max().item()
            tol = 1e-6
        err = (t - want).abs().max().item() / scale
        assert err <= tol, "%s terms: %s vs %s (err %.3e of scale)" % (tag, t.tolist(), want.tolist(), err)

        g0, gn = _grad_window(B, D, row0, nrows)
        grads = k.backward(g0, gn, mss, rowstats, ws)
        assert k.guard_intact(ws), "%s: backward wrote past dv_btcvae_workspace_bytes" % tag
        again = k.backward(g0, gn, mss, rowstats, ws)
        assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(grads, again)), tag + ": backward not deterministic"
        want = ref_grads(z, mu, lv, N_DATA, mss, g0, gn, COEF)
        tol = grad_tol(torch.cat([rowstats[1:2], rowstats[4:]])[:, g0:g0 + gn])
        for g, w, name in zip(grads, want, ["g_z", "g_mu", "g_logvar"]):
            _assert_rel(g.cpu(), w, tol, "%s %s rows (%d,%d)" % (tag, name, g0, gn))


def grad_tol(logs):
    """RTOL, unless the rows' log_qz or P are too large for fp32 to carry the gradient to RTOL.  The backward weighs
    every (i, j) pair by exp(A[i,j] - log_qz[i]) and exp(m[i,j,d] - P[i,d]), with log_qz and P read back from the fp32
    row statistics, which hold them only to half an ulp: 2^-24 of their magnitude.  For a sample tens of sigma away
    from every posterior, log_qz reaches -3.5e5 nats at D = 64 (an ulp of 0.03), so those weights, and the g_logvar
    they dominate, are only good to ~2^-24 |log_qz| relative.  The bound allows 8 such units for the backward's own
    fp32 sums over D.  Ordinary rows (|log_qz|, |P| < ~200 nats) keep RTOL."""
    return max(RTOL, 2.0 ** -21 * logs.abs().max().item())


def _splits(B, edges):
    edges = [0] + list(edges) + [B]
    return [(a, b - a) for a, b in zip(edges[:-1], edges[1:])]


WHOLE = lambda B: [(0, B)]   # noqa: E731

# (B, D, windows, path, interleaved)
CASES = [
    # cluster path: both capacity edges, both instantiations with a runtime D, the smallest batches
    (4096, 10, WHOLE(4096), CLUSTER, False),
    (1025, 10, WHOLE(1025), CLUSTER, False),
    (2048, 16, WHOLE(2048), CLUSTER, True),
    (2048, 12, WHOLE(2048), CLUSTER, False),
    (31, 15, WHOLE(31), CLUSTER, False),
    (3, 4, WHOLE(3), CLUSTER, False),
    (2, 1, WHOLE(2), CLUSTER, False),
    # tiled path, whole batch: one past each cluster capacity, D > 16, both column-tile widths
    (4097, 10, WHOLE(4097), TILED, False),
    (8192, 10, WHOLE(8192), TILED, False),
    (2049, 16, WHOLE(2049), TILED, False),
    (2049, 12, WHOLE(2049), TILED, True),
    (300, 33, WHOLE(300), TILED, False),
    (512, 32, WHOLE(512), TILED, False),
    (48, 65, WHOLE(48), TILED, False),
    # tiled path, row windows (uneven, a single row, a 32-row window; the 8-rank global batch of configs[4])
    (200, 1, _splits(200, [37]), TILED, False),
    (257, 7, _splits(257, [100, 101]), TILED, False),
    (130, 8, _splits(130, [64]), TILED, False),
    (600, 12, _splits(600, [250]), TILED, True),
    (1024, 10, [(512, 32), (0, 512)], TILED, False),
    (16384, 64, [(0, 2048), (14336, 2048)], TILED, False),
    # backward instantiations the cases above leave out: (4, T, F) at D = 4; (8, T, F) at 5; (16, T, F) at 9;
    # (16, F, T) at 48; (16, F, F) at 17
    (160, 4, WHOLE(160), CLUSTER, False),
    (160, 5, WHOLE(160), CLUSTER, False),
    (160, 9, WHOLE(160), CLUSTER, False),
    (160, 17, WHOLE(160), TILED, False),
    (160, 48, WHOLE(160), TILED, False),
]


@pytest.mark.gpu
@pytest.mark.parametrize("mss", [True, False])
@pytest.mark.parametrize("B,D,windows,path,interleaved", CASES,
                         ids=["%dx%d%s" % (c[0], c[1], "" if c[2] == WHOLE(c[0]) else "-windows") for c in CASES])
def test_btcvae_paths_match_the_fp64_reference(B, D, windows, path, interleaved, mss):
    z, mu, lv = _inputs(B, D, 1000 * D + B)
    run_case(z, mu, lv, windows, mss, path, interleaved)


def _outliers(B, D, kind):
    """The outlier construction of test_kernels_gpu.py::test_btcvae_outlier_rows_and_tiny_variances without its
    wide-variance row (which happened to keep every outlier row within range): tiny variances, row 9 shifted by 40
    sigma-ish in every dim (12 in "12sigma"), row 100 by 25 in one dim; "one_dim" shifts only row 9, in one dim."""
    g = torch.Generator().manual_seed(1)
    mu = torch.randn(B, D, generator=g)
    lv = torch.randn(B, D, generator=g) * 0.3 - 2.0
    lv[5] = -20.0
    lv[130, :3] = -16.0
    z = mu + torch.exp(0.5 * lv) * torch.randn(B, D, generator=g)
    if kind == "one_dim":
        z[9, D // 2] += 40.0
    else:
        z[9] += 40.0 if kind == "40sigma" else 12.0
        z[100, 2] -= 25.0
    return z, mu, lv


OUTLIER_CASES = [
    (192, 10, WHOLE(192), CLUSTER),
    (192, 20, WHOLE(192), TILED),
    (192, 64, WHOLE(192), TILED),
    (192, 10, _splits(192, [96]), TILED),
    (4097, 10, WHOLE(4097), TILED),
]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["40sigma", "12sigma", "one_dim"])
@pytest.mark.parametrize("mss", [True, False])
@pytest.mark.parametrize("B,D,windows,path", OUTLIER_CASES,
                         ids=["%dx%d%s" % (c[0], c[1], "" if c[2] == WHOLE(c[0]) else "-windows") for c in OUTLIER_CASES])
def test_btcvae_outlier_rows_on_every_forward_path(B, D, windows, path, mss, kind):
    """Every term of an outlier row lies far below the column-range bounds the tiled forward scales its sums by, so
    they all underflow there; its row statistics must still be finite and exact.  Gradients are held to grad_tol,
    which these rows' log_qz of up to -3.5e5 nats widen beyond RTOL."""
    z, mu, lv = _outliers(B, D, kind)
    run_case(z, mu, lv, windows, mss, path)
