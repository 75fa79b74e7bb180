"""The small kernels every training step runs between the decoder output and the weight update, against fp64
references written here, at training shapes and at the input edges where fp32 kernels go wrong.

- dv_vae_loss_fwd/bwd (csrc/dv_loss.cu): reconstruction loss + analytic KL.  The forward runs
  min(ceil(n/4 / 1024), 264) blocks (n = B x image elements) and the last block to finish combines the partials,
  through a counter in the workspace that it resets for the next launch.  Each case asserts the grid it ran by the
  recon partials it finds written in the workspace.
- dv_reparam_fwd/bwd: z = mu + exp(lv/2) eps, with eps injected or drawn on the device from Philox4x32-10 at the
  counters offset + i, restated on the host (`host_eps`).
- dv_factor_tc_*, dv_factor_ce_* (csrc/dv_factor.cu): the FactorVAE heads, one 256-thread block for any h.
- dv_adam_step, dv_adam_multi and disvae.fused.FusedAdam against CPU torch.optim.Adam(foreach=False).

Every direct C-ABI call here writes into buffers followed by a band of sentinel NaN bit patterns that must survive.
The references are first checked on the CPU against the oracle (oracle/disvae_oracle.py), fp64 autograd and torch;
everything else needs an H100 (pytest -m gpu).  Each GPU case prints its worst errors (pytest -s shows them)."""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import disvae_oracle as O

GUARD = 1024           # floats of sentinel after each output and workspace
SENTINEL = 0x7FBADBAD  # a NaN bit pattern no kernel writes
DV_ERR_BAD_SHAPE, DV_ERR_BAD_ARG = -1, -2     # include/disvae_b200.h
DISTS = {"bernoulli": 0, "gaussian": 1, "laplace": 2}
LOSS_BLOCKS = 264                             # dv_loss.cu: 2 x 132 SMs
LOSS_WS_FLOATS = 1 + LOSS_BLOCKS + 1024       # counter, recon partials, per-dimension KL
CHUNK = 1 << 22
U = 2.0 ** -24                                # fp32 unit roundoff

RECON_TOL = 1e-6       # recon loss, relative to the sum of |term| it adds up
KL_TOL = 1e-6          # KL per dimension and total, relative to 0.5 sum(1 + |lv| + mu^2 + e^lv) / B
GRAD_ULPS = 8          # gradients and z, per element, in units of U times the magnitude of the terms
EPS_TOL = 1e-6         # device noise, per element, relative to 1 + |eps|
FACTOR_TOL = 2e-7      # TC and CE values, relative to the magnitude summed
ADAM_ULPS = 2          # one Adam step from identical state, exp_avg and exp_avg_sq per element
ADAM_P_ULPS = 4        # ... p per element: m / denom, the step size and the subtraction each round once more
ADAM_CHAIN_TOL = 2e-6  # 200 Adam steps, per element, relative to |p0| + the path |p| travelled


# ---------------------------------------------------------------------------------------------------------------------
# fp64 references
# ---------------------------------------------------------------------------------------------------------------------
def _recon_terms(r, x, dist):
    """Per-element reconstruction terms as aten's losses compute them (before the final scaling)."""
    if dist == "bernoulli":
        return (x - 1) * torch.log1p(-r).clamp_min(-100) - x * torch.log(r).clamp_min(-100)
    if dist == "gaussian":
        return (r * 255 - x * 255) ** 2
    return (r - x).abs()


BCE_EPS = float(np.float32(1e-12))    # aten's binary_cross_entropy_backward clamps (1 - r) r at the fp32 1e-12


def _recon_scale(dist):
    return {"bernoulli": 1.0, "gaussian": 1 / 255, "laplace": 3.0}[dist]


SUBNORMAL = 2.0 ** -149      # fp32 spacing below 2^-126


def _recon_grad(r, x, dist, g_rec, laplace_live):
    """(d loss / d recon, the fp32 error scale of that element) per element, aten's backward formulas, where
    g_rec = upstream / B.  The scale is U times the magnitude of the terms combined, plus one subnormal spacing
    where aten's order of operations passes through g_rec (r - x), subnormal for a subnormal recon."""
    if dist == "bernoulli":
        den = ((1 - r) * r).clamp_min(BCE_EPS)
        return g_rec * (r - x) / den, (U * abs(g_rec) * (r.abs() + x.abs()) + SUBNORMAL) / den
    if dist == "gaussian":
        return g_rec * 2 * (r * 255 - x * 255), U * abs(g_rec) * 2 * 255 * (r.abs() + x.abs()) + SUBNORMAL
    s = g_rec * 3 if laplace_live else 0.0
    return s * torch.sign(r - x), torch.full_like(r, U * abs(s))


def ref_vae_loss(recon, data, mu, logvar, dist):
    """fp64 loss of the step, a chunk of elements at a time: dict of recon (as aten), its bound scale sum |term|
    (scaled alike), kl, kl_dims [D] and their bound scale 0.5 sum(1 + |lv| + mu^2 + e^lv) / B."""
    B = recon.shape[0]
    r, x = recon.reshape(-1), data.reshape(-1)
    tot = mag = 0.0
    for a in range(0, r.numel(), CHUNK):
        t = _recon_terms(r[a:a + CHUNK].double(), x[a:a + CHUNK].double(), dist)
        tot += t.sum().item()
        mag += t.abs().sum().item()
    s = _recon_scale(dist)
    loss = tot * s
    if dist == "laplace":
        loss = loss * (loss != 0)
    m, lv = mu.double(), logvar.double()
    kl_dims = 0.5 * (-1 - lv + m * m + lv.exp()).sum(0) / B
    kl_mag = 0.5 * (1 + lv.abs() + m * m + lv.exp()).sum(0) / B
    return dict(recon=loss / B, recon_mag=mag * s / B, kl=kl_dims.sum().item(), kl_mag=kl_mag.sum().item(),
                kl_dims=kl_dims, kl_dims_mag=kl_mag)


def ref_kl_grads(mu, logvar, g_kl):
    """(g_mu, |g_mu|, g_logvar, its magnitude) in fp64, g_kl = upstream / B."""
    m, lv = mu.double(), logvar.double()
    e = lv.exp()
    return g_kl * m, abs(g_kl) * m.abs(), g_kl * 0.5 * (e - 1), abs(g_kl) * 0.5 * (e + 1)


M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, seed):
    """Philox4x32-10 (dv_common.cuh) on uint64 arrays holding 32-bit counter words; key (seed_lo, seed_hi)."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & M32 for c in (c0, c1, c2, c3))
    k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64(seed >> 32)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & M32
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & M32, (k1 + np.uint64(0xBB67AE85)) & M32
    return c0, c1, c2, c3


def _unit_open(w):
    """u = (w >> 8) 2^-24 + 2^-25 in (0, 1], evaluated in fp32 as the kernel does (the sum rounds for w >> 8 >= 2^23;
    an fp64 u would move eps by up to 1e-4 where u is within 1e-3 of 1)."""
    k = (w >> np.uint64(8)).astype(np.float32)
    return (k * np.float32(2.0 ** -24) + np.float32(2.0 ** -25)).astype(np.float64)


def host_eps(n, seed, offset):
    """eps[i] of dv_reparam_fwd's device noise, i < n, in fp64: Philox at counter words (c_lo, c_hi, 0, 0) with
    c = offset + i, Box-Muller on words x and y."""
    c = np.uint64(offset) + np.arange(n, dtype=np.uint64)
    x, y, _, _ = philox4x32_10(c & M32, c >> np.uint64(32), np.zeros_like(c), np.zeros_like(c), seed)
    u1, u2 = _unit_open(x), _unit_open(y)
    return torch.from_numpy(np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2))


def ref_factor(d_z, d_perm, up_tc, up_ce):
    """fp64 FactorVAE heads: tc = mean(d_z[:, 0] - d_z[:, 1]), ce = (CE(d_z, 0) + CE(d_perm, 1)) / 2 and their input
    gradients for upstream gradients up_tc, up_ce, with the magnitudes the sums add up."""
    z, p = d_z.double(), d_perm.double()
    h = z.shape[0]
    lse_z, lse_p = torch.logsumexp(z, 1), torch.logsumexp(p, 1)
    tc = (z[:, 0] - z[:, 1]).mean().item()
    tc_mag = (z[:, 0].abs() + z[:, 1].abs()).mean().item()
    ce = 0.5 * ((lse_z - z[:, 0]).mean() + (lse_p - p[:, 1]).mean()).item()
    ce_mag = 0.5 * ((lse_z.abs() + z[:, 0].abs()).mean() + (lse_p.abs() + p[:, 1].abs()).mean()).item()
    g_tc = torch.full((h, 2), up_tc / h, dtype=torch.float64) * torch.tensor([1.0, -1.0], dtype=torch.float64)
    u = up_ce * 0.5 / h
    g_z = u * (torch.softmax(z, 1) - torch.tensor([1.0, 0.0], dtype=torch.float64))
    g_p = u * (torch.softmax(p, 1) - torch.tensor([0.0, 1.0], dtype=torch.float64))
    return dict(tc=tc, tc_mag=tc_mag, ce=ce, ce_mag=ce_mag, g_tc=g_tc, g_z=g_z, g_p=g_p, u=abs(u))


def torch_adam_step(p, g, m, v, step0, lr, betas, eps, grad_scale):
    """One step of CPU torch.optim.Adam(foreach=False) from state (m, v, step0), the gradient scaled in place first as
    the Trainer's non-fused path does.  -> (p, exp_avg, exp_avg_sq, step)."""
    q = p.detach().clone().requires_grad_(True)
    opt = torch.optim.Adam([q], lr=lr, betas=betas, eps=eps, foreach=False)
    opt.state[q] = {"step": torch.tensor(float(step0)), "exp_avg": m.clone(), "exp_avg_sq": v.clone()}
    q.grad = g.clone().mul_(grad_scale)
    opt.step()
    st = opt.state[q]
    return q.detach(), st["exp_avg"], st["exp_avg_sq"], float(st["step"])


def ulps(got, ref, *terms):
    """max |got - ref| in fp32 ulps of the largest magnitude among ref and `terms` per element."""
    got, ref = got.double().cpu(), ref.double().cpu()
    scale = ref.abs()
    for t in terms:
        scale = torch.maximum(scale, t.double().abs().cpu())
    s32 = scale.float()
    ulp = (torch.nextafter(s32, torch.tensor(float("inf"))) - s32).double()
    return ((got - ref).abs() / ulp).max().item()


# ---------------------------------------------------------------------------------------------------------------------
# CPU self-checks of the references
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dist", list(DISTS))
@pytest.mark.parametrize("regime", ["k255", "saturated", "equal"])
def test_loss_reference_matches_the_oracle_and_autograd(dist, regime):
    """ref_vae_loss and the analytic gradients equal O.reconstruction_loss / O.kl_normal and their fp64 autograd."""
    recon, data, mu, logvar = loss_inputs(5, (1, 8, 8), 7, regime, "extreme", 3)
    r, x, m, lv = (t.double().requires_grad_(True) for t in (recon, data, mu, logvar))
    rec = O.reconstruction_loss(x.detach(), r, dist)
    kl, kl_dims = O.kl_normal(m, lv)
    (1.7 * rec + 0.3 * kl).backward()
    ref = ref_vae_loss(recon, data, mu, logvar, dist)
    assert math.isclose(ref["recon"], rec.item(), rel_tol=1e-12, abs_tol=1e-300)
    assert math.isclose(ref["kl"], kl.item(), rel_tol=1e-12)
    assert torch.allclose(ref["kl_dims"], kl_dims.detach(), rtol=1e-12, atol=0)
    g_r, _ = _recon_grad(recon.double(), data.double(), dist, 1.7 / 5, ref["recon"] != 0)
    assert torch.allclose(g_r, r.grad.view_as(g_r), rtol=1e-12, atol=0)
    g_mu, _, g_lv, _ = ref_kl_grads(mu, logvar, 0.3 / 5)
    assert torch.allclose(g_mu, m.grad, rtol=1e-12, atol=0) and torch.allclose(g_lv, lv.grad, rtol=1e-12, atol=1e-300)


def test_laplace_reference_zero_loss():
    x = torch.rand(3, 1, 4, 4)
    ref = ref_vae_loss(x, x, torch.zeros(3, 2), torch.zeros(3, 2), "laplace")
    assert ref["recon"] == 0.0 and O.reconstruction_loss(x, x.clone(), "laplace").item() == 0.0
    g, _ = _recon_grad(x.double(), x.double(), "laplace", 1.0, False)
    assert torch.count_nonzero(g) == 0


def test_host_philox_known_answers():
    """philox4x32_10 against the Random123 known-answer vectors, and word x with counter word 0x5EED against the
    permutation test's restatement."""
    def one(ctr, key):
        return [int(w[0]) for w in philox4x32_10(*[np.array([c], dtype=np.uint64) for c in ctr], key)]
    assert one((0, 0, 0, 0), 0) == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    assert one((0xFFFFFFFF,) * 4, 0xFFFFFFFFFFFFFFFF) == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
    assert one((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0x299F31D0 << 32) | 0xA4093822) == \
        [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]
    from test_factor_global_gpu import philox_x
    c = np.array([0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 40 + 17], dtype=np.uint64)
    seed = 0x0123456789ABCDEF
    x = philox4x32_10(c & M32, c >> np.uint64(32), np.full_like(c, 0x5EED), np.zeros_like(c), seed)[0]
    assert np.array_equal(x, philox_x(c, seed))


def test_host_eps_is_standard_normal():
    e = host_eps(1 << 18, 99, 2 ** 32 - 5000)
    assert abs(e.mean().item()) < 0.01 and abs(e.std().item() - 1) < 0.01
    assert abs((e[1:] * e[:-1]).mean().item()) < 0.01


@pytest.mark.parametrize("regime", ["randn", "sat30", "sat1e4", "ties"])
def test_factor_reference_matches_torch(regime):
    d_z, d_perm = factor_inputs(37, regime)
    z, p = d_z.double().requires_grad_(True), d_perm.double().requires_grad_(True)
    tc = (z[:, 0] - z[:, 1]).mean()
    ones = torch.ones(37, dtype=torch.long)
    ce = 0.5 * (F.cross_entropy(z, torch.zeros_like(ones)) + F.cross_entropy(p, ones))
    (2 * tc + 3 * ce).backward()
    ref = ref_factor(d_z, d_perm, 2.0, 3.0)
    assert math.isclose(ref["tc"], tc.item(), rel_tol=1e-12, abs_tol=1e-12)
    assert math.isclose(ref["ce"], ce.item(), rel_tol=1e-12, abs_tol=1e-12)
    assert torch.allclose(ref["g_tc"] + ref["g_z"], z.grad, rtol=1e-12, atol=1e-15)
    assert torch.allclose(ref["g_p"], p.grad, rtol=1e-12, atol=1e-15)


def test_torch_adam_reference_restates_the_update():
    """torch_adam_step against the update written out in fp64 (a loose bar: torch works in fp32)."""
    g = torch.Generator().manual_seed(3)
    p, gr, m = (torch.randn(1000, generator=g) for _ in range(3))
    v = torch.rand(1000, generator=g)
    lr, (b1, b2), eps, s, step0 = 1e-2, (0.5, 0.9), 1e-6, 1 / 3, 999
    q, m1, v1, st = torch_adam_step(p, gr, m, v, step0, lr, (b1, b2), eps, s)
    gs = gr.double() * s
    m_ref = b1 * m.double() + (1 - b1) * gs
    v_ref = b2 * v.double() + (1 - b2) * gs * gs
    t = step0 + 1
    p_ref = p.double() - lr / (1 - b1 ** t) * m_ref / (v_ref.sqrt() / math.sqrt(1 - b2 ** t) + eps)
    assert st == t
    assert torch.allclose(m1.double(), m_ref, rtol=1e-6, atol=1e-7)
    assert torch.allclose(v1.double(), v_ref, rtol=1e-6, atol=1e-7)
    assert torch.allclose(q.double(), p_ref, rtol=1e-6, atol=1e-7)


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
SATURATED = torch.tensor([0.0, 1.0, 1e-30, 1 - 2.0 ** -24, 1e-40])    # 1e-40 is an fp32 subnormal


def loss_inputs(B, img, D, regime, latent, seed):
    """(recon, data [B, *img], mu, logvar [B, D]) fp32 CPU.
    Data regimes: 'binary' (dSprites-like 0/1), 'k255' (k/255), each with recon = sigmoid(3 randn); 'saturated'
    (every fourth recon from SATURATED, data 0/1); 'equal' (every other recon == data).
    Latent regimes: 'spread', 'extreme' (logvar over [-30, 20], |mu| up to 50), 'untrained' (mu, logvar ~ 1e-3)."""
    g = torch.Generator().manual_seed(seed)
    shape = (B,) + tuple(img)
    recon = torch.sigmoid(3 * torch.randn(shape, generator=g))
    if regime == "binary" or regime == "saturated":
        data = (torch.rand(shape, generator=g) < 0.3).float()
    else:
        data = torch.randint(0, 256, shape, generator=g).float() / 255
    flat = recon.view(-1)
    if regime == "saturated":
        idx = torch.arange(0, flat.numel(), 4)
        flat[idx] = SATURATED[torch.randint(0, len(SATURATED), (len(idx),), generator=g)]
    elif regime == "equal":
        flat[::2] = data.view(-1)[::2]
    if latent == "spread":
        mu, lv = torch.randn(B, D, generator=g) * 2, torch.randn(B, D, generator=g) - 1
    elif latent == "extreme":
        mu = (torch.rand(B, D, generator=g) * 2 - 1) * 50
        lv = torch.rand(B, D, generator=g) * 50 - 30
        lv.view(-1)[:2] = torch.tensor([-30.0, 20.0])[:lv.numel()]
    else:
        mu, lv = torch.randn(B, D, generator=g) * 1e-3, torch.randn(B, D, generator=g) * 1e-3
    return recon, data, mu, lv


def factor_inputs(h, regime, seed=0):
    g = torch.Generator().manual_seed(h * 7 + seed)
    if regime == "randn":
        return torch.randn(h, 2, generator=g), torch.randn(h, 2, generator=g)
    if regime in ("sat30", "sat1e4"):
        a = 30.0 if regime == "sat30" else 1e4
        return [(torch.randint(0, 2, (h, 2), generator=g).float() * 2 - 1) * a for _ in range(2)]
    v = torch.randn(h, 1, generator=g) * 5                 # exact ties: both logits of a row equal
    w = torch.randn(h, 1, generator=g) * 5
    return v.repeat(1, 2), w.repeat(1, 2)


# ---------------------------------------------------------------------------------------------------------------------
# device helpers
# ---------------------------------------------------------------------------------------------------------------------
def _bits(t):
    return t.contiguous().view(torch.int32)


def _guarded(n, fill=float("nan")):
    """n floats of `fill` followed by GUARD sentinel floats."""
    t = torch.full((n + GUARD,), fill, device="cuda")
    _bits(t)[n:] = SENTINEL
    return t


def _guarded_copy(src):
    t = _guarded(src.numel())
    t[:src.numel()] = src.reshape(-1).to("cuda")
    return t


def _intact(t, n):
    return bool((_bits(t)[n:] == SENTINEL).all())


def _native():
    from disvae import _native as N
    return N


def _loss_grid(n):
    """Blocks of vae_loss_fwd_kernel for n elements: min(ceil(floor(n / 4) / 1024), 264), at least 1."""
    return min(max(-(-(n // 4) // 1024), 1), LOSS_BLOCKS)


class LossCall:
    """Guarded device copies of one loss input and the raw dv_vae_loss_fwd/bwd calls on it, mu/logvar either
    interleaved [B, D, 2] as the encoder writes them (ld 2, row stride 2D) or contiguous [B, D] (ld 1, row stride D)."""

    def __init__(self, recon, data, mu, logvar):
        self.B, self.D = mu.shape
        self.n = recon.numel()
        self.n_img = self.n // self.B
        self.recon, self.data = _guarded_copy(recon), _guarded_copy(data)
        self.mu, self.lv = _guarded_copy(mu), _guarded_copy(logvar)
        self.ml = _guarded_copy(torch.stack([mu, logvar], -1))

    def layout(self, interleaved):
        if interleaved:
            return self.ml.data_ptr(), self.ml.data_ptr() + 4, 2, 2 * self.D
        return self.mu.data_ptr(), self.lv.data_ptr(), 1, self.D

    def fwd(self, dist, interleaved, ws=None):
        """-> (out [2 + D], workspace, launches); asserts every guard."""
        N = _native()
        mp, lp, ld, rs = self.layout(interleaved)
        if ws is None:
            ws = _guarded(LOSS_WS_FLOATS)
            ws[0] = 0.0                                  # the counter starts at 0, partials stay NaN until written
        out = _guarded(2 + self.D)
        before = N.lib().dv_launch_count()
        N.call("dv_vae_loss_fwd", self.recon.data_ptr(), self.data.data_ptr(), self.n_img, self.B, DISTS[dist], mp, lp,
               ld, rs, self.D, out.data_ptr(), ws.data_ptr(), N.stream())
        launches = N.lib().dv_launch_count() - before
        torch.cuda.synchronize()
        assert _intact(out, 2 + self.D) and _intact(ws, LOSS_WS_FLOATS), "loss forward wrote past its buffers"
        return out[:2 + self.D].clone(), ws, launches

    def bwd(self, dist, interleaved, fwd_out, upstream):
        N = _native()
        mp, lp, ld, rs = self.layout(interleaved)
        nz = self.B * self.D
        g_r, g_mu, g_lv = _guarded(self.n), _guarded(nz), _guarded(nz)
        up = torch.tensor(upstream, dtype=torch.float32, device="cuda")
        before = N.lib().dv_launch_count()
        N.call("dv_vae_loss_bwd", self.recon.data_ptr(), self.data.data_ptr(), self.n_img, self.B, DISTS[dist], mp, lp,
               ld, rs, self.D, fwd_out.data_ptr(), up.data_ptr(), g_r.data_ptr(), g_mu.data_ptr(), g_lv.data_ptr(),
               N.stream())
        assert N.lib().dv_launch_count() - before == 1
        torch.cuda.synchronize()
        assert _intact(g_r, self.n) and _intact(g_mu, nz) and _intact(g_lv, nz), "loss backward wrote past its outputs"
        return g_r[:self.n], g_mu[:nz].view(self.B, self.D), g_lv[:nz].view(self.B, self.D)


def _written_partials(ws):
    """Recon partials the forward wrote (the rest keep the NaN fill): the grid it ran."""
    part = ws[1:1 + LOSS_BLOCKS].cpu()
    k = int(torch.isfinite(part).sum())
    assert torch.isfinite(part[:k]).all(), "recon partials not a prefix"
    return k


UPSTREAM = (1.7, 0.3)


def check_loss_case(recon, data, mu, logvar, dist, tag, grads=True):
    """Forward in both layouts (bit-identical, repeatable), the grid from the workspace, forward vs ref_vae_loss and
    every gradient element vs fp64.  -> the worst errors."""
    k = LossCall(recon, data, mu, logvar)
    B, D, n = k.B, k.D, k.n
    grid = _loss_grid(n)
    out, ws, launches = k.fwd(dist, True)
    assert launches == 1
    assert _written_partials(ws) == grid, "%s: expected a %d-block grid" % (tag, grid)
    assert _bits(ws[:1])[0].item() == 0, tag + ": counter not reset"
    out_c, _, _ = k.fwd(dist, False)
    assert torch.equal(_bits(out), _bits(out_c)), tag + ": layouts differ"
    out_2, _, _ = k.fwd(dist, True, ws)
    assert torch.equal(_bits(out), _bits(out_2)), tag + ": repeat launch on one workspace differs"
    ref = ref_vae_loss(recon, data, mu, logvar, dist)
    o = out.double().cpu()
    e = dict(recon=abs(o[0].item() - ref["recon"]) / max(ref["recon_mag"], 1e-300),
             kl=abs(o[1].item() - ref["kl"]) / ref["kl_mag"],
             kl_dims=((o[2:] - ref["kl_dims"]).abs() / ref["kl_dims_mag"]).max().item())
    assert torch.isfinite(o).all(), tag + ": not finite"
    if grads:
        up = [float(np.float32(u)) for u in UPSTREAM]
        g_r, g_mu, g_lv = k.bwd(dist, True, out, UPSTREAM)
        g_r2, g_mu2, g_lv2 = k.bwd(dist, False, out, UPSTREAM)
        assert all(torch.equal(_bits(a), _bits(b)) for a, b in ((g_r, g_r2), (g_mu, g_mu2), (g_lv, g_lv2))), \
            tag + ": backward layouts differ"
        worst = 0.0
        rf, xf = recon.reshape(-1), data.reshape(-1)
        for a in range(0, n, CHUNK):
            want, scale = _recon_grad(rf[a:a + CHUNK].double(), xf[a:a + CHUNK].double(), dist, up[0] / B,
                                      ref["recon"] != 0)
            got = g_r[a:a + CHUNK].double().cpu()
            worst = max(worst, ((got - want).abs() / scale.clamp_min(1e-300)).max().item())
        e["g_recon"] = worst
        w_mu, m_mu, w_lv, m_lv = ref_kl_grads(mu, logvar, up[1] / B)
        e["g_mu"] = ((g_mu.double().cpu() - w_mu).abs() / m_mu.clamp_min(1e-300)).max().item() / U
        e["g_logvar"] = ((g_lv.double().cpu() - w_lv).abs() / m_lv).max().item() / U
    print("%s grid %d: recon %.2e, kl %.2e, kl dims %.2e%s" % (
        tag, grid, e["recon"], e["kl"], e["kl_dims"],
        ", grads (ulps) recon %.1f mu %.1f logvar %.1f" % (e["g_recon"], e["g_mu"], e["g_logvar"]) if grads else ""))
    assert e["recon"] <= RECON_TOL, "%s: recon err %.3e" % (tag, e["recon"])
    assert e["kl"] <= KL_TOL and e["kl_dims"] <= KL_TOL, "%s: kl err %.3e / %.3e" % (tag, e["kl"], e["kl_dims"])
    if grads:
        for name in ("g_recon", "g_mu", "g_logvar"):
            assert e[name] <= GRAD_ULPS, "%s: %s err %.1f ulps" % (tag, name, e[name])
    return e


# ---------------------------------------------------------------------------------------------------------------------
# 1. reconstruction + KL
# ---------------------------------------------------------------------------------------------------------------------
IMAGES = [(1, 32, 32), (3, 32, 32), (1, 64, 64), (3, 64, 64)]


@pytest.mark.gpu
@pytest.mark.parametrize("dist", list(DISTS))
@pytest.mark.parametrize("img", IMAGES, ids=["x".join(map(str, i)) for i in IMAGES])
@pytest.mark.parametrize("B", [1, 6, 257, 1024, 2048])
def test_vae_loss_training_shapes(B, img, dist):
    """From a 1-block grid (B 1, 1x32x32) to the 264-block cap with several grid-stride passes (2048 x 3x64x64, 25 M
    elements); dSprites-like binary data for one channel, k/255 for three, D = 10."""
    regime = "binary" if img[0] == 1 else "k255"
    check_loss_case(*loss_inputs(B, img, 10, regime, "spread", B + img[0] + img[1]), dist,
                    "B=%d %s %s %s" % (B, "x".join(map(str, img)), regime, dist))


@pytest.mark.gpu
@pytest.mark.parametrize("dist", list(DISTS))
@pytest.mark.parametrize("latent", ["spread", "extreme", "untrained"])
@pytest.mark.parametrize("regime", ["binary", "k255", "saturated", "equal"])
@pytest.mark.parametrize("B,img", [(1, (1, 32, 32)), (257, (1, 64, 64))], ids=["grid1", "grid257"])
def test_vae_loss_input_regimes(B, img, regime, latent, dist):
    check_loss_case(*loss_inputs(B, img, 10, regime, latent, 5 * B), dist,
                    "B=%d %s/%s %s" % (B, regime, latent, dist))


@pytest.mark.gpu
@pytest.mark.parametrize("dist", list(DISTS))
@pytest.mark.parametrize("D", [1, 10, 64, 300, 1024])
@pytest.mark.parametrize("B,img", [(4, (1, 32, 32)), (1024, (1, 64, 64))], ids=["grid1", "grid264"])
def test_vae_loss_latent_sizes(B, img, D, dist):
    """D up to 1024: on a 1-block grid one block reduces every dimension; on 264 blocks D = 300 and 1024 make
    blocks walk several dimensions."""
    check_loss_case(*loss_inputs(B, img, D, "k255", "extreme", D), dist, "B=%d D=%d %s" % (B, D, dist))


@pytest.mark.gpu
@pytest.mark.parametrize("dist", list(DISTS))
@pytest.mark.parametrize("B,n_img", [(1, 1), (3, 1027), (1, 4099), (7, 300001)])
def test_vae_loss_element_tail(B, n_img, dist):
    """n = B x n_img not a multiple of 4: block 0 adds the last n % 4 elements in its tail loop."""
    g = torch.Generator().manual_seed(n_img)
    recon = torch.sigmoid(3 * torch.randn(B, n_img, generator=g))
    data = torch.randint(0, 256, (B, n_img), generator=g).float() / 255
    tail = (B * n_img) % 4
    assert tail
    recon.view(-1)[-tail:] = 1e-30                     # a tail the sum cannot lose in rounding
    data.view(-1)[-tail:] = 1.0
    mu, lv = torch.randn(B, 5, generator=g), torch.randn(B, 5, generator=g)
    check_loss_case(recon, data, mu, lv, dist, "B=%d n_img=%d tail %d %s" % (B, n_img, tail, dist))


@pytest.mark.gpu
def test_laplace_all_equal_is_zero_with_zero_gradient():
    x = torch.rand(257, 1, 64, 64)
    mu, lv = torch.randn(257, 10), torch.randn(257, 10)
    k = LossCall(x, x, mu, lv)
    out, _, _ = k.fwd("laplace", True)
    assert out[0].item() == 0.0
    g_r, _, _ = k.bwd("laplace", True, out, UPSTREAM)
    assert torch.count_nonzero(g_r).item() == 0


@pytest.mark.gpu
def test_vae_loss_workspace_reuse_across_grids():
    """One workspace: a 264-block launch, a 1-block launch, a 264-block launch again.  The last block resets the
    counter, so each result is correct."""
    big = LossCall(*loss_inputs(2048, (1, 64, 64), 10, "binary", "spread", 1))
    small = LossCall(*loss_inputs(1, (1, 32, 32), 10, "binary", "spread", 2))
    ref_big = big.fwd("bernoulli", True)[0]
    ref_small = small.fwd("bernoulli", True)[0]
    ws = _guarded(LOSS_WS_FLOATS)
    ws[0] = 0.0
    for k, want, grid in ((big, ref_big, 264), (small, ref_small, 1), (big, ref_big, 264)):
        assert _loss_grid(k.n) == grid
        out, ws, _ = k.fwd("bernoulli", True, ws)
        assert torch.equal(_bits(out), _bits(want)), "grid %d after another grid on one workspace" % grid


@pytest.mark.gpu
def test_vae_loss_wrapper_is_the_raw_call():
    """ops.VaeLossFn on the encoder's interleaved views gives the raw call's bits, forward and backward."""
    from disvae import ops
    recon, data, mu, lv = loss_inputs(64, (1, 32, 32), 10, "binary", "spread", 9)
    k = LossCall(recon, data, mu, lv)
    out, _, _ = k.fwd("bernoulli", True)
    g_r, g_mu, g_lv = k.bwd("bernoulli", True, out, UPSTREAM)
    ml = torch.stack([mu, lv], -1).reshape(64, 20).cuda().requires_grad_(True)
    mud, lvd = ml.view(64, 10, 2).unbind(-1)
    rd = recon.cuda().requires_grad_(True)
    o = ops.VaeLossFn.apply(rd, data.cuda(), mud, lvd, DISTS["bernoulli"])
    assert torch.equal(_bits(o.detach()), _bits(out))
    (UPSTREAM[0] * o[0] + UPSTREAM[1] * o[1]).backward()
    assert torch.equal(_bits(rd.grad.view(-1)), _bits(g_r))
    g = ml.grad.view(64, 10, 2)
    assert torch.equal(_bits(g[..., 0]), _bits(g_mu)) and torch.equal(_bits(g[..., 1]), _bits(g_lv))


# ---------------------------------------------------------------------------------------------------------------------
# 2. reparameterisation
# ---------------------------------------------------------------------------------------------------------------------
def _reparam_call(mu, lv, interleaved, eps=None, seed=0, offset=None):
    """Raw dv_reparam_fwd on guarded copies -> (z, eps_out or None)."""
    N = _native()
    B, D = mu.shape
    n = B * D
    if interleaved:
        ml = _guarded_copy(torch.stack([mu, lv], -1))
        mp, lp, ld, rs = ml.data_ptr(), ml.data_ptr() + 4, 2, 2 * D
    else:
        m, v = _guarded_copy(mu), _guarded_copy(lv)
        mp, lp, ld, rs = m.data_ptr(), v.data_ptr(), 1, D
    z = _guarded(n)
    e_in = None if eps is None else _guarded_copy(eps)
    e_out = _guarded(n) if eps is None else None
    N.call("dv_reparam_fwd", mp, lp, ld, rs, None if e_in is None else e_in.data_ptr(), seed,
           None if offset is None else offset.data_ptr(), z.data_ptr(), None if e_out is None else e_out.data_ptr(),
           B, D, N.stream())
    torch.cuda.synchronize()
    assert _intact(z, n) and (e_out is None or _intact(e_out, n)), "reparam wrote past its outputs"
    return z[:n].view(B, D), None if e_out is None else e_out[:n].view(B, D)


def _reparam_inputs(B, D, seed):
    g = torch.Generator().manual_seed(seed)
    mu = torch.randn(B, D, generator=g) * 3
    lv = torch.rand(B, D, generator=g) * 50 - 30                # logvar over [-30, 20]
    lv.view(-1)[:2] = torch.tensor([-30.0, 20.0])[:lv.numel()]
    return mu, lv, torch.randn(B, D, generator=g)


@pytest.mark.gpu
@pytest.mark.parametrize("B,D", [(1, 1), (3, 7), (257, 10), (1024, 64), (4096, 64)])
def test_reparam_injected_eps(B, D):
    """z, g_mu, g_logvar vs fp64 in both layouts, B x D from 1 to past the 264 x 256-thread grid (4096 x 64)."""
    from disvae import ops
    N = _native()
    mu, lv, eps = _reparam_inputs(B, D, B * D)
    s = (0.5 * lv.double()).exp()
    want = mu.double() + s * eps.double()
    z_i, _ = _reparam_call(mu, lv, True, eps)
    z_c, _ = _reparam_call(mu, lv, False, eps)
    assert torch.equal(_bits(z_i), _bits(z_c)), "layouts differ"
    e_z = ulps(z_i, want, mu, s * eps.double())
    # backward through the wrapper (interleaved views), against fp64 and against the raw call on contiguous inputs
    ml = torch.stack([mu, lv], -1).reshape(B, 2 * D).cuda().requires_grad_(True)
    mud, lvd = ml.view(B, D, 2).unbind(-1)
    zd = ops.ReparamFn.apply(mud, lvd, eps.cuda(), 0, None)
    assert torch.equal(_bits(zd.detach()), _bits(z_i))
    g_z = torch.randn(B, D, generator=torch.Generator().manual_seed(1))
    zd.backward(g_z.cuda())
    g = ml.grad.view(B, D, 2)
    assert torch.equal(_bits(g[..., 0]), _bits(g_z.cuda())), "g_mu is not g_z"
    w_lv = g_z.double() * eps.double() * 0.5 * s
    e_lv = ulps(g[..., 1], w_lv)
    lvc, epsc, gzc = _guarded_copy(lv), _guarded_copy(eps), _guarded_copy(g_z)
    g_mu, g_lv = _guarded(B * D), _guarded(B * D)
    N.call("dv_reparam_bwd", gzc.data_ptr(), lvc.data_ptr(), 1, D, epsc.data_ptr(), g_mu.data_ptr(), g_lv.data_ptr(),
           B, D, N.stream())
    torch.cuda.synchronize()
    assert _intact(g_mu, B * D) and _intact(g_lv, B * D)
    assert torch.equal(_bits(g_lv[:B * D].view(B, D)), _bits(g[..., 1])), "backward layouts differ"
    print("reparam B=%d D=%d: z %.1f ulps, g_logvar %.1f ulps" % (B, D, e_z, e_lv))
    assert e_z <= GRAD_ULPS and e_lv <= GRAD_ULPS, (e_z, e_lv)


SEED = 0x9E3779B97F4A7C15      # both key halves nonzero


@pytest.mark.gpu
@pytest.mark.parametrize("start", [0, 2 ** 32 - 1000, 3 * 2 ** 32 + 12345], ids=["0", "2^32-1000", "3x2^32"])
@pytest.mark.parametrize("B,D", [(1, 1), (37, 10), (4096, 64)])
def test_reparam_device_noise_is_philox_box_muller(B, D, start):
    """Every eps against host_eps at counters start + i; the offset advances by B x D and the next call draws the
    following counters; a start of 2^32 - 1000 carries into the high counter word mid-call."""
    from disvae import ops
    n = B * D
    off = torch.tensor([start], dtype=torch.int64, device="cuda")
    zeros = torch.zeros(B, D, device="cuda")
    worst = 0.0
    for k in range(2):
        e = ops.ReparamFn.apply(zeros, zeros, None, SEED, off)          # z = 0 + 1 * eps
        assert off.item() == start + (k + 1) * n
        want = host_eps(n, SEED, start + k * n).view(B, D)
        err = ((e.double().cpu() - want).abs() / (1 + want.abs())).max().item()
        worst = max(worst, err)
        assert err <= EPS_TOL, "draw %d: eps err %.3e" % (k, err)
    # the raw call in both layouts writes the same eps it used for z
    mu, lv, _ = _reparam_inputs(B, D, 3)
    off.fill_(start)
    z, e_out = _reparam_call(mu, lv, True, None, SEED, off)
    off.fill_(start)
    z_c, e_c = _reparam_call(mu, lv, False, None, SEED, off)
    assert torch.equal(_bits(z), _bits(z_c)) and torch.equal(_bits(e_out), _bits(e_c))
    want = host_eps(n, SEED, start).view(B, D)
    assert ((e_out.double().cpu() - want).abs() / (1 + want.abs())).max().item() <= EPS_TOL
    z_inj, _ = _reparam_call(mu, lv, True, e_out.cpu())
    assert torch.equal(_bits(z), _bits(z_inj)), "z is not mu + std * eps_out"
    # the backward consumes the eps the forward drew
    off.fill_(start)
    ml = torch.stack([mu, lv], -1).reshape(B, 2 * D).cuda().requires_grad_(True)
    mud, lvd = ml.view(B, D, 2).unbind(-1)
    zd = ops.ReparamFn.apply(mud, lvd, None, SEED, off)
    g_z = torch.randn(B, D, generator=torch.Generator().manual_seed(2))
    zd.backward(g_z.cuda())
    w_lv = g_z.double() * want * 0.5 * (0.5 * lv.double()).exp()
    scale = g_z.double().abs() * (1 + want.abs()) * 0.5 * (0.5 * lv.double()).exp()
    e_lv = ((ml.grad.view(B, D, 2)[..., 1].double().cpu() - w_lv).abs() / scale).max().item()
    print("device noise B=%d D=%d start %d: eps err %.2e, g_logvar err %.2e" % (B, D, start, worst, e_lv))
    assert e_lv <= 2 * EPS_TOL, e_lv


@pytest.mark.gpu
def test_reparam_noise_is_not_reused_or_correlated():
    """Consecutive draws of one stream share no value, and neighbouring elements are uncorrelated."""
    from disvae import ops
    off = torch.zeros(1, dtype=torch.int64, device="cuda")
    zeros = torch.zeros(4096, 64, device="cuda")
    e1 = ops.ReparamFn.apply(zeros, zeros, None, SEED, off).view(-1).double()
    e2 = ops.ReparamFn.apply(zeros, zeros, None, SEED, off).view(-1).double()
    assert (e1 == e2).double().mean().item() < 1e-4
    for a, b in ((e1[1:], e1[:-1]), (e1, e2), (e1[64:], e1[:-64])):
        assert abs((a * b).mean().item()) < 0.01


# ---------------------------------------------------------------------------------------------------------------------
# 3. FactorVAE heads
# ---------------------------------------------------------------------------------------------------------------------
def _factor_raw(d_z, d_perm, up_tc, up_ce):
    """The four raw calls on guarded buffers -> (tc, ce, g_tc, g_z, g_p)."""
    N = _native()
    h = d_z.shape[0]
    z, p = _guarded_copy(d_z), _guarded_copy(d_perm)
    ut, uc = _guarded_copy(torch.tensor([up_tc])), _guarded_copy(torch.tensor([up_ce]))
    tc, ce = _guarded(1), _guarded(1)
    g_tc, g_z, g_p = _guarded(2 * h), _guarded(2 * h), _guarded(2 * h)
    before = N.lib().dv_launch_count()
    N.call("dv_factor_tc_fwd", z.data_ptr(), h, tc.data_ptr(), N.stream())
    N.call("dv_factor_ce_fwd", z.data_ptr(), p.data_ptr(), h, ce.data_ptr(), N.stream())
    N.call("dv_factor_tc_bwd", ut.data_ptr(), h, g_tc.data_ptr(), N.stream())
    N.call("dv_factor_ce_bwd", z.data_ptr(), p.data_ptr(), uc.data_ptr(), h, g_z.data_ptr(), g_p.data_ptr(), N.stream())
    assert N.lib().dv_launch_count() - before == 4
    torch.cuda.synchronize()
    assert all(_intact(t, 1) for t in (tc, ce)) and all(_intact(t, 2 * h) for t in (g_tc, g_z, g_p))
    return tc[0], ce[0], g_tc[:2 * h].view(h, 2), g_z[:2 * h].view(h, 2), g_p[:2 * h].view(h, 2)


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["randn", "sat30", "sat1e4", "ties"])
@pytest.mark.parametrize("h", [1, 2, 255, 256, 257, 1024, 4096])
def test_factor_heads_match_the_fp64_reference(h, regime):
    """TC and CE through ops.FactorTcFn / FactorCeFn against ref_factor, gradients element-wise; the raw calls on
    guarded buffers give the same bits, twice."""
    from disvae import ops
    d_z, d_perm = factor_inputs(h, regime)
    up_tc, up_ce = 2.0, 3.0
    ref = ref_factor(d_z, d_perm, up_tc, up_ce)
    z, p = d_z.cuda().requires_grad_(True), d_perm.cuda().requires_grad_(True)
    tc, ce = ops.FactorTcFn.apply(z), ops.FactorCeFn.apply(z, p)
    (up_tc * tc + up_ce * ce).backward()
    e_tc = abs(tc.item() - ref["tc"]) / max(ref["tc_mag"], 1e-30)
    e_ce = abs(ce.item() - ref["ce"]) / max(ref["ce_mag"], 1e-30)
    e_gz = ((z.grad.double().cpu() - ref["g_tc"] - ref["g_z"]).abs().max().item()) / (ref["u"] + up_tc / h) / U
    e_gp = (p.grad.double().cpu() - ref["g_p"]).abs().max().item() / ref["u"] / U
    raw = _factor_raw(d_z, d_perm, up_tc, up_ce)
    assert torch.equal(_bits(raw[0]), _bits(tc.detach())) and torch.equal(_bits(raw[1]), _bits(ce.detach()))
    e_gtc = ((raw[2].double().cpu() - ref["g_tc"]).abs().max().item()) / (up_tc / h) / U
    e_gz_raw = ((raw[3].double().cpu() - ref["g_z"]).abs().max().item()) / ref["u"] / U
    again = _factor_raw(d_z, d_perm, up_tc, up_ce)
    assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(raw, again)), "not deterministic"
    print("factor h=%d %s: tc %.2e, ce %.2e, grads (ulps) tc %.1f ce_z %.1f ce_perm %.1f both_z %.1f"
          % (h, regime, e_tc, e_ce, e_gtc, e_gz_raw, e_gp, e_gz))
    assert e_tc <= FACTOR_TOL and e_ce <= FACTOR_TOL, (e_tc, e_ce)
    assert max(e_gtc, e_gz_raw, e_gp, e_gz) <= GRAD_ULPS, (e_gtc, e_gz_raw, e_gp, e_gz)


# ---------------------------------------------------------------------------------------------------------------------
# 4. Adam
# ---------------------------------------------------------------------------------------------------------------------
def _adam_state(n, step0, seed):
    g = torch.Generator().manual_seed(seed)
    p, gr = torch.randn(n, generator=g), torch.randn(n, generator=g)
    gr[:3] = torch.tensor([0.0, 1e-20, 1e4])[:n]
    if step0 == 0:
        return p, gr, torch.zeros(n), torch.zeros(n)
    return p, gr, torch.randn(n, generator=g) * 0.1, torch.rand(n, generator=g) * 0.01


def _adam_multi_raw(ps, gs, ms, vs, step0, lr, betas, eps, grad_scale):
    """One dv_adam_multi call over guarded copies -> (params, exp_avgs, exp_avg_sqs, step after)."""
    N = _native()
    bufs = [[_guarded_copy(t) for t in ts] for ts in (ps, gs, ms, vs)]
    n = len(ps)
    arr = ctypes.c_void_p * n
    step = _guarded_copy(torch.tensor([float(step0)]))
    before = N.lib().dv_launch_count()
    N.call("dv_adam_multi", n, *[arr(*[t.data_ptr() for t in b]) for b in bufs],
           (ctypes.c_longlong * n)(*[t.numel() for t in ps]), step.data_ptr(), lr, betas[0], betas[1], eps, grad_scale,
           N.stream())
    assert N.lib().dv_launch_count() - before == 2
    torch.cuda.synchronize()
    for b in bufs:
        assert all(_intact(t, s.numel()) for t, s in zip(b, ps)), "adam_multi wrote past a tensor"
    assert _intact(step, 1)
    out = [[t[:s.numel()].cpu() for t, s in zip(b, ps)] for b in (bufs[0], bufs[2], bufs[3])]
    return out[0], out[1], out[2], step[0].item()


def _check_one_step(got, want, state, hyper, grad_scale, step0, tag):
    """got/want = (p, exp_avg, exp_avg_sq) after one step from state = (p, grad, exp_avg, exp_avg_sq): ulps of each
    against the largest operand it combines.  exp_avg = lerp(m, g, 1 - b1) of m and the scaled g (both of which
    cancel when m ~ g); exp_avg_sq of b2 v and (1 - b2) g^2; p of p and the step lr / bc1 * M / denom, M the larger of
    |m| and |g| that exp_avg came from."""
    lr, (b1, b2), eps = hyper
    p0, m0, v0 = state[0].double(), state[2].double(), state[3].double()
    gs = (state[1] * grad_scale).double()                    # scaled in fp32 first, as torch's reference does
    t = step0 + 1
    denom = want[2].double().sqrt() / math.sqrt(1 - b2 ** t) + eps
    step = lr / (1 - b1 ** t) * torch.maximum(m0.abs(), gs.abs()) / denom
    e = (ulps(got[0], want[0], p0, step), ulps(got[1], want[1], m0, gs),
         ulps(got[2], want[2], b2 * v0, (1 - b2) * gs * gs))
    assert e[0] <= ADAM_P_ULPS and max(e[1:]) <= ADAM_ULPS, \
        "%s: p %.1f, exp_avg %.1f, exp_avg_sq %.1f ulps" % ((tag,) + e)
    return e


HYPER = [(5e-4, (0.9, 0.999), 1e-8), (1e-2, (0.5, 0.9), 1e-6), (1e-2, (0.0, 0.99), 1e-8)]


@pytest.mark.gpu
@pytest.mark.parametrize("step0", [0, 1, 999, 100000])
@pytest.mark.parametrize("grad_scale", [1.0, 0.5, 1 / 3, 0.125])
@pytest.mark.parametrize("hyper", HYPER, ids=["default", "lr1e-2_b0.5_0.9_eps1e-6", "lr1e-2_b0_0.99"])
def test_adam_one_step_matches_torch(hyper, grad_scale, step0):
    """dv_adam_step and dv_adam_multi from the same state as CPU torch.optim.Adam: p, exp_avg, exp_avg_sq within
    ADAM_ULPS per element, step counter advanced by one."""
    from disvae import ops
    lr, betas, eps = hyper
    n = 70001
    p, gr, m, v = _adam_state(n, step0, int(grad_scale * 1000) + step0)
    want = torch_adam_step(p, gr, m, v, step0, lr, betas, eps, grad_scale)
    tag = "lr %g betas %s eps %g scale %g step0 %d" % (lr, betas, eps, grad_scale, step0)
    pd, md, vd = p.cuda(), m.cuda(), v.cuda()
    sd = torch.tensor([float(step0)], device="cuda")
    ops.adam_step(pd, gr.cuda(), md, vd, sd, lr, betas, eps, grad_scale)
    assert sd.item() == want[3]
    e1 = _check_one_step((pd, md, vd), want, (p, gr, m, v), hyper, grad_scale, step0, "adam_step " + tag)
    ps, ms, vs, st = _adam_multi_raw([p], [gr], [m], [v], step0, lr, betas, eps, grad_scale)
    assert st == want[3]
    e2 = _check_one_step((ps[0], ms[0], vs[0]), want, (p, gr, m, v), hyper, grad_scale, step0, "adam_multi " + tag)
    print("adam %s: p %.1f, exp_avg %.1f, exp_avg_sq %.1f ulps (adam_step), %.1f %.1f %.1f (adam_multi)"
          % ((tag,) + e1 + e2))


@pytest.mark.gpu
@pytest.mark.parametrize("hyper", HYPER, ids=["default", "lr1e-2_b0.5_0.9_eps1e-6", "lr1e-2_b0_0.99"])
def test_adam_chain_of_200_steps(hyper):
    """200 steps of dv_adam_step (gradient scale 1/3) against torch, each element within ADAM_CHAIN_TOL of
    |p0| + the path its torch value travelled."""
    from disvae import ops
    lr, betas, eps = hyper
    n = 20000
    g = torch.Generator().manual_seed(7)
    p0 = torch.randn(n, generator=g)
    q = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([q], lr=lr, betas=betas, eps=eps, foreach=False)
    pd, sd = p0.cuda(), torch.zeros(1, device="cuda")
    md, vd = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    path = torch.zeros(n, dtype=torch.float64)
    for _ in range(200):
        gr = torch.randn(n, generator=g) + 0.3 * torch.sin(q.detach())
        prev = q.detach().clone()
        q.grad = gr.clone().mul_(1 / 3)
        opt.step()
        path += (q.detach().double() - prev.double()).abs()
        ops.adam_step(pd, gr.cuda(), md, vd, sd, lr, betas, eps, 1 / 3)
    assert sd.item() == 200.0
    e = ((pd.double().cpu() - q.detach().double()).abs() / (p0.double().abs() + path)).max().item()
    print("adam chain lr %g betas %s: worst err %.2e of |p0| + path" % (lr, betas, e))
    assert e <= ADAM_CHAIN_TOL, e


@pytest.mark.gpu
@pytest.mark.parametrize("numels", [[1, 4095, 4096, 4097, 3 * 4096 + 1], [1 + (i * 997) % 9000 for i in range(48)]],
                         ids=["chunk_edges", "48_tensors"])
def test_adam_multi_tensor_table(numels):
    """One dv_adam_multi call over tensors that end on, before and after the 4096-element chunk boundaries, and over
    a full table of 48 tensors, against torch per element; 49 tensors are refused."""
    lr, betas, eps, scale, step0 = 1e-2, (0.5, 0.9), 1e-6, 1 / 3, 5
    states = [_adam_state(n, step0, i) for i, n in enumerate(numels)]
    got = _adam_multi_raw(*[[s[k] for s in states] for k in range(4)], step0, lr, betas, eps, scale)
    assert got[3] == step0 + 1
    worst = (0.0, 0.0, 0.0)
    for i, s in enumerate(states):
        want = torch_adam_step(*s, step0, lr, betas, eps, scale)
        e = _check_one_step((got[0][i], got[1][i], got[2][i]), want, s, (lr, betas, eps), scale, step0,
                            "tensor %d (%d)" % (i, numels[i]))
        worst = tuple(max(a, b) for a, b in zip(worst, e))
    print("adam_multi %d tensors: p %.1f, exp_avg %.1f, exp_avg_sq %.1f ulps" % ((len(numels),) + worst))


def _torch_and_fused(shapes, seed, lr=5e-4):
    from disvae.fused import FusedAdam
    g = torch.Generator().manual_seed(seed)
    ps_ref = [torch.randn(s, generator=g).requires_grad_(True) for s in shapes]
    ps = [p.detach().clone().cuda().requires_grad_(True) for p in ps_ref]
    opt_ref = torch.optim.Adam(ps_ref, lr=lr, betas=(0.8, 0.95), foreach=False)
    opt = torch.optim.Adam(ps, lr=lr, betas=(0.8, 0.95))
    return g, ps_ref, ps, opt_ref, opt, FusedAdam


def _compare_adams(ps_ref, ps, opt_ref, opt, fused, p0, path, tag):
    fused.flush_state()
    worst = 0.0
    for i, (a, b) in enumerate(zip(ps_ref, ps)):
        assert float(opt.state[b]["step"]) == float(opt_ref.state[a]["step"]), "%s: param %d step count" % (tag, i)
        e = ((b.detach().double().cpu() - a.detach().double()).abs() / (p0[i].abs() + path[i])).max().item()
        worst = max(worst, e)
        assert e <= ADAM_CHAIN_TOL, "%s: param %d err %.3e" % (tag, i, e)
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("count", [49, 100])
def test_fused_adam_beyond_one_table(count):
    """FusedAdam over more tensors than one dv_adam_multi call takes (48): one call per 48 tensors, the step counter
    rewound between them, so every chunk steps at the same count as torch."""
    N = _native()
    assert N.lib().dv_adam_multi_max_tensors() == 48
    shapes = [(1 + (i * 613) % 5000,) for i in range(count)]
    g, ps_ref, ps, opt_ref, opt, FusedAdam = _torch_and_fused(shapes, count)
    fused = FusedAdam(opt)
    p0 = [p.detach().double().clone() for p in ps_ref]
    path = [torch.zeros_like(p) for p in p0]
    for _ in range(5):
        for a, b in zip(ps_ref, ps):
            gr = torch.randn(a.shape, generator=g)
            a.grad, b.grad = gr.clone(), gr.cuda()
        prev = [a.detach().double().clone() for a in ps_ref]
        before = N.lib().dv_launch_count()
        opt_ref.step()
        fused.step()
        assert N.lib().dv_launch_count() - before == 2 * math.ceil(count / 48)
        for i, a in enumerate(ps_ref):
            path[i] += (a.detach().double() - prev[i]).abs()
    e = _compare_adams(ps_ref, ps, opt_ref, opt, fused, p0, path, "%d tensors" % count)
    print("FusedAdam %d tensors, 5 steps: worst err %.2e" % (count, e))


@pytest.mark.gpu
def test_fused_adam_skipped_parameters_follow_torch():
    """torch.optim.Adam keeps one step count per parameter and leaves a parameter without a gradient alone.  Starting
    from a loaded state whose parameters have taken 0 to 3 steps, with some parameters skipping some steps (60
    tensors, so the skips cross the 48-tensor tables), FusedAdam must give torch's parameters, moments and counts."""
    count = 60
    shapes = [(1 + (i * 389) % 3000,) for i in range(count)]
    g, ps_ref, ps, opt_ref, opt, FusedAdam = _torch_and_fused(shapes, 11)
    for t in range(3):                                            # unequal step counts: param i took min(i % 4, 3)
        for i, a in enumerate(ps_ref):
            a.grad = torch.randn(a.shape, generator=g) if i % 4 > t else None
        opt_ref.step()
    assert sorted({float(s["step"]) for s in opt_ref.state.values()}) == [1.0, 2.0, 3.0]
    for a, b in zip(ps_ref, ps):
        b.data.copy_(a.detach())
    opt.load_state_dict(opt_ref.state_dict())
    fused = FusedAdam(opt)
    p0 = [p.detach().double().clone() for p in ps_ref]
    path = [torch.zeros_like(p) for p in p0]
    for t in range(8):
        for i, (a, b) in enumerate(zip(ps_ref, ps)):
            live = t == 3 or (i + t) % 3 != 0 and not (t == 5 and i < 50)
            gr = torch.randn(a.shape, generator=g) if live else None
            a.grad, b.grad = gr, None if gr is None else gr.cuda()
        prev = [a.detach().double().clone() for a in ps_ref]
        opt_ref.step()
        fused.step()
        for i, a in enumerate(ps_ref):
            path[i] += (a.detach().double() - prev[i]).abs()
    e = _compare_adams(ps_ref, ps, opt_ref, opt, fused, p0, path, "skipped parameters")
    for a, b in zip(ps_ref, ps):
        assert torch.allclose(opt.state[b]["exp_avg_sq"].cpu(), opt_ref.state[a]["exp_avg_sq"], rtol=1e-5, atol=0)
    print("FusedAdam with skipped parameters and unequal loaded counts: worst err %.2e" % e)


# ---------------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_refusals_launch_nothing():
    """Bad shapes and NULL pointers come back as status codes from the raw calls, with no launch."""
    N = _native()
    L = N.lib()
    B, D, n_img = 4, 3, 64
    buf = torch.zeros(4096, device="cuda")
    a = buf.data_ptr()
    out = torch.full((2 + D,), 7.0, device="cuda")

    def refused(rc_want, fn, *args):
        before = L.dv_launch_count()
        rc = getattr(L, fn)(*args)
        torch.cuda.synchronize()
        assert rc == rc_want and L.dv_launch_count() == before, (fn, args, rc)

    S = N.stream()
    loss = dict(recon=a, data=a, mu=a, lv=a, out=out.data_ptr(), ws=a)

    def loss_args(n_=n_img, B_=B, dist=0, D_=D, **null):
        q = dict(loss, **null)
        return (q["recon"], q["data"], n_, B_, dist, q["mu"], q["lv"], 1, D, D_, q["out"], q["ws"], S)
    for shape in (dict(n_=0), dict(B_=0), dict(B_=-1), dict(D_=0), dict(D_=1025)):
        refused(DV_ERR_BAD_SHAPE, "dv_vae_loss_fwd", *loss_args(**shape))
    for name in loss:
        refused(DV_ERR_BAD_ARG, "dv_vae_loss_fwd", *loss_args(**{name: None}))
    refused(DV_ERR_BAD_ARG, "dv_vae_loss_fwd", *loss_args(dist=3))
    refused(DV_ERR_BAD_ARG, "dv_vae_loss_fwd", *loss_args(recon=a + 4))
    assert torch.equal(out, torch.full((2 + D,), 7.0, device="cuda"))
    bwd = (a, a, n_img, B, 0, a, a, 1, D, D, a, a, a, a, a, S)
    for i in (0, 1, 5, 6, 10, 11):
        refused(DV_ERR_BAD_ARG, "dv_vae_loss_bwd", *(bwd[:i] + (None,) + bwd[i + 1:]))
    for i in (2, 3, 9):
        refused(DV_ERR_BAD_SHAPE, "dv_vae_loss_bwd", *(bwd[:i] + (0,) + bwd[i + 1:]))

    refused(DV_ERR_BAD_ARG, "dv_reparam_fwd", None, a, 1, D, a, 0, None, a, None, B, D, S)
    refused(DV_ERR_BAD_ARG, "dv_reparam_fwd", a, a, 1, D, None, 0, None, a, None, B, D, S)
    refused(DV_ERR_BAD_SHAPE, "dv_reparam_fwd", a, a, 1, D, a, 0, None, a, None, 0, D, S)
    refused(DV_ERR_BAD_SHAPE, "dv_reparam_fwd", a, a, 1, D, a, 0, None, a, None, B, 0, S)
    refused(DV_ERR_BAD_ARG, "dv_reparam_bwd", a, a, 1, D, None, a, a, B, D, S)
    refused(DV_ERR_BAD_SHAPE, "dv_reparam_bwd", a, a, 1, D, a, a, a, B, -1, S)

    for h in (0, -1):
        refused(DV_ERR_BAD_SHAPE, "dv_factor_tc_fwd", a, h, a, S)
        refused(DV_ERR_BAD_SHAPE, "dv_factor_tc_bwd", a, h, a, S)
        refused(DV_ERR_BAD_SHAPE, "dv_factor_ce_fwd", a, a, h, a, S)
        refused(DV_ERR_BAD_SHAPE, "dv_factor_ce_bwd", a, a, a, h, a, a, S)
    refused(DV_ERR_BAD_ARG, "dv_factor_tc_fwd", None, 4, a, S)
    refused(DV_ERR_BAD_ARG, "dv_factor_ce_fwd", a, None, 4, a, S)
    refused(DV_ERR_BAD_ARG, "dv_factor_ce_bwd", a, a, None, 4, a, a, S)

    ws = a
    refused(DV_ERR_BAD_SHAPE, "dv_act_bwd_chansum", a, a, a, B, 5, 64, 2, 0.0, a, ws, S)
    refused(DV_ERR_BAD_SHAPE, "dv_act_bwd_chansum", a, a, a, B, 1, 6, 2, 0.0, a, ws, S)
    refused(DV_ERR_BAD_SHAPE, "dv_act_bwd_chansum", a, a, a, 0, 1, 64, 2, 0.0, a, ws, S)
    refused(DV_ERR_BAD_ARG, "dv_act_bwd_chansum", a, a, a, B, 1, 64, 2, 0.0, None, ws, S)

    refused(DV_ERR_BAD_SHAPE, "dv_adam_step", a, a, a, a, a, 0, 1e-3, 0.9, 0.999, 1e-8, 1.0, S)
    refused(DV_ERR_BAD_ARG, "dv_adam_step", a, a, a, a, None, 16, 1e-3, 0.9, 0.999, 1e-8, 1.0, S)

    def multi(count, numel=16, null=False):
        k = max(count, 1)
        arr = (ctypes.c_void_p * k)(*([a] * k))
        if null:
            arr[k - 1] = None
        return (count, arr, arr, arr, arr, (ctypes.c_longlong * k)(*([numel] * k)), a, 1e-3, 0.9, 0.999, 1e-8, 1.0, S)
    refused(DV_ERR_BAD_SHAPE, "dv_adam_multi", *multi(0))
    refused(DV_ERR_BAD_SHAPE, "dv_adam_multi", *multi(49))
    refused(DV_ERR_BAD_ARG, "dv_adam_multi", *multi(3, numel=0))
    refused(DV_ERR_BAD_ARG, "dv_adam_multi", *multi(3, numel=1 << 31))
    refused(DV_ERR_BAD_ARG, "dv_adam_multi", *multi(3, null=True))
