"""Per-kernel parity: every C-ABI entry point against the oracle's plain-PyTorch CPU ops on the
same seeded inputs.  Tolerance: the north_star's 1e-4 relative (fp32); most kernels are far
inside it.  Run on an H100:  pytest -m gpu."""

import pytest
import torch
import torch.nn.functional as F

from oracle import disvae_oracle as O

pytestmark = pytest.mark.gpu

RTOL = 1e-4


def dev():
    return torch.device("cuda")


def rel_err(a, b):
    """max |a-b| relative to the scale of b (fp32 sums of mixed sign: judge against max |b|)."""
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def assert_close(a, b, tol=RTOL, what=""):
    assert a.shape == b.shape, (what, a.shape, b.shape)
    e = rel_err(a, b)
    assert e <= tol, "%s: rel err %.3e > %.1e" % (what, e, tol)


@pytest.fixture(scope="module")
def ops():
    from disvae import ops as _ops
    return _ops


@pytest.mark.parametrize("dist", ["bernoulli", "gaussian", "laplace"])
def test_vae_loss_kernel(ops, golden, dist):
    from disvae._native import DIST
    i = golden("losses.pt")["inputs"]
    data, recon0, mu0, lv0 = i["data"], i["recon"], i["mu"], i["logvar"]
    ml = torch.stack([mu0, lv0], dim=-1).reshape(mu0.size(0), -1)        # interleaved like the encoder output
    recon = recon0.clone().requires_grad_(True)
    mu = mu0.clone().requires_grad_(True)
    lv = lv0.clone().requires_grad_(True)
    rec = O.reconstruction_loss(data, recon, dist)
    kl, kl_dims = O.kl_normal(mu, lv)
    (1.7 * rec + 0.3 * kl).backward()
    mld = ml.to(dev()).requires_grad_(True)
    mud, lvd = mld.view(-1, mu0.size(1), 2).unbind(-1)
    rd = recon0.to(dev()).requires_grad_(True)
    out = ops.VaeLossFn.apply(rd, data.to(dev()), mud, lvd, DIST[dist])
    assert_close(out[0:1].cpu(), rec.detach().view(1), tol=2e-6, what="recon loss")
    assert_close(out[1:2].cpu(), kl.detach().view(1), tol=2e-6, what="kl")
    assert_close(out[2:].cpu(), kl_dims.detach(), tol=2e-6, what="kl dims")
    (1.7 * out[0] + 0.3 * out[1]).backward()
    assert_close(rd.grad.cpu(), recon.grad, tol=1e-5, what="d recon")
    g_ml = mld.grad.cpu().view(-1, mu0.size(1), 2)
    assert_close(g_ml[..., 0], mu.grad, tol=1e-5, what="d mu")
    assert_close(g_ml[..., 1], lv.grad, tol=1e-5, what="d logvar")


def test_laplace_zero_loss_mask(ops):
    from disvae._native import DIST
    x = torch.rand(2, 1, 32, 32, device=dev())
    r = x.clone().requires_grad_(True)
    z = torch.zeros(2, 3, device=dev())
    out = ops.VaeLossFn.apply(r, x, z, z, DIST["laplace"])
    assert out[0].item() == 0.0
    out[0].backward()
    assert torch.count_nonzero(r.grad).item() == 0


def test_reparam_fwd_bwd_and_device_noise(ops):
    torch.manual_seed(11)
    B, D = 37, 10
    ml = torch.randn(B, 2 * D)
    eps = torch.randn(B, D)
    mlc = ml.clone().requires_grad_(True)
    mu, lv = mlc.view(B, D, 2).unbind(-1)
    z = O.reparameterize(mu, lv, eps)
    (z * torch.arange(B * D).view(B, D).float()).sum().backward()
    mld = ml.to(dev()).requires_grad_(True)
    mud, lvd = mld.view(B, D, 2).unbind(-1)
    zd = ops.ReparamFn.apply(mud, lvd, eps.to(dev()), 0, None)
    assert_close(zd.cpu(), z.detach(), tol=1e-6)
    (zd * torch.arange(B * D, device=dev()).view(B, D).float()).sum().backward()
    assert_close(mld.grad.cpu(), mlc.grad, tol=1e-6)
    # device Philox noise: N(0,1) moments, reproducible per (seed, offset), offset advances
    Bn, Dn = 4096, 64
    zeros = torch.zeros(Bn, Dn, device=dev())
    off = torch.zeros(1, dtype=torch.int64, device=dev())
    e1 = ops.ReparamFn.apply(zeros, zeros, None, 1234, off)
    assert off.item() == Bn * Dn
    e2 = ops.ReparamFn.apply(zeros, zeros, None, 1234, off)
    off.zero_()
    e3 = ops.ReparamFn.apply(zeros, zeros, None, 1234, off)
    assert torch.equal(e1, e3) and not torch.equal(e1, e2)
    assert abs(e1.mean().item()) < 0.01 and abs(e1.std().item() - 1) < 0.01
    assert abs((e1 ** 3).mean().item()) < 0.03 and abs((e1 ** 4).mean().item() - 3) < 0.1


BT_CASES = ["b64_d10", "b256_d64", "b7_d3", "b2_d1"]


@pytest.mark.parametrize("key", BT_CASES)
@pytest.mark.parametrize("mss", [1, 0])
def test_btcvae_kernel_against_reference_golden(ops, golden, key, mss):
    g = golden("btcvae_density.pt")["%s_mss%d" % (key, mss)]
    B, D = g["b"], g["d"]
    z = g["z"].to(dev()).requires_grad_(True)
    ml = torch.stack([g["mu"], g["logvar"]], dim=-1).reshape(B, -1).to(dev()).requires_grad_(True)
    mu, lv = ml.view(B, D, 2).unbind(-1)
    stats = ops.btcvae_rowstats(z, mu, lv, g["n_data"], bool(mss))
    for got, name in zip(stats, ["log_pz", "log_qz", "log_prod_qzi", "log_q_zCx"]):
        assert_close(got.cpu(), g[name], tol=2e-5, what=name)
    terms = ops.BtcvaeFn.apply(z, mu, lv, g["n_data"], bool(mss))
    c = g["coef"]          # probe = c0*mean(log_pz) + c1*mean(log_qz) + c2*mean(log_prod) + c3*mean(log_qzCx)
    mi_ref = (g["log_q_zCx"] - g["log_qz"]).mean()
    tc_ref = (g["log_qz"] - g["log_prod_qzi"]).mean()
    dw_ref = (g["log_prod_qzi"] - g["log_pz"]).mean()
    assert_close(terms.cpu(), torch.stack([mi_ref, tc_ref, dw_ref]), tol=5e-5, what="terms")
    # probe in terms of (mi, tc, dw): a*mi + b*tc + e*dw with lqc coef = a = c3; lqz: -a + b = c1; lprod: -b + e = c2;
    # lpz: -e = c0  => only consistent if c0+c1+c2+c3 == 0; use autograd on the oracle instead.
    zo = g["z"].clone().requires_grad_(True)
    muo = g["mu"].clone().requires_grad_(True)
    lvo = g["logvar"].clone().requires_grad_(True)
    mi, tc, dw = O.btcvae_terms(zo, muo, lvo, g["n_data"], bool(mss))
    (1.0 * mi + 6.0 * tc - 2.5 * dw).backward()
    (1.0 * terms[0] + 6.0 * terms[1] - 2.5 * terms[2]).backward()
    assert_close(z.grad.cpu(), zo.grad, what="g_z")
    gml = ml.grad.cpu().view(B, D, 2)
    assert_close(gml[..., 0], muo.grad, what="g_mu")
    assert_close(gml[..., 1], lvo.grad, what="g_logvar")


@pytest.mark.parametrize("B,D", [(1024, 10), (256, 64), (512, 16), (129, 5), (1000, 8), (96, 20), (2048, 64)])
def test_btcvae_kernel_against_oracle_sizes(ops, B, D):
    torch.manual_seed(B + D)
    mu = torch.randn(B, D)
    lv = torch.randn(B, D) * 0.5 - 1
    z = mu + torch.exp(0.5 * lv) * torch.randn(B, D)
    n_data = 737280
    zo, muo, lvo = [t.clone().requires_grad_(True) for t in (z, mu, lv)]
    big = B * B * D > 5e7
    if big:           # oracle materialises B*B*D floats: keep the big case forward-only + properties
        with torch.no_grad():
            ref = O.btcvae_log_densities(z, mu, lv, n_data)
    else:
        ref = O.btcvae_log_densities(zo, muo, lvo, n_data)
    zd, mud, lvd = [t.to(dev()).requires_grad_(True) for t in (z, mu, lv)]
    stats = ops.btcvae_rowstats(zd, mud, lvd, n_data, True)
    for got, r, name in zip(stats, ref, ["log_pz", "log_qz", "log_prod_qzi", "log_q_zCx"]):
        assert_close(got.cpu(), r.detach(), tol=2e-5, what=name)
    terms = ops.BtcvaeFn.apply(zd, mud, lvd, n_data, True)
    (terms[0] + 6 * terms[1] + terms[2]).backward()
    if not big:
        mi = (ref[3] - ref[1]).mean(); tc = (ref[1] - ref[2]).mean(); dw = (ref[2] - ref[0]).mean()
        (mi + 6 * tc + dw).backward()
        assert_close(zd.grad.cpu(), zo.grad, what="g_z")
        assert_close(mud.grad.cpu(), muo.grad, what="g_mu")
        assert_close(lvd.grad.cpu(), lvo.grad, what="g_logvar")
    # size-independent property: run-to-run bit-exactness (fixed reduction order)
    terms2 = ops.BtcvaeFn.apply(zd, mud, lvd, n_data, True)
    assert torch.equal(terms, terms2)


def test_btcvae_extreme_variances_stay_finite(ops):
    """Trained models have tiny variances: logsumexp must not under/overflow (exact max)."""
    torch.manual_seed(0)
    B, D = 128, 10
    mu = torch.randn(B, D) * 3
    lv = torch.full((B, D), -14.0)
    lv[::7] = 3.0
    z = mu + torch.exp(0.5 * lv) * torch.randn(B, D)
    ref = O.btcvae_log_densities(z, mu, lv, 10000)
    stats = ops.btcvae_rowstats(z.to(dev()), mu.to(dev()), lv.to(dev()), 10000, True)
    for got, r in zip(stats, ref):
        assert torch.isfinite(got).all()
        assert_close(got.cpu(), r, tol=2e-5)


def test_btcvae_outlier_rows_and_tiny_variances(ops):
    """Rows far (100s of sigma) from every other column, tiny and huge variances mixed: the single-sweep
    logsumexp (bounded reference exponent) must agree with the exact-max oracle and stay finite."""
    torch.manual_seed(1)
    B, D = 192, 10
    mu = torch.randn(B, D)
    lv = torch.randn(B, D) * 0.3 - 2.0
    lv[5] = -20.0; lv[77] = 6.0; lv[130, :3] = -16.0
    z = mu + torch.exp(0.5 * lv) * torch.randn(B, D)
    z[9] += 40.0; z[100, 2] -= 25.0
    ref = O.btcvae_log_densities(z, mu, lv, 50000)
    stats = ops.btcvae_rowstats(z.to(dev()), mu.to(dev()), lv.to(dev()), 50000, True)
    for got, r, name in zip(stats, ref, ["log_pz", "log_qz", "log_prod_qzi", "log_q_zCx"]):
        assert torch.isfinite(got).all(), name
        assert_close(got.cpu(), r, tol=2e-5, what=name)


def test_permute_dims(ops, golden):
    g = golden("permute.pt")
    torch.manual_seed(1234 + 7)
    perms = torch.stack([torch.randperm(16) for _ in range(10)])
    got = ops.permute_dims(g["z"].to(dev()), perms)
    assert torch.equal(got.cpu(), g["z_perm"])
    # device-generated permutations: every column is a permutation of the input column
    B, D = 1000, 12
    z = torch.randn(B, D, device=dev())
    off = torch.zeros(1, dtype=torch.int64, device=dev())
    p1 = ops.permute_dims(z, None, 99, off)
    assert off.item() == B * D
    assert torch.equal(p1.sort(0).values, z.sort(0).values)
    assert not torch.equal(p1, z)
    p2 = ops.permute_dims(z, None, 99, off)
    assert not torch.equal(p1, p2)
    # uniformity smoke: mean displacement of a uniform random permutation ~ B/3
    idx = torch.arange(B, device=dev(), dtype=torch.float32).unsqueeze(1).repeat(1, D)
    pi = ops.permute_dims(idx, None, 5, off)
    disp = (pi - idx).abs().mean().item()
    assert abs(disp - B / 3) < 0.05 * B


def test_factor_heads(ops):
    torch.manual_seed(2)
    h = 130
    dz = torch.randn(h, 2, requires_grad=True)
    dp = torch.randn(h, 2, requires_grad=True)
    tc = (dz[:, 0] - dz[:, 1]).mean()
    ones = torch.ones(h, dtype=torch.long)
    ce = 0.5 * (F.cross_entropy(dz, torch.zeros_like(ones)) + F.cross_entropy(dp, ones))
    (2 * tc + 3 * ce).backward()
    dzd = dz.detach().to(dev()).requires_grad_(True)
    dpd = dp.detach().to(dev()).requires_grad_(True)
    tcd = ops.FactorTcFn.apply(dzd)
    ced = ops.FactorCeFn.apply(dzd, dpd)
    assert abs(tcd.item() - tc.item()) < 1e-6 and abs(ced.item() - ce.item()) < 1e-6
    (2 * tcd + 3 * ced).backward()
    assert_close(dzd.grad.cpu(), dz.grad, tol=1e-5)
    assert_close(dpd.grad.cpu(), dp.grad, tol=1e-5)


def test_adam_step_matches_torch(ops):
    torch.manual_seed(4)
    n = 100003
    p = torch.randn(n)
    po = p.clone().requires_grad_(True)
    opt = torch.optim.Adam([po], lr=5e-4)
    pd = p.to(dev())
    m = torch.zeros(n, device=dev()); v = torch.zeros(n, device=dev()); step = torch.zeros(1, device=dev())
    for i in range(3):
        g = torch.randn(n)
        po.grad = g.clone()
        opt.step()
        ops.adam_step(pd, g.to(dev()), m, v, step, 5e-4, (0.9, 0.999), 1e-8)
    assert step.item() == 3
    assert_close(pd.cpu(), po.detach(), tol=1e-6)


def test_fused_adam_multi_matches_torch_adam():
    """disvae.fused.FusedAdam (dv_adam_multi, one launch for all tensors) == torch.optim.Adam, incl. shared state."""
    from disvae.fused import FusedAdam
    torch.manual_seed(6)
    shapes = [(32, 1, 4, 4), (32,), (256, 512), (20, 256), (1000, 1000), (3,)]
    ps_ref = [torch.randn(s, requires_grad=True) for s in shapes]
    ps = [p.detach().clone().to(dev()).requires_grad_(True) for p in ps_ref]
    opt_ref = torch.optim.Adam(ps_ref, lr=5e-4)
    opt = torch.optim.Adam(ps, lr=5e-4)
    assert FusedAdam.supports(opt) and not FusedAdam.supports(torch.optim.Adam(ps, lr=1e-3, weight_decay=0.1))
    fused = FusedAdam(opt)
    for _ in range(4):
        for a, b in zip(ps_ref, ps):
            g = torch.randn(a.shape)
            a.grad = g.clone(); b.grad = g.to(dev())
        opt_ref.step(); fused.step()
    for a, b in zip(ps_ref, ps):
        assert_close(b.detach().cpu(), a.detach(), tol=1e-6)
        assert_close(opt.state[b]["exp_avg_sq"].cpu(), opt_ref.state[a]["exp_avg_sq"], tol=1e-6)
    fused.flush_state()
    assert float(opt.state[ps[0]]["step"]) == 4.0


@pytest.mark.parametrize("B,D,world", [(256, 64, 2), (96, 10, 3), (2048, 64, 8), (130, 5, 2)])
def test_btcvae_row_windows_compose_to_the_full_batch(ops, B, D, world):
    """SURVEY.md 8f-1 kernels: the estimator over row windows of one (all-gathered) batch.  Window r evaluates rows
    [r*b, (r+1)*b) against ALL B columns; rowstats of the windows == the oracle's full-batch values; the mean of the
    windows' terms == the full-batch terms; g_z windows stack to the full g_z and the column-side partial sums add up to
    the full g_mu / g_logvar (what the reduce-scatter over ranks computes)."""
    from disvae import _native as N
    torch.manual_seed(B + D + world)
    b = B // world
    B = b * world
    mu = torch.randn(B, D)
    lv = torch.randn(B, D) * 0.5 - 1
    z = mu + torch.exp(0.5 * lv) * torch.randn(B, D)
    n_data = 202599
    big = B * B * D > 5e7
    zo, muo, lvo = [t.clone().requires_grad_(not big) for t in (z, mu, lv)]
    with torch.set_grad_enabled(not big):
        ref = O.btcvae_log_densities(zo, muo, lvo, n_data)
    coef = (1.0, 6.0, -2.5)
    if not big:
        mi, tc, dw = (ref[3] - ref[1]).mean(), (ref[1] - ref[2]).mean(), (ref[2] - ref[0]).mean()
        (coef[0] * mi + coef[1] * tc + coef[2] * dw).backward()
    zd, mud, lvd = z.to(dev()), mu.to(dev()), lv.to(dev())
    nbytes = N.lib().dv_btcvae_workspace_bytes(B, D)
    g_terms = torch.tensor(coef, device=dev())
    terms_mean = torch.zeros(3)
    g_z, g_mu, g_lv = torch.zeros(B, D), torch.zeros(B, D), torch.zeros(B, D)
    for r in range(world):
        ws = torch.zeros((nbytes + 3) // 4, device=dev())
        rowstats = torch.full((4 + D, B), float("nan"), device=dev())
        terms = torch.empty(3, device=dev())
        N.call("dv_btcvae_fwd_rows", N.ptr(zd), N.ptr(mud), N.ptr(lvd), 1, D, B, D, r * b, b, n_data, 1, N.ptr(rowstats),
               N.ptr(terms), N.ptr(ws), N.stream())
        for got, rf, name in zip(rowstats[:4], ref, ["log_pz", "log_qz", "log_prod_qzi", "log_q_zCx"]):
            assert_close(got[r * b:(r + 1) * b].cpu(), rf.detach()[r * b:(r + 1) * b], tol=2e-5, what="%s window %d" % (name, r))
        if r * b > 0:
            assert torch.isnan(rowstats[1:3, :r * b]).all()          # rows outside the window are not touched
        terms_mean += terms.cpu() / world
        gz = torch.empty(b, D, device=dev())
        gm, gl = torch.empty(B, D, device=dev()), torch.empty(B, D, device=dev())
        N.call("dv_btcvae_bwd_rows", B, D, r * b, b, n_data, 1, N.ptr(rowstats), N.ptr(ws), N.ptr(g_terms), N.ptr(gz), N.ptr(gm),
               N.ptr(gl), N.stream())
        g_z[r * b:(r + 1) * b] = gz.cpu()
        g_mu += gm.cpu()
        g_lv += gl.cpu()
    full = ops.BtcvaeFn.apply(zd, mud, lvd, n_data, True)
    assert_close(terms_mean, full.cpu(), tol=2e-5, what="mean of window terms")
    if not big:
        # gradients of the MEAN-over-windows loss: each window's backward used 1/b, the full batch uses 1/B
        assert_close(g_z / world, zo.grad, what="g_z")
        assert_close(g_mu / world, muo.grad, what="g_mu")
        assert_close(g_lv / world, lvo.grad, what="g_logvar")


def test_u8_to_f32_is_totensor(ops):
    """dv_u8_to_f32 == torchvision ToTensor's `img.float().div(255)` bit for bit (utils/datasets.py:182,247,364-367)."""
    torch.manual_seed(0)
    for n in (16, 1 << 20, 12345 * 16 + 7, 3):
        u = torch.randint(0, 256, (n,), dtype=torch.uint8)
        got = ops.u8_to_f32(u.to(dev())).cpu()
        assert torch.equal(got, u.float().div(255))
    u = torch.arange(256, dtype=torch.uint8).repeat(64)          # every byte value
    assert torch.equal(ops.u8_to_f32(u.to(dev())).cpu(), u.float().div(255))


def test_conv_pack_multi_equals_per_layer_pack(ops):
    """dv_conv_pack_multi (all conv layers of a node, one launch) writes exactly the buffers of dv_conv_pack_weights."""
    torch.manual_seed(9)
    chans = [1, 32, 32, 32, 3, 32, 32, 32, 32, 1]        # > 8 layers: the library splits the table
    ws = [(torch.randn(32, ch, 4, 4) * 0.1).to(dev()) for ch in chans]
    for pk, w, ch in zip(ops.conv_pack_multi(ws, chans), ws, chans):
        assert torch.equal(pk, ops.conv_pack(w, ch)), ch
