"""The marginal-entropy estimator of the MIG / AAM metrics (csrc/dv_entropy.cu) on every path it can take, against a
chunked fp64 reference.

dv_latent_entropy splits the N posteriors into n-splits (pick_nsplit: one to 64, at least four 256-posterior chunks
each), walks each split in 256-posterior chunks, covers the S samples in 512-sample tiles, and merges the splits in a
fixed order in entropy_finalize_kernel.  Each case below asserts its split count (read back from
dv_latent_entropy_workspace_bytes) and checks every log q(z) entry and H, or a fixed set of sample columns at dSprites
size, against `ref_logq`, which evaluates the Gaussian mixture in fp64 a block of samples at a time, so that N up to
737,280 can be checked.  The inputs come in four regimes: spread posteriors, a trained model's (tiny variances in
active dimensions, near-identical posteriors in inactive ones), exact ties, and samples 40 sigma from every posterior.

The reference is first checked against the oracle (oracle/disvae_oracle.py) on the CPU; everything else needs an H100
(pytest -m gpu).  Each GPU case prints its worst errors (pytest -s shows them)."""
import math

import pytest
import torch

from oracle import disvae_oracle as O

LOGQ_TOL = 2e-5      # per log q(z) entry, relative to max(1, |ref|)
H_TOL = 1e-5         # per H[d], relative to max(1, |ref|)
MI_TOL = 1e-4        # MI entries, MIG and AAM, absolute (nats)
CHUNK_ELEMS = 1 << 22
GUARD = 4096           # floats of sentinel after each output and the workspace
SENTINEL = 0x7FBADBAD  # a NaN bit pattern no kernel writes
DV_ERR_BAD_SHAPE, DV_ERR_BAD_ARG = -1, -2     # include/disvae_b200.h


# ---------------------------------------------------------------------------------------------------------------------
# fp64 reference, a block of samples at a time
# ---------------------------------------------------------------------------------------------------------------------
def ref_logq(zs, mean, logvar, cols=None):
    """log q(z[d][s]) = -log N + logsumexp_n log N(z[d][s]; mean[n][d], exp(logvar[n][d])) in fp64, [D, S] or
    [D, len(cols)] for the chosen sample columns.  Evaluates one dimension and N x block <= 2^22 pairs at a time."""
    zs, mean, logvar = zs.double(), mean.double(), logvar.double()
    if cols is not None:
        zs = zs[:, torch.as_tensor(cols, dtype=torch.long)]
    N = mean.shape[0]
    D, S = zs.shape
    block = max(1, CHUNK_ELEMS // N)
    out = torch.empty(D, S, dtype=torch.float64)
    for d in range(D):
        mu, lv = mean[:, d:d + 1], logvar[:, d:d + 1]
        for a in range(0, S, block):
            dens = O.log_density_gaussian(zs[d, a:a + block].unsqueeze(0), mu, lv)        # [N, block]
            out[d, a:a + block] = torch.logsumexp(dens, dim=0)
    return out - math.log(N)


def ref_H(logq):
    return -logq.mean(1)


# ---------------------------------------------------------------------------------------------------------------------
# CPU self-check of the reference against the oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,D,S", [(1, 1, 1), (7, 4, 7), (300, 3, 200), (20000, 3, 500)])
def test_reference_matches_the_oracle(N, D, S):
    """H from ref_logq on the oracle's reshaped (not transposed) draw equals O.estimate_latent_entropies in fp64;
    (20000, 3, 500) runs three sample blocks per dimension.  A column subset gives the same entries."""
    g = torch.Generator().manual_seed(N + D + S)
    mean = torch.randn(N, D, generator=g, dtype=torch.float64)
    logvar = torch.randn(N, D, generator=g, dtype=torch.float64) * 0.7 - 1.5
    samples = mean + torch.exp(0.5 * logvar) * torch.randn(N, D, generator=g, dtype=torch.float64)
    draw = torch.randperm(N, generator=g)[:S]
    zs = samples.index_select(0, draw).view(D, S)               # evaluate.py:270, as the Evaluator passes it
    logq = ref_logq(zs, mean, logvar)
    want = O.estimate_latent_entropies(samples, mean, logvar, draw)
    err = ((ref_H(logq) - want).abs().max() / want.abs().max()).item()
    assert err <= 1e-12, err
    cols = sorted({0, S // 2, S - 1})
    assert torch.equal(ref_logq(zs, mean, logvar, cols), logq[:, cols])


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def _spread(N, D, S, g):
    mean = torch.randn(N, D, generator=g)
    logvar = torch.randn(N, D, generator=g) * 0.7 - 1.5
    zs = torch.randn(D, S, generator=g) * 1.3
    return zs, mean, logvar


def _trained(N, D, S, g):
    """Even dimensions active: logvar in [-12, -6], means spread over +-3.  Odd ones inactive: logvar and means
    within ~0.05 of 0.  Every sample is drawn from the posterior of a random example."""
    active = torch.arange(D) % 2 == 0
    mean = torch.where(active, torch.rand(N, D, generator=g) * 6 - 3, torch.randn(N, D, generator=g) * 0.05)
    logvar = torch.where(active, torch.rand(N, D, generator=g) * 6 - 12, torch.randn(N, D, generator=g) * 0.05)
    src = torch.randint(N, (D, S), generator=g)
    mu, lv = mean.t().gather(1, src), logvar.t().gather(1, src)
    zs = mu + torch.exp(0.5 * lv) * torch.randn(D, S, generator=g)
    return zs, mean, logvar


def _ties(N, D, S, g):
    """Spread, except dimension D // 2: every posterior N(0.375, exp(-0.5)), and every third sample exactly 0.375."""
    zs, mean, logvar = _spread(N, D, S, g)
    t = D // 2
    mean[:, t], logvar[:, t] = 0.375, -0.5
    zs[t, ::3] = 0.375
    return zs, mean, logvar


def _outliers(N, D, S, g):
    """Spread, with logvar -20 and +6 entries mixed in, and every fifth sample at least 40 sigma from every posterior
    of its dimension (alternately above and below all of them)."""
    zs, mean, logvar = _spread(N, D, S, g)
    nd = torch.arange(N).unsqueeze(1) + torch.arange(D).unsqueeze(0)
    logvar[nd % 7 == 0] = -20.0
    logvar[nd % 11 == 5] = 6.0
    reach = 40 * torch.exp(0.5 * logvar)
    hi, lo = (mean + reach).max(0).values, (mean - reach).min(0).values
    for k, s in enumerate(range(0, S, 5)):
        zs[:, s] = hi if k % 2 == 0 else lo
    return zs, mean, logvar


REGIMES = {"spread": _spread, "trained": _trained, "ties": _ties, "outliers": _outliers}


def _inputs(N, D, S, regime):
    return REGIMES[regime](N, D, S, torch.Generator().manual_seed(N * 131 + D * 7 + S))


# ---------------------------------------------------------------------------------------------------------------------
# the kernel
# ---------------------------------------------------------------------------------------------------------------------
def _bits(t):
    return t.contiguous().view(torch.int32)


def _guarded(n):
    """n NaN floats followed by GUARD sentinel floats."""
    t = torch.full((n + GUARD,), float("nan"), device="cuda")
    _bits(t)[n:] = SENTINEL
    return t


def _intact(t, n):
    return bool((_bits(t)[n:] == SENTINEL).all())


class Kernel:
    """Device copies of (zs, mean, logvar), the posteriors either contiguous [N, D] or interleaved [N, D, 2] as
    Evaluator._compute_q_zCx leaves them (ld = 2, row stride 2D), and the C-ABI call on them with every output and
    the workspace (sized by dv_latent_entropy_workspace_bytes alone) followed by a sentinel guard."""

    def __init__(self, zs, mean, logvar):
        from disvae import _native as N
        self.N = N
        self.n, self.D = mean.shape
        self.S = zs.shape[1]
        self.zs = zs.cuda()
        self.mean, self.logvar = mean.cuda(), logvar.cuda()
        self.ml = torch.stack([mean, logvar], dim=-1).reshape(self.n, 2 * self.D).cuda()
        self.ws_bytes = N.lib().dv_latent_entropy_workspace_bytes(self.n, self.D, self.S)
        assert self.ws_bytes % (8 * self.D * self.S) == 0
        self.nsplit = self.ws_bytes // (8 * self.D * self.S)

    def run(self, interleaved=False, with_logq=True, mean=None):
        """-> (H [D], logq [D, S] or None, kernel launches); asserts every guard survived."""
        N, D, S = self.N, self.D, self.S
        if interleaved:
            mp, lp, ld, rs = self.ml.data_ptr(), self.ml.data_ptr() + 4, 2, 2 * D
        else:
            mp, lp, ld, rs = (mean if mean is not None else self.mean).data_ptr(), self.logvar.data_ptr(), 1, D
        ws_floats = self.ws_bytes // 4
        ws, H = _guarded(ws_floats), _guarded(D)
        logq = _guarded(D * S) if with_logq else None
        before = N.lib().dv_launch_count()
        N.call("dv_latent_entropy", N.ptr(self.zs), mp, lp, ld, rs, self.n, D, S, N.ptr(H), N.ptr(logq), N.ptr(ws),
               N.stream())
        launches = N.lib().dv_launch_count() - before
        torch.cuda.synchronize()
        assert _intact(ws, ws_floats), "wrote past dv_latent_entropy_workspace_bytes"
        assert _intact(H, D), "wrote past H[D]"
        assert logq is None or _intact(logq, D * S), "wrote past logq[D, S]"
        return H[:D].clone(), None if logq is None else logq[:D * S].view(D, S).clone(), launches


def _err(got, ref):
    """max |got - ref| / max(1, |ref|), over finite-checked fp64 copies."""
    got, ref = got.double().cpu(), ref.double().cpu()
    assert torch.isfinite(ref).all()
    return ((got - ref).abs() / ref.abs().clamp_min(1.0)).max().item()


def _columns(S, count=64):
    """Both ends, the 512-sample tile boundaries around 512 and 1024, the middle, and seeded fill to `count`."""
    fixed = sorted(c for c in {0, 1, 255, 256, 511, 512, 513, 1023, 1024, S // 2, S - 2, S - 1} if 0 <= c < S)
    g = torch.Generator().manual_seed(S)
    extra = [c for c in torch.randperm(S, generator=g).tolist() if c not in fixed]
    return sorted(fixed + extra[:count - len(fixed)])


# (N, D, S, n-splits): the split count pick_nsplit gives with 132 SMs
CASES = [
    (1, 1, 1, 1),             # single posterior, single sample
    (255, 3, 7, 1),           # one partial chunk
    (1024, 10, 513, 1),       # four full chunks, two sample tiles, a 1-sample tail
    (1025, 10, 500, 2),       # splits of 513: split 0 ends in a 1-posterior chunk
    (100003, 1, 512, 64),     # the 64-split cap: splits of 1563 = 6 * 256 + 27, the last of 1534
    (5000, 64, 2000, 3),      # D = 64 (the c5 latent size), four tiles with a tail, splits of 1667
    (2000, 300, 64, 2),       # large D (grid.y)
]
LARGE_CASES = [
    (23040, 10, 10000, 3),    # one dSprites posX slice (a conditional-entropy call)
    (737280, 10, 10000, 3),   # the marginal call at dSprites size
]


def run_case(n, D, S, nsplit, regime, cols=None):
    zs, mean, logvar = _inputs(n, D, S, regime)
    k = Kernel(zs, mean, logvar)
    tag = "N=%d D=%d S=%d %s" % (n, D, S, regime)
    assert k.nsplit == nsplit, "%s: %d n-splits, expected %d" % (tag, k.nsplit, nsplit)

    H, logq, launches = k.run()
    assert launches == 2, "%s: %d launches" % (tag, launches)
    H_i, logq_i, launches = k.run(interleaved=True)
    assert launches == 2
    assert torch.equal(_bits(H_i), _bits(H)) and torch.equal(_bits(logq_i), _bits(logq)), tag + ": layouts differ"
    H_n, none, launches = k.run(with_logq=False)
    assert launches == 2 and none is None
    assert torch.equal(_bits(H_n), _bits(H)), tag + ": H depends on logq_out"
    H_2, logq_2, _ = k.run()
    assert torch.equal(_bits(H_2), _bits(H)) and torch.equal(_bits(logq_2), _bits(logq)), tag + ": not deterministic"

    assert torch.isfinite(logq).all() and torch.isfinite(H).all(), tag + ": not finite"
    if cols is None:
        ref = ref_logq(zs, mean, logvar)
        e_logq = _err(logq, ref)
        e_H = _err(H, ref_H(ref))
    else:
        ref = ref_logq(zs, mean, logvar, cols)
        e_logq = _err(logq[:, torch.tensor(cols).cuda()], ref)
        e_H = _err(H, ref_H(logq.double().cpu()))          # the kernel's own mean of its log q
    print("%s: n-splits %d, worst logq err %.2e, H err %.2e" % (tag, nsplit, e_logq, e_H))
    assert e_logq <= LOGQ_TOL, "%s: logq err %.3e > %.1e" % (tag, e_logq, LOGQ_TOL)
    assert e_H <= H_TOL, "%s: H err %.3e > %.1e" % (tag, e_H, H_TOL)


def _id(c):
    return "%dx%dx%d" % c[:3]


@pytest.mark.gpu
@pytest.mark.parametrize("regime", list(REGIMES))
@pytest.mark.parametrize("n,D,S,nsplit", CASES, ids=[_id(c) for c in CASES])
def test_entropy_paths_match_the_fp64_reference(n, D, S, nsplit, regime):
    run_case(n, D, S, nsplit, regime)


@pytest.mark.gpu
@pytest.mark.parametrize("regime", list(REGIMES))
@pytest.mark.parametrize("n,D,S,nsplit", LARGE_CASES, ids=[_id(c) for c in LARGE_CASES])
def test_entropy_at_dsprites_size_matches_the_fp64_reference(n, D, S, nsplit, regime):
    """log q on 64 sample columns against the reference, H against the kernel's own log q.  Every regime runs here:
    at N = 737280 a single running fp32 (max, sum) per split, in place of the per-chunk states merged afterwards,
    breaks the log q bar on spread posteriors but not on the trained ones."""
    run_case(n, D, S, nsplit, regime, cols=_columns(S))


# ---------------------------------------------------------------------------------------------------------------------
# NaN propagation and refusals
# ---------------------------------------------------------------------------------------------------------------------
NAN_CASES = [CASES[1], CASES[3], CASES[4], CASES[5]]     # one split, two, the 64-split cap, D = 64


@pytest.mark.gpu
@pytest.mark.parametrize("n,D,S,nsplit", NAN_CASES, ids=[_id(c) for c in NAN_CASES])
def test_nan_mean_poisons_only_its_dimension(n, D, S, nsplit):
    """A NaN mean of one posterior makes every log q of its dimension NaN, as torch.logsumexp does, wherever it sits
    (first posterior, a later split, the last posterior); the other dimensions stay bit-identical."""
    zs, mean, logvar = _inputs(n, D, S, "spread")
    k = Kernel(zs, mean, logvar)
    H, logq, _ = k.run()
    d = D // 2
    for row in sorted({0, n // 2, n - 1}):
        bad = k.mean.clone()
        bad[row, d] = float("nan")
        H_b, logq_b, _ = k.run(mean=bad)
        assert torch.isnan(H_b[d]) and torch.isnan(logq_b[d]).all(), "NaN at posterior %d lost" % row
        keep = torch.arange(D, device="cuda") != d
        assert torch.equal(_bits(H_b[keep]), _bits(H[keep])), "posterior %d: other dimensions changed" % row
        assert torch.equal(_bits(logq_b[keep]), _bits(logq[keep])), "posterior %d: other dimensions changed" % row
    assert torch.isnan(torch.logsumexp(torch.tensor([0.0, float("nan"), 1.0]), 0))


@pytest.mark.gpu
def test_refusals_launch_nothing():
    """Shape and NULL-pointer refusals return their status through the raw C call, launch nothing, leave H alone."""
    from disvae import _native as N
    L = N.lib()
    n, D, S = 64, 4, 16
    zs = torch.randn(D, S, device="cuda")
    mean, logvar = torch.randn(n, D, device="cuda"), torch.zeros(n, D, device="cuda")
    ws = torch.empty(L.dv_latent_entropy_workspace_bytes(n, D, S) // 4, device="cuda")
    H = torch.full((D,), 7.0, device="cuda")
    p = dict(zs=zs.data_ptr(), mean=mean.data_ptr(), logvar=logvar.data_ptr(), H=H.data_ptr(), ws=ws.data_ptr())

    def call(n_=n, D_=D, S_=S, **null):
        q = dict(p, **null)
        before = L.dv_launch_count()
        rc = L.dv_latent_entropy(q["zs"], q["mean"], q["logvar"], 1, D, n_, D_, S_, q["H"], None, q["ws"],
                                 N.stream())
        torch.cuda.synchronize()
        assert L.dv_launch_count() == before
        assert torch.equal(H, torch.full((D,), 7.0, device="cuda"))
        return rc

    for shape in [dict(n_=0), dict(n_=-1), dict(D_=0), dict(D_=-3), dict(S_=0), dict(S_=-1), dict(D_=65536)]:
        assert call(**shape) == DV_ERR_BAD_SHAPE, shape
    for name in p:
        assert call(**{name: None}) == DV_ERR_BAD_ARG, name
    before = L.dv_launch_count()
    assert L.dv_latent_entropy(p["zs"], p["mean"], p["logvar"], 1, D, n, D, S, p["H"], None, p["ws"], N.stream()) == 0
    assert L.dv_launch_count() - before == 2


# ---------------------------------------------------------------------------------------------------------------------
# the Evaluator's MIG / AAM against the fp64 oracle
# ---------------------------------------------------------------------------------------------------------------------
LAT_SIZES = (3, 6, 8, 8, 8)
ENCODES = (2, 5, 7, 0, 9)       # the latent that encodes each factor
EV_D, EV_S = 10, 1000


def _factor_posteriors():
    """Posteriors of the 9216 images of the LAT_SIZES grid: latent ENCODES[k] places factor k's value on a line over
    [-2, 2] with logvar ~ -4; the other latents are inactive (means and logvar within ~0.05 of 0).  Samples are drawn
    from each image's posterior.

    The estimator reshapes rather than transposes the drawn samples (evaluate.py:270), so the samples it scores
    against latent j come from every latent.  An encoding latent's narrow conditional posteriors then score most of
    them far worse than its marginal does: its MI with its own factor is about -30 nats and clamps to 0.  MIG and AAM
    rest on the small positive MI entries of the other latents instead; the seeds keep every one of them clear of
    the clamps (checked in the test)."""
    g = torch.Generator().manual_seed(0)
    n = math.prod(LAT_SIZES)
    grid = torch.meshgrid(*[torch.arange(s) for s in LAT_SIZES], indexing="ij")
    mean = torch.randn(n, EV_D, generator=g) * 0.05
    logvar = torch.randn(n, EV_D, generator=g) * 0.05
    for k, d in enumerate(ENCODES):
        v = grid[k].reshape(-1).float()
        mean[:, d] = (v / (LAT_SIZES[k] - 1) - 0.5) * 4 + 0.05 * torch.randn(n, generator=g)
        logvar[:, d] = -4 + 0.3 * torch.randn(n, generator=g)
    z = mean + torch.exp(0.5 * logvar) * torch.randn(n, EV_D, generator=g)
    return z, mean, logvar


@pytest.mark.gpu
def test_evaluator_metrics_match_the_fp64_oracle(tmp_path):
    """Marginal and conditional entropies, every MI entry, MIG and AAM of the Evaluator (the marginal call on the
    interleaved views _compute_q_zCx produces, 34 kernel calls in all) against the oracle run in fp64 on the same
    draws.  The oracle's per-factor MIG and AAM are checked to sit clear of their clamps, so the comparison sees
    the kernel's values rather than a clamped 0."""
    import logging

    import disvae
    z, mean, logvar = _factor_posteriors()
    n = z.shape[0]
    g = torch.Generator().manual_seed(1)
    draws = [torch.randperm(n, generator=g)]                                   # H(z_j), then H(z_j | v_k) per value
    draws += [torch.randperm(n // s, generator=g) for s in LAT_SIZES for _ in range(s)]

    model = disvae.init_specific_model("Burgess", (1, 32, 32), EV_D)
    ev = disvae.Evaluator(model, None, device=torch.device("cuda"), logger=logging.getLogger("t"),
                          save_dir=str(tmp_path), is_progress_bar=False)
    ev._perm_queue = list(draws)
    fn = disvae.Evaluator._estimate_latent_entropies
    old = fn.__defaults__
    fn.__defaults__ = (EV_S,)
    try:
        samples = z.cuda()
        params = torch.stack([mean, logvar], dim=-1).cuda().unbind(-1)
        H_z = ev._estimate_latent_entropies(samples, params)
        H_zCv = ev._estimate_H_zCv(samples.view(*LAT_SIZES, EV_D), tuple(p.view(*LAT_SIZES, EV_D) for p in params),
                                   LAT_SIZES, ["f%d" % k for k in range(len(LAT_SIZES))])
    finally:
        fn.__defaults__ = old
    assert not ev._perm_queue
    H_z, H_zCv = H_z.cpu(), H_zCv.cpu()
    mut_info = -H_zCv + H_z                                                    # as Evaluator.compute_metrics
    sorted_mut_info = torch.sort(mut_info, dim=1, descending=True)[0].clamp(min=0)
    st = {}
    mig = ev._mutual_information_gap(sorted_mut_info, LAT_SIZES, st)
    aam = ev._axis_aligned_metric(sorted_mut_info, st)

    z64, m64, lv64 = z.double(), mean.double(), logvar.double()
    H_z_ref = O.estimate_latent_entropies(z64, m64, lv64, draws[0][:EV_S])
    H_zCv_ref = O.estimate_H_zCv(z64, m64, lv64, LAT_SIZES, iter([p[:EV_S] for p in draws[1:]]))
    mig_ref, aam_ref, mig_k_ref, aam_k_ref = O.mig_aam(H_z_ref, H_zCv_ref, LAT_SIZES)
    assert (mig_k_ref > 0.02).all() and (aam_k_ref > 0.1).all(), (mig_k_ref, aam_k_ref)

    e_H = max(_err(H_z, H_z_ref), _err(H_zCv, H_zCv_ref))
    e_mi = (mut_info.double() - (H_z_ref - H_zCv_ref)).abs().max().item()
    e_metric = max((st["mig_k"].double() - mig_k_ref).abs().max().item(),
                   (st["aam_k"].double() - aam_k_ref).abs().max().item(),
                   abs(mig.item() - mig_ref.item()), abs(aam.item() - aam_ref.item()))
    print("Evaluator %s: worst H err %.2e, MI err %.2e, MIG/AAM err %.2e (MIG %.4f, AAM %.4f)"
          % (LAT_SIZES, e_H, e_mi, e_metric, mig_ref.item(), aam_ref.item()))
    assert e_H <= H_TOL, e_H
    assert e_mi <= MI_TOL, e_mi
    assert e_metric <= MI_TOL, e_metric
