"""IRS on the host (no GPU, no kernel): the restatement of tests/irs_reference.py bins factors as np.histogram and
np.digitize do and takes quantiles bit for bit as np.percentile does; it agrees with disentanglement_lib's float32
computation; every refusal happens before any GPU work; and the host path of `irs_score` (with `irs_fit` replaced by
the restatement) draws SAP's training rows and finishes the matrix as the definition does."""
import numpy as np
import pytest
import torch

import irs_reference as R
from disvae import evaluate
from score_stubs import _evaluator, _Grid, no_gpu  # noqa: F401


def test_bins_equal_numpy_histogram_and_digitize():
    """Every integer range lo in [0, 4], hi in [lo, 399]: the fp64 edges are np.histogram's bit for bit, and the bins
    np.digitize's (less one); the equal range is widened by 0.5 each way."""
    for lo in range(5):
        for hi in range(lo, 400):
            v = np.arange(lo, hi + 1, dtype=np.int64)
            e = R.edges(v)
            want = np.histogram(v, 20)[1]
            assert np.array_equal(e.view(np.int64), want.view(np.int64)), (lo, hi)
            assert np.array_equal(R.bins(v, e) + 1, np.digitize(v, want[:-1])), (lo, hi)
    assert R.edges([3, 3])[0] == 2.5 and R.edges([3, 3])[-1] == 3.5


def test_fp32_edges_would_bin_some_ranges_differently():
    """Why the factor edges are fp64: numpy's fp32 linspace rule (dv_common.cuh's histogram_edges) moves some value to
    another bin on some of those ranges."""
    import modularity_reference as MR
    differ = 0
    for lo in range(5):
        for hi in range(lo, 400):
            v = np.arange(lo, hi + 1, dtype=np.int64)
            differ += not np.array_equal(R.bins(v, R.edges(v)) + 1, MR.bins(v, MR.edges(v)))
    assert differ > 0


@pytest.mark.parametrize("dq", [0.0, 0.5, 0.9, 0.99, 1.0, 0.123456789, 0.3141592653589793, 0.999, 0.01, 0.75])
def test_quantile_equals_np_percentile_bitwise(dq):
    g = np.random.default_rng(int(dq * 1e6))
    for m in range(1, 301):
        a = np.abs(g.standard_normal(m)) * 10.0 ** g.integers(-3, 4)
        want = np.percentile(a, dq * 100)
        got = R.quantile(a, dq)
        assert np.float64(got).view(np.int64) == np.float64(want).view(np.int64), (m, dq, got, want)


def test_random_quantiles_equal_np_percentile_bitwise():
    g = np.random.default_rng(5)
    for dq in g.random(40):
        for m in (1, 2, 3, 7, 100, 101, 256, 300):
            a = np.abs(g.standard_normal(m))
            assert np.float64(R.quantile(a, dq)).view(np.int64) == np.float64(
                np.percentile(a, dq * 100)).view(np.int64), (m, dq)


def _codes(lat_sizes, rows, D, seed, noise=0.2):
    """Latent d follows scored factor d (scaled to [0, 1)) plus noise; further latents are noise."""
    g = np.random.default_rng(seed)
    factors, v = R.draw_values(lat_sizes, rows)
    x = g.standard_normal((len(rows), D)).astype(np.float32)
    for d in range(min(D, len(factors))):
        x[:, d] = v[d] / lat_sizes[factors[d]] + noise * x[:, d]
    return x.astype(np.float32), v


@pytest.mark.parametrize("dq", [0.99, 0.5])
def test_restatement_agrees_with_the_float32_library(dq):
    """dSprites-like factors (3, 6, 40, 32, 32 values: 40 and 32 merge bins), aligned and noise latents and one
    constant latent: IRS within 1e-5; num_active_dims is the count here, the sum of the active codes there."""
    lat = [3, 6, 40, 32, 32]
    rows = np.random.default_rng(1).integers(0, int(np.prod(lat)), 10000)
    x, v = _codes(lat, rows, 8, 2)
    x[:, 6] = 0.25
    f = R.fit(x, v, dq)
    irs, per, parents = R.score(f["irs_matrix"], f["max_deviation"], f["active"])
    lib = R.library_irs(x.T, v, dq)
    assert abs(irs - lib["IRS"]) < 1e-5, (irs, lib["IRS"])
    assert f["active"].sum() == 7 and parents[6] == -1 and np.isnan(per[6])
    assert lib["num_active_dims"] != 7
    assert abs(lib["num_active_dims"] - np.delete(x, 6, 1).sum()) <= 1e-3 * abs(np.delete(x, 6, 1)).sum()
    assert parents[:5].tolist() == [0, 1, 2, 3, 4]


def test_all_constant_codes_score_zero():
    lat = [4, 5]
    rows = np.arange(20)
    x = np.zeros((20, 3), np.float32)
    x[:10, 1] = -0.0
    f = R.fit(x, R.draw_values(lat, rows)[1], 0.99)
    assert not f["active"].any() and np.isnan(f["irs_matrix"]).all()
    assert R.score(f["irs_matrix"], f["max_deviation"], f["active"])[0] == 0.0
    assert R.library_irs(x.T, R.draw_values(lat, rows)[1])["IRS"] == 0.0


# ---- refusals ----------------------------------------------------------------------------------------------------
REFUSALS = [
    (_Grid([4, 5], factors=False), 10, {}, "no lat_sizes / lat_names"),
    (_Grid([4, 5], n=21), 10, {}, "has 21 items, not the 20 of the full grid"),
    (_Grid([1, 1, 1]), 10, {}, r"every factor of \[1, 1, 1\] has one value"),
    (_Grid([4, 5]), 0, {}, r"latent_dim must be in \[1, 1024\], got 0"),
    (_Grid([4, 5]), 1025, {}, r"latent_dim must be in \[1, 1024\], got 1025"),
    (_Grid([4, 5]), 10, {"num_train": 0}, r"num_train must be in \[1, 32768\], got 0"),
    (_Grid([4, 5]), 10, {"num_train": 32769}, r"num_train must be in \[1, 32768\], got 32769"),
    (_Grid([4, 5]), 10, {"diff_quantile": -0.01}, r"diff_quantile must be in \[0, 1\], got -0.01"),
    (_Grid([4, 5]), 10, {"diff_quantile": 1.5}, r"diff_quantile must be in \[0, 1\], got 1.5"),
    (_Grid([4, 5]), 10, {"diff_quantile": float("nan")}, r"diff_quantile must be in \[0, 1\], got nan"),
]


@pytest.mark.parametrize("case", range(len(REFUSALS)))
def test_refusals_before_gpu_work(tmp_path, no_gpu, case):
    ds, latent_dim, settings, msg = REFUSALS[case]
    loader = torch.utils.data.DataLoader(ds, batch_size=10)
    with pytest.raises(ValueError, match=msg):
        _evaluator(tmp_path, latent_dim).compute_irs_score(loader, **settings)
    with pytest.raises(ValueError, match=msg):
        evaluate.check_irs_score(ds, latent_dim, **settings)
    if hasattr(ds, "lat_sizes"):
        with pytest.raises(ValueError, match=msg):
            evaluate.irs_score(torch.zeros(len(ds), latent_dim), ds.lat_sizes, **settings)
    assert not list(tmp_path.iterdir())


# ---- the host path with the restatement standing in for the kernel -----------------------------------------------
@pytest.fixture
def host_fit(monkeypatch):
    calls = []

    def fit(mu, rows, values, diff_quantile):
        calls.append((rows.clone(), values.clone(), diff_quantile))
        assert values.dtype == torch.int32
        f = R.fit(mu.numpy()[rows.numpy()], values.numpy(), diff_quantile)
        t = {k: torch.from_numpy(np.asarray(v)) for k, v in f.items()}
        return (t["max_deviation"], t["active"].int(), t["irs_matrix"], t["group_deviation"], t["group_count"].int(),
                t["edges"])
    monkeypatch.setattr(evaluate, "irs_fit", fit)
    monkeypatch.setattr(evaluate.N, "require_cuda_f32", lambda *t: None)
    return calls


def test_host_path_equals_the_definition(host_fit, monkeypatch):
    """Factors of 3, 1, 40 and 5 values (the size-1 factor is not scored); the rows are SAP's training rows."""
    lat = [3, 1, 40, 5]
    n = int(np.prod(lat))
    g = torch.Generator().manual_seed(3)
    mu = torch.randn(n, 6, generator=g)
    mu[:, 0] = torch.from_numpy(np.unravel_index(np.arange(n), lat)[2] / 40.0).float() + 0.05 * mu[:, 0]
    mu[:, 5] = 1.5
    score, helpers = evaluate.irs_score(mu, lat, num_train=500, diff_quantile=0.9, seed=11)
    rows, values, dq = host_fit[0]
    assert dq == 0.9
    sap_rows = evaluate._sap_draws(mu, lat, 500, 7, 11)[0]
    assert torch.equal(rows, sap_rows)
    factors, want_values = R.draw_values(lat, rows.numpy())
    assert factors == [0, 2, 3] and np.array_equal(values.numpy(), want_values)
    f = R.fit(mu.numpy()[rows.numpy()], want_values, 0.9)
    irs, per, parents = R.score(f["irs_matrix"], f["max_deviation"], f["active"])
    assert score == {"IRS": irs, "num_active_dims": 5}
    assert helpers["factors"].tolist() == [0, 2, 3]
    assert helpers["parents"].tolist() == parents.tolist() and helpers["parents"][0] == 1 and helpers["parents"][5] == -1
    assert np.array_equal(helpers["disentanglement_scores"].numpy(), per, equal_nan=True)
    assert helpers["active_dims"].dtype == torch.bool and helpers["active_dims"].tolist() == [True] * 5 + [False]
    assert helpers["group_counts"].dtype == torch.int64 and helpers["group_counts"].sum(1).tolist() == [500] * 3
    assert tuple(helpers["group_deviations"].shape) == (3, 20, 6) and tuple(helpers["bin_edges"].shape) == (3, 21)
    assert tuple(helpers["irs_matrix"].shape) == (6, 3) and helpers["max_deviations"].shape == (6,)


def test_irs_from_matrix_ties_and_no_active_latent():
    M = torch.tensor([[0.5, 0.7, 0.7], [0.2, 0.1, 0.2], [float("nan")] * 3], dtype=torch.float64)
    dev = torch.tensor([2.0, 1.0, 0.0], dtype=torch.float64)
    irs, per, parents = evaluate.irs_from_matrix(M, dev, torch.tensor([1, 1, 0], dtype=torch.int32))
    assert parents.tolist() == [1, 0, -1] and per[:2].tolist() == [0.7, 0.2] and torch.isnan(per[2])
    assert irs == (2.0 * 0.7 + 1.0 * 0.2) / 3.0
    irs, per, parents = evaluate.irs_from_matrix(M, dev, torch.zeros(3, dtype=torch.bool))
    assert irs == 0.0 and parents.tolist() == [-1] * 3 and torch.isnan(per).all()
