"""GPU parity tests: CUDA kernels (through the C ABI) vs the CPU oracle on seeded inputs.

Tolerances (stated once, used everywhere):
  LS     |P_gpu - P_oracle_slow64| <= 1e-5 * max(P) + 1e-4 * P      (fp32 kernel arithmetic, fp32 output)
  BLS    per-sample bin indices and winning (start bin, duration bins): bit-exact;
         sums / objective / depth ...: rtol 1e-9 (fp64, different summation order)
  flatten, regression: rtol 1e-9 vs the scipy/numpy oracle (fp64 kernels)
"""
import numpy as np
import pytest

from oracle import bls as obls
from oracle import detrend as odet
from oracle import ls as ols

pytestmark = pytest.mark.gpu


def assert_ls_close(p_gpu, p_ref):
    p_ref = np.asarray(p_ref, dtype=np.float64)
    p_gpu = np.asarray(p_gpu, dtype=np.float64)
    tol = 1e-5 * np.nanmax(p_ref) + 1e-4 * np.abs(p_ref)
    bad = np.abs(p_gpu - p_ref) > tol
    assert not bad.any(), "LS mismatch: %d/%d bins, worst excess %.3g" % (
        bad.sum(), bad.size, np.max(np.abs(p_gpu - p_ref) / tol))


def make_lc(rng, n, baseline=80.0, irregular=True, dtype=np.float64):
    t = np.sort(rng.uniform(0, baseline, n)) if irregular else np.arange(n) * (baseline / n)
    y = 1.0 + 3e-3 * np.sin(2 * np.pi * t / 3.7 + 0.4) + 1e-3 * np.sin(2 * np.pi * t * 1.9) + 5e-4 * rng.normal(size=n)
    return t + 2000.0, y.astype(dtype)


# ---------------------------------------------------------------- Lomb-Scargle, K1
@pytest.mark.parametrize("normalization", ["amplitude", "psd", "psd_raw"])
def test_ls_ragged_vs_oracle(engine, normalization):
    rng = np.random.default_rng(11)
    ns = [1000, 37, 4099, 1537, 5]
    lcs = [make_lc(rng, n) for n in ns]
    freq = np.linspace(0.01, 12.0, 777)
    scale = np.array([2.0 / (n * 1.0 * 0.013) for n in ns])
    out = engine.ls_power_ragged([l[0] for l in lcs], [l[1] for l in lcs], freq, normalization,
                                 norm_scale=scale if normalization == "psd" else None)
    assert out.shape == (len(ns), len(freq)) and out.dtype == np.float32
    for b, (t, y) in enumerate(lcs):
        p = ols.ls_slow_psd(t, y, freq)
        if normalization == "amplitude":
            p = np.sqrt(p) * np.sqrt(4.0 / len(t))
        elif normalization == "psd":
            p = p * scale[b]
        assert_ls_close(out[b], p)


def test_ls_ragged_per_lc_grids_and_f32(engine):
    rng = np.random.default_rng(12)
    lcs = [make_lc(rng, n, dtype=np.float32) for n in (800, 1200, 64)]
    grids = [ols.default_frequency_grid(l[0])[0] for l in lcs]
    out = engine.ls_power_ragged([l[0] for l in lcs], [l[1] for l in lcs], grids, "amplitude")
    for (t, y), g, o in zip(lcs, grids, out):
        assert o.shape == g.shape
        p = np.sqrt(ols.ls_slow_psd(t, y.astype(np.float64), g)) * np.sqrt(4.0 / len(t))
        assert_ls_close(o, p)


@pytest.mark.parametrize("nterms", [1, 2, 3, 4])
def test_ls_chi2_vs_oracle(engine, nterms):
    rng = np.random.default_rng(14)
    lcs = [make_lc(rng, n) for n in (900, 257, 3000)]
    for t, y in lcs:
        y += 2e-3 * np.sin(2 * np.pi * 2 * (t - t[0]) / 3.7)        # a second harmonic
    freq = np.linspace(0.02, 3.0, 150)
    out, theta = engine.ls_power_chi2([l[0] for l in lcs], [l[1] for l in lcs], freq, nterms, "psd_raw",
                                      return_theta=True)
    for b, (t, y) in enumerate(lcs):
        ref = ols.ls_chi2_psd(t - t[0], y, freq, nterms)
        np.testing.assert_allclose(out[b], ref, rtol=2e-4, atol=1e-5 * ref.max())
        k = int(np.argmax(ref))
        X = ols.design_matrix(t - t[0], freq[k], True, nterms)
        th_ref = np.linalg.solve(X.T @ X, X.T @ (y - y.mean()))
        np.testing.assert_allclose(theta[b, k], th_ref, rtol=1e-5, atol=1e-9)
    if nterms == 1:      # chi2 with one term == the closed-form kernel
        np.testing.assert_allclose(out, engine.ls_power_ragged([l[0] for l in lcs], [l[1] for l in lcs], freq, "psd_raw"),
                                   rtol=5e-4, atol=1e-5 * out.max())


def test_ls_very_low_frequencies(engine):
    """f * baseline << 1: CC'/SS' cancel to ~1e-6 of their terms; the kernels take a full-fp64 path
    for those bins (ragged, shared-SIMT and shared-tcgen05 window terms)."""
    rng = np.random.default_rng(13)
    N = 6000
    t = np.sort(rng.uniform(0, 27.4, N)) + 1325
    y = 1 + 1e-3 * np.sin(2 * np.pi * 3.1 * t) + 3e-4 * rng.normal(size=N)
    T = t[-1] - t[0]
    # (below f * baseline ~ 0.01 the fp64 reference formula itself is ill-conditioned: CC' ~ 1e-11)
    freq = np.concatenate([np.array([0.01, 0.02, 0.03, 0.05, 0.1, 0.3, 1.0, 1.9, 2.1, 3.0]) / T,
                           np.linspace(5 / T, 8.0, 390)])
    ref = np.sqrt(ols.ls_slow_psd(t, y, freq)) * np.sqrt(4.0 / N)
    out = engine.ls_power_ragged([t], [y], freq, "amplitude")[0]
    np.testing.assert_allclose(out, ref, rtol=2e-4, atol=1e-5 * ref.max())
    reg = (1 + np.arange(400)) * (0.05 / T)                       # regular grid starting at 0.05 cycles/baseline
    ref = np.sqrt(ols.ls_slow_psd(t, y, reg)) * np.sqrt(4.0 / N)
    out = engine.ls_power_ragged([t], [y], reg, "amplitude")[0]
    np.testing.assert_allclose(out, ref, rtol=2e-4, atol=1e-5 * ref.max())
    Y = np.stack([y + 1e-4 * rng.normal(size=N) for _ in range(70)])
    for algo in ("simt", "tcgen05"):
        out = engine.ls_power_shared(t, Y, reg, "amplitude", algo=algo)
        for b in (0, 69):
            ref = np.sqrt(ols.ls_slow_psd(t, Y[b], reg)) * np.sqrt(4.0 / N)
            np.testing.assert_allclose(out[b], ref, rtol=2e-4, atol=1e-5 * ref.max(), err_msg=algo)


def test_edge_cases_empty_and_tiny_light_curves(engine):
    freq = np.linspace(0.1, 1.0, 40)
    t2, y2 = np.array([0.0, 1.0]), np.array([1.0, 2.0])
    t7 = np.arange(7.0) * 1.37                                      # (integer times x f=1.0 would be 0/0 in the reference too)
    out = engine.ls_power_ragged([np.zeros(0), t2, t7], [np.zeros(0), y2, np.arange(7.0) ** 2], freq, "psd_raw")
    assert np.isnan(out[0]).all()                                   # empty light curve
    ref = ols.ls_slow_psd(t7, np.arange(7.0) ** 2, freq)
    np.testing.assert_allclose(out[2], ref, rtol=2e-4, atol=1e-5 * ref.max())
    assert out[1].shape == freq.shape                               # 2 points: degenerate (0/0 bins), must not crash
    one = engine.ls_power_ragged([np.arange(50.0)], [np.sin(np.arange(50.0))], np.array([0.05]), "amplitude")
    assert one.shape == (1, 1) and np.isfinite(one).all()           # a single frequency bin
    res = engine.bls_power([np.zeros(0), np.arange(0, 30, 0.1)], [np.zeros(0), np.ones(300)], None, [1.0, 2.0], [0.2])
    assert np.isnan(res["power"][0]).all() and np.isfinite(res["power"][1]).all()
    med, sd = engine.nanmedian_std([np.array([np.nan, np.nan]), np.array([3.0])])
    assert np.isnan(med[0]) and np.isnan(sd[0]) and med[1] == 3.0 and sd[1] == 0.0


def test_ls_constant_flux_is_exactly_zero(engine):
    """reference tests/test_periodogram.py:445-457 (masked NaN -> [1,1,1] must give power == 0)."""
    t = np.array([1.0, 3.0, 4.0])
    y = np.array([1.0, 1.0, 1.0])
    freq = ols.default_frequency_grid(t)[0]
    out = engine.ls_power_ragged([t], [y], freq, "amplitude")
    assert (out == 0).all()


def test_ls_period_recovery_default_grid(engine):
    """reference tests/test_periodogram.py:102-114."""
    rng = np.random.default_rng(1001)
    t = np.arange(1000.0)
    y = rng.normal(1, 0.1, 1000) + np.sin(t / t.max() * 20 * np.pi)
    y /= np.median(y)
    freq = ols.default_frequency_grid(t)[0]
    assert len(freq) == 2497
    out = engine.ls_power_ragged([t], [y], freq, "amplitude")[0]
    assert np.isclose(1.0 / freq[np.nanargmax(out)], 100, rtol=1e-3)
    # and the reference's default (fast, FFT-approximate) method agrees on the peak
    _, pf, _ = ols.lombscargle(t, y)
    assert np.nanargmax(pf) == np.nanargmax(out)


# ---------------------------------------------------------------- Lomb-Scargle, K2 (shared grid)
@pytest.mark.parametrize("algo", ["simt", "auto"])
@pytest.mark.parametrize("B,N,F", [(5, 1000, 300), (130, 2500, 257), (64, 777, 129)])
def test_ls_shared_vs_oracle(engine, algo, B, N, F):
    rng = np.random.default_rng(21)
    keep = np.sort(rng.choice(int(N * 1.1), N, replace=False))
    t = 131.5 + keep * 0.0204336
    amp = 10 ** rng.uniform(-4, -2, (B, 1))
    f_sig = rng.uniform(0.05, 20, (B, 1))
    Y = (1 + amp * np.sin(2 * np.pi * f_sig * t[None, :] + rng.uniform(0, 6, (B, 1)))
         + 10 ** rng.uniform(-4.3, -3, (B, 1)) * rng.normal(size=(B, N))).astype(np.float32)
    baseline = t[-1] - t[0]
    freq = (1 + np.arange(F)) * (1.0 / (5 * baseline)) * 40
    out = engine.ls_power_shared(t, Y, freq, "amplitude", algo=algo)
    assert out.shape == (B, F)
    for b in rng.choice(B, min(B, 6), replace=False):
        p = np.sqrt(ols.ls_slow_psd(t, Y[b].astype(np.float64), freq)) * np.sqrt(4.0 / N)
        assert_ls_close(out[b], p)


def test_ls_tcgen05_long_accumulation(engine):
    """tcgen05 path at the full Kepler cadence count: 65 000-term fp32 register accumulation of split-fp16
    products must still meet the LS tolerance (weak signals in noise are the hard case)."""
    rng = np.random.default_rng(23)
    B, N, F = 70, 65000, 200
    keep = np.sort(rng.choice(71500, N, replace=False))
    t = 131.5 + keep * 0.0204336
    Y = (1 + 10 ** rng.uniform(-4, -2, (B, 1)) * np.sin(2 * np.pi * rng.uniform(0.05, 13, (B, 1)) * t[None, :])
         + 10 ** rng.uniform(-4.3, -3, (B, 1)) * rng.normal(size=(B, N))).astype(np.float32)
    freq = np.sort(rng.uniform(0.01, 13.6, F))
    out = engine.ls_power_shared(t, Y, freq, "amplitude", algo="tcgen05")
    sim = engine.ls_power_shared(t, Y, freq, "amplitude", algo="simt")
    for b in (0, 33, 69):
        p = np.sqrt(ols.ls_slow_psd(t, Y[b].astype(np.float64), freq)) * np.sqrt(4.0 / N)
        assert_ls_close(out[b], p)
        assert_ls_close(sim[b], p)


def test_ls_tcgen05_ragged_tiles(engine):
    """The tensor-core kernel with partly filled frequency and light-curve tiles must meet the same tolerance."""
    rng = np.random.default_rng(23)
    B, N, F = 300, 4100, 700                     # ragged tiles in every dimension, 2 flux tiles, 3 frequency pairs
    t = np.sort(rng.uniform(0, 80, N))
    Y = (1 + 1e-3 * np.sin(2 * np.pi * 1.7 * t)[None, :] + 3e-4 * rng.normal(size=(B, N))).astype(np.float32)
    freq = 0.01 + np.arange(F) * 0.01
    out = engine.ls_power_shared(t, Y, freq, "psd_raw", algo="tcgen05")
    for b in (0, 127, 128, 255, 256, 299):
        assert_ls_close(out[b], ols.ls_slow_psd(t, Y[b].astype(np.float64), freq))


def test_ls_shared_host_pipeline_matches_single_shot(engine, monkeypatch):
    """Host-mode calls with B > 256 are chunk-pipelined (copies overlap compute): same numbers as one shot."""
    rng = np.random.default_rng(24)
    B, N, F = 600, 1500, 300
    t = np.sort(rng.uniform(0, 90, N))
    Y = (1 + 1e-3 * np.sin(2 * np.pi * 0.9 * t)[None, :] + 3e-4 * rng.normal(size=(B, N))).astype(np.float32)
    freq = 0.02 + np.arange(F) * 0.02
    piped = engine.ls_power_shared(t, Y, freq, "amplitude")
    monkeypatch.setenv("LKB_LS_NO_PIPELINE", "1")
    single = engine.ls_power_shared(t, Y, freq, "amplitude")
    np.testing.assert_array_equal(piped, single)
    for b in (0, 255, 256, 511, 512, 599):
        assert_ls_close(piped[b], np.sqrt(ols.ls_slow_psd(t, Y[b].astype(np.float64), freq)) * np.sqrt(4.0 / N))


@pytest.mark.parametrize("algo", ["auto", "simt"])
def test_ls_shared_plan_cache(engine, algo):
    """The y-independent tables of the shared-grid call are cached between calls on the same (times, regular grid,
    family): a second call must return bitwise the same powers, a call with other time stamps of the same count, or
    another grid, must not see stale tables, and an unrelated entry point in between invalidates the cache."""
    rng = np.random.default_rng(5)
    N, B, F = 3000, 9, 20000
    t = 100.0 + np.sort(rng.uniform(0, 80.0, N))
    df = 1.0 / (5.0 * (t[-1] - t[0]))
    freq = df * (1 + np.arange(F))
    Y = (1 + 1e-3 * np.sin(2 * np.pi * 1.7 * t)[None, :] + 3e-4 * rng.normal(size=(B, N))).astype(np.float32)
    a = engine.ls_power_shared(t, Y, freq, "amplitude", algo=algo)
    b = engine.ls_power_shared(t, Y, freq, "amplitude", algo=algo)              # plan found cached
    assert np.array_equal(a, b)
    c = engine.ls_power_shared(t, Y[:4], freq, "amplitude", algo=algo)          # another batch on the cached plan
    assert np.array_equal(c, a[:4])
    t2 = t.copy()
    t2[1000:2000] += 1e-3                                                       # same count, same ends, other stamps
    d = engine.ls_power_shared(t2, Y, freq, "amplitude", algo=algo)
    ref = np.sqrt(ols.ls_slow_psd(t2, Y[2].astype(np.float64), freq[:3000])) * np.sqrt(4.0 / N)
    assert_ls_close(d[2][:3000], ref)
    assert not np.array_equal(d, a)
    engine.nanmedian_std([Y[0].astype(np.float64)])                             # unrelated entry point (re-uses workspace)
    e = engine.ls_power_shared(t2, Y, freq, "amplitude", algo=algo)
    assert np.array_equal(e, d)
    f = engine.ls_power_shared(t2, Y, 2 * freq, "amplitude", algo=algo)         # other grid
    ref = np.sqrt(ols.ls_slow_psd(t2, Y[5].astype(np.float64), 2 * freq[:3000])) * np.sqrt(4.0 / N)
    assert_ls_close(f[5][:3000], ref)


def test_ls_shared_equals_ragged(engine):
    rng = np.random.default_rng(22)
    N, B, F = 1500, 9, 200
    t = np.sort(rng.uniform(0, 50, N))
    Y = 1 + 1e-3 * rng.normal(size=(B, N))
    Y[3] = 1.0   # constant light curve -> exactly zero
    freq = np.linspace(0.02, 10, F)
    a = engine.ls_power_shared(t, Y, freq, "psd_raw", algo="simt")
    b = engine.ls_power_ragged([t] * B, list(Y), freq, "psd_raw")
    assert (a[3] == 0).all() and (b[3] == 0).all()
    assert_ls_close(a, b)


# ---------------------------------------------------------------- BLS, K3
def make_transit_lc(rng, n=2000, dt=0.02, period=2.0, t0=0.5, dur=0.1, depth=0.02, sig=1e-3, gap=True):
    t = np.arange(n) * dt
    if gap:
        t = t[(t < 15) | (t > 16.3)]
    y = np.ones_like(t)
    y[np.abs((t - t0 + 0.5 * period) % period - 0.5 * period) < 0.5 * dur] -= depth
    y += sig * rng.normal(size=len(t))
    return t + 1325.0, y


def assert_bls_close(got, ref, t, y, dy, period, duration, objective="likelihood", max_tied_frac=0.02):
    """Winning (start bin, duration bins) must be IDENTICAL to the oracle's, except where the
    oracle itself has a mathematical tie (the GPU's box, evaluated in the oracle's arithmetic,
    reaches the oracle's best objective to 1e-10): bls.c breaks those by rounding noise only.
    All value outputs rtol 1e-9; transit_time / duration only where the boxes coincide."""
    same = np.all(got["bins"] == ref["bins"], axis=1)
    for p_idx in np.flatnonzero(~same):
        n, dur = got["bins"][p_idx]
        o = obls.objective_at(t, y, dy, period[p_idx], duration, int(n), int(dur), objective=objective)
        assert abs(o - ref["power"][p_idx]) <= 1e-10 * abs(ref["power"][p_idx]), \
            "period %d: GPU box (%d,%d) is not tied with the oracle's %s" % (p_idx, n, dur, ref["bins"][p_idx])
    assert (~same).mean() <= max_tied_frac, "too many tie-broken periods: %d" % (~same).sum()
    for k in ("power", "depth", "depth_err", "depth_snr", "log_likelihood"):
        np.testing.assert_allclose(got[k], ref[k], rtol=1e-9, atol=1e-12, err_msg=k)
    for k in ("duration", "transit_time"):
        np.testing.assert_allclose(got[k][same], ref[k][same], rtol=1e-12, atol=1e-9, err_msg=k)
    return int((~same).sum())


def test_bls_bin_index_bit_exact(engine):
    rng = np.random.default_rng(31)
    t = np.sort(rng.uniform(0, 27.4, 20000))
    t -= t.min()
    for period in (0.3314, 1.0, 2.718281828, 9.26, 0.5 + 1e-13, 1.0 / 3.0):
        for bd in (0.005, 0.0123, 1.0 / 720):
            ref = obls.bin_index_c(t, 0.0, period, bd)
            got = engine.bls_bin_index(t, 0.0, period, bd)
            assert np.array_equal(ref, got), (period, bd, np.flatnonzero(ref != got)[:5])
            assert np.array_equal(ref, obls.bin_index(t, 0.0, period, bd))
    # adversarial: times that are exact multiples of the bin width / period
    t2 = np.arange(4000) * 0.005
    for period in (0.5, 1.0, 0.375):
        assert np.array_equal(obls.bin_index_c(t2, 0.0, period, 0.005), engine.bls_bin_index(t2, 0.0, period, 0.005))


@pytest.mark.parametrize("objective", ["likelihood", "snr"])
@pytest.mark.parametrize("with_dy", [True, False])
def test_bls_vs_oracle(engine, objective, with_dy):
    rng = np.random.default_rng(32)
    lcs = [make_transit_lc(rng, n=n, period=p) for n, p in ((2000, 2.0), (1500, 3.3), (700, 1.234))]
    dys = [np.full(len(t), 1e-3) * rng.uniform(0.8, 1.2, len(t)) for t, _ in lcs] if with_dy else None
    duration = np.linspace(0.05, 0.33, 10)
    period = obls.autoperiod(lcs[0][0], duration, 0.4, 8.0, frequency_factor=30)
    res = engine.bls_power([l[0] for l in lcs], [l[1] for l in lcs], dys, period, duration,
                           objective=objective, return_bins=True)
    for b, (t, y) in enumerate(lcs):
        dyb = None if dys is None else dys[b]
        ref = obls.bls_power_c(t, y, dyb, period, duration, objective=objective, return_bins=True)
        assert_bls_close({k: v[b] for k, v in res.items() if k != "period"}, ref, t, y, dyb, period, duration,
                         objective)
    # period recovery (reference tests/test_periodogram.py:331-361 style)
    assert abs(period[np.argmax(res["power"][0])] - 2.0) < 0.01


def test_bls_lightkurve_defaults_recovery(engine):
    """reference tests/test_periodogram.py:331-361: P=2.0 recovered to 2 decimals on the default grid."""
    rng = np.random.default_rng(33)
    time = np.arange(0, 20, 0.02)
    flux = np.ones_like(time)
    flux[np.abs((time - 0.5 + 1.0) % 2.0 - 1.0) < 0.05] = 0.8
    flux += 0.01 * rng.normal(size=len(time))
    lo, hi = obls.lk_default_period_bounds(time, obls.DEFAULT_DURATIONS)
    period = obls.autoperiod(time, obls.DEFAULT_DURATIONS, lo, hi, frequency_factor=10)
    res = engine.bls_power([time], [flux], None, period, obls.DEFAULT_DURATIONS)
    np.testing.assert_almost_equal(period[np.argmax(res["power"][0])], 2.0, decimal=2)


@pytest.mark.parametrize("density", ["0", "1e31", None])
def test_bls_dense_sampling_boundary_path(engine, density, monkeypatch):
    """TESS-like 2-min sampling (3.6 cadences per bin): the bin-boundary path (prefix-sum differences between
    exactly located run starts) must give the oracle's boxes and values; forced on ("0"), off ("1e31"), auto."""
    if density is not None:
        monkeypatch.setenv("LKB_BLS_MIN_DENSITY", density)
    rng = np.random.default_rng(35)
    lcs, dys = [], []
    for n_keep, p_true in ((9000, 2.17), (7000, 0.9), (3000, 4.4)):
        grid = 1325.0 + np.arange(10000) / 720.0
        grid = np.concatenate([grid[:4200], grid[4900:]])                    # a data gap
        keep = np.sort(rng.choice(len(grid), n_keep, replace=False))
        t = grid[keep] + rng.uniform(-2e-4, 2e-4, n_keep)
        t.sort()
        y = 1 + 5e-4 * rng.normal(size=n_keep)
        y[np.abs((t - 1326.0 + 0.5 * p_true) % p_true - 0.5 * p_true) < 0.06] -= 3e-3
        lcs.append((t, y))
        dys.append(5e-4 * rng.uniform(0.8, 1.2, n_keep))
    # adversarial: cadences that sit (to an ulp) ON the bin edges - decided by the exact fmod/division walk
    t_adv = 1325.0 + np.arange(9000) * (0.005 / 4)
    lcs.append((t_adv, 1 + 5e-4 * rng.normal(size=len(t_adv))))
    dys.append(np.full(len(t_adv), 5e-4))
    duration = np.linspace(0.05, 0.33, 10)
    period = np.concatenate([obls.autoperiod(lcs[0][0], duration, 0.3314, 9.26, frequency_factor=10),
                             [0.3314, 0.335 + 1e-13, 0.5, 1.0, 0.4 + 0.005 / 3, 2.5, 13.0]])
    res = engine.bls_power([l[0] for l in lcs], [l[1] for l in lcs], dys, period, duration, return_bins=True)
    for b, (t, y) in enumerate(lcs):
        ref = obls.bls_power_c(t, y, dys[b], period, duration, return_bins=True)
        assert_bls_close({k: v[b] for k, v in res.items() if k != "period"}, ref, t, y, dys[b], period, duration,
                         max_tied_frac=0.02 if b < 3 else 0.5)
    assert abs(period[np.argmax(res["power"][0])] - 2.17) < 0.01


def test_bls_global_histograms_in_light_curve_groups(engine, monkeypatch):
    """Global-memory histograms with a tiny workspace cap: the light curves are launched in groups; same results."""
    rng = np.random.default_rng(37)
    lcs = [make_transit_lc(rng, n=1200, period=2.0 + 0.3 * k) for k in range(5)]
    duration = np.linspace(0.05, 0.2, 4)
    period = obls.autoperiod(lcs[0][0], duration, 0.5, 6.0, frequency_factor=40)
    ref = engine.bls_power([l[0] for l in lcs], [l[1] for l in lcs], None, period, duration, return_bins=True)
    monkeypatch.setenv("LKB_BLS_GHIST_BINS", "0")
    monkeypatch.setenv("LKB_BLS_HIST_CAP_MB", "1")
    got = engine.bls_power([l[0] for l in lcs], [l[1] for l in lcs], None, period, duration, return_bins=True)
    for k in ("power", "depth", "bins", "transit_time"):
        np.testing.assert_array_equal(got[k], ref[k])


def test_bls_unsorted_times_fall_back_to_cadence_path(engine):
    rng = np.random.default_rng(36)
    t = 1325.0 + np.arange(8000) / 720.0
    y = 1 + 5e-4 * rng.normal(size=len(t))
    perm = rng.permutation(len(t))
    duration = np.linspace(0.05, 0.2, 4)
    period = obls.autoperiod(t, duration, 0.5, 5.0, frequency_factor=20)
    res = engine.bls_power([t[perm]], [y[perm]], None, period, duration, return_bins=True)
    ref = obls.bls_power_c(t[perm], y[perm], None, period, duration, return_bins=True)
    assert_bls_close({k: v[0] for k, v in res.items() if k != "period"}, ref, t[perm], y[perm], None, period, duration)


def test_bls_long_period_global_histograms(engine):
    """n_bins too large for shared memory -> global-memory histogram path."""
    rng = np.random.default_rng(34)
    t = np.sort(rng.uniform(0, 400, 6000))
    y = 1 + 1e-3 * rng.normal(size=len(t))
    duration = [0.02, 0.05]
    period = np.array([35.0, 120.1, 133.3])       # 120/0.002 = 60000 bins
    res = engine.bls_power([t], [y], None, period, duration, return_bins=True)
    ref = obls.bls_power_c(t, y, None, period, duration, return_bins=True)
    assert_bls_close({k: v[0] for k, v in res.items() if k != "period"}, ref, t, y, None, period, duration,
                     max_tied_frac=0.34)


def test_bls_errors(engine):
    t = np.arange(100.0)
    y = np.ones(100)
    with pytest.raises(ValueError, match="maximum transit duration"):
        engine.bls_power([t], [y], None, [0.1, 1.0], [0.2])
    with pytest.raises(ValueError, match="period"):
        engine.bls_power([t], [y], None, [1.0, np.nan], [0.2])


# ---------------------------------------------------------------- flatten, K4
def make_trend_lc(rng, n, gaps=True):
    t = np.arange(n) * 0.0204336 + 131.5
    if gaps:
        keep = np.ones(n, bool)
        for s in rng.choice(n - 200, 3, replace=False):
            keep[s:s + rng.integers(20, 150)] = False
        t = t[keep]
    f = 1 + 0.01 * np.sin(2 * np.pi * t / 11.0) + 2e-3 * np.cos(2 * np.pi * t / 2.3) + 3e-4 * rng.normal(size=len(t))
    out = rng.choice(len(t), max(1, len(t) // 300), replace=False)
    f[out] += 8 * 3e-4 * rng.choice([-1, 1], len(out))
    fe = 3e-4 * rng.uniform(0.8, 1.2, len(t))
    return t, f, fe


@pytest.mark.parametrize("window_length,polyorder,niters", [(101, 2, 3), (401, 2, 3), (51, 3, 2), (7, 1, 1)])
def test_flatten_vs_oracle(engine, window_length, polyorder, niters):
    rng = np.random.default_rng(41)
    lcs = [make_trend_lc(rng, n) for n in (6000, 3000, 900, 450)]
    lcs[1][1][100:110] = np.nan                     # NaN flux passes through
    masks = [None, None, rng.uniform(size=len(lcs[2][0])) < 0.05, None]
    masks = [np.zeros(len(l[0]), bool) if m is None else m for l, m in zip(lcs, masks)]
    flat, flat_err, trend = engine.flatten([l[0] for l in lcs], [l[1] for l in lcs], [l[2] for l in lcs], masks,
                                           window_length=window_length, polyorder=polyorder, niters=niters)
    for b, (t, f, fe) in enumerate(lcs):
        rf, rfe, rtr = odet.flatten(t, f, fe, window_length=window_length, polyorder=polyorder, niters=niters,
                                    mask=masks[b])
        np.testing.assert_allclose(trend[b], rtr, rtol=1e-9, err_msg="trend lc %d" % b)
        np.testing.assert_allclose(flat[b], rf, rtol=1e-9, equal_nan=True)
        np.testing.assert_allclose(flat_err[b], rfe, rtol=1e-9, equal_nan=True)


def test_flatten_kernel_generations_agree(engine, monkeypatch):
    """The streaming kernel (flatten_v2.cuh, default) and the round-1 FIR kernel (LKB_FLATTEN_V1=1) on the same light
    curves; a light curve with more gap segments than the streaming kernel's shared-memory list (status 2) makes the
    whole call re-run on the first kernel - the result is the oracle's either way; polyorder 6 is first-kernel only."""
    rng = np.random.default_rng(77)
    lcs = [make_trend_lc(rng, n) for n in (5000, 2500)]
    args = dict(window_length=101, polyorder=2, niters=3)
    a = engine.flatten([l[0] for l in lcs], [l[1] for l in lcs], [l[2] for l in lcs], None, **args)
    monkeypatch.setenv("LKB_FLATTEN_V1", "1")
    b = engine.flatten([l[0] for l in lcs], [l[1] for l in lcs], [l[2] for l in lcs], None, **args)
    monkeypatch.delenv("LKB_FLATTEN_V1")
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            np.testing.assert_allclose(u, v, rtol=1e-9, equal_nan=True)
    # 1500 gaps of 10 cadence steps each, segments of 8 cadences: all median fallbacks, more than 1023 segments
    n_seg, seg_len = 1500, 8
    idx = (np.arange(n_seg)[:, None] * (seg_len + 10) + np.arange(seg_len)[None, :]).ravel()
    t = 100.0 + idx * 0.02
    f = 1 + 1e-3 * np.sin(t) + 1e-4 * rng.normal(size=len(t))
    fe = np.full(len(t), 1e-4)
    flat, _, trend = engine.flatten([t, lcs[0][0]], [f, lcs[0][1]], [fe, lcs[0][2]], None, window_length=5, polyorder=2)
    rf, _, rt = odet.flatten(t, f, fe, window_length=5, polyorder=2)
    np.testing.assert_allclose(trend[0], rt, rtol=1e-9)
    np.testing.assert_allclose(flat[0], rf, rtol=1e-9)
    flat6, _, trend6 = engine.flatten([lcs[1][0]], [lcs[1][1]], [lcs[1][2]], None, window_length=51, polyorder=6)
    np.testing.assert_allclose(trend6[0], odet.flatten(lcs[1][0], lcs[1][1], lcs[1][2], window_length=51, polyorder=6,
                                                       savgol=odet.savgol_lsq)[2], rtol=1e-9)


def test_flatten_reference_known_answers(engine):
    """reference tests/test_lightcurve.py:1297-1317."""
    t = np.arange(6.0)
    f = np.array([10, 20, 30, 40, 50, 60], dtype=np.float64)
    flat, _, trend = engine.flatten([t], [f], None, None, window_length=3, polyorder=1)
    np.testing.assert_allclose(flat[0], 1.0, rtol=1e-12)
    # window_length > len -> median fallback
    flat, _, trend = engine.flatten([t], [f], None, None, window_length=7, polyorder=1)
    np.testing.assert_allclose(trend[0], np.median(f))
    # polyorder >= window_length is clamped; break_tolerance=None accepted
    engine.flatten([t], [f], None, None, window_length=3, polyorder=5, break_tolerance=None)


def test_iterative_flatten_reference(engine):
    """reference tests/test_lightcurve.py:1344-1360."""
    x = np.arange(2000.0)
    y = np.sin(np.arange(2000) / 200) / 100 + 1
    y[250] -= 0.01
    flat, _, _ = engine.flatten([x], [y], None, None, window_length=25, niters=2, sigma=3)
    assert np.isclose(flat[0], 1, rtol=1e-5).sum() == 1999
    m = np.zeros(2000, bool)
    m[250] = True
    flat, _, _ = engine.flatten([x], [y], None, [m], window_length=25, niters=1, sigma=3)
    assert np.isclose(flat[0], 1, rtol=1e-5).sum() == 1999


# ---------------------------------------------------------------- regression, K5
def test_regress_reference_known_answers(engine):
    """reference tests/correctors/test_regressioncorrector.py:13-48."""
    X = np.array([[1.0, 1.0], [1.0, 2.0]])
    y = np.array([[5.0, 10.0]])
    r = engine.regress(X, y)
    np.testing.assert_almost_equal(r["coefficients"][0], [0, 5])
    r = engine.regress(X, y, flux_err=np.array([[0.1, 0.1]]))
    np.testing.assert_almost_equal(r["coefficients"][0], [0, 5])
    r = engine.regress(X, y, prior_mu=np.array([99.0, 99.0]), prior_sigma=np.array([1e-9, 1e-9]))
    np.testing.assert_almost_equal(r["coefficients"][0], [99, 99])
    r = engine.regress(X, y, prior_mu=np.array([99.0, 99.0]), prior_sigma=np.array([1e9, 1e9]))
    np.testing.assert_almost_equal(r["coefficients"][0], [0, 5])


@pytest.mark.parametrize("K,N,B", [(7, 500, 3), (151, 3000, 4), (64, 1000, 2), (151, 2011, 9), (13, 777, 70),
                                   (163, 900, 8)])
def test_regress_vs_oracle(engine, K, N, B):
    rng = np.random.default_rng(51)
    X = np.cumsum(rng.normal(size=(N, K - 1)), axis=0)
    X, _ = np.linalg.qr(X)
    X = np.hstack([X * np.sqrt(N), np.ones((N, 1))])
    W = rng.normal(size=(B, K)) * 1e-3
    Y = 1 + W @ X.T + 3e-4 * rng.normal(size=(B, N))
    for b in range(B):
        o = rng.choice(N, 6, replace=False)
        Y[b, o] += 8 * 3e-4
    fe = 3e-4 * rng.uniform(0.8, 1.2, (B, N))
    cm = np.ones((B, N), bool)
    cm[0, 10:30] = False
    pm = np.zeros(K)
    ps = np.full(K, np.inf)
    ps[:3] = 0.5
    r = engine.regress(X, Y, fe, cm, pm, ps, sigma=5, niters=5)
    assert (r["status"] == 0).all()
    for b in range(B):
        ref = odet.regress(X, Y[b], fe[b], cm[b], pm, ps, sigma=5, niters=5)
        assert np.array_equal(r["outlier_mask"][b], ref["outlier_mask"])
        np.testing.assert_allclose(r["coefficients"][b], ref["coefficients"], rtol=1e-7, atol=1e-10)
        np.testing.assert_allclose(r["model"][b], ref["model"], rtol=1e-7, atol=1e-10)


def test_regress_tcgen05_gram_vs_fp64(engine, monkeypatch):
    """The first fit's Gram matrices as one tcgen05 GEMM (regress_tc.cu) against the fp64 DMMA kernel on the same
    batch: K = 37 (three column blocks, the last one partly empty), 70 light curves (a partly filled light-curve
    tile), per-cadence errors, a cadence mask and outliers that later iterations downdate.  Identical outlier masks,
    coefficients to SURVEY 8c's 1e-4."""
    rng = np.random.default_rng(202)
    N, K, B = 6000, 37, 70
    X = np.cumsum(rng.normal(size=(N, K - 1)), axis=0)
    X, _ = np.linalg.qr(X - X.mean(0))
    X = np.hstack([X * np.sqrt(N) * 10 ** rng.uniform(-2, 2, K - 1), np.ones((N, 1))])     # columns of very different scale
    Wt = rng.normal(size=(B, K)) * 1e-3 / np.abs(X).max(axis=0)
    Wt[:, -1] = 0
    Y = 1 + Wt @ X.T + 3e-4 * rng.normal(size=(B, N))
    for b in range(B):
        Y[b, rng.choice(N, 20, replace=False)] += 8 * 3e-4
    fe = 3e-4 * rng.uniform(0.7, 1.4, (B, N))
    cm = rng.uniform(size=(B, N)) > 0.03
    monkeypatch.setenv("LKB_REGRESS_TC", "1")
    a = engine.regress(X, Y, fe, cm, None, None, sigma=5, niters=4)
    monkeypatch.setenv("LKB_REGRESS_TC", "0")
    b_ = engine.regress(X, Y, fe, cm, None, None, sigma=5, niters=4)
    assert (a["status"] == 0).all() and (b_["status"] == 0).all()
    assert np.array_equal(a["outlier_mask"], b_["outlier_mask"])
    scale = np.abs(b_["coefficients"] * np.abs(X).max(axis=0)).max(axis=1, keepdims=True) / np.abs(X).max(axis=0)
    assert np.all(np.abs(a["coefficients"] - b_["coefficients"]) <= 1e-4 * np.abs(b_["coefficients"]) + 1e-5 * scale)
    np.testing.assert_allclose(a["model"], b_["model"], atol=2e-7)
    ref = odet.regress(X, Y[3], fe[3], cm[3], None, None, sigma=5, niters=4)
    assert np.array_equal(a["outlier_mask"][3], ref["outlier_mask"])
    np.testing.assert_allclose(a["model"][3], ref["model"], atol=2e-7)


def test_regress_singular_reports_status(engine):
    X = np.ones((50, 2))                           # duplicate columns, no priors -> singular
    y = np.arange(50.0)[None, :]
    r = engine.regress(X, y)
    assert r["status"][0] == -4 and np.isnan(r["coefficients"]).all()


# ---------------------------------------------------------------- K6
def test_nanmedian_std(engine):
    rng = np.random.default_rng(61)
    arrs = [rng.normal(size=n) for n in (1, 2, 3, 1000, 4097)]
    arrs[3][::7] = np.nan
    arrs.append(np.array([1.0, 1.0, 1.0, 2.0]))
    arrs.append(np.array([-0.0, 0.0, 5.0, -3.0, np.inf]))
    med, sd = engine.nanmedian_std(arrs)
    for a, m, s in zip(arrs, med, sd):
        assert m == np.nanmedian(a)
        np.testing.assert_allclose(s, np.nanstd(a), rtol=1e-12, equal_nan=True)


# ---------------------------------------------------------------- periodogram background (K6 reuse)
@pytest.mark.parametrize("F,B,fw", [(2497, 3, 0.1), (20000, 5, 0.01), (777, 2, 0.033)])
def test_pg_logmedian_vs_oracle(engine, F, B, fw):
    """Periodogram.smooth(method="logmedian") (periodogram.py:260-284): exact window medians, reference summation order."""
    from oracle import pg as opg
    rng = np.random.default_rng(61)
    freq = (np.arange(F) + 1) * 0.0137 if F != 777 else np.sort(rng.uniform(0.01, 300, F))
    power = rng.chisquare(2, size=(B, F)) * (1 + 5.0 / (1 + freq))
    power[0, 5] = np.nan                                            # nanmedian semantics
    got = engine.pg_logmedian(freq, power, fw)
    for b in range(B):
        ref = opg.smooth_logmedian(freq, power[b], fw)
        np.testing.assert_allclose(got[b], ref, rtol=1e-13, atol=0, equal_nan=True)
    # an unsorted grid is handled by sorting (the window sets are order independent)
    perm = rng.permutation(F)
    got_p = engine.pg_logmedian(freq[perm], power[1][perm], fw)
    if freq[perm][0] == freq.min() and freq[perm][-1] == freq.max():
        np.testing.assert_allclose(got_p, got[1][perm], rtol=1e-13)
