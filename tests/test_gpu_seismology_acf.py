"""K7 windowed autocorrelation on the GPU (lkb_acf_windows, engine.acf_windows) and the batched ACF2D estimators
built on it (seismology.estimate_numax_acf2d_batch / estimate_deltanu_acf2d_batch), against np.correlate and the
per-periodogram host estimators."""
import warnings

import numpy as np
import pytest

import lightkurve_b200 as lk
from lightkurve_b200 import units as u
from lightkurve_b200.periodogram import SNRPeriodogram
from lightkurve_b200.seismology import (estimate_deltanu_acf2d, estimate_deltanu_acf2d_batch, estimate_numax_acf2d,
                                        estimate_numax_acf2d_batch)
from test_seismology_batch_host import red_giant_snr

pytestmark = pytest.mark.gpu

KEPLER_F, KEPLER_NYQ = 35749, 283.2            # 4-year long-cadence grid, oversample 1 (uHz)
KEPLER_FS = KEPLER_NYQ / KEPLER_F


def ref_acf(x, start, n):
    sel = np.array(x[start:start + n], dtype=np.float64)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        sel -= np.nanmean(sel)
    acf = np.correlate(sel, sel, mode="full")[n - 1:]
    return acf, (np.sum(np.abs(acf)) - 1) / n


def assert_acf_close(got, ref):
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    ok = ~np.isnan(ref)
    if ok.any():
        scale = abs(ref[0]) if ok[0] else np.nanmax(np.abs(ref))
        assert np.max(np.abs(got[ok] - ref[ok])) <= 1e-12 * scale


def ms_spectrum(nmx, fmax=4000.0, df=0.4):
    """A main-sequence SNR spectrum in the form of test_seismology.generate_test_spectrum at numax `nmx`."""
    f = np.arange(0, fmax, df)
    fs = f.max() / len(f)
    s = 0.25 * nmx / 2.335
    p = 10 * np.exp(-0.5 * (f - nmx) ** 2 / s ** 2)
    m = np.zeros(len(f))
    lo, hi = int(np.floor(0.5 * nmx / fs)), int(np.floor(1.5 * nmx / fs))
    for modeloc in np.arange(lo, hi, 0.294 * nmx ** 0.772 / 2, dtype=int):
        m[modeloc] += 1
    p = p * m + 1
    return SNRPeriodogram(u.Quantity(f, u.microhertz), u.Quantity(p, None))


def test_acf_windows_vs_np_correlate(engine):
    """Random windows of ragged series: numax-sized windows, the 68 k-lag deltanu window of an oversample-5 Kepler
    grid, lengths around the 1152-lag tile, NaN windows (one NaN, all NaN)."""
    rng = np.random.default_rng(11)
    lengths = [3154, 68164, 1, 1151, 1152, 1153, 63, 500]
    series, starts = [], []
    for n in lengths:
        F = n + int(rng.integers(1, 4000))
        x = rng.exponential(size=F) * (1 + 5 * np.exp(-0.5 * ((np.arange(F) - F / 2) / (F / 8)) ** 2))
        st = np.sort(rng.integers(0, F - n + 1, size=1 if n > 10000 else 4)).astype(np.int64)
        series.append(x)
        starts.append(st)
    series[7][starts[7][1] + 17] = np.nan                  # one NaN inside a window
    series[7][starts[7][2]:starts[7][2] + 500] = np.nan    # an all-NaN window
    metrics, acfs = engine.acf_windows(series, starts, lengths, return_acf=True)
    for b, (x, st, n) in enumerate(zip(series, starts, lengths)):
        assert acfs[b].shape == (len(st), n) and metrics[b].shape == (len(st),)
        for k, s in enumerate(st):
            ra, rm = ref_acf(x, int(s), n)
            assert_acf_close(acfs[b][k], ra)
            np.testing.assert_allclose(metrics[b][k], rm, rtol=1e-10, equal_nan=True)
    assert np.isnan(metrics[7][1]) and np.isnan(acfs[7][2]).all()
    m_only = engine.acf_windows(series, starts, lengths)
    for b in range(len(series)):
        np.testing.assert_array_equal(m_only[b], metrics[b])
    with pytest.raises(ValueError, match="leaves the series"):
        engine.acf_windows([np.ones(10)], [np.array([5])], [6])
    with pytest.raises(ValueError, match=">= 1"):
        engine.acf_windows([np.ones(10)], [np.array([0])], [0])


def _catalog_like(rng, numaxs, F=KEPLER_F, fs=KEPLER_FS):
    return [red_giant_snr(rng, nm, F=F, fs=fs) for nm in numaxs]


def _near_tie(ms):
    top = np.sort(ms)[-2:]
    return abs(top[1] - top[0]) <= 1e-9 * abs(top[1])


def test_numax_deltanu_batch_equal_the_host_loop(engine):
    rng = np.random.default_rng(12)
    pgs = _catalog_like(rng, [35.0, 60.0, 90.0, 120.0, 150.0, 180.0, 210.0, 240.0])
    pgs += [ms_spectrum(nm) for nm in (1000.0, 1500.0, 2000.0, 2500.0)]
    pgs += [red_giant_snr(rng, nm) for nm in (50.0, 100.0, 170.0, 220.0)]
    got = estimate_numax_acf2d_batch(pgs, return_acf2d=True)
    refs = [estimate_numax_acf2d(pg) for pg in pgs]
    for g, r in zip(got, refs):
        dg, dr = g.diagnostics, r.diagnostics
        assert g.unit == r.unit and (g.name, g.method) == ("numax", "ACF2D")
        np.testing.assert_array_equal(dg["numaxs"], dr["numaxs"])
        assert dg["window_width"] == dr["window_width"]
        np.testing.assert_allclose(dg["metric"], dr["metric"], rtol=1e-10)
        np.testing.assert_allclose(dg["metric_smooth"], dr["metric_smooth"], rtol=1e-10)
        assert dg["acf2d"].shape == dr["acf2d"].shape
        for k in range(dr["acf2d"].shape[1]):
            assert_acf_close(dg["acf2d"][:, k], dr["acf2d"][:, k])
        if not _near_tie(dr["metric_smooth"]):
            assert g.value == r.value
    dn = estimate_deltanu_acf2d_batch(pgs, refs)
    for d, pg, r in zip(dn, pgs, refs):
        assert d.value == estimate_deltanu_acf2d(pg, r).value
    for g, nm in zip(got[:8], [35.0, 60.0, 90.0, 120.0, 150.0, 180.0, 210.0, 240.0]):
        assert abs(g.value - nm) < 0.1 * nm


def test_bitwise_repeatable_and_independent_of_the_batch(engine):
    rng = np.random.default_rng(13)
    pgs = _catalog_like(rng, [70.0, 110.0, 160.0])
    a = estimate_numax_acf2d_batch(pgs, return_acf2d=True)
    b = estimate_numax_acf2d_batch(pgs, return_acf2d=True)
    alone = estimate_numax_acf2d_batch([pgs[1]], return_acf2d=True)[0]
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x.diagnostics["metric"], y.diagnostics["metric"])
        np.testing.assert_array_equal(x.diagnostics["acf2d"], y.diagnostics["acf2d"])
    np.testing.assert_array_equal(alone.diagnostics["metric"], a[1].diagnostics["metric"])
    np.testing.assert_array_equal(alone.diagnostics["acf2d"], a[1].diagnostics["acf2d"])
    d1 = estimate_deltanu_acf2d_batch(pgs, a)
    d2 = estimate_deltanu_acf2d_batch([pgs[2]], [a[2]])[0]
    np.testing.assert_array_equal(d1[2].diagnostics["acf"], d2.diagnostics["acf"])


def test_chain_from_light_curves(engine):
    """Light curves in the style of test_seismology_from_lightcurve at several numax: the batched periodogram and
    background, then the batched estimators."""
    N, dt = 12000, 1765.5 / 86400.0
    t = np.arange(N) * dt
    keep = np.ones(N, bool)
    keep[5000:5200] = False
    truths, lcs = [], []
    for i, numax_true in enumerate((110.0, 150.0, 190.0)):
        rng = np.random.default_rng(50 + i)
        dnu = 0.294 * numax_true ** 0.772
        modes = numax_true + dnu * np.arange(-5, 6)
        modes = np.concatenate([modes, modes + 0.5 * dnu - 1.2])
        amp = 3e-5 * np.exp(-0.5 * ((modes - numax_true) / (0.66 * numax_true ** 0.88 / 2.355)) ** 2)
        y = 1 + sum(a * np.sin(2 * np.pi * (m * 1e-6 * 86400) * t + rng.uniform(0, 2 * np.pi)) for a, m in zip(amp, modes))
        y = y + 2e-5 * rng.normal(size=N)
        lcs.append(lk.LightCurve(time=t[keep], flux=y[keep], flux_err=np.full(keep.sum(), 2e-5)))
        truths.append((numax_true, dnu))
    np.random.seed(11)
    prepared = lk.LightCurveCollection([lc.normalize().remove_nans().fill_gaps() for lc in lcs])
    pgs = [pg.flatten() for pg in prepared.to_periodogram(normalization="psd")]
    numaxs = estimate_numax_acf2d_batch(pgs)
    deltanus = estimate_deltanu_acf2d_batch(pgs, numaxs)
    for (nm, dnu), n_est, d_est in zip(truths, numaxs, deltanus):
        assert n_est.unit == u.microhertz
        assert abs(n_est.value - nm) < 0.1 * nm
        assert abs(d_est.value - dnu) < 0.25 * dnu


def test_catalog_size(engine):
    """2048 red giants x 35 749 bins x 257 windows in one call; four stars from different places in the batch
    equal the host estimator."""
    rng = np.random.default_rng(14)
    B = 2048
    f = KEPLER_FS * (1 + np.arange(KEPLER_F))
    templates = [np.asarray(red_giant_snr(np.random.default_rng(k), nm, F=KEPLER_F, fs=KEPLER_FS).power.value)
                 for k, nm in enumerate((45.0, 80.0, 130.0, 200.0))]
    fq = u.Quantity(f, u.microhertz)
    pgs = [SNRPeriodogram(fq, u.Quantity(templates[b % 4] * rng.uniform(0.5, 1.5, KEPLER_F), None)) for b in range(B)]
    got = estimate_numax_acf2d_batch(pgs)
    assert len(got) == B and len(got[0].diagnostics["numaxs"]) == 257
    for b in (0, 701, 1366, 2047):
        ref = estimate_numax_acf2d(pgs[b])
        np.testing.assert_allclose(got[b].diagnostics["metric"], ref.diagnostics["metric"], rtol=1e-10)
        if not _near_tie(ref.diagnostics["metric_smooth"]):
            assert got[b].value == ref.value
