"""LightCurveCollection.fill_gaps and .to_seismology on the GPU (K15, the ragged log-median) against the single-curve
loop under the same np.random seed:
  fill_gaps      times, flux_err and the flux of original cadences bitwise; inserted flux within the CDPP difference
                 of lkb_cdpp and estimate_cdpp (measured 1.9e-9 relative for K12) times |z|, plus the rounding of the
                 mean; the RNG left where the loop leaves it
  to_seismology  frequency grids bitwise; SNR power within the Lomb-Scargle parity tolerance carried through the
                 background: the collection runs the exact direct sums per light curve while the loop's one-curve call
                 may take the NUFFT kernels (both within 1e-5 of max power + 1e-4 relative of the fp64 sums,
                 DESIGN.md section 2), and the log-median background divides that out up to the same order, so the
                 SNR is compared at 1e-3 relative + 1e-3 absolute; the multi-term periodogram and a descending
                 (period) grid likewise;  numax / deltanu from the batch estimators equal the loop's except where the
                 loop's smoothed ACF2D metric has a near-tie, and lie within 10 % / 25 % of the injected values."""
import numpy as np
import pytest

import lightkurve_b200 as lk
from lightkurve_b200 import units as u
from lightkurve_b200.seismology import Seismology, estimate_deltanu_acf2d_batch, estimate_numax_acf2d_batch

pytestmark = pytest.mark.gpu

DT = 1765.5 / 86400.0


def red_giant_lc(seed, numax, N=6000, gaps=((2000, 2150),), unit=None, scale=1.0):
    rng = np.random.default_rng(seed)
    t = np.arange(N) * DT
    keep = np.ones(N, bool)
    for a, b in gaps:
        keep[a:b] = False
    dnu = 0.294 * numax ** 0.772
    modes = numax + dnu * np.arange(-5, 6)
    modes = np.concatenate([modes, modes + 0.5 * dnu - 1.2])
    amp = 3e-5 * np.exp(-0.5 * ((modes - numax) / (0.66 * numax ** 0.88 / 2.355)) ** 2)
    y = 1 + sum(a * np.sin(2 * np.pi * (m * 1e-6 * 86400) * t + rng.uniform(0, 2 * np.pi)) for a, m in zip(amp, modes))
    y = scale * (y + 2e-5 * rng.normal(size=N))
    e = scale * np.full(N, 2e-5) * rng.uniform(0.9, 1.1, N)
    y[rng.integers(0, N, 5)] = np.nan
    kw = dict(flux=y[keep], flux_err=e[keep]) if unit is None else \
        dict(flux=u.Quantity(y[keep], unit), flux_err=u.Quantity(e[keep], unit))
    return lk.LightCurve(time=t[keep], **kw), (numax, dnu)


def edge_cases():
    t = np.arange(40) * DT
    y = 1 + 1e-4 * np.sin(t)
    e = np.full(40, 1e-4)
    e2 = e.copy()
    e2[19] = np.nan                                  # NaN error next to a gap
    e3 = e.copy()
    e3[21] = e3[19]                                  # equal errors on both sides of a gap
    cases = [
        (t, y, e),                                                            # no gap
        (np.delete(t, 20), np.delete(y, 20), np.delete(e, 20)),               # a gap of one cadence
        (np.concatenate([t[:10], t[10:] + 0.2 * DT]), y, e),                  # a step of exactly 1.2 dt: no insert
        (np.concatenate([t[:10], t[10:] + 1200 * DT]), y, e),                 # more than 1 000 inserts
        (np.concatenate([t[:5], t[4:39]]), y, e),                             # duplicate times
        (np.delete(t, [20]), np.delete(y, [20]), np.delete(e2, [20])),
        (np.delete(t, [20]), np.delete(y, [20]), np.delete(e3, [20])),
        (t[:0], y[:0], e[:0]), (t[:1], y[:1], e[:1]), (t[:2], y[:2], e[:2]),
    ]
    return [lk.LightCurve(time=a, flux=b, flux_err=c) for a, b, c in cases]


def collection(n=64):
    numaxs = np.linspace(60.0, 220.0, n)
    lcs, truths = [], []
    for i, nm in enumerate(numaxs):
        gaps = ((1000 + 37 * i, 1100 + 37 * i),) if i % 3 else ((1000, 1100), (4000, 4400))
        lc, tr = red_giant_lc(100 + i, nm, N=5000 + 13 * i, gaps=gaps)
        lcs.append(lc)
        truths.append(tr)
    return lcs, truths


def loop_fill(lcs, seed):
    np.random.seed(seed)
    out = [lc.fill_gaps() for lc in lcs]
    return out, np.random.get_state()


def assert_filled_equal(got, ref, srcs, cdpp_rel=1e-8):
    """Times and flux_err bitwise; original cadences' flux bitwise; inserted flux m + s * z within the CDPP difference
    of lkb_cdpp and estimate_cdpp (1.9e-9 relative for K12, bounded here by `cdpp_rel`) times |s * z|, plus the
    rounding of the mean (a plain sum against numpy's pairwise one: 1e-13 relative)."""
    assert len(got) == len(ref)
    for b, (g, r, src) in enumerate(zip(got, ref, srcs)):
        tg, tr = np.asarray(g.time.value), np.asarray(r.time.value)
        np.testing.assert_array_equal(tg, tr, err_msg="time, light curve %d" % b)
        np.testing.assert_array_equal(np.asarray(g.flux_err.value), np.asarray(r.flux_err.value),
                                      err_msg="flux_err, light curve %d" % b)
        assert g.flux.unit == r.flux.unit
        fg, fr = np.asarray(g.flux.value), np.asarray(r.flux.value)
        src = src.remove_nans()
        if len(src) < 2:
            np.testing.assert_array_equal(fg, fr)
            continue
        ino = np.isin(tr, np.asarray(src.time.value))
        np.testing.assert_array_equal(fg[ino], fr[ino], err_msg="original flux, light curve %d" % b)
        m = np.mean(np.asarray(src.flux.value, dtype=np.float64))
        tol = cdpp_rel * np.abs(fr[~ino] - m) + 1e-13 * abs(m)
        assert np.all(np.abs(fg[~ino] - fr[~ino]) <= tol), "inserted flux, light curve %d" % b


def test_fill_gaps_equals_the_loop(engine):
    lcs, _ = collection(64)
    lcs = lcs + edge_cases()
    lcs.append(red_giant_lc(7, 90.0, N=22000, gaps=((9000, 9720),))[0])       # a TESS-orbit-like 720-cadence gap
    ref, st_ref = loop_fill(lcs, 3)
    np.random.seed(3)
    got = lk.LightCurveCollection(lcs).fill_gaps()
    st = np.random.get_state()
    assert st[0] == st_ref[0] and np.array_equal(st[1], st_ref[1]) and st[2:] == st_ref[2:]
    assert_filled_equal(list(got), ref, lcs)


def test_fill_gaps_electron_per_second_uses_nanstd(engine):
    lcs = [red_giant_lc(20 + i, 120.0, N=3000, unit=u.electron / u.s, scale=5e4)[0] for i in range(5)]
    ref, _ = loop_fill(lcs, 5)
    np.random.seed(5)
    got = lk.LightCurveCollection(lcs).fill_gaps()
    assert_filled_equal(list(got), ref, lcs, cdpp_rel=0.0)       # std is numpy's nanstd here


def test_fill_gaps_repeatable(engine):
    lcs, _ = collection(12)
    np.random.seed(9)
    a = lk.LightCurveCollection(lcs).fill_gaps()
    np.random.seed(9)
    b = lk.LightCurveCollection(lcs).fill_gaps()
    for x, y in zip(a, b):
        np.testing.assert_array_equal(np.asarray(x.flux.value), np.asarray(y.flux.value))


def test_fill_gaps_rejects(engine):
    t = np.arange(20) * DT
    bad = lk.LightCurve(time=t[::-1].copy(), flux=np.ones(20), flux_err=np.ones(20))
    good = lk.LightCurve(time=t, flux=np.ones(20), flux_err=np.ones(20))
    with pytest.raises(ValueError, match="light curve 1"):
        lk.LightCurveCollection([good, bad]).fill_gaps()
    zero = lk.LightCurve(time=np.array([0.0, 0, 0, 0, 1.0]), flux=np.ones(5), flux_err=np.ones(5))
    with pytest.raises(ValueError, match="light curve 0"):
        lk.LightCurveCollection([zero]).fill_gaps()
    inf = lk.LightCurve(time=np.array([0.0, np.inf, 2.0]), flux=np.ones(3), flux_err=np.ones(3))
    with pytest.raises(ValueError, match="non-finite"):
        lk.LightCurveCollection([good, inf]).fill_gaps()


def test_to_seismology_equals_the_loop(engine):
    lcs, truths = collection(64)
    np.random.seed(21)
    ref = [Seismology.from_lightcurve(lc, normalization="psd") for lc in lcs]
    st_ref = np.random.get_state()
    np.random.seed(21)
    got = lk.LightCurveCollection(lcs).to_seismology(normalization="psd")
    st = np.random.get_state()
    assert np.array_equal(st[1], st_ref[1]) and st[2] == st_ref[2]
    assert len(got) == len(ref)
    for b, (g, r) in enumerate(zip(got, ref)):
        pg, pr = g.periodogram, r.periodogram
        assert type(pg) is type(pr)
        np.testing.assert_array_equal(np.asarray(pg.frequency.value), np.asarray(pr.frequency.value))
        assert pg.frequency.unit == pr.frequency.unit and pg.power.unit == pr.power.unit
        assert pg.nyquist == pr.nyquist and pg.label == pr.label and pg.targetid == pr.targetid
        assert pg.meta == pr.meta
        a, c = np.asarray(pg.power.value), np.asarray(pr.power.value)
        np.testing.assert_allclose(a, c, rtol=1e-3, atol=1e-3, err_msg="SNR, light curve %d" % b)
    nm_g = estimate_numax_acf2d_batch([s.periodogram for s in got])
    nm_r = estimate_numax_acf2d_batch([s.periodogram for s in ref])
    dn_g = estimate_deltanu_acf2d_batch([s.periodogram for s in got], nm_g)
    dn_r = estimate_deltanu_acf2d_batch([s.periodogram for s in ref], nm_r)
    for b, ((nm, dnu), x, y, d, e) in enumerate(zip(truths, nm_g, nm_r, dn_g, dn_r)):
        if not _near_tie(y.diagnostics["metric_smooth"]):
            assert x.value == y.value, "numax differs from the loop at light curve %d (%r vs %r)" % (b, x, y)
            assert d.value == e.value, "deltanu differs from the loop at light curve %d (%r vs %r)" % (b, d, e)
        assert abs(x.value - nm) < 0.1 * nm, (b, x, nm)
        assert abs(d.value - dnu) < 0.25 * dnu, (b, d, dnu)


def _near_tie(ms):
    """Two smoothed ACF2D metrics within 1e-3 relative: the SNR spectra agree to the parity tolerance, which can
    pick the other of two near-equal maxima."""
    top = np.sort(np.asarray(ms))[-2:]
    return abs(top[1] - top[0]) <= 1e-3 * abs(top[1])


def assert_seismology_close(got, ref):
    for g, r in zip(got, ref):
        np.testing.assert_array_equal(np.asarray(g.periodogram.frequency.value),
                                      np.asarray(r.periodogram.frequency.value))
        assert g.periodogram.power.unit == r.periodogram.power.unit
        np.testing.assert_allclose(np.asarray(g.periodogram.power.value), np.asarray(r.periodogram.power.value),
                                   rtol=1e-3, atol=1e-3)


def test_to_seismology_multiterm_and_descending_grid(engine):
    lcs, _ = collection(4)
    for kw in (dict(ls_method="fastchi2", nterms=2, normalization="psd"),
               dict(period=np.linspace(1.0 / 250.0, 1.0 / 20.0, 3000), freq_unit=u.microhertz,
                    normalization="psd")):
        np.random.seed(4)
        ref = [Seismology.from_lightcurve(lc, **kw) for lc in lcs]
        np.random.seed(4)
        assert_seismology_close(lk.LightCurveCollection(lcs).to_seismology(**kw), ref)


def test_to_seismology_amplitude_and_kwargs(engine):
    lcs, _ = collection(6)
    kw = dict(minimum_frequency=20.0, maximum_frequency=250.0, oversample_factor=2, freq_unit=u.microhertz)
    np.random.seed(4)
    ref = [Seismology.from_lightcurve(lc, **kw) for lc in lcs]
    np.random.seed(4)
    got = lk.LightCurveCollection(lcs).to_seismology(**kw)
    assert_seismology_close(got, ref)


def test_to_seismology_repeatable_and_errors(engine):
    lcs, _ = collection(5)
    np.random.seed(1)
    a = lk.LightCurveCollection(lcs).to_seismology(normalization="psd")
    np.random.seed(1)
    b = lk.LightCurveCollection(lcs).to_seismology(normalization="psd")
    for x, y in zip(a, b):
        np.testing.assert_array_equal(np.asarray(x.periodogram.power.value), np.asarray(y.periodogram.power.value))
    assert lk.LightCurveCollection([]).to_seismology() == []
    with pytest.raises(ValueError, match="light curve 0"):
        lk.LightCurveCollection(lcs).to_seismology(minimum_frequency=300.0, maximum_frequency=100.0)
