"""LightCurveCollection.fill_gaps / .to_seismology on the host, with numpy stand-ins for the engine's device calls
(as in test_bls_find_host.py): argument handling, fill_gaps' refusals naming the light curve, the nanstd fallback,
the RNG state, the loop's first periodogram error, and LombScarglePeriodogram._prepare unchanged by its grid helper."""
import numpy as np
import pytest

import lightkurve_b200 as lk
from lightkurve_b200 import engine
from lightkurve_b200 import units as u
from lightkurve_b200.periodogram import LombScarglePeriodogram as LS

DT = 1765.5 / 86400.0


def np_fill(times, fluxes, errs, std):
    """numpy stand-in of engine.fill_gaps: the loop's statements, one standard_normal draw."""
    for b, t in enumerate(times):
        if len(t) > 1:
            d = np.diff(t)
            e = engine._gap_reject(b, (1 if np.any(d < 0) else 0) | (2 if np.any(d > 0) else 0), np.median(d))
            if e is not None:
                raise e
    s = std(np.full(len(times), 50.0))
    plans = []
    for t, e in zip(times, errs):
        if len(t) < 2:
            plans.append((t, None, e))
            continue
        dt = np.nanmedian(np.diff(t))
        nt = [t[0]]
        for x in t[1:]:
            while x - nt[-1] > 1.2 * dt:
                nt.append(nt[-1] + dt)
            nt.append(x)
        nt = np.asarray(nt)
        ino = np.isin(nt, t)
        ne = np.zeros(len(nt))
        ne[ino] = e
        ne[~ino] = np.interp(nt[~ino], t, e)
        plans.append((nt, ino, ne))
    z = np.random.standard_normal(sum(int((~p[1]).sum()) for p in plans if p[1] is not None))
    k, to, yo, eo = 0, [], [], []
    for b, (nt, ino, ne) in enumerate(plans):
        if ino is None:
            to.append(nt), yo.append(fluxes[b]), eo.append(ne)
            continue
        y = np.zeros(len(nt))
        y[ino] = fluxes[b]
        m = int((~ino).sum())
        y[~ino] = np.mean(fluxes[b]) + s[b] * z[k:k + m]
        k += m
        to.append(nt), yo.append(y), eo.append(ne)
    return to, yo, eo


@pytest.fixture
def fake(monkeypatch):
    monkeypatch.setattr(engine, "fill_gaps", np_fill)
    monkeypatch.setattr(engine, "nanmedian_std", lambda xs: (np.array([np.nanmedian(x) for x in xs]),
                                                             np.array([np.nanstd(x) for x in xs])))
    calls = {}

    def spectra(times, fluxes, errs, grid, on_median=None, filter_width=0.01):
        med = np.array([np.nanmedian(f) if np.any(~np.isnan(f)) else np.nan for f in fluxes])
        if on_median is not None:
            on_median(med, np.array([np.nanstd(f) for f in fluxes]))
        ts, ys, es = [], [], []
        for t, f, e, m in zip(times, fluxes, errs, med):
            keep = ~np.isnan(f / m)
            if not np.isfinite(t[keep]).all():
                raise ValueError("light curve %d has non-finite times" % len(ts))
            ts.append(t[keep]), ys.append(f[keep] / m), es.append(e[keep] / m)
        ts, ys, es = np_fill(ts, ys, es, lambda c: c * 1e-6)
        grids = []
        for b, t in enumerate(ts):
            grids.append(grid(b, np.median(np.diff(t)) if len(t) > 1 else np.nan, t[0] if len(t) else None,
                              t[-1] if len(t) else None, len(t)))
        calls["grids"] = grids
        return [np.ones(len(g["frequency"])) for g in grids]

    monkeypatch.setattr(engine, "seismology_spectra", spectra)
    return calls


def lc(n=300, unit=None, seed=0, t=None):
    rng = np.random.default_rng(seed)
    t = np.arange(n) * DT if t is None else t
    t = np.delete(t, np.arange(100, 120)) if len(t) > 150 else t
    y = 1 + 1e-3 * rng.normal(size=len(t))
    e = np.full(len(t), 1e-3)
    if unit is not None:
        return lk.LightCurve(time=t, flux=u.Quantity(y * 5e4, unit), flux_err=u.Quantity(e * 5e4, unit))
    return lk.LightCurve(time=t, flux=y, flux_err=e)


def test_fill_gaps_method_and_empty(fake):
    with pytest.raises(NotImplementedError, match="No such method"):
        lk.LightCurveCollection([lc()]).fill_gaps(method="linear")
    assert len(lk.LightCurveCollection([]).fill_gaps()) == 0
    assert lk.LightCurveCollection([]).to_seismology() == []


def test_fill_gaps_rng_state_and_short(fake):
    lcs = [lc(seed=1), lc(n=1), lc(n=0), lc(seed=2)]
    np.random.seed(3)
    got = lk.LightCurveCollection(lcs).fill_gaps()
    st = np.random.get_state()
    np.random.seed(3)
    np.random.standard_normal(40)                   # the two light curves' 20 inserted cadences each
    assert np.array_equal(np.random.get_state()[1], st[1]) and np.random.get_state()[2] == st[2]
    assert len(got[1]) == 1 and len(got[2]) == 0
    assert len(got[0]) == len(lcs[0]) + 20


@pytest.mark.parametrize("unit", [u.electron / u.s, u.electron, u.K])
def test_fill_gaps_nanstd_where_ppm_does_not_convert(fake, unit):
    """estimate_cdpp().to(flux.unit) raises for a unit ppm does not convert to; the noise is then nanstd(flux)."""
    x = lc(unit=unit, seed=4)
    with pytest.raises(Exception):
        u.Quantity(1.0, u.ppm).to(x.flux.unit)
    np.random.seed(0)
    got = lk.LightCurveCollection([x]).fill_gaps()[0]
    np.random.seed(0)
    z = np.random.standard_normal(20)
    ins = ~np.isin(got.time.value, x.time.value)
    f = np.asarray(x.flux.value)
    np.testing.assert_allclose(got.flux.value[ins], np.mean(f) + np.nanstd(f) * z, rtol=1e-14)


def test_fill_gaps_cdpp_in_the_flux_unit(fake):
    x = lc(seed=5)
    np.random.seed(0)
    got = lk.LightCurveCollection([x]).fill_gaps()[0]
    np.random.seed(0)
    z = np.random.standard_normal(20)
    ins = ~np.isin(got.time.value, x.time.value)
    np.testing.assert_allclose(got.flux.value[ins], np.mean(x.flux.value) + 50e-6 * z, rtol=1e-14)


def test_rejects_name_the_light_curve(fake):
    t = np.arange(30) * DT
    with pytest.raises(ValueError, match="light curve 1: its times decrease"):
        lk.LightCurveCollection([lc(), lc(t=t[::-1].copy())]).fill_gaps()
    with pytest.raises(ValueError, match="light curve 0: the median time step"):
        lk.LightCurveCollection([lc(t=np.array([0.0, 0, 0, 0, 1]))]).fill_gaps()
    with pytest.raises(ValueError, match="light curve 1 has non-finite times"):
        lk.LightCurveCollection([lc(), lc(t=np.array([0.0, np.nan, 2]))]).fill_gaps()
    with pytest.raises(ValueError, match="light curve 1 has non-finite times"):
        lk.LightCurveCollection([lc(), lc(t=np.array([0.0, np.inf, 2]))]).to_seismology()


def test_to_seismology_errors_and_grids(fake):
    lcs = [lc(seed=1), lc(seed=2)]
    lk.LightCurveCollection(lcs).to_seismology(ls_method="fastchi2", nterms=2)
    assert all(g["multiterm"] and g["nterms"] == 2 for g in fake["grids"])
    with pytest.raises(ValueError, match="light curve 0: minimum_frequency cannot be larger"):
        lk.LightCurveCollection(lcs).to_seismology(minimum_frequency=300.0, maximum_frequency=100.0)
    with pytest.raises(TypeError, match="light curve 0"):
        lk.LightCurveCollection(lcs).to_seismology(bogus=1)
    with pytest.raises(IndexError, match="light curve 1"):
        lk.LightCurveCollection([lcs[0], lc(n=0)]).to_seismology()
    np.random.seed(1)
    seis = lk.LightCurveCollection(lcs).to_seismology(normalization="psd")
    np.random.seed(1)
    for s, x in zip(seis, lcs):
        filled = x.normalize().remove_nans().fill_gaps()
        ref = LS._prepare(filled, normalization="psd")
        np.testing.assert_array_equal(s.periodogram.frequency.value, ref["frequency"].value)
        assert s.periodogram.frequency.unit == ref["frequency"].unit
        assert s.periodogram.nyquist == ref["nyquist"]
        assert s.periodogram.meta["NORMALIZED"] is True


def test_prepare_grid_against_its_formula():
    """_prepare's grid, from the formula of periodogram.py:784-958 written out independently of `_grid`: a frequency
    step of 1 / (t[-1] - t[0]) / oversample, up to the Nyquist frequency of the median step."""
    x = lc(seed=7)
    t = np.asarray(x.time.value, dtype=np.float64)
    nyq = 0.5 / np.median(np.diff(t))
    for kw, conv, over in ((dict(), 1.0, 5.0), (dict(normalization="psd"), 1e6 / 86400.0, 1.0),
                           (dict(oversample_factor=3, nyquist_factor=2), 1.0, 3.0)):
        p = LS._prepare(x, **kw)
        fs = conv / (t[-1] - t[0]) / over
        ref = np.arange(fs, nyq * conv * kw.get("nyquist_factor", 1), fs)
        assert len(p["frequency"]) == len(ref)
        np.testing.assert_allclose(p["frequency"].value, ref, rtol=1e-13)
        np.testing.assert_allclose(float(p["nyquist"].value), nyq * conv, rtol=1e-14)
        assert p["lc"] is x and np.array_equal(p["time"], t)
    p = LS._prepare(x, minimum_period=0.5, maximum_period=9.0)
    np.testing.assert_allclose(p["frequency"].value, np.arange(1 / 9.0, 2.0, 1 / (t[-1] - t[0]) / 5.0), rtol=1e-13)
    assert p["default_view"] == "period"
    p = LS._prepare(x, frequency=np.linspace(1, 5, 50), ls_method="slow")
    np.testing.assert_array_equal(p["frequency"].value, np.linspace(1, 5, 50))
    assert p["ls_method"] == "slow"
