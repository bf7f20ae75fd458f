"""`LightCurveCollection.to_periodogram("bls")` on the host: one engine call for the whole collection, with
`engine.bls_power` replaced by an oracle-backed stand-in (oracle/bls_c.c through oracle.bls.bls_power_c) that
honours both the shared-grid and the per-light-curve-grid forms.  tests/test_gpu_bls_ragged.py runs the kernel."""
import numpy as np
import pytest

import lightkurve_b200 as lk
from oracle import bls as obls

CALLS = []


def oracle_bls_power(times, fluxes, flux_errs, period, duration, oversample=10, objective="likelihood",
                     return_bins=False):
    """`engine.bls_power`'s contract on the oracle: a shared grid gives [B, P] arrays, a list of grids lists."""
    CALLS.append(isinstance(period, (list, tuple)))
    B = len(times)
    per_lc = isinstance(period, (list, tuple))
    grids = list(period) if per_lc else [np.asarray(period, dtype=np.float64)] * B
    rs = [obls.bls_power_c(times[b], fluxes[b], None if flux_errs is None else flux_errs[b], grids[b], duration,
                           oversample=oversample, objective=objective, return_bins=return_bins) for b in range(B)]
    keys = ("power", "depth", "depth_err", "duration", "transit_time", "depth_snr", "log_likelihood") + \
        (("bins",) if return_bins else ())
    if per_lc:
        res = {k: [r[k] for r in rs] for k in keys}
        res["period"] = [np.asarray(g, dtype=np.float64) for g in grids]
    else:
        res = {k: np.stack([r[k] for r in rs]) for k in keys}
        res["period"] = grids[0]
    return res


@pytest.fixture
def engine(monkeypatch):
    from lightkurve_b200 import engine as eng
    monkeypatch.setattr(eng, "bls_power", oracle_bls_power)
    CALLS.clear()
    yield eng


def make_lc(seed, t0=1325.0, days=27.0, cadence=10.0 / 1440, keep=0.9, finite_err=True, transit=True):
    r = np.random.default_rng(seed)
    t = t0 + np.arange(0, days, cadence)
    t = np.sort(t[r.random(len(t)) < keep])
    f = 1 + 5e-4 * r.standard_normal(len(t))
    if transit:
        per, dur = r.uniform(1.5, 5), r.uniform(0.08, 0.2)
        f[np.abs((t - t[0] - 0.4 + 0.5 * per) % per - 0.5 * per) < 0.5 * dur] -= 3e-3
    fe = np.full(len(t), 5e-4) if finite_err else np.full(len(t), np.nan)
    return lk.LightCurve(time=t, flux=f, flux_err=fe)


def assert_same(pgs, loop):
    assert len(pgs) == len(loop)
    for a, b in zip(pgs, loop):
        np.testing.assert_array_equal(np.asarray(a.period.value), np.asarray(b.period.value))
        np.testing.assert_array_equal(np.asarray(a.power.value), np.asarray(b.power.value))
        for k in ("duration", "depth", "snr"):
            np.testing.assert_array_equal(np.asarray(getattr(a, k).value), np.asarray(getattr(b, k).value))
        np.testing.assert_array_equal(np.asarray(a.transit_time.value), np.asarray(b.transit_time.value))
        assert set(a._BLS_result) == set(b._BLS_result)
        for k in a._BLS_result:
            np.testing.assert_array_equal(a._BLS_result[k], b._BLS_result[k])
        assert (a._dy is None) == (b._dy is None)
        if a._dy is not None:
            np.testing.assert_array_equal(a._dy, b._dy)


def collection_vs_loop(lcs, **kw):
    coll = lk.LightCurveCollection(lcs)
    CALLS.clear()
    pgs = coll.to_periodogram("bls", **kw)
    assert len(CALLS) == 1, "the collection made %d engine calls" % len(CALLS)
    ragged = CALLS[0]
    loop = [lc.to_periodogram("bls", **kw) for lc in lcs]
    assert_same(pgs, loop)
    return ragged, pgs


def test_different_baselines_and_cadences(engine):
    lcs = [make_lc(0), make_lc(1, days=20.0), make_lc(2, cadence=30.0 / 1440), make_lc(3, t0=2000.0, days=13.0)]
    ragged, pgs = collection_vs_loop(lcs, duration=[0.05, 0.1, 0.2], frequency_factor=40)
    assert ragged
    assert len({len(pg.period) for pg in pgs}) > 1


def test_mixed_dy_and_snr(engine):
    lcs = [make_lc(4), make_lc(5, finite_err=False), make_lc(6, days=19.0, finite_err=False), make_lc(7, days=22.0)]
    ragged, pgs = collection_vs_loop(lcs, duration=[0.08, 0.16], frequency_factor=40, objective="snr")
    assert ragged
    assert pgs[1]._dy is None and pgs[0]._dy is not None
    # the same light curves on one shared grid take the shared entry, still one call
    ragged, _ = collection_vs_loop(lcs, duration=[0.08, 0.16], period=np.linspace(0.5, 6.0, 700))
    assert not ragged


def test_all_without_flux_err(engine):
    lcs = [make_lc(8, finite_err=False), make_lc(9, days=21.0, finite_err=False)]
    collection_vs_loop(lcs, duration=0.1, frequency_factor=50)


def test_explicit_period_and_bounds(engine):
    lcs = [make_lc(10), make_lc(11, days=16.0)]
    collection_vs_loop(lcs, duration=[0.05, 0.1], period=np.linspace(0.6, 5.0, 500), oversample=5)
    ragged, _ = collection_vs_loop(lcs, duration=[0.05, 0.1], minimum_period=0.7, maximum_period=4.0,
                                   frequency_factor=30)
    assert ragged


def test_one_light_curve_and_empty(engine):
    collection_vs_loop([make_lc(12)], duration=[0.1], frequency_factor=60)
    assert lk.LightCurveCollection([]).to_periodogram("bls") == []


@pytest.mark.parametrize("kw,match", [
    (dict(duration=[0.1, np.nan]), "illegal nan"),
    (dict(duration=[0.1], period=[0.05, 1.0]), "shorter than the minimum period"),
    (dict(duration=[0.1], objective="bic"), "objective|bic"),
    (dict(duration=[0.1], frequency_factor=1e-7), "too large to evaluate"),
    (dict(duration=[0.1], oversample=0), "oversample must be"),
])
def test_prepare_errors_before_engine(engine, kw, match):
    lcs = [make_lc(13), make_lc(14, days=18.0)]
    CALLS.clear()
    with pytest.raises(Exception, match=match):
        lk.LightCurveCollection(lcs).to_periodogram("bls", **kw)
    assert CALLS == []
