"""The shim of the batched BLS follow-ups (BoxLeastSquaresPeriodogram.compute_stats_batch / get_transit_mask_batch)
on a numpy stand-in for engine.bls_stats: candidate defaults and their warnings, broadcasting, the transit-mask rule,
the transit-slot bound and the errors.  Where astropy is installed, the host compute_stats is also checked against
astropy's BoxLeastSquares.compute_stats."""
import logging
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _bls_stats_cases as C  # noqa: E402

from lightkurve_b200 import _lib as L  # noqa: E402
from lightkurve_b200 import engine  # noqa: E402
from lightkurve_b200.periodogram import BoxLeastSquaresPeriodogram as BLS  # noqa: E402


def numpy_bls_stats(times, fluxes, flux_errs, period, duration, transit_time, return_mask=False, offsets=None,
                    transit_offsets=None):
    """engine.bls_stats (host mode) restated with the host compute_stats and numpy."""
    numpy_bls_stats.calls.append(dict(period=np.array(period), duration=np.array(duration),
                                      transit_time=np.array(transit_time), flux_errs=flux_errs))
    B = len(times)
    per, dur, tts = (np.broadcast_to(np.asarray(x, dtype=float), (B,)) for x in (period, duration, transit_time))
    toff = engine.bls_transit_slots(times, per, tts)
    offs = np.r_[0, np.cumsum([len(t) for t in times])]
    stats = np.zeros((B, len(engine.BLS_STATS_COLUMNS)))
    first, n_tr, status = np.zeros(B, np.int64), np.zeros(B, np.int32), np.zeros(B, np.int32)
    cnt, lls, mask = np.zeros(toff[-1], np.int32), np.zeros(toff[-1]), np.zeros(offs[-1], bool)
    for b in range(B):
        t_abs, y = np.asarray(times[b], float), np.asarray(fluxes[b], float)
        dy = None if flux_errs is None else np.asarray(flux_errs[b], float)
        p, d, tt = per[b], dur[b], tts[b]
        pg = C.make_pg(t_abs, y, dy, p, d, tt)
        t, ttr = t_abs - t_abs[0], tt - t_abs[0]
        m_in = np.abs((t - ttr + 0.5 * p) % p - 0.5 * p) < 0.5 * d
        if m_in.any():
            ids = np.round((t[m_in] - ttr) / p).astype(int)
            first[b], n_tr[b] = ids.min(), ids.max() - ids.min() + 1
        try:
            r = pg.compute_stats(p, d, tt)
            for k, key in enumerate(("depth", "depth_odd", "depth_even", "depth_half", "depth_phased")):
                stats[b, 2 * k:2 * k + 2] = r[key][0].value, r[key][1].value
            stats[b, 10], stats[b, 11] = r["harmonic_amplitude"].value, r["harmonic_delta_log_likelihood"]
            cnt[toff[b]:toff[b] + n_tr[b]] = r["per_transit_count"]
            lls[toff[b]:toff[b] + n_tr[b]] = r["per_transit_log_likelihood"]
        except np.linalg.LinAlgError:
            status[b] = L.E_SINGULAR
        ivar = np.ones_like(y) if dy is None else 1.0 / dy ** 2
        mm = np.abs((t_abs - tt + 0.5 * p) % p - 0.5 * p) < 0.5 * d
        with np.errstate(divide="ignore", invalid="ignore"):
            stats[b, 12] = np.sum(y[mm] * ivar[mm]) / np.sum(ivar[mm])
            stats[b, 13] = np.sum(y[~mm] * ivar[~mm]) / np.sum(ivar[~mm])
        stats[b, 14] = mm.sum()
        mask[offs[b]:offs[b + 1]] = mm
    res = dict(stats=stats, transit_first=first, transit_n=n_tr, per_transit_count=cnt, per_transit_log_likelihood=lls,
               status=status, offsets=offs, transit_offsets=toff)
    if return_mask:
        res["in_transit"] = mask
    return res


@pytest.fixture
def stand_in(monkeypatch):
    numpy_bls_stats.calls = []
    monkeypatch.setattr(engine, "bls_stats", numpy_bls_stats)
    return numpy_bls_stats


def test_cases_through_the_shim(stand_in):
    C.check_batch(C.cases(), BLS.compute_stats_batch, BLS.get_transit_mask_batch)


def test_defaults_warn_once_per_call(stand_in, caplog):
    cs = C.cases()
    pgs = C.pgs_of(cs)
    with caplog.at_level(logging.WARNING):
        BLS.compute_stats_batch(pgs)
    msgs = [r.getMessage() for r in caplog.records]
    assert msgs == ["No period specified. Using period at max power",
                    "No duration specified. Using duration at max power",
                    "No transit time specified. Using transit time at max power"]
    call = stand_in.calls[-1]
    np.testing.assert_array_equal(call["period"], [c[4] for c in cs])
    np.testing.assert_array_equal(call["duration"], [c[5] for c in cs])
    np.testing.assert_array_equal(call["transit_time"], [c[6] for c in cs])
    caplog.clear()
    with caplog.at_level(logging.WARNING):
        BLS.get_transit_mask_batch(pgs, period=[c[4] for c in cs])
    assert len(caplog.records) == 2 and "period" not in caplog.records[0].getMessage().split(".")[0]


def test_broadcasting_and_quantities(stand_in):
    from lightkurve_b200 import units as u
    cs = C.cases()[:3]
    pgs = C.pgs_of(cs)
    got = BLS.compute_stats_batch(pgs, period=u.Quantity(2.5, u.day), duration=0.1,
                                  transit_time=[c[6] for c in cs])
    call = stand_in.calls[-1]
    np.testing.assert_array_equal(call["period"], [2.5] * 3)
    np.testing.assert_array_equal(call["duration"], [0.1] * 3)
    for pg, g, c in zip(pgs, got, cs):
        C.assert_stats_match(g, pg.compute_stats(2.5, 0.1, c[6]), pg, 2.5, 0.1, c[6])
    with pytest.raises(ValueError, match="3 periodograms"):
        BLS.compute_stats_batch(pgs, period=[1.0, 2.0])
    assert BLS.compute_stats_batch([]) == [] and BLS.get_transit_mask_batch([]) == []


def test_flux_err_mixed(stand_in):
    """Periodograms without flux_err get unit weights next to ones with it."""
    cs = C.cases()
    pgs = C.pgs_of(cs)
    BLS.get_transit_mask_batch(pgs)
    errs = stand_in.calls[-1]["flux_errs"]
    for c, e in zip(cs, errs):
        np.testing.assert_array_equal(e, np.ones(len(c[1])) if c[3] is None else c[3])
    pgs = C.pgs_of([c for c in cs if c[3] is None])
    BLS.get_transit_mask_batch(pgs)
    assert stand_in.calls[-1]["flux_errs"] is None


def test_mask_rule(stand_in):
    """model != median(model) for the two-valued box model: fewer than half in transit -> m_in, more -> ~m_in,
    exactly half -> all True, none or y_in == y_out -> all False."""
    cs = {c[0]: c for c in C.cases()}
    for name, expect in (("sorted_dy", "m_in"), ("majority_in_transit", "~m_in"), ("exactly_half", "all"),
                         ("no_transit_cadence", "none")):
        _, t, y, dy, p, d, tt = cs[name]
        pg = C.make_pg(t, y, dy, p, d, tt)
        m = BLS.get_transit_mask_batch([pg])[0]
        m_in = np.abs((t - tt + 0.5 * p) % p - 0.5 * p) < 0.5 * d
        want = {"m_in": m_in, "~m_in": ~m_in, "all": np.ones(len(t), bool), "none": np.zeros(len(t), bool)}[expect]
        np.testing.assert_array_equal(m, want, err_msg=name)
        np.testing.assert_array_equal(m, pg.get_transit_mask(), err_msg=name)
    t = np.arange(100) * 0.01
    pg = C.make_pg(t, np.ones(100), None, 0.3, 0.05, 0.1)        # flat light curve: y_in == y_out
    assert not BLS.get_transit_mask_batch([pg])[0].any() and not pg.get_transit_mask().any()


def test_transit_slot_bound():
    """bls_transit_slots bounds (and for a candidate inside sorted data, equals) the transit ids compute_stats uses."""
    for name, t, y, dy, p, d, tt in C.cases() + [C.kepler_case()]:
        toff = engine.bls_transit_slots([t], [p], [tt])
        r = C.make_pg(t, y, dy, p, d, tt).compute_stats(p, d, tt)
        assert len(r["per_transit_count"]) <= toff[1], name
        ids = np.round(((t - t[0]) - (tt - t[0])) / p)
        assert toff[1] == ids.max() - ids.min() + 1, name
    # ids rint(0 / 2) .. rint(9 / 2) = 0 .. 4 (half to even), and 0 .. rint(4 / 10) = 0
    toff = engine.bls_transit_slots([np.arange(10.0), np.arange(5.0) + 3], [2.0, 10.0], [0.0, 3.0])
    np.testing.assert_array_equal(toff, [0, 5, 6])


def test_errors(stand_in):
    cs = C.cases()
    pgs = C.pgs_of(cs[:2])
    empty = C.make_pg(np.zeros(0), np.zeros(0))
    with pytest.raises(ValueError, match="no cadences"):
        BLS.compute_stats_batch(pgs + [empty], 1.0, 0.1, 0.0)
    with pytest.raises(ValueError, match="no cadences"):
        BLS.get_transit_mask_batch([empty], 1.0, 0.1, 0.0)
    assert stand_in.calls == []                                   # raised before any device work
    sing = C.singular_cases()
    pgs = C.pgs_of(cs[:2] + sing)
    with pytest.raises(np.linalg.LinAlgError, match="periodogram 2"):
        BLS.compute_stats_batch(pgs, [c[4] for c in cs[:2] + sing], [c[5] for c in cs[:2] + sing],
                                [c[6] for c in cs[:2] + sing])


def test_engine_rejects_bad_candidates_without_a_gpu():
    t = np.arange(10.0)
    for bad in ((0.0, 0.1, 0.0), (np.nan, 0.1, 0.0), (1.0, -0.1, 0.0), (1.0, 0.1, np.inf)):
        with pytest.raises(ValueError):
            engine.bls_stats([t], [np.ones(10)], None, *bad)
    with pytest.raises(ValueError, match="no cadences"):
        engine.bls_stats([t, np.zeros(0)], [np.ones(10), np.zeros(0)], None, 1.0, 0.1, 0.0)


def test_host_compute_stats_against_astropy():
    astropy_ts = pytest.importorskip("astropy.timeseries")
    for name, t, y, dy, p, d, tt in C.cases():
        if name in ("exactly_half",):
            continue
        ref = astropy_ts.BoxLeastSquares(t, y, dy).compute_stats(p, d, tt)
        got = C.make_pg(t, y, dy, p, d, tt).compute_stats(p, d, tt)
        for k in ("depth", "depth_odd", "depth_even", "depth_half", "depth_phased"):
            np.testing.assert_allclose(got[k][0].value, ref[k][0], rtol=1e-9, atol=1e-12, err_msg=name + k)
        np.testing.assert_array_equal(got["per_transit_count"], ref["per_transit_count"], err_msg=name)
        np.testing.assert_allclose(got["per_transit_log_likelihood"], ref["per_transit_log_likelihood"], rtol=1e-9,
                                   atol=1e-9, err_msg=name)
        np.testing.assert_allclose(got["harmonic_delta_log_likelihood"], ref["harmonic_delta_log_likelihood"],
                                   rtol=1e-9, err_msg=name)
