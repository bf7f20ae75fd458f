"""LightCurveCollection.find_transit_candidates (K3 + K14 + K10 + K6) on the GPU against the loop of single-curve
methods it stands for (tests/_bls_find_cases.loop): every candidate field and masked_in bitwise, the statistics to
compute_stats_batch's tolerance, a light curve alone / in the batch / in a permuted batch bitwise alike, the injected
periods recovered, and the loop's first error."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _bls_find_cases as F  # noqa: E402
import _bls_stats_cases as C  # noqa: E402

from lightkurve_b200 import LightCurve, LightCurveCollection  # noqa: E402

pytestmark = pytest.mark.gpu

FIELDS = ("period", "duration", "transit_time", "depth", "depth_err", "depth_snr", "power")
N_LC = 120


@pytest.fixture(scope="module")
def lcs(engine):
    return F.make_lcs(N_LC)


def _complement_lc():
    """A box of 0.4 d on periods of 0.45 - 0.7 d: most cadences are in transit (the complement is removed)."""
    t = 100.0 + np.arange(3000) * 0.00694
    y = 1 + 1e-3 * np.random.default_rng(5).standard_normal(len(t))
    y[np.abs((t - 100.1 + 0.25) % 0.5 - 0.25) < 0.2] -= 0.01
    return LightCurve(time=t, flux=y, flux_err=np.full(len(t), 1e-3))


SETTINGS = [
    ("autoperiod", dict(), 3),
    ("autoperiod_snr_os5", dict(objective="snr", oversample=5, frequency_factor=20), 2),
    ("period_grid", dict(period=np.exp(np.linspace(np.log(0.6), np.log(9.0), 1500)), duration=[0.05, 0.1, 0.2]), 3),
]


def _check_against_loop(batch, lcs, n, return_stats=False, **kw):
    res = LightCurveCollection(batch).find_transit_candidates(n_candidates=n, return_stats=return_stats, **kw)
    for k in FIELDS:
        assert res[k].shape == (len(batch), n) and res[k].dtype == np.float64
    for b, lc in enumerate(lcs):
        rows, masked, stats, pgs = F.loop(lc, n, return_stats=return_stats, **kw)
        for j, k in enumerate(FIELDS):
            np.testing.assert_array_equal(res[k][b], rows[:, j], err_msg="light curve %d %s" % (b, k))
        assert res["masked_in"][b].dtype == np.int8
        np.testing.assert_array_equal(res["masked_in"][b], masked, err_msg="light curve %d masked_in" % b)
        if return_stats:
            for r, (got, ref, (pg, p, d, tt)) in enumerate(zip(res["stats"][b], stats, pgs)):
                C.assert_stats_match(got, ref, pg, p, d, tt, "light curve %d round %d " % (b, r))
    return res


@pytest.mark.parametrize("name,kw,n", SETTINGS, ids=[s[0] for s in SETTINGS])
def test_against_loop(lcs, name, kw, n):
    batch = lcs[0] if name == "autoperiod" else lcs[0][:40]
    _check_against_loop(batch, batch, n, **kw)


def test_stats_and_complement_mask(lcs):
    batch = lcs[0][:30] + [_complement_lc()]
    _check_against_loop(batch, batch, 2, return_stats=True)
    extra = dict(period=np.linspace(0.45, 0.7, 60), duration=[0.4])
    res = _check_against_loop([_complement_lc()] + lcs[0][:5], [_complement_lc()] + lcs[0][:5], 2, **extra)
    assert np.sum(res["masked_in"][0] == 0) > 0


def test_weights_switch_after_round_0(lcs):
    """A light curve whose NaN flux_err all lie in the first transit searches with flux_err after round 0."""
    got = [b for b, lc in enumerate(lcs[0]) if np.isnan(lc.flux_err.value).any() and not
           np.isnan(lc.flux_err.value[~np.isnan(lc.flux.value)][F.loop(lc, 1)[1] == -1]).any()]
    assert got, "the generator must give a light curve whose NaN flux_err are all removed in round 0"
    batch = [lcs[0][b] for b in got[:8]]
    _check_against_loop(batch, batch, 3)


def test_alone_batched_permuted(lcs):
    batch = lcs[0][:40]
    full = LightCurveCollection(batch).find_transit_candidates(n_candidates=3)
    perm = np.random.default_rng(3).permutation(len(batch))
    pres = LightCurveCollection([batch[i] for i in perm]).find_transit_candidates(n_candidates=3)
    for j, i in enumerate(perm):
        for k in FIELDS:
            np.testing.assert_array_equal(pres[k][j], full[k][i])
        np.testing.assert_array_equal(pres["masked_in"][j], full["masked_in"][i])
    for i in (0, 7, 39):
        one = LightCurveCollection([batch[i]]).find_transit_candidates(n_candidates=3)
        for k in FIELDS:
            np.testing.assert_array_equal(one[k][0], full[k][i])
        np.testing.assert_array_equal(one["masked_in"][0], full["masked_in"][i])


def test_injected_periods_recovered(lcs):
    batch, truth = lcs
    res = LightCurveCollection(batch).find_transit_candidates(n_candidates=3)
    found = total = 0
    for b, planets in enumerate(truth):
        for per, dur, dep, t0 in planets:
            if dep < 0.004:
                continue
            total += 1
            ratio = res["period"][b] / per
            found += bool(np.any(np.abs(ratio - np.rint(ratio)) < 0.01 * np.rint(ratio)) or
                          np.any(np.abs(1 / ratio - np.rint(1 / ratio)) < 0.01))
    assert total > 10 and found >= 0.75 * total, (found, total)


def test_first_error_matches_loop(lcs):
    """Light curve 2 (three cadences) cannot be searched, nor can light curve 4 (no cadence left by remove_nans); the
    loop meets light curve 2 first."""
    t = np.linspace(0, 10, 400)
    tiny = LightCurve(time=t[:3], flux=np.array([1.0, 0.5, 1.0]))
    empty = LightCurve(time=t[:2], flux=np.array([np.nan, np.nan]))
    batch = list(lcs[0][:2]) + [tiny] + [lcs[0][3], empty]
    with pytest.raises(Exception) as ref:
        for lc in batch:
            F.loop(lc, 3)
    with pytest.raises(type(ref.value)) as got:
        LightCurveCollection(batch).find_transit_candidates(n_candidates=3)
    assert "light curve 2, round" in str(got.value) and str(ref.value) in str(got.value)
    with pytest.raises(ValueError, match="light curve 0, round 0"):
        LightCurveCollection([empty]).find_transit_candidates(n_candidates=1)
