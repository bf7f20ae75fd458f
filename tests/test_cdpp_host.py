"""LightCurveCollection.remove_outliers / estimate_cdpp on oracle-backed stand-ins for engine.sigma_clip / engine.cdpp
(and, for the single-curve loop they must equal, engine.flatten / engine.nanmedian_std): argument handling, shapes,
the empty collection, column="flux_err", keyword errors, float32 flux and the polyorder clamp."""
import logging
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _cdpp_cases as C  # noqa: E402
import _cdpp_oracle as O  # noqa: E402

import lightkurve_b200 as lk  # noqa: E402
from lightkurve_b200 import engine  # noqa: E402
from oracle import detrend as odet  # noqa: E402


@pytest.fixture
def calls(monkeypatch):
    log = []

    def sigma_clip(arrays, sigma_lower=3.0, sigma_upper=3.0, maxiters=5, offsets=None):
        log.append(("sigma_clip", len(arrays), sigma_lower, sigma_upper, maxiters))
        mi = None if maxiters < 0 else maxiters
        masks = [O.sigma_clip_mask(a, sigma_lower=sigma_lower, sigma_upper=sigma_upper, maxiters=mi) for a in arrays]
        return dict(mask=masks)

    def cdpp(times, fluxes, durations=13, savgol_window=101, savgol_polyorder=2, sigma=5.0, offsets=None):
        log.append(("cdpp", len(times), list(np.atleast_1d(durations)), savgol_window, savgol_polyorder, sigma,
                    [np.asarray(f).dtype for f in fluxes]))
        for d in np.atleast_1d(durations):
            if d < 1:
                raise ValueError("lkb_cdpp: transit durations must be >= 1 cadence")
        return np.array([[O.cdpp(t, f, int(d), savgol_window, savgol_polyorder, sigma)
                          for d in np.atleast_1d(durations)] for t, f in zip(times, fluxes)])

    def flatten(times, fluxes, flux_errs=None, masks=None, window_length=101, polyorder=2, break_tolerance=5,
                niters=3, sigma=3):
        out = [odet.flatten(t, f, e, window_length, polyorder, break_tolerance, niters, sigma)
               for t, f, e in zip(times, fluxes, flux_errs)]
        return [o[0] for o in out], [o[1] for o in out], [o[2] for o in out]

    def nanmedian_std(arrays):
        with np.errstate(all="ignore"), _quiet():
            return (np.array([np.nanmedian(a) if np.isfinite(a).any() else np.nan for a in arrays]),
                    np.array([np.nanstd(a) if np.isfinite(a).any() else np.nan for a in arrays]))

    for name, fn in (("sigma_clip", sigma_clip), ("cdpp", cdpp), ("flatten", flatten),
                     ("nanmedian_std", nanmedian_std)):
        monkeypatch.setattr(engine, name, fn)
    return log


class _quiet:
    def __enter__(self):
        import warnings
        self._w = warnings.catch_warnings()
        self._w.__enter__()
        warnings.simplefilter("ignore", RuntimeWarning)

    def __exit__(self, *a):
        return self._w.__exit__(*a)


def _coll(dtype=np.float64, n=(600, 1500, 400)):
    rng = np.random.default_rng(4)
    lcs = []
    for k, m in enumerate(n):
        t, f = C.light_curve(rng, m, 200, ["everything", "transit", "flares"][k % 3])
        lcs.append(lk.LightCurve(time=t, flux=f.astype(dtype), flux_err=np.full(m, 2e-4, dtype)))
    return lk.LightCurveCollection(lcs)


def test_estimate_cdpp_equals_the_loop(calls):
    coll = _coll()
    got = coll.estimate_cdpp()
    assert got.unit == lk.units.ppm and got.shape == (3,)
    ref = [lc.estimate_cdpp().value for lc in coll]
    np.testing.assert_allclose(got.value, ref, rtol=1e-9)
    assert [c for c in calls if c[0] == "cdpp"] == [("cdpp", 3, [13], 101, 2, 5.0, [np.dtype(np.float64)] * 3)]


def test_sequence_durations_give_b_by_d(calls):
    coll = _coll()
    got = coll.estimate_cdpp(transit_duration=[13, 1, 30], savgol_window=51, sigma=4.0)
    assert got.shape == (3, 3)
    for b, lc in enumerate(coll):
        for d, dur in enumerate((13, 1, 30)):
            np.testing.assert_allclose(got.value[b, d], lc.estimate_cdpp(dur, 51, 2, 4.0).value, rtol=1e-9)
    assert coll.estimate_cdpp(transit_duration=np.array([5, 7])).shape == (3, 2)
    assert coll.estimate_cdpp(transit_duration=(5,)).shape == (3, 1)
    assert sum(c[0] == "cdpp" for c in calls) == 3              # one engine call each


@pytest.mark.parametrize("bad", [13.0, np.int64(13), "13", [13, 2.5], None])
def test_non_int_duration_raises_like_the_single_curve(calls, bad):
    coll = _coll(n=(300,))
    with pytest.raises(ValueError, match="transit_duration must be an integer"):
        coll.estimate_cdpp(transit_duration=bad)
    if np.ndim(bad) == 0:
        with pytest.raises(ValueError, match="transit_duration must be an integer"):
            coll[0].estimate_cdpp(transit_duration=bad)
    assert not [c for c in calls if c[0] == "cdpp"]


def test_duration_below_one_raises(calls):
    with pytest.raises(ValueError):
        _coll(n=(300,)).estimate_cdpp(transit_duration=[13, 0])


def test_empty_collection(calls):
    empty = lk.LightCurveCollection([])
    assert empty.estimate_cdpp().shape == (0,)
    assert empty.estimate_cdpp(transit_duration=[1, 2]).shape == (0, 2)
    assert len(empty.remove_outliers()) == 0
    out, masks = empty.remove_outliers(return_mask=True)
    assert len(out) == 0 and masks == []
    assert not calls


def test_polyorder_clamp_is_logged_once(calls, caplog):
    coll = _coll(n=(300, 300))
    with caplog.at_level(logging.WARNING):
        coll.estimate_cdpp(savgol_window=3, savgol_polyorder=5)
    assert sum("polyorder must be smaller than window_length" in r.message for r in caplog.records) == 1
    assert calls[-1][3:5] == (3, 2)


def test_float32_works_in_float64(calls):
    """The single-curve method keeps float32 flux through normalize and running_mean's cumulative sum: on float32
    input it differs from the loop on a float64 copy.  The collection casts to float64 and equals the latter."""
    c32 = _coll(np.float32)
    c64 = lk.LightCurveCollection([lk.LightCurve(time=lc.time.value, flux=lc.flux.value.astype(np.float64),
                                                 flux_err=lc.flux_err.value.astype(np.float64)) for lc in c32])
    got = c32.estimate_cdpp().value
    assert calls[-1][-1] == [np.dtype(np.float64)] * 3
    loop64 = np.array([lc.estimate_cdpp().value for lc in c64])
    loop32 = np.array([lc.estimate_cdpp().value for lc in c32])
    np.testing.assert_allclose(got, loop64, rtol=1e-9)
    assert np.max(np.abs(loop32 / loop64 - 1)) > 1e-6          # the float32 path's own rounding
    mean_f32 = lk.utils.running_mean(c32[0].normalize("ppm").flux.value, 13)
    assert mean_f32.dtype == np.float32


@pytest.mark.parametrize("kw", [dict(), dict(sigma=3.0), dict(sigma_lower=2.0, sigma_upper=np.inf),
                                dict(maxiters=None), dict(maxiters=1), dict(maxiters=2.5), dict(maxiters=-1),
                                dict(column="flux_err"), dict(cenfunc="median", stdfunc=np.std)])
def test_remove_outliers_equals_the_loop(calls, kw):
    coll = _coll()
    for lc in coll:                                            # give flux_err outliers of its own
        lc.flux_err.view(np.ndarray)[::37] *= 50
    out, masks = coll.remove_outliers(return_mask=True, **kw)
    assert isinstance(out, lk.LightCurveCollection) and len(out) == len(coll)
    for lc, o, m in zip(coll, out, masks):
        ref_lc, ref_m = lc.remove_outliers(return_mask=True, **kw)
        assert np.array_equal(m, ref_m)
        assert np.array_equal(o.time.value, ref_lc.time.value)
        assert np.array_equal(o.flux.value, ref_lc.flux.value, equal_nan=True)
    plain = coll.remove_outliers(**kw)
    assert all(np.array_equal(a.flux.value, b.flux.value, equal_nan=True) for a, b in zip(plain, out))
    mi = kw.get("maxiters", 5)
    want = -1 if mi is None else max(0, int(np.ceil(mi)))
    assert calls[-1][4] == want


def test_remove_outliers_keyword_errors(calls):
    coll = _coll(n=(300,))
    with pytest.raises(TypeError, match="unsupported sigma_clip keyword"):
        coll.remove_outliers(grow=2)
    with pytest.raises(NotImplementedError):
        coll.remove_outliers(cenfunc="mean")
    with pytest.raises(NotImplementedError):
        coll.remove_outliers(stdfunc="mad_std")
    with pytest.raises(AttributeError):
        coll.remove_outliers(column="no_such_column")
    assert not calls


def test_test_oracle_equals_the_oracle_where_they_overlap():
    """tests/_cdpp_oracle.sigma_clip_mask adds asymmetric sigmas and maxiters=None to oracle.detrend.sigma_clip_mask;
    with equal sigmas and an integer maxiters the two give the same mask."""
    for name, x, sl, su, mi in C.clip_cases():
        for sigma, k in ((sl, mi), (su, 5), (3.0, 1)):
            if k is None or not np.isfinite(sigma):
                continue
            assert np.array_equal(O.sigma_clip_mask(x, sigma, k), odet.sigma_clip_mask(x, sigma, k)), name
