"""LightCurveCollection.fold / bin on a numpy stand-in for engine.fold and engine.bin (no GPU): scalar and
per-light-curve arguments with Quantity units, the JD warning once per call, the single-curve methods' errors and
messages, the aggregate_func fallback, and empty collections and zero-length light curves.  The stand-ins restate
the kernels' contract (lightkurve_b200/csrc/foldbin.cuh) in numpy, so these tests check the Python layer only."""
import os
import sys
import warnings

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lightkurve_b200 as lk  # noqa: E402
from lightkurve_b200 import engine, units as u  # noqa: E402
from lightkurve_b200.units import Quantity, Time  # noqa: E402
from lightkurve_b200.utils import LightkurveWarning  # noqa: E402


def fake_fold(times, t0, shift, period, wrap, normalize=False, offsets=None):
    phase, perm = [], []
    for t, a, s, p, w in zip(times, t0, shift, period, wrap):
        assert p > 0
        rel = ((np.asarray(t) - a) + s + (p - w)) % p - (p - w)
        o = np.argsort(rel, kind="stable")
        phase.append(rel[o] / p if normalize else rel[o])
        perm.append(o.astype(np.int32))
    return dict(phase=phase, perm=perm)


def fake_bin(times, fluxes, flux_errs, starts, ends, index_edges=False, aggregate="nanmean", offsets=None,
             bin_offsets=None):
    agg = {"nanmean": np.nanmean, "nanmedian": np.nanmedian}[aggregate]
    res = dict(time=[], flux=[], flux_err=[], count=[])
    for b, t in enumerate(times):
        o = np.argsort(t, kind="stable")
        ts, f, fe = np.asarray(t)[o], np.asarray(fluxes[b])[o], np.asarray(flux_errs[b])[o]
        s, e = (ts[starts[b]], ts[ends[b]]) if index_edges else (starts[b], ends[b])
        nb = len(s)
        which = np.searchsorted(s, ts, side="right") - 1
        inside = (which >= 0) & ((ts < e[np.clip(which, 0, nb - 1)]) | ((which == nb - 1) & (ts <= e[-1])))
        fl, er = np.full(nb, np.nan), np.full(nb, np.nan)
        have = np.any(np.isfinite(fe))
        with warnings.catch_warnings(), np.errstate(all="ignore"):
            warnings.simplefilter("ignore", RuntimeWarning)
            for j in np.unique(which[inside]):
                sel = inside & (which == j)
                fl[j] = agg(f[sel])
                if have:
                    er[j] = np.sqrt(np.nansum(fe[sel] ** 2) / np.sum(np.isfinite(fe[sel]))) \
                        if np.any(np.isfinite(fe[sel])) else np.nan
                else:
                    er[j] = np.nanstd(f[sel]) if np.any(np.isfinite(f[sel])) else np.nan
        res["time"].append(s + 0.5 * (e - s))
        res["flux"].append(fl)
        res["flux_err"].append(er)
        res["count"].append(np.bincount(which[inside], minlength=nb).astype(np.int32))
    return res


@pytest.fixture
def calls(monkeypatch):
    log = []

    def wrap(fn, name):
        def inner(*a, **k):
            log.append(name)
            return fn(*a, **k)
        return inner

    monkeypatch.setattr(engine, "fold", wrap(fake_fold, "fold"))
    monkeypatch.setattr(engine, "bin", wrap(fake_bin, "bin"))
    return log


def _coll(B=5, seed=0, fmt="btjd"):
    rng = np.random.default_rng(seed)
    lcs = []
    for b in range(B):
        n = 200 + 37 * b
        t = rng.permutation(1500.0 + np.arange(n) * 0.0208 + rng.normal(0, 1e-4, n))
        f = 1 + 1e-3 * rng.standard_normal(n)
        lcs.append(lk.LightCurve(time=Time(t, format=fmt, scale="tdb"), flux=f, flux_err=np.full(n, 1e-3),
                                 cadenceno=np.arange(n), targetid=100 + b, label="star %d" % b))
    return lk.LightCurveCollection(lcs)


def _same_lc(a, b):
    assert type(a) is type(b)
    for k in ("time", "flux", "flux_err"):
        x, y = getattr(a, k), getattr(b, k)
        assert np.array_equal(np.asarray(x.value), np.asarray(y.value), equal_nan=True), k
        assert str(getattr(x, "unit", None)) == str(getattr(y, "unit", None)), k
        assert np.asarray(x.value).dtype == np.asarray(y.value).dtype, k
    assert a._columns.keys() == b._columns.keys()
    for k in a._columns:
        assert np.array_equal(a._columns[k], b._columns[k])
    if hasattr(b, "time_original"):
        assert np.array_equal(a.time_original.value, b.time_original.value)
        assert a.time_original.format == b.time_original.format
    assert a.meta.keys() == b.meta.keys()
    for k, v in b.meta.items():
        w = a.meta[k]
        if v is None:
            assert w is None, k
        elif hasattr(v, "value"):
            assert np.array_equal(np.asarray(w.value), np.asarray(v.value)), k
            assert str(getattr(w, "unit", None)) == str(getattr(v, "unit", None)), k
        else:
            assert w == v, k


FOLD_ARGS = [dict(period=0.7),
             dict(period=0.7 * u.day, epoch_time=1500.3, epoch_phase=0.1, wrap_phase=0.2 * u.day),
             dict(period=16.8 * u.hour, epoch_phase=-0.25, normalize_phase=True, wrap_phase=0.75),
             dict(period=[0.5, 0.6, 0.7, 0.8, 0.9], epoch_time=[1500.1, 1500.2, 1500.3, 1500.4, 1500.5]),
             dict(period=[0.5 * u.day, 13.0 * u.hour, 0.7 * u.day, 0.8 * u.day, 0.9 * u.day],
                  epoch_time=Time([1500.1, 1500.2, 1500.3, 1500.4, 1500.5], format="btjd"), wrap_phase=0.0),
             dict(period=Quantity([0.5, 0.6, 0.7, 0.8, 0.9], u.day), epoch_phase=[0.0, 0.1, -0.2, 0.3, 0.4],
                  wrap_phase=[0.5, 0.6, 0.7, 0.8, 0.9] * u.day)]


@pytest.mark.parametrize("kw", FOLD_ARGS, ids=range(len(FOLD_ARGS)))
def test_fold_equals_loop(calls, kw):
    coll = _coll()
    got = coll.fold(**kw)
    assert calls == ["fold"]
    per = lambda v, b: v[b] if isinstance(v, (list, Quantity)) and np.ndim(getattr(v, "value", v)) == 1 else v
    for b, lc in enumerate(coll):
        want = lc.fold(**{k: per(v, b) for k, v in kw.items()})
        _same_lc(got[b], want)
        assert isinstance(got[b], lk.FoldedLightCurve)


def test_fold_jd_warning_once_per_call(calls):
    coll = _coll()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        coll.fold(period=0.7, epoch_time=2458000.5)
    msgs = [str(x.message) for x in w if issubclass(x.category, LightkurveWarning)]
    assert msgs == ["`epoch_time` appears to be given in JD, however the light curve time uses BTJD "
                    "(i.e. JD - 2457000)."]
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        coll.fold(period=0.7, epoch_time=1500.5)
    assert not [x for x in w if issubclass(x.category, LightkurveWarning)]


def _raises_like_loop(coll, meth, kw):
    with pytest.raises(Exception) as single:
        for lc in coll:
            getattr(lc, meth)(**kw)
    with pytest.raises(type(single.value)) as batch:
        getattr(coll, meth)(**kw)
    assert str(batch.value) == str(single.value)


@pytest.mark.parametrize("kw", [dict(), dict(period=0.7, wrap_phase=0.9), dict(period=0.7, wrap_phase=-0.1),
                                dict(period=0.7, wrap_phase=1.5, normalize_phase=True)])
def test_fold_errors_like_loop(calls, kw):
    _raises_like_loop(_coll(), "fold", kw)


def test_fold_per_light_curve_length_checked(calls):
    with pytest.raises(ValueError, match="3 values for 5 light curves"):
        _coll().fold(period=[1.0, 2.0, 3.0])


def test_fold_nonpositive_period_goes_through_the_loop(calls):
    coll = _coll(3)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        got = coll.fold(period=[0.7, -0.7, 0.0])
        for b, p in enumerate((0.7, -0.7, 0.0)):
            _same_lc(got[b], coll[b].fold(period=p))
    assert calls == ["fold"]


def test_fold_empty_and_zero_length(calls):
    assert len(lk.LightCurveCollection([]).fold(period=1.0)) == 0
    coll = lk.LightCurveCollection([_coll(1)[0], lk.LightCurve(time=np.zeros(0), flux=np.zeros(0))])
    got = coll.fold(period=0.7, epoch_time=1500.0)
    for b, lc in enumerate(coll):
        _same_lc(got[b], lc.fold(period=0.7, epoch_time=1500.0))
    _raises_like_loop(coll, "fold", dict(period=0.7))                     # t[0] of a zero-length light curve


BIN_ARGS = [dict(), dict(time_bin_size=0.1), dict(time_bin_size=3 * u.hour), dict(time_bin_size=0.2, n_bins=500),
            dict(time_bin_size=0.2, time_bin_start=1499.0, time_bin_end=1502.0), dict(bins=17), dict(binsize=9),
            dict(bins=[0, 5, 10, 100, -1]), dict(aggregate_func=np.nanmedian, time_bin_size=0.05)]


@pytest.mark.parametrize("kw", BIN_ARGS, ids=range(len(BIN_ARGS)))
def test_bin_equals_loop(calls, kw):
    coll = _coll()
    got = coll.bin(**kw)
    assert calls == ["bin"]
    for b, lc in enumerate(coll):
        _same_lc(got[b], lc.bin(**kw))


def test_bin_of_folded_collection(calls):
    folded = _coll().fold(period=0.7, normalize_phase=True)
    got = folded.bin(time_bin_size=0.02)
    for b, lc in enumerate(folded):
        _same_lc(got[b], lc.bin(time_bin_size=0.02))
        assert str(got[b].time.unit) == str(u.dimensionless_unscaled)


@pytest.mark.parametrize("kw", [dict(bins=3, binsize=2), dict(bins=3, time_bin_size=0.1), dict(bins=2.5),
                                dict(bins="scott"), dict(bins="auto"), dict(aggregate_func=3),
                                dict(time_bin_size=-1.0), dict(bins=[0, 10, 100000]), dict(binsize=0),
                                dict(n_bins=0)])
def test_bin_errors_like_loop(calls, kw):
    _raises_like_loop(_coll(), "bin", kw)


def test_bin_aggregate_fallback(calls):
    coll = _coll()
    got = coll.bin(time_bin_size=0.1, aggregate_func=np.nanmax)
    assert calls == []
    for b, lc in enumerate(coll):
        _same_lc(got[b], lc.bin(time_bin_size=0.1, aggregate_func=np.nanmax))


def test_bin_descending_indices_go_through_the_loop(calls):
    coll = _coll(2)
    got = coll.bin(bins=[0, 50, 20, 100])
    for b, lc in enumerate(coll):
        _same_lc(got[b], lc.bin(bins=[0, 50, 20, 100]))
    assert calls == []


def test_bin_empty_and_zero_length(calls):
    assert len(lk.LightCurveCollection([]).bin()) == 0
    empty = lk.LightCurve(time=np.zeros(0), flux=np.zeros(0))
    coll = lk.LightCurveCollection([empty, _coll(1)[0]])
    got = coll.bin(time_bin_size=0.1)
    for b, lc in enumerate(coll):
        _same_lc(got[b], lc.bin(time_bin_size=0.1))
    assert got[0] is not empty


def test_bin_signed_zero_and_nan_ends():
    """The first and last stably sorted time, as the edges use them: -0.0 / +0.0 in their order, NaN last."""
    from lightkurve_b200.collections import _sorted_first_last
    ts = [np.array([0.0, -0.0, -1.0, 0.0]), np.array([-0.0, 0.0, 3.0]), np.array([2.0, np.nan, 1.0]),
          np.array([np.nan, np.nan]), np.array([-0.0, 0.0])]
    first, last = _sorted_first_last(ts)
    for b, t in enumerate(ts):
        s = np.sort(t, kind="stable")
        assert np.array_equal(np.array([first[b], last[b]]).view(np.int64) if not np.isnan(s[0]) else
                              np.isnan([first[b], last[b]]), np.array([s[0], s[-1]]).view(np.int64)
                              if not np.isnan(s[0]) else np.isnan([s[0], s[-1]]))
    assert np.isnan(last[2]) and first[2] == 1.0
