"""K13 on the GPU: LightCurveCollection.fold / bin against the per-light-curve loop on 300 config-5 light curves plus
the edge cases of the emulated tests and one light curve past both shared-memory caps.  fold is bitwise equal in
phase, flux, flux_err, time_original, columns and meta; bin and fold-then-bin are equal within 4 n 2^-52 max|x|, n the light
curve's length (exact NaN pattern and centres); repeated and permuted runs are bitwise equal; device mode is bitwise
equal to host mode; bad arguments return LKB_E_ARG."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -52


@pytest.fixture(scope="module")
def coll():
    import lightkurve_b200 as lk
    from bench_bls_ragged import make_c5_bls
    times, fluxes, errs = make_c5_bls(B=300)
    lcs = [lk.LightCurve(time=t, flux=f, flux_err=e, cadenceno=np.arange(len(t))) for t, f, e in
           zip(times, fluxes, errs)]
    rng = np.random.default_rng(9)
    n = 20000                                                       # past both shared-memory caps
    t = rng.permutation(2000.0 + np.arange(n) * 0.0013889)
    f = 1 + 1e-3 * rng.standard_normal(n)
    f[::97] = np.nan
    f[5] = np.inf
    lcs.append(lk.LightCurve(time=t, flux=f, flux_err=np.full(n, np.nan)))
    t2 = np.repeat(np.arange(300) * 0.25, 2)                        # duplicates, a period dividing the step
    lcs.append(lk.LightCurve(time=t2, flux=rng.standard_normal(len(t2)), flux_err=np.where(t2 < 20, np.nan, 0.1)))
    lcs.append(lk.LightCurve(time=np.array([3.0]), flux=np.array([1.0])))
    lcs.append(lk.LightCurve(time=np.array([3.5, 3.0]), flux=np.array([1.0, 2.0])))
    return lk.LightCurveCollection(lcs)


def _bits(x):
    return np.asarray(x, np.float64).view(np.int64)


def _same_fold(a, b):
    for k in ("time", "flux", "flux_err", "time_original"):
        assert np.array_equal(_bits(getattr(a, k).value), _bits(getattr(b, k).value)), k
    for k in b._columns:
        assert np.array_equal(a._columns[k], b._columns[k])
    for k, v in b.meta.items():
        w = a.meta[k]
        assert (w is None and v is None) or np.array_equal(np.asarray(getattr(w, "value", w)),
                                                           np.asarray(getattr(v, "value", v))), k


def _close_bin(a, b, n):
    """Centres bitwise, NaN pattern exact, values within 4 n 2^-52 max|x| (n >= any bin's count)."""
    assert np.array_equal(_bits(a.time.value), _bits(b.time.value))
    for k in ("flux", "flux_err"):
        x, y = np.asarray(getattr(a, k).value), np.asarray(getattr(b, k).value)
        assert np.array_equal(np.isnan(x), np.isnan(y)), k
        m = ~np.isnan(y)
        tol = 4 * n * EPS * np.abs(y[m]).max(initial=0.0)
        assert np.all((x[m] == y[m]) | (np.abs(x[m] - y[m]) <= tol)), k


@pytest.mark.parametrize("kw", [dict(period=1.37), dict(period=0.25, wrap_phase=0.25, epoch_time=0.0),
                                dict(period=2.1, epoch_phase=-0.3, normalize_phase=True)])
def test_fold_equals_loop_bitwise(coll, kw):
    got = coll.fold(**kw)
    for b, lc in enumerate(coll):
        _same_fold(got[b], lc.fold(**kw))
    again = coll.fold(**kw)
    for b in range(len(coll)):
        _same_fold(again[b], got[b])


def test_fold_per_light_curve_periods(coll):
    per = [0.5 + 0.01 * b for b in range(len(coll))]
    got = coll.fold(period=per, epoch_time=[float(np.min(lc.time.value)) for lc in coll])
    for b, lc in enumerate(coll):
        _same_fold(got[b], lc.fold(period=per[b], epoch_time=float(np.min(lc.time.value))))


@pytest.mark.parametrize("agg", [np.nanmean, np.nanmedian], ids=["nanmean", "nanmedian"])
@pytest.mark.parametrize("kw", [dict(time_bin_size=10 / 1440.0), dict(time_bin_size=0.3, n_bins=400), dict(bins=50),
                                dict(binsize=13), dict(bins=[0, 1, 2, 50, -1])])
def test_bin_equals_loop(coll, kw, agg):
    if np.size(kw.get("bins", 0)) > 1:          # edge index 50: not on the one- and two-cadence light curves
        coll = coll[:-2]
    got = coll.bin(aggregate_func=agg, **kw)
    for b, lc in enumerate(coll):
        _close_bin(got[b], lc.bin(aggregate_func=agg, **kw), len(lc))


@pytest.mark.parametrize("agg", [np.nanmean, np.nanmedian], ids=["nanmean", "nanmedian"])
def test_fold_then_bin_equals_loop(coll, agg):
    got = coll.fold(period=1.37, epoch_time=1.0).bin(time_bin_size=0.02, aggregate_func=agg)
    for b, lc in enumerate(coll):
        _close_bin(got[b], lc.fold(period=1.37, epoch_time=1.0).bin(time_bin_size=0.02, aggregate_func=agg), len(lc))


def test_repeat_and_permutation_bitwise(coll):
    import lightkurve_b200 as lk
    kw = dict(time_bin_size=0.05, aggregate_func=np.nanmedian)
    base = coll.bin(**kw)
    perm = np.random.default_rng(1).permutation(len(coll))
    shuffled = lk.LightCurveCollection([coll[int(p)] for p in perm]).bin(**kw)
    again = coll.bin(**kw)
    for j, p in enumerate(perm):
        for k in ("time", "flux", "flux_err"):
            assert np.array_equal(_bits(getattr(shuffled[j], k).value), _bits(getattr(base[int(p)], k).value))
            assert np.array_equal(_bits(getattr(again[int(p)], k).value), _bits(getattr(base[int(p)], k).value))


def test_device_mode_equals_host_mode(coll):
    import torch
    from lightkurve_b200 import engine
    lcs = list(coll)[:40] + list(coll)[-4:]
    times = [np.asarray(lc.time.value, np.float64) for lc in lcs]
    fl = [np.asarray(lc.flux.value, np.float64) for lc in lcs]
    fe = [np.asarray(lc.flux_err.value, np.float64) for lc in lcs]
    off = np.zeros(len(lcs) + 1, np.int64)
    off[1:] = np.cumsum([len(t) for t in times])
    cat = lambda xs, dt=np.float64: torch.from_numpy(np.concatenate(xs).astype(dt)).cuda()
    B = len(lcs)
    pars = dict(t0=np.array([t[0] for t in times]), shift=np.zeros(B), period=np.full(B, 0.9), wrap=np.full(B, 0.45))
    h = engine.fold(times, **pars)
    d = engine.fold(cat(times), offsets=off, **pars)
    torch.cuda.synchronize()
    assert np.array_equal(_bits(np.concatenate(h["phase"])), _bits(d["phase"].cpu().numpy()))
    assert np.array_equal(np.concatenate(h["perm"]), d["perm"].cpu().numpy())
    starts = [np.arange(0, len(t), 7) for t in times]
    ends = [np.append(s[1:], len(t) - 1) for s, t in zip(starts, times)]
    boff = np.zeros(B + 1, np.int64)
    boff[1:] = np.cumsum([len(s) for s in starts])
    for agg in ("nanmean", "nanmedian"):
        h = engine.bin(times, fl, fe, starts, ends, index_edges=True, aggregate=agg)
        d = engine.bin(cat(times), cat(fl), cat(fe), cat(starts, np.int32), cat(ends, np.int32), index_edges=True,
                       aggregate=agg, offsets=off, bin_offsets=boff)
        for k in ("time", "flux", "flux_err"):
            assert np.array_equal(_bits(np.concatenate(h[k])), _bits(d[k].cpu().numpy())), (agg, k)
        assert np.array_equal(np.concatenate(h["count"]), d["count"].cpu().numpy())


def test_bad_arguments_return_e_arg():
    """LKB_E_ARG is raised as ValueError with the library's message."""
    from lightkurve_b200 import engine
    t = [np.arange(10.0), np.arange(5.0)]
    with pytest.raises(ValueError, match="light curve 1 has a non-positive period"):
        engine.fold(t, [0.0, 0.0], [0.0, 0.0], [1.0, 0.0], [0.5, 0.0])
    f = [np.ones(10), np.ones(5)]
    with pytest.raises(ValueError, match="light curve 1 has a bin edge index outside"):
        engine.bin(t, f, None, [np.array([0, 5]), np.array([0, 7])], [np.array([5, 9]), np.array([2, 4])],
                   index_edges=True)
    with pytest.raises(ValueError, match="bin starts of light curve 1 do not ascend"):
        engine.bin(t, f, None, [np.array([0.0, 5.0]), np.array([3.0, 1.0])], [np.array([5.0, 9.0]),
                                                                               np.array([2.0, 4.0])])
