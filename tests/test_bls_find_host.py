"""The shim of LightCurveCollection.find_transit_candidates on a numpy stand-in for engine.bls_find_candidates, which
runs the rounds light curve by light curve over the oracle BLS (oracle/bls.py, through tests/_oracle_engine.py) and
the host mask rule: the result layout and units, return_stats, keyword validation, warnings and errors naming the
light curve and round; and BoxLeastSquaresPeriodogram._grid, the grid helper the driver shares with _prepare, against
_prepare and tools/bench_bls_ragged.default_grid."""
import logging
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import _oracle_engine as OE  # noqa: E402
from test_bls_stats_host import numpy_bls_stats  # noqa: E402

from lightkurve_b200 import LightCurve, LightCurveCollection, engine  # noqa: E402
from lightkurve_b200.periodogram import BoxLeastSquaresPeriodogram as BLS  # noqa: E402


def stand_in_find(times, fluxes, flux_errs, grid, n_candidates, shared_grid=False, return_stats=False):
    """engine.bls_find_candidates restated: per light curve, per round, the oracle search and the host mask."""
    B = len(times)
    out = {k: np.full((B, n_candidates), np.nan) for k in engine.BLS_CANDIDATE_FIELDS}
    out["masked_in"], per_round = [], [[] for _ in range(n_candidates)]
    for b in range(B):
        t, y, dy = (np.asarray(a, dtype=np.float64) for a in (times[b], fluxes[b], flux_errs[b]))
        idx = np.arange(len(t))
        masked = np.full(len(t), -1, np.int8)
        for r in range(n_candidates):
            try:
                g = grid(b, r, np.min(t) if len(t) else None, np.max(t) if len(t) else None,
                         np.median(np.diff(t)) if len(t) > 1 else np.nan)
                w = dy if np.isfinite(dy).all() else np.ones(len(t))
                res = OE.bls_power([t], [y], [w], g["period"], g["duration"], oversample=g["oversample"],
                                   objective=g["objective"])
                k = np.nanargmax(res["power"][0])
            except Exception as e:
                raise engine._named_error(e, b, r) from e
            cand = [1.0 / (1.0 / g["period"][k])] + [res[f][0][k] for f in engine.BLS_CANDIDATE_FIELDS[1:]]
            for f, v in zip(engine.BLS_CANDIDATE_FIELDS, cand):
                out[f][b, r] = v
            st = numpy_bls_stats([t], [y], [w], cand[0], cand[1], cand[2], return_mask=True)
            st["tstart"] = np.array([t[0]])
            per_round[r].append(st)
            s = st["stats"][0]
            n, n_in, y_in, y_out = len(t), int(s[14]), s[12], s[13]
            med = y_out if 2 * n_in < n else (y_in if 2 * n_in > n else np.mean([y_in, y_out]))
            m = np.where(st["in_transit"], y_in != med, y_out != med)
            masked[idx[m]] = r
            idx, t, y, dy = idx[~m], t[~m], y[~m], dy[~m]
        out["masked_in"].append(masked)
    if return_stats:
        out["stats"] = [_stack(rs) for rs in per_round]
    return out


def _stack(rs):
    """One host-mode bls_stats result of B light curves from B one-light-curve results."""
    toff = np.r_[0, np.cumsum([r["transit_offsets"][-1] for r in rs])]
    return dict(stats=np.concatenate([r["stats"] for r in rs]), transit_n=np.concatenate([r["transit_n"] for r in rs]),
                transit_first=np.concatenate([r["transit_first"] for r in rs]), transit_offsets=toff,
                per_transit_count=np.concatenate([r["per_transit_count"] for r in rs]),
                per_transit_log_likelihood=np.concatenate([r["per_transit_log_likelihood"] for r in rs]),
                tstart=np.concatenate([r["tstart"] for r in rs]))


@pytest.fixture
def stand_in(monkeypatch):
    numpy_bls_stats.calls = []
    monkeypatch.setattr(engine, "bls_find_candidates", stand_in_find)


def _lcs(n=3, seed=4):
    rng = np.random.default_rng(seed)
    out = []
    for b in range(n):
        t = 500.0 + np.sort(rng.uniform(0, 10, 600))
        y = 1 + 1e-4 * rng.normal(size=len(t))
        for per, dep in ((1.3 + b, 0.01), (2.9 + b, 0.006)):
            y[np.abs((t - 500.2 + 0.5 * per) % per - 0.5 * per) < 0.05] -= dep
        y[5] = np.nan
        out.append(LightCurve(time=t, flux=y, flux_err=np.full(len(t), 1e-4)))
    return out


def test_layout_units_and_stats(stand_in):
    lcs = _lcs()
    res = LightCurveCollection(lcs).find_transit_candidates(n_candidates=2, return_stats=True, duration=[0.05, 0.1])
    for k in engine.BLS_CANDIDATE_FIELDS:
        assert res[k].shape == (3, 2) and res[k].dtype == np.float64
    for b, lc in enumerate(lcs):
        assert len(res["masked_in"][b]) == len(lc.remove_nans()) and res["masked_in"][b].dtype == np.int8
        assert set(np.unique(res["masked_in"][b])) <= {-1, 0, 1}
        assert len(res["stats"][b]) == 2
        for r, s in enumerate(res["stats"][b]):
            assert s["depth"][0].unit == lc.flux.unit
            assert s["transit_times"].format == lc.time.format
            assert len(s["transit_times"]) == len(s["per_transit_count"])
        assert min(abs(res["period"][b, 0] - p) for p in (1.3 + b, 2.9 + b)) < 0.05, res["period"][b]


def test_keyword_errors_name_light_curve_and_round(stand_in):
    coll = LightCurveCollection(_lcs(2))
    with pytest.raises(TypeError, match="light curve 0, round 0: unexpected keyword"):
        coll.find_transit_candidates(n_candidates=1, bogus=3)
    with pytest.raises(ValueError, match="light curve 0, round 0: .*time_unit"):
        coll.find_transit_candidates(n_candidates=1, time_unit="week")
    with pytest.raises(ValueError, match="round 0: The maximum transit duration"):
        coll.find_transit_candidates(n_candidates=1, period=[1.0, 1.5], duration=[2.0])
    with pytest.raises(ValueError, match="n_candidates"):
        coll.find_transit_candidates(n_candidates=0)
    t = np.arange(10.0)
    t[3] = np.nan
    with pytest.raises(ValueError, match="light curve 1 has non-finite times"):
        LightCurveCollection([_lcs(1)[0], LightCurve(time=t, flux=np.ones(10))]).find_transit_candidates()


def test_empty_collection():
    res = LightCurveCollection([]).find_transit_candidates(n_candidates=2, return_stats=True)
    assert res["period"].shape == (0, 2) and res["masked_in"] == [] and res["stats"] == []


def test_npoints_warning_each_round(stand_in, caplog):
    with caplog.at_level(logging.WARNING):
        LightCurveCollection(_lcs(1)).find_transit_candidates(n_candidates=2, frequency_factor=0.05,
                                                              duration=[0.05, 0.1])
    assert sum("Periodogram is likely to be large" in r.getMessage() for r in caplog.records) == 2


def _varied_times():
    rng = np.random.default_rng(9)
    out = [np.sort(rng.uniform(0, 27, 3000)), 1000 + np.arange(2000) * 0.0208, np.arange(6) * 2.0,
           np.sort(rng.uniform(0, 12, 1001))]
    t = 300 + np.arange(1500) * 0.02
    out.append(np.r_[t[:700], t[900:]])
    return out


@pytest.mark.parametrize("kw", [dict(), dict(frequency_factor=3, duration=[0.1, 0.2]), dict(minimum_period=1.0),
                                dict(maximum_period=4.0, time_unit="h"), dict(period=[1.0, 2.0, 3.5])])
def test_grid_helper_equals_prepare(kw):
    for t in _varied_times():
        lc = LightCurve(time=t, flux=np.ones(len(t)))
        try:
            p = BLS._prepare(lc, **dict(kw))
        except ValueError as e:
            with pytest.raises(ValueError, match=str(e)[:30]):
                BLS._grid(np.min(t), np.max(t), np.median(np.diff(t)), **dict(kw))
            continue
        g = BLS._grid(np.min(t), np.max(t), np.median(np.diff(t)), **dict(kw))
        np.testing.assert_array_equal(g["period"], p["period"])
        for k in ("duration", "objective", "oversample", "time_unit"):
            assert np.array_equal(g[k], p[k])


def test_grid_helper_equals_bench_default_grid():
    from tools.bench_bls_ragged import default_grid
    for t in _varied_times()[:2] + _varied_times()[3:]:
        np.testing.assert_array_equal(BLS._grid(np.min(t), np.max(t), np.median(np.diff(t)))["period"],
                                      default_grid(t))


def test_grid_helper_empty_light_curve():
    with pytest.raises(ValueError, match="zero-size array"):
        BLS._prepare(LightCurve(time=np.zeros(0), flux=np.zeros(0)))
    with pytest.raises(ValueError, match="zero-size array"):
        BLS._grid(None, None, np.nan)
    with pytest.raises(ValueError, match="illegal nan"):        # keyword errors come first, as in _prepare
        BLS._grid(None, None, np.nan, duration=[np.nan])
