"""Light curves for LightCurveCollection.find_transit_candidates and the single-curve loop it must equal.

make_lcs: config-5-like light curves (TESS 2-min cadence, 1 500 - 4 000 cadences over ~27 days, +-20 s jitter, gaps)
with 0 - 3 injected box transits of different periods, plus:
  - NaN flux at scattered cadences;
  - flux_err NaN only inside the deepest transit (round 0 searches with unit weights, the next rounds with flux_err);
  - light curves without flux_err (unit weights in every round).
"""
import numpy as np

from lightkurve_b200 import LightCurve


def make_lcs(n=120, seed=2024):
    rng = np.random.default_rng(seed)
    lcs, truth = [], []
    for b in range(n):
        m = int(rng.integers(1500, 4000))
        t = 2000.0 + np.sort(rng.uniform(0, 27.0, m))
        t = t[(t < 2013.0) | (t > 2014.0)]                      # the mid-sector gap
        sig = 10 ** rng.uniform(-4, -3)
        y = 1 + sig * rng.standard_normal(len(t))
        planets = []
        for k in range(int(rng.integers(0, 4))):
            per = rng.uniform(1.0, 8.0) * (1.7 ** k)
            per = min(per, 8.5)
            dur, dep, t0 = rng.uniform(0.06, 0.25), 10 ** rng.uniform(-2.7, -1.7), 2000.0 + rng.uniform(0, per)
            y[np.abs((t - t0 + 0.5 * per) % per - 0.5 * per) < 0.5 * dur] -= dep
            planets.append((per, dur, dep, t0))
        e = np.full(len(t), sig)
        if b % 7 == 3:
            y[rng.choice(len(t), 20, replace=False)] = np.nan
        if b % 5 == 2 and planets:
            per, dur, dep, t0 = max(planets, key=lambda p: p[2])
            e[np.abs((t - t0 + 0.5 * per) % per - 0.5 * per) < 0.2 * dur] = np.nan
        lcs.append(LightCurve(time=t, flux=y, flux_err=None if b % 6 == 5 else e))
        truth.append(planets)
    return lcs, truth


def loop(lc, n_candidates, return_stats=False, **kw):
    """The contract of find_transit_candidates for one light curve: (candidate rows [n, 7], masked_in, stats, pgs)."""
    lc = lc.remove_nans()
    masked = np.full(len(lc), -1, np.int8)
    idx = np.arange(len(lc))
    rows, stats, pgs = [], [], []
    for r in range(n_candidates):
        pg = lc.to_periodogram("bls", **kw)
        k = np.nanargmax(pg.power.value)
        P, D, T0 = pg.period_at_max_power, pg.duration_at_max_power, pg.transit_time_at_max_power
        rows.append([P.value, D.value, T0.value, pg.depth[k].value, pg._BLS_result["depth_err"][k], pg.snr[k].value,
                     pg.power[k].value])
        if return_stats:
            stats.append(pg.compute_stats(P, D, T0))
            pgs.append((pg, float(P.value), float(D.value), float(T0.value)))
        m = pg.get_transit_mask(period=P, duration=D, transit_time=T0)
        masked[idx[m]] = r
        idx = idx[~m]
        lc = lc[~m]
    return np.array(rows), masked, stats, pgs
