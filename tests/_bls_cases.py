"""Box Least Squares fixtures shared by tests/test_bls_emulated.py (CPU emulator) and tests/test_gpu_bls_paths.py (H100).

Exact-arithmetic ("dyadic") fixtures: times are multiples of 2^-10 d, fluxes small integers times 2^-6 and flux errors
None or powers of two.  Every sum either side forms (weighted fluxes, weights, their prefix sums and totals) is then
exact in fp64, so the order of summation cannot matter and the kernel must equal oracle/bls_c.c bit for bit, ties
included.  The fixtures contain real ties: constant flux (every box ties at 0), a few cadences whose empty bins make
several boxes cover the same samples, and two identical transits."""
import numpy as np

from oracle import bls as obls

FIELDS = obls.RESULT_FIELDS
DUR = np.array([0.0625, 0.125, 0.25])
T0 = 1325.0


def dyadic_times(rng, n, span, unique=True):
    """n times on the 2^-10 d grid within [T0, T0 + span), sorted."""
    cells = int(span * 1024)
    k = rng.choice(cells, n, replace=False) if unique else rng.integers(0, cells, n)
    return T0 + np.sort(k) / 1024.0


def dyadic_flux(rng, t, period=None, duration=0.125, depth=24, epoch=0.5):
    """Small integers times 2^-6, with a box of `depth` / 64 at `period` if given."""
    y = rng.integers(-6, 7, len(t)).astype(np.float64)
    if period is not None:
        ph = (t - T0 - epoch) % period
        y[ph < duration] -= depth
    return y / 64.0


def pow2_errors(rng, n):
    return 2.0 ** rng.integers(-4, -1, n).astype(np.float64)


def matrix_batch(scale=1, seed=0):
    """Light curves of the oversample x objective x path matrix: (name, t, y, dy).  scale multiplies the cadence
    counts and spans (1 on the emulator)."""
    rng = np.random.default_rng(seed)
    out = []
    t = dyadic_times(rng, 120 * scale, 16.0 * scale)
    out.append(("sparse", t, dyadic_flux(rng, t, 2.25), None))
    t = T0 + np.arange(640 * scale) / 128.0                      # 11.25-min cadence
    y = rng.integers(-3, 4, len(t)).astype(np.float64)
    dy = pow2_errors(rng, len(t))
    for a in (1.0, 3.0):                                         # two identical transits
        w = (t - T0 >= a) & (t - T0 < a + 0.125)
        y[w] = -20.0
        dy[w] = 0.125
    out.append(("dense_twin_transits", t, y / 64.0, dy))
    t = dyadic_times(rng, 200 * scale, 12.0 * scale)
    out.append(("constant", t, np.full(len(t), 5.0 / 64.0), np.full(len(t), 0.25)))
    t = dyadic_times(rng, 9, 10.0)
    out.append(("nine_cadences", t, dyadic_flux(rng, t), None))
    t = dyadic_times(rng, 150 * scale, 14.0 * scale)
    out.append(("unsorted", rng.permutation(t), rng.permutation(dyadic_flux(rng, t, 1.75)), None))
    return out


def matrix_grid(n=24, lo=0.4, hi=4.0):
    return np.linspace(lo, hi, n)


def exact_ties(t, y, dy, period, duration, oversample, objective):
    """Per period: how many boxes attain the oracle's best objective exactly (numpy restatement of bls.c, exact on
    dyadic inputs).  A value > 1 is a real tie that only the first-maximum rule separates."""
    trel, yc, ivar, _ = obls._prepare(t, y, dy)
    duration = np.atleast_1d(np.asarray(duration, dtype=np.float64))
    bd = duration.min() / float(oversample)
    wy = yc * ivar
    sum_y, sum_ivar = wy.sum(), ivar.sum()
    eps = np.finfo(np.float64).eps
    out = np.zeros(len(period), dtype=np.int64)
    for p, per in enumerate(period):
        n_bins = int(np.ceil(per / bd)) + oversample
        ind = obls.bin_index(trel, 0.0, per, bd)
        my = np.zeros(n_bins + 1)
        mi = np.zeros(n_bins + 1)
        np.add.at(my, ind, wy)
        np.add.at(mi, ind, ivar)
        lo = n_bins - oversample
        my[lo:lo + oversample] = my[1:oversample + 1].copy()
        mi[lo:lo + oversample] = mi[1:oversample + 1].copy()
        my, mi = np.cumsum(my), np.cumsum(mi)
        objs = []
        for d in duration:
            dur = int(np.round(d / bd))
            n_max = n_bins - dur
            y_in = my[dur:dur + n_max + 1] - my[:n_max + 1]
            i_in = mi[dur:dur + n_max + 1] - mi[:n_max + 1]
            y_out, i_out = sum_y - y_in, sum_ivar - i_in
            ok = ~((i_in < eps) | (i_out < eps))
            with np.errstate(divide="ignore", invalid="ignore"):
                yi, yo = y_in / i_in, y_out / i_out
                if objective == "snr":
                    o = (yo - yi) / np.sqrt(1.0 / i_in + 1.0 / i_out)
                else:
                    o = 0.5 * i_in * (yo - yi) * (yo - yi)
            objs.append(np.where(ok & (yo >= yi), o, -np.inf))
        objs = np.concatenate(objs)
        best = objs.max()
        out[p] = 0 if best == -np.inf else int((objs == best).sum())
    return out


def bin_multiple_periods(oversample, duration=DUR):
    """Periods that are exact integer multiples k * bin_duration, all longer than the longest duration."""
    bd = np.min(duration) / oversample
    k0 = int(np.ceil(np.max(duration) / bd)) + 1
    return np.array([k * bd for k in (k0, 2 * k0, 23 * k0 + 3)])


def assert_bls_close(got, ref, t, y, dy, period, duration, oversample, objective="likelihood", max_tied_frac=0.02):
    """The tie rule and tolerances of test_gpu_engine.assert_bls_close for inputs whose sums round (the kernel adds in
    another order than the C loop), with the tie check evaluated at `oversample`.  Returns the tie-broken count."""
    same = np.all(got["bins"] == ref["bins"], axis=1)
    for p_idx in np.flatnonzero(~same):
        n, dur = got["bins"][p_idx]
        o = obls.objective_at(t, y, dy, period[p_idx], duration, int(n), int(dur), oversample=oversample,
                              objective=objective)
        assert abs(o - ref["power"][p_idx]) <= 1e-10 * abs(ref["power"][p_idx]), "period %d not tied" % p_idx
    assert (~same).mean() <= max_tied_frac, "too many tie-broken periods: %d" % (~same).sum()
    for k in ("power", "depth", "depth_err", "depth_snr", "log_likelihood"):
        np.testing.assert_allclose(got[k], ref[k], rtol=1e-9, atol=1e-12, err_msg=k)
    for k in ("duration", "transit_time"):
        np.testing.assert_allclose(got[k][same], ref[k][same], rtol=1e-12, atol=1e-9, err_msg=k)
    return int((~same).sum())


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.int64 if a.dtype == np.float64 else a.dtype)


def assert_exact(got, t, y, dy, period, duration, oversample, objective, what="", count_ties=True):
    """Bins and all seven outputs bitwise equal to bls_power_c; returns (periods with an exact tie, boxes tied),
    or (0, 0) without count_ties."""
    ref = obls.bls_power_c(t, y, dy, period, duration, oversample=oversample, objective=objective, return_bins=True)
    np.testing.assert_array_equal(got["bins"], ref["bins"], err_msg="%s bins" % what)
    for k in FIELDS:
        g, r = bits(got[k]), bits(ref[k])
        bad = np.flatnonzero(g != r)
        assert len(bad) == 0, "%s %s differs at periods %s: %r vs %r" % (what, k, bad[:5], got[k][bad[:3]],
                                                                         ref[k][bad[:3]])
    if not count_ties:
        return 0, 0
    ties = exact_ties(t, y, dy, period, duration, oversample, objective)
    return int((ties > 1).sum()), int(ties[ties > 1].sum())
