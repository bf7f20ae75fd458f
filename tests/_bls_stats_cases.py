"""Light curves and candidates for the batched BLS follow-ups (compute_stats_batch / get_transit_mask_batch), the
comparison with the host compute_stats / get_transit_mask at the K10 tolerances, and a periodogram factory that needs
no GPU.  Shared by the emulator, host and GPU tests."""
import numpy as np

from lightkurve_b200 import units as u
from lightkurve_b200.periodogram import BoxLeastSquaresPeriodogram
from lightkurve_b200.units import Quantity, Time


def make_pg(t, y, dy=None, period=1.0, duration=0.1, transit_time=0.0):
    """A BoxLeastSquaresPeriodogram over (t, y, dy) whose maximum power sits at (period, duration, transit_time)."""
    per = np.array([0.8, 1.0, 1.25]) * period
    pg = BoxLeastSquaresPeriodogram(
        frequency=1.0 / Quantity(per, u.day), power=Quantity(np.array([0.1, 1.0, 0.2]), u.dimensionless_unscaled),
        default_view="period", transit_time=Time(np.full(3, float(transit_time)), "btjd", "tdb"),
        duration=Quantity(np.full(3, float(duration)), u.day), depth=Quantity(np.zeros(3), u.electron / u.s),
        snr=Quantity(np.zeros(3), u.dimensionless_unscaled), time=Time(np.asarray(t, dtype=float), "btjd", "tdb"),
        flux=Quantity(np.asarray(y, dtype=float), u.electron / u.s), time_unit="day")
    pg._dy = None if dy is None else np.asarray(dy, dtype=float)
    return pg


def box(t, period, duration, t0, depth):
    return np.where(np.abs((t - t0 + 0.5 * period) % period - 0.5 * period) < 0.5 * duration, -depth, 0.0)


def cases(seed=0):
    """(name, t, y, dy, period, duration, transit_time): every edge the kernel has to get right."""
    rng = np.random.default_rng(seed)
    out = []
    t = 1325.0 + np.arange(0, 27.0, 2.0 / 1440)
    t = t[rng.random(len(t)) < 0.97]
    y = 1 + 5e-4 * rng.standard_normal(len(t)) + box(t, 3.1, 0.12, 1326.7, 3e-3)
    out.append(("sorted_dy", t, y, np.full(len(t), 5e-4) * rng.uniform(0.8, 1.2, len(t)), 3.1, 0.12, 1326.7))
    t = 1400.0 + np.arange(0, 20.0, 10.0 / 1440)
    y = 1 + 4e-4 * rng.standard_normal(len(t)) + box(t, 0.4, 0.05, 1400.13, 2e-3)
    p = rng.permutation(len(t))
    out.append(("unsorted_no_dy", t[p], y[p], None, 0.4, 0.05, 1400.13))
    out.append(("unsorted_dy", t[p], y[p], np.full(len(t), 4e-4), 0.4, 0.05, 1400.13))
    t = 1500.0 + np.arange(0, 30, 0.02)
    t = t[np.abs((t - 1501.0 + 1.5) % 3.0 - 1.5) > 0.3]           # every transit falls in a gap
    y = 1 + 1e-3 * rng.standard_normal(len(t))
    out.append(("no_transit_cadence", t, y, np.full(len(t), 1e-3), 3.0, 0.5, 1501.0))
    t = 1600.0 + np.arange(0, 12.0, 0.01)
    y = 1 + 1e-3 * rng.standard_normal(len(t)) + box(t, 1.0, 0.8, 1600.2, 4e-3)
    out.append(("majority_in_transit", t, y, None, 1.0, 0.8, 1600.2))
    t = (np.arange(160) + 0.5) / 8.0           # phases (j + 1/2) / 8: exactly 4 of every 8 within 0.25 of a transit
    y = 1 + 1e-3 * rng.standard_normal(len(t)) + box(t, 1.0, 0.5, 0.0, 3e-3)
    out.append(("exactly_half", t, y, np.full(len(t), 1e-3), 1.0, 0.5, 0.0))
    t = 1700.0 + np.arange(0, 15.0, 0.02)
    y = 1 + 1e-3 * rng.standard_normal(len(t)) + box(t, 2.3, 0.2, 1700.9, 3e-3)
    out.append(("transit_time_after_data", t, y, None, 2.3, 0.2, 1700.9 + 40 * 2.3))
    out.append(("transit_time_before_data", t, y, np.full(len(t), 1e-3), 2.3, 0.2, 1700.9 - 55 * 2.3))
    return out


def kepler_case(seed=1):
    """A Kepler-length light curve (65 000 long cadences, about 1 330 days) and a 0.4-day candidate: > 3 000 transits."""
    rng = np.random.default_rng(seed)
    t = 131.5 + np.arange(65000) * 0.0204336
    y = 1 + 2e-4 * rng.standard_normal(len(t)) + box(t, 0.4, 0.05, 131.61, 4e-4)
    return ("kepler_3000_transits", t, y, np.full(len(t), 2e-4), 0.4, 0.05, 131.61)


def singular_cases():
    """Sine fits numpy cannot solve: one cadence, and time stamps that all equal t[0] (the sine column is 0)."""
    return [("one_cadence", np.array([1234.5]), np.array([1.0]), None, 2.0, 0.1, 1234.5),
            ("all_equal_times", np.full(50, 1234.5), 1 + 1e-3 * np.arange(50.0), np.full(50, 1e-3), 2.0, 0.1, 1234.4)]


def pgs_of(cs):
    return [make_pg(t, y, dy, p, d, tt) for _, t, y, dy, p, d, tt in cs]


def _ll_scale(pg, period, duration, transit_time):
    """sum ivar (y - y_out)^2 of compute_stats: the scale of its log-likelihoods."""
    t = np.asarray(pg.time.value, dtype=float)
    y = np.asarray(pg.flux.value, dtype=float)
    ivar = np.ones_like(y) if pg._dy is None else 1.0 / pg._dy ** 2
    t0 = t[0]
    hp = 0.5 * period
    m_in = np.abs(((t - t0) - (transit_time - t0) + hp) % period - hp) < 0.5 * duration
    y_out = np.sum(y[~m_in] * ivar[~m_in]) / np.sum(ivar[~m_in]) if np.any(~m_in) else 0.0
    return np.sum(ivar * (y - y_out) ** 2)


def assert_stats_match(got, ref, pg, period, duration, transit_time, name=""):
    """The K10 contract: exact transit times and counts; depths within 1e-11 max|y|; errors and the harmonic amplitude
    rtol 1e-10; log-likelihoods within 1e-10 sum ivar (y - y_out)^2.  The amplitude also gets an absolute floor of
    1e-12 max|y|: its sine and cosine coefficients are differences of sums of y sin and y cos, whose rounding is of
    order eps max|y| whatever the amplitude (a config-5 light curve at flux 1 with a 2.5e-6 amplitude differs by
    6.4e-16, 2.5e-10 relative)."""
    assert got.keys() == ref.keys(), name
    np.testing.assert_array_equal(np.asarray(got["transit_times"].value), np.asarray(ref["transit_times"].value),
                                  err_msg=name)
    assert got["transit_times"].format == ref["transit_times"].format
    np.testing.assert_array_equal(got["per_transit_count"], ref["per_transit_count"], err_msg=name)
    assert got["per_transit_count"].dtype == ref["per_transit_count"].dtype, name
    ymax = np.max(np.abs(np.asarray(pg.flux.value)))
    for k in ("depth", "depth_phased", "depth_half", "depth_odd", "depth_even"):
        assert got[k][0].unit == ref[k][0].unit
        np.testing.assert_allclose(got[k][0].value, ref[k][0].value, rtol=0, atol=1e-11 * ymax, err_msg=name + k)
        np.testing.assert_allclose(got[k][1].value, ref[k][1].value, rtol=1e-10, err_msg=name + k + " err")
    np.testing.assert_allclose(got["harmonic_amplitude"].value, ref["harmonic_amplitude"].value, rtol=1e-10,
                               atol=1e-12 * ymax, err_msg=name)
    scale = _ll_scale(pg, period, duration, transit_time)
    np.testing.assert_allclose(got["harmonic_delta_log_likelihood"], ref["harmonic_delta_log_likelihood"], rtol=0,
                               atol=1e-10 * scale, err_msg=name)
    np.testing.assert_allclose(got["per_transit_log_likelihood"], ref["per_transit_log_likelihood"], rtol=0,
                               atol=1e-10 * scale, err_msg=name)


def check_batch(cs, stats_batch, mask_batch):
    """compute_stats_batch / get_transit_mask_batch on the cases against the host loop."""
    pgs = pgs_of(cs)
    got = stats_batch(pgs)
    masks = mask_batch(pgs)
    for (name, _, _, _, p, d, tt), pg, g, m in zip(cs, pgs, got, masks):
        ref = pg.compute_stats(p, d, tt)
        assert_stats_match(g, ref, pg, p, d, tt, name)
        mref = pg.get_transit_mask(p, d, tt)
        assert m.dtype == bool and m.shape == mref.shape, name
        np.testing.assert_array_equal(m, mref, err_msg=name)
    return pgs, got, masks
