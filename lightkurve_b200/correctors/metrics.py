"""Over-fitting metric of a systematics correction: /root/reference/src/lightkurve/correctors/metrics.py:23-123
(``overfit_metric_lombscargle``; SURVEY.md section 8(f) rank 4).  Same definition and the same use of numpy's
global random stream; the difference is where the arithmetic runs: the original / corrected periodograms are
computed once (the reference recomputes the identical pair in every iteration) and the ``n_samples`` white-noise
periodograms, which share one cadence grid, go through the batched GPU call in one launch.

Under-fitting metric: ``underfit_metric_neighbors`` (metrics.py:125-255) with the neighbouring light curves handed
over (``neighbors=``) instead of searched and downloaded from MAST; the correlations run in one K9 call
(``lkb_underfit_metric``).
"""
import numpy as np
from scipy.interpolate import PchipInterpolator

from ..collections import LightCurveCollection
from ..lightcurve import LightCurve

__all__ = ["overfit_metric_lombscargle", "underfit_metric_neighbors", "MinTargetsError"]

MAST_MESSAGE = ("the under-fitting metric needs a MAST search of neighbouring targets, which is outside the scope of "
                "lightkurve_b200: pass the neighbouring light curves with `neighbors=`")


class MinTargetsError(Exception):
    """Fewer than `min_targets` neighbours are available (metrics.py:258-260)."""


def _overfit_from_terms(n_positive, sum_positive, noise_means):
    """overfit_metric_lombscargle's metric from its terms (n_positive, sum of positive changes, mean noise powers)."""
    metric_per_iter = []
    for mean_noise_power in noise_means:
        if n_positive == 0:
            metric_per_iter.append(0.0)
        else:
            denominator = n_positive * mean_noise_power
            metric_per_iter.append(np.inf if denominator == 0 else sum_positive / denominator)
    with np.errstate(over="ignore"):
        return float(2.0 / (1 + np.exp(np.max([np.mean(metric_per_iter), 0.0]))))


def _centred(lc):
    """``lc.remove_nans().normalize() - 1``: the flux the metrics correlate / transform."""
    lc = lc.copy().remove_nans().normalize()
    return lc, np.asarray(lc.flux.value, dtype=np.float64) - 1.0


# The common cadence grid of the under-fitting metric: cadence numbers from a multiple of GRID_ALIGN on.  The K9 kernel
# sums a cadence in the lane and partial sum its grid position (mod 256) selects, so with this alignment a target's
# metric does not depend on which other light curves set the extent of the grid.
GRID_ALIGN = 256


def _cadence_grid(cadence_arrays):
    lo = min(int(np.min(c)) for c in cadence_arrays if len(c))
    hi = max(int(np.max(c)) for c in cadence_arrays if len(c))
    c0 = (lo // GRID_ALIGN) * GRID_ALIGN
    return c0, hi - c0 + 1


def _require_cadenceno(lc):
    if "cadenceno" not in lc.__dict__.get("_columns", {}):
        raise ValueError("aligning neighbours needs cadence numbers (`cadenceno`) on every light curve")


def _on_grid(cadenceno, values, c0, G):
    """`values` at their cadence numbers on the grid, NaN elsewhere (_align_to_lc: cadences off the grid drop)."""
    row = np.full(G, np.nan)
    pos = np.asarray(cadenceno, dtype=np.int64) - c0
    keep = (pos >= 0) & (pos < G)
    row[pos[keep]] = values[keep]
    return row


def _neighbor_rows(neighbors, target_lc, target_cad, c0, G, interpolate=False, extrapolate=False):
    """Pool rows of the neighbours: remove_nans().normalize() - 1, aligned by cadence number or, with `interpolate`,
    PCHIP-interpolated to the target's times (metrics.py:343-360)."""
    rows = np.empty((len(neighbors), G))
    for i, lc in enumerate(neighbors):
        n, f = _centred(lc)
        if interpolate:
            vals = PchipInterpolator(np.asarray(n.time.value, dtype=np.float64), f,
                                     extrapolate=extrapolate)(np.asarray(target_lc.time.value, dtype=np.float64))
            rows[i] = _on_grid(target_cad, vals, c0, G)
        else:
            rows[i] = _on_grid(n.cadenceno, f, c0, G)
    return rows


def underfit_metric_neighbors(corrected_lc, radius=6000, min_targets=30, max_targets=50, interpolate=False,
                              extrapolate=False, quality_bitmask="default", neighbors=None):
    """Residual correlation of the corrected light curve with its neighbours, mapped to (0, 1] (0 bad, 1 good; 0.95:
    the correlations of white Gaussian noise).  `neighbors`: the neighbouring light curves (a list or
    `LightCurveCollection`) in place of the reference's MAST search; the first `max_targets` are used, fewer than
    `min_targets` raise `MinTargetsError`.  They are aligned to `corrected_lc` by cadence number, or PCHIP-interpolated
    to its times with `interpolate=True`.  `radius` only appears in the error text; `quality_bitmask` is not used (the
    light curves are given, not downloaded)."""
    from .. import engine
    if neighbors is None:
        raise NotImplementedError(MAST_MESSAGE)
    if extrapolate and (extrapolate != interpolate):
        raise Exception("interpolate must be True if extrapolate is True")
    target, tflux = _centred(corrected_lc)
    neighbors = list(neighbors)[:max_targets]
    if len(neighbors) < min_targets:
        raise MinTargetsError("Unable to find at least {} neighbors within {} arcseconds radius.".format(min_targets,
                                                                                                         radius))
    if interpolate:
        cad = np.arange(len(target))
    else:
        for lc in [target] + neighbors:
            _require_cadenceno(lc)
        cad = target.cadenceno
    c0, G = _cadence_grid([cad])
    pool = _neighbor_rows(neighbors, target, cad, c0, G, interpolate, extrapolate)
    row = _on_grid(cad, tflux, c0, G)[None, :]
    M = len(neighbors)
    return float(engine.underfit_metric(pool, row, np.array([0, M]), np.arange(M))["metric"][0])


def overfit_metric_lombscargle(original_lc, corrected_lc, n_samples=10):
    """Change in broad-band Lomb-Scargle power introduced by a correction, mapped to [0, 1] (0 bad, 1 good);
    0.5 means the introduced noise has the power level of the light curve's uncertainties."""
    orig_lc = original_lc.copy()
    orig_lc = orig_lc.remove_nans().normalize()
    orig_lc -= 1.0
    corrected_lc = corrected_lc.copy()
    corrected_lc = corrected_lc.remove_nans().normalize()
    corrected_lc -= 1.0
    if len(corrected_lc) == 0:
        return 1.0

    pg_orig = orig_lc.to_periodogram()
    pg_corrected = corrected_lc.to_periodogram(frequency=pg_orig.frequency)
    pg_change = np.asarray(pg_corrected.power.value) - np.asarray(pg_orig.power.value)
    pg_change = pg_change[~np.isnan(pg_change)]
    n_positive = len(np.nonzero(pg_change > 0.0)[0])

    n_cad = len(orig_lc)
    mean_err = np.nanmean(np.asarray(corrected_lc.flux_err.value))
    # the reference draws randn(n, 1) once per iteration, in order: same stream
    noise = [(np.random.randn(n_cad, 1) * mean_err).T[0] for _ in range(n_samples)]
    noise_lcs = LightCurveCollection([LightCurve(time=orig_lc.time, flux=w, flux_err=np.zeros(n_cad)) for w in noise])
    noise_pgs = noise_lcs.to_periodogram() if n_samples > 0 else []

    metric_per_iter = []
    for pg_noise in noise_pgs:
        mean_noise_power = np.nanmean(np.asarray(pg_noise.power.value))
        if n_positive == 0:
            metric_per_iter.append(0.0)
        else:
            denominator = n_positive * mean_noise_power
            metric_per_iter.append(np.inf if denominator == 0 else np.sum(pg_change[pg_change > 0.0]) / denominator)
    with np.errstate(over="ignore"):
        metric = np.mean(metric_per_iter)
        return float(2.0 / (1 + np.exp(np.max([metric, 0.0]))))
