"""TEST INFRASTRUCTURE: the fp64 reference of K11 / K12 (lightkurve_b200/csrc/clip.cuh), built on oracle/detrend.py.

sigma_clip_mask : astropy.stats.sigma_clip(data, sigma, sigma_lower, sigma_upper, maxiters).mask with the default
                  cenfunc/stdfunc, restated with the semantics of oracle.detrend.sigma_clip_mask (which it equals for
                  sigma_lower == sigma_upper and an integer maxiters, tests/test_cdpp_host.py) plus the asymmetric
                  sigmas and maxiters=None (until a round clips nothing) of LightCurve.remove_outliers.
cdpp            : lightcurve.py:1764-1833 (estimate_cdpp) on oracle.detrend.flatten, sigma_clip_mask above,
                  oracle.detrend.normalize and utils.py:374-387 (running_mean, a cumsum).
Nothing in the product imports this module."""
import warnings

import numpy as np

from oracle import detrend as odet


def sigma_clip_mask(data, sigma=3.0, maxiters=5, sigma_lower=None, sigma_upper=None):
    data = np.asarray(data, dtype=np.float64)
    sigma_lower = sigma if sigma_lower is None else sigma_lower
    sigma_upper = sigma if sigma_upper is None else sigma_upper
    mask = ~np.isfinite(data)
    nchanged = 1
    it = 0
    while nchanged != 0 and (maxiters is None or it < maxiters):
        it += 1
        good = data[~mask]
        size = good.size
        if size == 0:
            break
        c = np.median(good)
        s = np.std(good)
        lo = c - s * sigma_lower
        hi = c + s * sigma_upper
        with np.errstate(invalid="ignore"):
            mask = mask | (data < lo) | (data > hi)
        nchanged = size - int((~mask).sum())
    return mask


def running_mean(data, window_size):
    """utils.py:374-387: top-hat running mean by cumulative sums."""
    if window_size > len(data):
        window_size = len(data)
    cumsum = np.cumsum(np.insert(data, 0, 0))
    return (cumsum[window_size:] - cumsum[:-window_size]) / float(window_size)


def cdpp(time, flux, transit_duration=13, savgol_window=101, savgol_polyorder=2, sigma=5.0):
    """The Savitzky-Golay CDPP proxy in ppm: flatten, remove_outliers(sigma) (maxiters 5), normalize("ppm"), then the
    standard deviation of the running means over transit_duration cadences."""
    flat = odet.flatten(time, flux, window_length=savgol_window, polyorder=savgol_polyorder)[0]
    return cdpp_of_flat(flat, transit_duration, sigma)


def cdpp_of_flat(flat, transit_duration=13, sigma=5.0):
    """The part of cdpp after flatten, on the flattened flux."""
    flat = np.asarray(flat, dtype=np.float64)
    cleaned = flat[~sigma_clip_mask(flat, sigma=sigma)]
    normalized = odet.normalize(cleaned)[0] * 1e6
    with warnings.catch_warnings(), np.errstate(all="ignore"):
        warnings.simplefilter("ignore", RuntimeWarning)
        return float(np.std(running_mean(normalized, transit_duration)))
