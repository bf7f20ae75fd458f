"""Oracle: flatten / sigma_clip / RegressionCorrector numerics (TEST INFRASTRUCTURE ONLY).

flatten   : /root/reference/src/lightkurve/lightcurve.py:996-1070 restated on plain
            ndarrays; calls the REAL scipy.signal.savgol_filter (:1040) and
            scipy.interpolate.interp1d (:1053) the reference calls.  savgol=savgol_lsq
            swaps in the same filter from a well-conditioned least-squares basis:
            scipy builds its taps from the unscaled Vandermonde matrix of the window
            offsets, which loses accuracy at polyorder >= 4 and long windows (taps off
            by 1e-8 relative at window 201, 1e-6 at 1001, for polyorder 5).
sigma_clip: astropy.stats.sigma_clip defaults (maxiters=5, median, std) as used at
            correctors/regressioncorrector.py:269 -- restated (astropy absent).
regress   : correctors/regressioncorrector.py:127-189 (_fit_coefficients, dense
            branch) and :244-279 (correct loop), on the REAL numpy.linalg.solve.
normalize : lightcurve.py:1253-1254.
Pinned by the reference's known-answer tests (tests/test_lightcurve.py:1284-1360,
tests/correctors/test_regressioncorrector.py:13-83) ported under tests/.
"""
import functools
import warnings

import numpy as np
from numpy.polynomial import legendre
from scipy.interpolate import interp1d
from scipy.signal import savgol_filter


@functools.lru_cache(maxsize=64)
def _savgol_basis(window_length, polyorder):
    """Orthonormal basis [window_length, polyorder + 1] of the polynomials of degree <= polyorder on the window:
    QR of the Legendre Vandermonde matrix on u = (k - half) / half, whose columns are nearly orthogonal."""
    half = window_length // 2
    u = (np.arange(window_length) - half) / max(half, 1)
    q, _ = np.linalg.qr(legendre.legvander(u, polyorder))
    q.setflags(write=False)
    return q


def savgol_lsq(x, window_length, polyorder):
    """scipy.signal.savgol_filter(x, window_length, polyorder) (mode="interp", len(x) >= window_length): the
    least-squares polynomial of the window around each interior point evaluated at its centre, and the fits of the
    first and last windows evaluated at the edge points; the projections come from _savgol_basis."""
    x = np.asarray(x, dtype=np.float64)
    n, w, half = len(x), window_length, window_length // 2
    q = _savgol_basis(w, polyorder)
    taps = q @ q[half]
    y = np.empty(n)
    y[half:n - half] = np.convolve(x, taps[::-1], mode="valid")
    y[:half] = q[:half] @ (q.T @ x[:w])
    y[n - half:] = q[w - half:] @ (q.T @ x[n - w:])
    return y


def flatten(time, flux, flux_err=None, window_length=101, polyorder=2, break_tolerance=5,
            niters=3, sigma=3, mask=None, savgol=savgol_filter):
    """Returns (flat_flux, flat_flux_err, trend).  `mask` True = exclude (lightcurve.py:980-1000).  `savgol`: the
    Savitzky-Golay filter, called as savgol(x, window_length, polyorder)."""
    time = np.asarray(time, dtype=np.float64)
    flux = np.asarray(flux)
    if not np.issubdtype(flux.dtype, np.floating):
        fluxf = flux.astype(np.float64)
    else:
        fluxf = flux
    if flux_err is None:
        flux_err = np.full(len(fluxf), np.nan)
    if mask is None:
        mask = np.ones(len(time), dtype=bool)
    else:
        mask = ~np.asarray(mask, dtype=bool)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        extra_mask = np.isfinite(fluxf)
        extra_mask &= np.nan_to_num(np.abs(fluxf - np.nanmedian(fluxf))) <= (np.nanstd(fluxf) * sigma)
    mask = mask & extra_mask

    trend_signal = None
    for _ in range(niters):
        if break_tolerance is None:
            break_tolerance = np.nan
        if polyorder >= window_length:
            polyorder = window_length - 1
        tm = time[mask]
        fm = fluxf[mask]
        dt = tm[1:] - tm[0:-1]
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)
            cut = np.where(dt > break_tolerance * np.nanmedian(dt))[0] + 1
        low = np.append([0], cut)
        high = np.append(cut, len(tm))
        trend_signal = np.zeros(len(tm))
        for l, h in zip(low, high):
            if np.any([window_length > (h - l), (h - l) < break_tolerance]):
                trend_signal[l:h] = np.nanmedian(fm[l:h])
            else:
                trend_signal[l:h] = savgol(fm[l:h], window_length, polyorder)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)
            mask1 = np.nan_to_num(np.abs(fm - trend_signal)) < (np.nanstd(fm - trend_signal) * sigma + 1e-14)
        f = interp1d(tm[mask1], trend_signal[mask1], fill_value="extrapolate")
        trend_signal = f(time)
        mask[mask] &= mask1
    with np.errstate(divide="ignore", invalid="ignore"):
        return fluxf / trend_signal, np.asarray(flux_err, dtype=np.float64) / trend_signal, trend_signal


def sigma_clip_mask(data, sigma=3.0, maxiters=5):
    """astropy.stats.sigma_clip(data, sigma).mask with default cenfunc/stdfunc."""
    data = np.asarray(data, dtype=np.float64)
    mask = ~np.isfinite(data)
    nchanged = 1
    it = 0
    while nchanged != 0 and it < maxiters:
        it += 1
        good = data[~mask]
        size = good.size
        if size == 0:
            break
        c = np.median(good)
        s = np.std(good)
        lo = c - s * sigma
        hi = c + s * sigma
        with np.errstate(invalid="ignore"):
            mask = mask | (data < lo) | (data > hi)
        nchanged = size - int((~mask).sum())
    return mask


def fit_coefficients(X, y, flux_err, cadence_mask, prior_mu=None, prior_sigma=None):
    """regressioncorrector.py:127-189 dense branch."""
    if np.all(~np.isfinite(flux_err)):
        fe = np.ones(int(cadence_mask.sum()))
    else:
        fe = flux_err[cadence_mask]
    Xm = X[cadence_mask]
    sigma_w_inv = Xm.T.dot(Xm / fe[:, None] ** 2)
    B = np.dot(Xm.T, y[cadence_mask] / fe ** 2)
    if prior_sigma is not None:
        sigma_w_inv = sigma_w_inv + np.diag(1.0 / prior_sigma ** 2)
        B = B + (prior_mu / prior_sigma ** 2)
    return np.linalg.solve(sigma_w_inv, B).T


def regress(X, y, flux_err=None, cadence_mask=None, prior_mu=None, prior_sigma=None,
            sigma=5, niters=5):
    """regressioncorrector.py:238-279.  Returns dict(coefficients, model, corrected,
    outlier_mask).  model is median-subtracted (:278-279)."""
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    N = len(y)
    if flux_err is None:
        flux_err = np.full(N, np.nan)
    flux_err = np.asarray(flux_err, dtype=np.float64)
    if cadence_mask is None:
        cadence_mask = np.ones(N, bool)
    outlier_mask = np.zeros(N, bool)
    coefficients = None
    for _ in range(niters):
        tmp = cadence_mask & ~outlier_mask
        coefficients = fit_coefficients(X, y, flux_err, tmp, prior_mu, prior_sigma)
        model = X.dot(coefficients)
        residuals = np.where(tmp, y - model, np.nan)  # masked -> NaN (:258-266)
        outlier_mask |= sigma_clip_mask(residuals, sigma=sigma)
    model_flux = X.dot(coefficients)
    model_flux = model_flux - np.median(model_flux)
    return dict(coefficients=coefficients, model=model_flux, corrected=y - model_flux,
                outlier_mask=outlier_mask)


def normalize(flux, flux_err=None):
    """lightcurve.py:1253-1254,1281-1283."""
    flux = np.asarray(flux, dtype=np.float64)
    med = np.nanmedian(flux)
    fe = None if flux_err is None else np.asarray(flux_err, dtype=np.float64) / med
    return flux / med, fe
