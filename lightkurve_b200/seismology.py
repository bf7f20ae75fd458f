"""Asteroseismology on top of the periodogram: the step after Lomb-Scargle + `Periodogram.flatten`
(SURVEY.md 8(f) rank 3; /root/reference/src/lightkurve/seismology/{core,numax_estimators,deltanu_estimators,
stellar_estimators,utils}.py).

``Seismology.from_lightcurve`` runs the GPU path (``to_periodogram`` = K1/K2, ``flatten`` = the batched log-median
background, K6); the estimators themselves work on the resulting signal-to-noise spectrum on the host, like the
reference: numax by the 2-D autocorrelation ("ACF2D") collapsed metric, deltanu by the autocorrelation of the
mode envelope, radius / mass / logg by the solar scaling relations with first-order error propagation (the
reference uses the `uncertainties` package for that; the formulae below are its linear propagation written out).
``estimate_numax_acf2d_batch`` / ``estimate_deltanu_acf2d_batch`` give the same results for many periodograms with
every autocorrelation in one GPU pass (K7, ``engine.acf_windows``); validation, window placement and the final
smoothing / peak search are the same functions as the per-periodogram estimators'.
Plotting / echelle diagrams are out of scope.
"""
import logging
import warnings

import numpy as np
from scipy.signal import find_peaks

from . import units as u
from .units import Quantity
from .utils import LightkurveWarning, validate_method

log = logging.getLogger(__name__)

__all__ = ["Seismology", "SeismologyQuantity", "estimate_numax_acf2d", "estimate_deltanu_acf2d",
           "estimate_numax_acf2d_batch", "estimate_deltanu_acf2d_batch", "estimate_radius", "estimate_mass", "estimate_logg", "NUMAX_SOL", "DELTANU_SOL", "TEFF_SOL", "G_SOL"]


class _UFloat:
    """Value with a standard error (`.n`, `.s`), the two attributes the reference's constants expose."""

    def __init__(self, n, s):
        self.n, self.s = float(n), float(s)

    def __repr__(self):
        return "{}+/-{}".format(self.n, self.s)


NUMAX_SOL = _UFloat(3090, 30)        # microhertz, Huber et al. 2011
DELTANU_SOL = _UFloat(135.1, 0.1)    # microhertz, Huber et al. 2011
TEFF_SOL = _UFloat(5772.0, 0.8)      # Kelvin, Prsa et al. 2016
# G M_sun / R_sun^2 in cm s^-2 (CODATA 2018 G M_sun = 1.3271244e20 m^3 s^-2, IAU nominal R_sun = 6.957e8 m)
G_SOL = Quantity(1.3271244e20 / 6.957e8 ** 2 * 100.0, u.cm / u.second ** 2)


class SeismologyQuantity(Quantity):
    """A Quantity that remembers its name, error, method and diagnostics (seismology/utils.py:11-66)."""

    def __new__(cls, quantity, name=None, error=None, method=None, diagnostics=None, diagnostics_plot_method=None):
        base = Quantity(quantity)
        obj = np.asarray(base.value, dtype=float).view(cls)
        obj._unit = base.unit
        obj.name = name
        obj.error = error
        obj.method = method
        obj.diagnostics = diagnostics
        obj.diagnostics_plot_method = diagnostics_plot_method
        return obj

    def __array_finalize__(self, obj):
        super().__array_finalize__(obj)
        for attr in ("name", "error", "method", "diagnostics", "diagnostics_plot_method"):
            setattr(self, attr, getattr(obj, attr, None))

    def __repr__(self):
        if self.name is None or self.ndim != 0:
            return super().__repr__()
        return "{}: {} {} (method: {})".format(self.name, "{:.2f}".format(float(self.value)),
                                               self.unit.to_string(), self.method)


# ---- helpers (seismology/utils.py) ------------------------------------------------------------------
def _in_microhertz(x):
    return float(np.asarray(Quantity(x, u.microhertz).value))


def get_fwhm(periodogram, numax):
    """Expected FWHM of the mode envelope: 0.25 numax for main-sequence spectra (highest frequency above
    500 uHz, Lund et al. 2017), 0.66 numax^0.88 for red giants (Mosser et al. 2010)."""
    if _in_microhertz(periodogram.frequency[-1]) > 500.0:
        return 0.25 * numax
    return 0.66 * numax ** 0.88


def _window_slices(F, f0, numaxs, window_width, fs):
    """(start, length) arrays of the reference's windows ``power[centre - spread : centre + spread]`` with
    spread = int(window_width / 2 / fs) and centre = int(numax / fs) - int(f0 / fs) (the same fp64 expressions,
    truncated toward zero like int()), under Python's slice rules: a negative end counts from the end of the
    array, then both ends are clipped to [0, F]; the slice may come out truncated or empty."""
    spread = int(window_width / 2 / fs)
    centre = np.trunc(np.asarray(numaxs, dtype=float) / fs).astype(np.int64) - int(f0 / fs)

    def resolve(e):
        return np.where(e < 0, np.maximum(e + F, 0), np.minimum(e, F))

    start, stop = resolve(centre - spread), resolve(centre + spread)
    return start, np.maximum(stop - start, 0)


def _correlate(sel):
    """Non-negative lags of the autocorrelation of the mean-subtracted window (np.correlate "full")."""
    sel = np.array(sel, dtype=float)
    sel -= np.nanmean(sel)
    return np.correlate(sel, sel, mode="full")[len(sel) - 1:]


def autocorrelate(periodogram, numax, window_width=25.0, frequency_spacing=None):
    """Autocorrelation (non-negative lags) of the mean-subtracted power in a window of `window_width` around
    `numax` (both in the periodogram's frequency unit)."""
    freq = np.asarray(periodogram.frequency.value, dtype=float)
    if frequency_spacing is None:
        frequency_spacing = np.median(np.diff(freq))
    start, length = _window_slices(len(freq), freq[0], [numax], window_width, frequency_spacing)
    return _correlate(np.asarray(periodogram.power.value, dtype=float)[start[0]:start[0] + length[0]])


def _gaussian_smooth_extend(x, stddev):
    """astropy ``convolve(x, Gaussian1DKernel(stddev), boundary="extend")``: normalised Gaussian sampled at
    integer offsets out to 4 sigma (kernel size 8 sigma rounded up to odd), edges padded with the end values."""
    half = int(np.ceil(8 * stddev)) // 2
    if (2 * half + 1) < int(np.ceil(8 * stddev)):
        half += 1
    offsets = np.arange(-half, half + 1)
    kernel = np.exp(-0.5 * (offsets / stddev) ** 2)
    kernel /= kernel.sum()
    padded = np.concatenate([np.full(half, x[0]), x, np.full(half, x[-1])])
    return np.convolve(padded, kernel, mode="valid")


def _check_evenly_spaced(periodogram):
    if not periodogram._is_evenly_spaced():
        raise ValueError("the ACF 2D method requires that the periodogram "
                         "has a grid of uniformly spaced frequencies.")


def _which(index):
    return "" if index is None else " (periodogram {})".format(index)


# ---- numax (seismology/numax_estimators.py:15-215) ---------------------------------------------------
def _numax_setup(periodogram, numaxs, window_width, spacing, index=None):
    """Validation and window placement of the ACF2D numax estimator: the trial numaxs, the window width, the
    lag count and the first bin of every window.  A window the reference's slice would truncate (or leave empty)
    makes its loop fail; it raises ValueError here, before any autocorrelation."""
    _check_evenly_spaced(periodogram)
    funit = periodogram.frequency.unit
    freq = np.asarray(periodogram.frequency.value, dtype=float)
    main_sequence = _in_microhertz(periodogram.frequency[-1]) > 500.0
    if window_width is None:
        window_width = Quantity(250.0 if main_sequence else 25.0, u.microhertz).to(funit).value
    if spacing is None:
        spacing = Quantity(10.0 if main_sequence else 1.0, u.microhertz).to(funit).value
    window_width = float(np.asarray(Quantity(window_width, funit).value))
    spacing = float(np.asarray(Quantity(spacing, funit).value))
    if numaxs is None:
        numaxs = np.arange(np.ceil(np.nanmin(freq)) + window_width / 2,
                           np.floor(np.nanmax(freq)) - window_width / 2, spacing)
    numaxs = np.atleast_1d(np.asarray(Quantity(numaxs, funit).value, dtype=float))
    fs = np.median(np.diff(freq))
    for var, label in ((window_width, "window_width"), (spacing, "spacing")):
        if var < fs:
            raise ValueError("You can't have {} smaller than the frequency separation!".format(label))
        if var > freq[-1] - freq[0]:
            raise ValueError("You can't have {} wider than the entire power spectrum!".format(label))
        if var < 0:
            raise ValueError("Please pass an entirely positive {}.".format(label))
    if np.any(numaxs < fs):
        raise ValueError("A custom range of numaxs can not extend below a single frequency bin.")
    if np.any(numaxs > np.nanmax(freq)):
        raise ValueError("A custom range of numaxs can not extend above "
                         "the highest frequency value in the periodogram.")
    if len(numaxs) == 0:
        raise ValueError("No trial numax fits in the periodogram{}.".format(_which(index)))
    nlags = int(window_width / 2 / fs) * 2
    starts, lengths = _window_slices(len(freq), freq[0], numaxs, window_width, fs)
    bad = np.flatnonzero(lengths != nlags) if nlags >= 1 else [0]
    if len(bad):
        raise ValueError("The {}-bin window around numax = {} {} does not fit in the periodogram{}.".format(
            nlags, numaxs[bad[0]], funit.to_string(), _which(index)))
    return dict(funit=funit, power=np.asarray(periodogram.power.value, dtype=float), numaxs=numaxs,
                window_width=window_width, nlags=nlags, starts=starts)


def _numax_finish(setup, metric, acf2d):
    """numax = the trial numax of the largest smoothed metric; the diagnostics of the reference."""
    numaxs = setup["numaxs"]
    if len(numaxs) > 10:
        metric_smooth = _gaussian_smooth_extend(metric, np.sqrt(len(numaxs)))
    else:
        metric_smooth = metric
    best = Quantity(numaxs[np.argmax(metric_smooth)], setup["funit"])
    diagnostics = {"numaxs": numaxs, "acf2d": acf2d, "window_width": setup["window_width"], "metric": metric,
                   "metric_smooth": metric_smooth}
    return SeismologyQuantity(best, name="numax", method="ACF2D", diagnostics=diagnostics)


def estimate_numax_acf2d(periodogram, numaxs=None, window_width=None, spacing=None):
    """numax = centre of the window whose autocorrelation carries the most (smoothed) collapsed power."""
    setup = _numax_setup(periodogram, numaxs, window_width, spacing)
    nlags, power = setup["nlags"], setup["power"]
    acf2d = np.zeros([nlags, len(setup["numaxs"])])
    metric = np.zeros(len(setup["numaxs"]))
    for idx, start in enumerate(setup["starts"]):
        acf = _correlate(power[start:start + nlags])
        acf2d[:, idx] = acf
        metric[idx] = (np.sum(np.abs(acf)) - 1) / len(acf)
    return _numax_finish(setup, metric, acf2d)


def estimate_numax_acf2d_batch(periodograms, numaxs=None, window_width=None, spacing=None, return_acf2d=False):
    """`estimate_numax_acf2d` of many periodograms with every autocorrelation in one GPU pass (K7,
    ``engine.acf_windows``).  Element b equals ``estimate_numax_acf2d(periodograms[b], numaxs, window_width,
    spacing)``: value, unit and diagnostics.  The diagnostic "acf2d" ([nlags, len(numaxs)]) is only filled with
    `return_acf2d` (a catalog of red giants at oversample 5 holds tens of GB of it); otherwise it is None.
    Every periodogram is validated before the GPU runs; a failure raises the loop's ValueError."""
    from . import engine
    setups = [_numax_setup(pg, numaxs, window_width, spacing, index=b) for b, pg in enumerate(periodograms)]
    if not setups:
        return []
    res = engine.acf_windows([s["power"] for s in setups], [s["starts"] for s in setups],
                             [s["nlags"] for s in setups], return_acf=return_acf2d)
    metrics, acfs = res if return_acf2d else (res, [None] * len(setups))
    return [_numax_finish(s, np.asarray(m), None if a is None else np.asarray(a).T)
            for s, m, a in zip(setups, metrics, acfs)]


# ---- deltanu (seismology/deltanu_estimators.py:15-129) -------------------------------------------------
def _deltanu_setup(periodogram, numax, index=None):
    """Validation and window placement of the ACF2D deltanu estimator.  The reference's slice may be truncated
    by the end of the spectrum (a shorter autocorrelation); an empty one makes it fail and raises ValueError."""
    _check_evenly_spaced(periodogram)
    funit = periodogram.frequency.unit
    freq = np.asarray(periodogram.frequency.value, dtype=float)
    numax = Quantity(numax, funit)
    numax_value = float(np.asarray(numax.value))
    fs = np.median(np.diff(freq))
    if numax_value < fs:
        raise ValueError("The input numax can not be lower than a single frequency bin.")
    if numax_value > np.nanmax(freq):
        raise ValueError("The input numax can not be higher than"
                         "the highest frequency value in the periodogram.")
    deltanu_emp = float(np.asarray(Quantity(0.294 * _in_microhertz(numax) ** 0.772, u.microhertz).to(funit).value))
    window_width = 2 * int(np.floor(get_fwhm(periodogram, numax_value)))
    start, length = (int(v[0]) for v in _window_slices(len(freq), freq[0], [numax_value], window_width, fs))
    if length < 1:
        raise ValueError("The window around numax = {} {} is empty{}.".format(numax_value, funit.to_string(),
                                                                               _which(index)))
    return dict(funit=funit, power=np.asarray(periodogram.power.value, dtype=float), numax=numax, fs=fs,
                deltanu_emp=deltanu_emp, start=start, length=length)


def _deltanu_finish(setup, aacf):
    """deltanu = the autocorrelation peak closest to the empirical deltanu; the diagnostics of the reference."""
    fs, deltanu_emp = setup["fs"], setup["deltanu_emp"]
    acf = (np.abs(aacf ** 2) / np.abs(aacf[0] ** 2)) / (3 / (2 * len(aacf)))
    lags = np.linspace(0.0, len(acf) * fs, len(acf))
    sel = (lags > 0.75 * deltanu_emp) & (lags < 1.25 * deltanu_emp)
    peaks, _ = find_peaks(acf[sel], distance=np.floor(deltanu_emp / 2.0 / fs))
    candidates = lags[sel][peaks]
    best = Quantity(candidates[np.argmin(np.abs(candidates - deltanu_emp))], setup["funit"])
    diagnostics = {"lags": lags, "acf": acf, "peaks": peaks, "sel": sel, "numax": setup["numax"],
                   "deltanu_emp": deltanu_emp}
    return SeismologyQuantity(best, name="deltanu", method="ACF2D", diagnostics=diagnostics)


def estimate_deltanu_acf2d(periodogram, numax):
    """deltanu = the autocorrelation peak of the mode envelope closest to 0.294 numax^0.772 (Stello et al. 2009)."""
    setup = _deltanu_setup(periodogram, numax)
    start, length = setup["start"], setup["length"]
    return _deltanu_finish(setup, _correlate(setup["power"][start:start + length]))


def estimate_deltanu_acf2d_batch(periodograms, numaxs):
    """`estimate_deltanu_acf2d` of many (periodogram, numax) pairs with the autocorrelations in one GPU pass (K7,
    ``engine.acf_windows``); the peak search stays on the host.  Element b equals
    ``estimate_deltanu_acf2d(periodograms[b], numaxs[b])``."""
    from . import engine
    if len(numaxs) != len(periodograms):
        raise ValueError("Pass one numax per periodogram ({} periodograms, {} numaxs).".format(
            len(periodograms), len(numaxs)))
    setups = [_deltanu_setup(pg, nm, index=b) for b, (pg, nm) in enumerate(zip(periodograms, numaxs))]
    if not setups:
        return []
    _, acfs = engine.acf_windows([s["power"] for s in setups], [[s["start"]] for s in setups],
                                 [s["length"] for s in setups], return_acf=True)
    return [_deltanu_finish(s, np.asarray(a)[0]) for s, a in zip(setups, acfs)]


# ---- scaling relations (seismology/stellar_estimators.py) ----------------------------------------------
def _power_law(terms):
    """prod (x_i / ref_i)^p_i with first-order error propagation over (x, sigma_x, ref, sigma_ref, p)."""
    value, rel2 = 1.0, 0.0
    for x, sx, ref, sref, p in terms:
        value *= (x / ref) ** p
        rel2 += (p * sx / x) ** 2 + (p * sref / ref) ** 2
    return value, abs(value) * np.sqrt(rel2)


def _value(x, unit):
    return float(np.asarray(Quantity(x, unit).value))


def _errors(pairs):
    """The reference propagates the observational errors only when ALL of them are given."""
    if all(e is not None for _, e in pairs):
        return [_value(e, unit) for unit, e in pairs]
    return [0.0 for _ in pairs]


def estimate_radius(numax, deltanu, teff, numax_err=None, deltanu_err=None, teff_err=None):
    """R / Rsun = (numax / numax_sun) (deltanu / deltanu_sun)^-2 (Teff / Teff_sun)^0.5."""
    numax, deltanu, teff = _value(numax, u.microhertz), _value(deltanu, u.microhertz), _value(teff, u.Kelvin)
    en, ed, et = _errors([(u.microhertz, numax_err), (u.microhertz, deltanu_err), (u.Kelvin, teff_err)])
    val, err = _power_law([(numax, en, NUMAX_SOL.n, NUMAX_SOL.s, 1.0), (deltanu, ed, DELTANU_SOL.n, DELTANU_SOL.s, -2.0),
                           (teff, et, TEFF_SOL.n, TEFF_SOL.s, 0.5)])
    return SeismologyQuantity(Quantity(val, u.solRad), error=Quantity(err, u.solRad), name="radius",
                              method="Uncorrected Scaling Relations")


def estimate_mass(numax, deltanu, teff, numax_err=None, deltanu_err=None, teff_err=None):
    """M / Msun = (numax / numax_sun)^3 (deltanu / deltanu_sun)^-4 (Teff / Teff_sun)^1.5."""
    numax, deltanu, teff = _value(numax, u.microhertz), _value(deltanu, u.microhertz), _value(teff, u.Kelvin)
    en, ed, et = _errors([(u.microhertz, numax_err), (u.microhertz, deltanu_err), (u.Kelvin, teff_err)])
    val, err = _power_law([(numax, en, NUMAX_SOL.n, NUMAX_SOL.s, 3.0), (deltanu, ed, DELTANU_SOL.n, DELTANU_SOL.s, -4.0),
                           (teff, et, TEFF_SOL.n, TEFF_SOL.s, 1.5)])
    return SeismologyQuantity(Quantity(val, u.solMass), error=Quantity(err, u.solMass), name="mass",
                              method="Uncorrected Scaling Relations")


def estimate_logg(numax, teff, numax_err=None, teff_err=None):
    """log10 of g = g_sun (numax / numax_sun) (Teff / Teff_sun)^0.5 in cgs, returned in dex."""
    numax, teff = _value(numax, u.microhertz), _value(teff, u.Kelvin)
    en, et = _errors([(u.microhertz, numax_err), (u.Kelvin, teff_err)])
    ratio, ratio_err = _power_law([(numax, en, NUMAX_SOL.n, NUMAX_SOL.s, 1.0), (teff, et, TEFF_SOL.n, TEFF_SOL.s, 0.5)])
    g = float(G_SOL.value) * ratio
    logg = np.log10(g)
    logg_err = ratio_err / ratio / np.log(10.0)
    return SeismologyQuantity(Quantity(logg, u.dex), error=Quantity(logg_err, u.dex), name="logg",
                              method="Uncorrected Scaling Relations")


# ---- the front end (seismology/core.py) ------------------------------------------------------------------
class Seismology(object):
    """Estimate numax, deltanu, radius, mass and logg from a background-corrected periodogram
    (seismology/core.py:21-920 without the plotting / echelle parts)."""

    periodogram = None

    def __init__(self, periodogram):
        from .periodogram import SNRPeriodogram
        if not isinstance(periodogram, SNRPeriodogram):
            warnings.warn("Seismology received a periodogram which does not appear "
                          "to have been background-corrected. Please consider calling "
                          "`periodogram.flatten()` prior to extracting seismological parameters.", LightkurveWarning)
        self.periodogram = periodogram

    def __repr__(self):
        attrs = np.asarray(["numax", "deltanu", "mass", "radius", "logg"])
        have = np.asarray([hasattr(self, attr) for attr in attrs])
        if have.sum() == 0:
            tail = " - no values have been computed so far."
        else:
            tail = " - computed values:\n * " + "\n * ".join([getattr(self, attr).__repr__() for attr in attrs[have]])
        return "Seismology(ID: {}){}".format(self.periodogram.label, tail)

    @staticmethod
    def from_lightcurve(lc, **kwargs):
        """`Seismology` of ``lc.normalize().remove_nans().fill_gaps().to_periodogram(**kwargs).flatten()``
        (core.py:97-110); the periodogram and its log-median background run on the GPU."""
        log.info("Building a Seismology object directly from a light curve "
                 "uses default periodogram parameters. For further tuneability, "
                 "create a periodogram object first, using `to_periodogram`.")
        return Seismology(periodogram=lc.normalize().remove_nans().fill_gaps().to_periodogram(**kwargs).flatten())

    def _validate_numax(self, numax):
        if numax is None:
            try:
                return self.numax
            except AttributeError:
                raise AttributeError("You need to call `Seismology.estimate_numax()` first.")
        return numax

    def _validate_deltanu(self, deltanu):
        if deltanu is None:
            try:
                return self.deltanu
            except AttributeError:
                raise AttributeError("You need to call `Seismology.estimate_deltanu()` first.")
        return deltanu

    def _validate_teff(self, teff):
        if teff is None:
            teff = self.periodogram.meta.get("TEFF")
            if teff is None:
                raise ValueError(
                    "You must provide an effective temperature argument (`teff`) to `estimate_radius`,"
                    "because the Periodogram object does not contain it in its meta data (i.e. `pg.meta['TEFF']` is missing")
            log.info("Using value for effective temperature from the Kepler Input Catalogue."
                     "These temperatue values may sometimes differ significantly from modern estimates.")
        return teff

    def estimate_numax(self, method="acf2d", **kwargs):
        validate_method(method, supported_methods=["acf2d"])
        self.numax = estimate_numax_acf2d(self.periodogram, **kwargs)
        return self.numax

    def estimate_deltanu(self, method="acf2d", numax=None):
        validate_method(method, supported_methods=["acf2d"])
        numax = self._validate_numax(numax)
        self.deltanu = estimate_deltanu_acf2d(self.periodogram, numax=numax)
        return self.deltanu

    def estimate_radius(self, teff=None, numax=None, deltanu=None):
        numax, deltanu = self._validate_numax(numax), self._validate_deltanu(deltanu)
        self.radius = estimate_radius(numax, deltanu, self._validate_teff(teff))
        return self.radius

    def estimate_mass(self, teff=None, numax=None, deltanu=None):
        numax, deltanu = self._validate_numax(numax), self._validate_deltanu(deltanu)
        self.mass = estimate_mass(numax, deltanu, self._validate_teff(teff))
        return self.mass

    def estimate_logg(self, teff=None, numax=None):
        numax = self._validate_numax(numax)
        self.logg = estimate_logg(numax, self._validate_teff(teff))
        return self.logg
