"""`LightCurve`: the slice of /root/reference/src/lightkurve/lightcurve.py that sits on the hot path.

Mirrors the reference's names, defaults, warnings and error behaviour for: the constructor
(:355-488), ``normalize`` (:1216-1298), ``remove_nans`` (:1300-1327), ``flatten`` (:943-1078),
``to_periodogram`` (:2490-2535), ``remove_outliers`` (:1429-1549, sigma_clip on the GPU select
kernel), ``estimate_cdpp`` (:1764-1833), ``fold``-free arithmetic used by the correctors, and
``to_corrector``.  The container is numpy-backed (the reference subclasses astropy TimeSeries,
which cannot be imported here); plotting, FITS export, binning and archive access are out of
scope (SURVEY.md section 2).  The arithmetic of flatten / periodograms / sigma-clip statistics is
NOT done here: it is routed through ``engine`` into the CUDA kernels.
"""
import copy as _copy
import logging
import warnings

import numpy as np

from . import units as u
from .units import Quantity, Time
from .utils import LightkurveWarning, validate_method, running_mean

log = logging.getLogger(__name__)

__all__ = ["LightCurve", "FoldedLightCurve"]


def _as_flux_quantity(x, unit=None):
    if isinstance(x, Quantity):
        return x if unit is None else x.to(unit)
    if hasattr(x, "unmasked") and hasattr(x, "mask"):            # astropy Masked -> NaN where masked
        data = np.array(getattr(x.unmasked, "value", x.unmasked), dtype=float)
        data[np.asarray(x.mask, dtype=bool)] = np.nan
        return Quantity(data, u._as_unit(getattr(x.unmasked, "unit", unit)))
    if isinstance(x, np.ma.MaskedArray):
        data = np.array(x.filled(np.nan), dtype=float)
        return Quantity(data, unit)
    if u.is_quantity(x):
        return Quantity(x)
    arr = np.asarray(x)
    if arr.dtype.kind not in "f":
        arr = arr.astype(float)
    return Quantity(arr, unit, dtype=arr.dtype)


def _fold_params(t, time, period, epoch_time, epoch_phase, wrap_phase, normalize_phase):
    """(period, t0, shift, wrap, JD warning or None) of `LightCurve.fold` in days, for the float64 times `t` of a
    light curve whose time object is `time`: phase = ((t - t0) + shift + (period - wrap)) % period - (period - wrap).
    Raises the errors of the single-curve method; the caller issues the warning."""
    if period is None:
        raise ValueError("`period` must be given")
    per = float(np.asarray(Quantity(period, u.day).value)) if u.is_quantity(period) else float(period)
    t0 = t[0] if epoch_time is None else float(np.asarray(getattr(epoch_time, "value", epoch_time)))
    jd_warning = None
    if epoch_time is not None and t0 > 2450000:
        if time.format == "bkjd":
            jd_warning = ("`epoch_time` appears to be given in JD, "
                          "however the light curve time uses BKJD "
                          "(i.e. JD - 2454833).")
        elif time.format == "btjd":
            jd_warning = ("`epoch_time` appears to be given in JD, "
                          "however the light curve time uses BTJD "
                          "(i.e. JD - 2457000).")
    ep = float(np.asarray(getattr(epoch_phase, "value", epoch_phase)))
    ep_days = ep * per if normalize_phase else (float(np.asarray(Quantity(epoch_phase, u.day).value))
                                                if u.is_quantity(epoch_phase) else ep)
    if wrap_phase is None:
        wrap = per / 2.0
    else:
        wv = float(np.asarray(getattr(wrap_phase, "value", wrap_phase)))
        if normalize_phase:
            if wv < 0 or wv > 1:
                raise ValueError("wrap_phase should be between 0 and 1")
            wrap = wv * per
        else:
            wrap = float(np.asarray(Quantity(wrap_phase, u.day).value)) if u.is_quantity(wrap_phase) else wv
            if wrap < 0 or wrap > per:
                raise ValueError("wrap_phase should be between 0 and the period")
    return per, t0, ep_days, wrap, jd_warning


def _bin_check_args(time_bin_size, n_bins, aggregate_func, bins, binsize):
    """Checks the keywords of `LightCurve.bin` as the single-curve method does; returns the aggregate function."""
    if binsize is not None and bins is not None:
        raise ValueError("Only one of ``bins`` and ``binsize`` can be specified.")
    if (binsize is not None or bins is not None) and (time_bin_size is not None or n_bins is not None):
        raise ValueError("``bins`` or ``binsize`` conflicts with ``n_bins`` or ``time_bin_size``.")
    if bins is not None:
        if isinstance(bins, str):
            if bins in ("blocks", "knuth", "scott", "freedman"):
                raise NotImplementedError("adaptive ``bins`` rules need astropy.stats, which is not available")
            raise TypeError("``bins`` must have integer type.")
        if np.array(bins).dtype.kind not in "iu":
            raise TypeError("``bins`` must have integer type.")
    if aggregate_func is None:
        aggregate_func = np.nanmean
    if not callable(aggregate_func):
        raise TypeError("`aggregate_func` must be callable")
    return aggregate_func


def _bin_edges(n, t_first, t_last, time_bin_size, time_bin_start, time_bin_end, n_bins, bins, binsize):
    """The bin edges of `LightCurve.bin` for a light curve of n > 0 cadences whose stably time-sorted times start with
    `t_first` and end with `t_last`: ("time", starts, ends) as times, or ("index", starts, ends) as indices into the
    time-sorted cadences (`binsize` and `bins=<indices>`, whose edges are cadence times)."""
    as_days = lambda x: float(np.asarray(Quantity(x, u.day).value)) if u.is_quantity(x) else float(x)
    if binsize is not None:
        starts = np.arange(n)[::int(binsize)]
        return "index", starts, np.append(starts[1:], n - 1)
    if bins is not None and np.size(bins) == 1:
        edges = np.linspace(t_first, t_last, int(bins) + 1)
        starts = edges[:-1]
        return "time", starts, np.append(starts[1:], t_last)
    if bins is not None:
        idx = np.asarray(bins, dtype=int)
        cad = np.arange(n)
        return "index", cad[idx[:-1]], cad[idx[1:]]
    size = 0.5 if time_bin_size is None else as_days(time_bin_size)
    if not size > 0:
        raise ValueError("`time_bin_size` must be positive")
    start = t_first if time_bin_start is None else float(getattr(time_bin_start, "value", time_bin_start))
    if n_bins is None:
        stop = t_last if time_bin_end is None else float(getattr(time_bin_end, "value", time_bin_end))
        n_bins = max(1, int(np.ceil((stop - start) / size)))
    starts = start + size * np.arange(int(n_bins))
    return "time", starts, starts + size


def _normalize_warnings(median_flux, std_flux):
    """The LightkurveWarnings of `LightCurve.normalize` for a flux of this nanmedian and nanstd."""
    if (median_flux == 0) or (np.isfinite(std_flux) and (np.abs(median_flux) < 0.5 * std_flux)):
        warnings.warn(
            "The light curve appears to be zero-centered "
            "(median={:.2e} +/- {:.2e}); `normalize()` will divide "
            "the light curve by a value close to zero, which is "
            "probably not what you want."
            "".format(median_flux, std_flux),
            LightkurveWarning,
        )
    if median_flux < 0:
        warnings.warn(
            "The light curve has a negative median flux ({:.2e});"
            " `normalize()` will therefore divide by a negative "
            "number and invert the light curve, which is probably"
            "not what you want".format(median_flux),
            LightkurveWarning,
        )


class LightCurve:
    """Time series of flux values (subset of lightkurve.LightCurve).

    Parameters mirror the reference: ``LightCurve(data=None, *, time=None, flux=None,
    flux_err=None, **kwargs)``; deprecated keywords ``flux_unit``, ``time_format``,
    ``time_scale``, ``targetid``, ``label`` are accepted (lightcurve.py:327-333).
    """

    _default_time_format = "jd"
    _default_time_scale = "tdb"

    def __init__(self, data=None, *args, time=None, flux=None, flux_err=None, meta=None, **kwargs):
        if len(args) in (1, 2):                       # deprecated positional form (time, flux[, flux_err])
            time, flux, data = data, args[0], None
            if len(args) == 2:
                flux_err = args[1]
        extra = {}
        if isinstance(data, dict):
            time = data.get("time", time)
            flux = data.get("flux", flux)
            flux_err = data.get("flux_err", flux_err)
            extra.update({k: v for k, v in data.items() if k in self._extra_column_names})
        elif data is not None:
            raise TypeError("`data` must be a dict with 'time'/'flux'[/'flux_err'] in this build")
        for name in self._extra_column_names:                  # optional per-cadence columns (cadenceno, quality, ...)
            if name in kwargs:
                extra[name] = kwargs.pop(name)
        flux_unit = kwargs.pop("flux_unit", None)
        time_format = kwargs.pop("time_format", self._default_time_format)
        time_scale = kwargs.pop("time_scale", self._default_time_scale)
        self.meta = dict(meta) if meta else {}
        for kw in ("targetid", "label"):
            if kw in kwargs:
                self.meta[kw.upper()] = kwargs.pop(kw)
        self.meta.update({k.upper(): v for k, v in kwargs.items() if k.isupper() or k in ("mission", "sector")})

        if time is None and flux is not None:
            time = np.arange(len(flux))                              # :388-389
        if time is None:
            time = np.zeros(0)
        if not isinstance(time, Time):
            time = Time(time, format=time_format, scale=time_scale)
        if flux is None:
            flux = np.full(len(time), np.nan)
        if np.ndim(getattr(flux, "value", flux)) == 0:               # scalars broadcast (astropy TimeSeries column semantics)
            flux = np.full(len(time), float(getattr(flux, "value", flux))) * (flux.unit if u.is_quantity(flux) else 1)
        if flux_err is not None and np.ndim(getattr(flux_err, "value", flux_err)) == 0:
            flux_err = np.full(len(time), float(getattr(flux_err, "value", flux_err))) * \
                (flux_err.unit if u.is_quantity(flux_err) else 1)
        flux = _as_flux_quantity(flux, flux_unit)
        if flux_err is None:
            flux_err = np.full(len(flux), np.nan)                     # :458-460
        flux_err = _as_flux_quantity(flux_err, None if u.is_quantity(flux_err) else flux.unit)
        if not (len(time) == len(flux) == len(flux_err)):
            raise ValueError("time, flux and flux_err must have the same length")
        self.time = time
        self.flux = flux
        self.flux_err = flux_err
        self._columns = {}
        for name, col in extra.items():
            col = np.asarray(getattr(col, "value", col))
            if len(col) != len(time):
                raise ValueError("column `{}` must have as many entries as `time`".format(name))
            self._columns[name] = col

    # per-cadence columns carried along besides time / flux / flux_err (the reference's LightCurve is a table with
    # arbitrary columns, lightcurve.py:490-539; these are the ones the hot path's neighbours use)
    _extra_column_names = ("cadenceno", "quality", "centroid_col", "centroid_row")

    def __getattr__(self, name):
        cols = self.__dict__.get("_columns")
        if cols is not None and name in cols:
            return cols[name]
        raise AttributeError("{!r} object has no attribute {!r}".format(type(self).__name__, name))

    # ------------------------------------------------------------------ container protocol
    def __len__(self):
        return len(self.time)

    def __repr__(self):
        return "<LightCurve length={} label={!r}>".format(len(self), self.label)

    @property
    def targetid(self):
        return self.meta.get("TARGETID")

    @property
    def label(self):
        return self.meta.get("LABEL")

    def copy(self, copy_data=True):
        new = self.__class__.__new__(self.__class__)
        new.meta = _copy.deepcopy(self.meta)
        new.time = self.time.copy() if copy_data else self.time
        new.flux = self.flux.copy() if copy_data else self.flux
        new.flux_err = self.flux_err.copy() if copy_data else self.flux_err
        new._columns = {k: (v.copy() if copy_data else v) for k, v in self.__dict__.get("_columns", {}).items()}
        return new

    def __getitem__(self, key):
        if isinstance(key, str):
            return getattr(self, key)
        if isinstance(key, (int, np.integer)):
            key = slice(key, key + 1 if key != -1 else None)
        new = self.copy(copy_data=False)
        new.time = Time(self.time.value[key], self.time.format, self.time.scale)
        new.flux = Quantity(self.flux.value[key], self.flux.unit, dtype=self.flux.dtype)
        new.flux_err = Quantity(self.flux_err.value[key], self.flux_err.unit, dtype=self.flux_err.dtype)
        new._columns = {k: v[key] for k, v in self.__dict__.get("_columns", {}).items()}
        return new

    def __setitem__(self, key, value):
        if isinstance(key, str):
            setattr(self, key, value)
            return
        # row assignment, e.g. lc[400:500] = np.nan (tests/test_periodogram.py:39)
        self.flux.view(np.ndarray)[key] = value
        self.flux_err.view(np.ndarray)[key] = value

    def _binop(self, other, op):
        new = self.copy()
        if isinstance(other, LightCurve):
            if len(other) != len(self):
                raise ValueError("Cannot combine LightCurve objects of different length.")
            a, b = self.flux, other.flux
            if op in ("add", "sub"):
                new.flux = a + b if op == "add" else a - b
                new.flux_err = np.hypot(self.flux_err, other.flux_err)
            elif op == "mul":
                new.flux = a * b
                new.flux_err = abs(new.flux) * np.hypot((self.flux_err / a).value, (other.flux_err / b).value)
            else:
                new.flux = a / b
                new.flux_err = abs(new.flux) * np.hypot((self.flux_err / a).value, (other.flux_err / b).value)
            return new
        if op == "add":
            new.flux = self.flux + other
        elif op == "sub":
            new.flux = self.flux - other
        elif op == "mul":
            new.flux = self.flux * other
            new.flux_err = self.flux_err * abs(other)
        else:
            new.flux = self.flux / other
            new.flux_err = self.flux_err / abs(other)
        return new

    def __add__(self, other):
        return self._binop(other, "add")

    __radd__ = __add__

    def __sub__(self, other):
        return self._binop(other, "sub")

    def __rsub__(self, other):
        return (-1 * self).__add__(other)

    def __mul__(self, other):
        return self._binop(other, "mul")

    __rmul__ = __mul__

    def __truediv__(self, other):
        return self._binop(other, "div")

    # ------------------------------------------------------------------ cleaning
    def remove_nans(self, column="flux"):
        """Removes cadences where ``column`` is a NaN (lightcurve.py:1300-1327)."""
        return self[~np.isnan(np.asarray(getattr(self, column).value))]

    def normalize(self, unit="unscaled"):
        """Divide flux and flux_err by the median flux (lightcurve.py:1216-1298).
        The median/std are batched-select kernel results (K6)."""
        validate_method(unit, ["unscaled", "percent", "ppt", "ppm"])
        from . import engine
        med, sd = engine.nanmedian_std([np.asarray(self.flux.value, dtype=np.float64)])
        median_flux, std_flux = float(med[0]), float(sd[0])
        _normalize_warnings(median_flux, std_flux)
        lc = self.copy()
        with np.errstate(divide="ignore", invalid="ignore"):
            lc.flux = Quantity(self.flux.value / median_flux, u.dimensionless_unscaled)
            lc.flux_err = Quantity(self.flux_err.value / median_flux, u.dimensionless_unscaled)
        if unit == "percent":
            lc.flux, lc.flux_err = lc.flux.to(u.percent), lc.flux_err.to(u.percent)
        elif unit in ("ppt", "ppm"):
            lc.flux, lc.flux_err = lc.flux.to(unit), lc.flux_err.to(unit)
        lc.meta["NORMALIZED"] = True
        return lc

    def bin(self, time_bin_size=None, time_bin_start=None, time_bin_end=None, n_bins=None, aggregate_func=None,
            bins=None, binsize=None):
        """Bin the light curve in time (lightcurve.py:1558-1763, a wrapper of astropy's `aggregate_downsample`).

        Bins are half-open intervals [start, end) in time, the last one closed; `flux` is aggregated with
        `aggregate_func` (default `numpy.nanmean`), `flux_err` combines as the root mean square of the errors in a
        bin (or, without errors, is the standard deviation of the binned fluxes); a bin's time is its centre and
        bins that hold no cadence come out as NaN.  `time_bin_size` is in days (default 0.5), `time_bin_start`
        defaults to the first cadence, `n_bins` to the number needed to reach the last one.  The v1.x keywords:
        `binsize` = a new bin every `binsize` cadences, `bins` = a number of equal-width bins or an array of cadence
        indices of the bin edges (astropy's adaptive rules "blocks"/"knuth"/"scott"/"freedman" are not available
        here).  O(N) host code, like the reference's."""
        aggregate_func = _bin_check_args(time_bin_size, n_bins, aggregate_func, bins, binsize)
        order = np.argsort(np.asarray(self.time.value, dtype=np.float64), kind="stable")
        t = np.asarray(self.time.value, dtype=np.float64)[order]
        f = np.asarray(self.flux.value, dtype=np.float64)[order]
        fe = np.asarray(self.flux_err.value, dtype=np.float64)[order]
        if len(t) == 0:
            return self.copy()
        kind, starts, ends = _bin_edges(len(t), t[0], t[-1], time_bin_size, time_bin_start, time_bin_end, n_bins,
                                        bins, binsize)
        if kind == "index":
            starts, ends = t[starts], t[ends]
        nb = len(starts)
        which = np.searchsorted(starts, t, side="right") - 1                  # last bin starting at or before t
        inside = (which >= 0) & ((t < ends[np.clip(which, 0, nb - 1)]) | ((which == nb - 1) & (t <= ends[-1])))
        bflux = np.full(nb, np.nan)
        berr = np.full(nb, np.nan)
        have_err = bool(np.any(np.isfinite(fe)))
        with warnings.catch_warnings(), np.errstate(all="ignore"):
            warnings.simplefilter("ignore", RuntimeWarning)
            for j in np.unique(which[inside]):
                sel = inside & (which == j)
                bflux[j] = aggregate_func(f[sel])
                if have_err:
                    e = fe[sel]
                    berr[j] = np.sqrt(np.nansum(e ** 2) / np.sum(np.isfinite(e))) if np.any(np.isfinite(e)) else np.nan
                else:
                    v = f[sel]
                    berr[j] = np.nanstd(v) if np.any(np.isfinite(v)) else np.nan
        return self._binned(starts + 0.5 * (ends - starts), bflux, berr)

    def _binned(self, centres, bflux, berr):
        """The light curve of bin centres, aggregated flux and errors that `bin` returns."""
        new = self.__class__.__new__(self.__class__)
        new.meta = _copy.deepcopy(self.meta)
        new._columns = {}
        if isinstance(self.time, Time):
            new.time = Time(centres, self.time.format, self.time.scale)
        else:                                                   # a folded light curve: "time" is the phase
            new.time = Quantity(centres, self.time.unit)
        new.flux = Quantity(bflux, self.flux.unit)
        new.flux_err = Quantity(berr, self.flux_err.unit)
        return new

    def remove_outliers(self, sigma=5.0, sigma_lower=None, sigma_upper=None, return_mask=False, column="flux", **kwargs):
        """Sigma-clip outliers of `column` (lightcurve.py:1429-1549; astropy sigma_clip defaults:
        maxiters=5, median centre, std).  Centre/spread come from the GPU select kernel; of astropy's further
        ``sigma_clip`` keywords only ``maxiters`` and the defaults ``cenfunc="median"`` / ``stdfunc="std"`` are
        implemented - anything else raises instead of being silently ignored."""
        from . import engine
        maxiters = kwargs.pop("maxiters", 5)
        if kwargs.pop("cenfunc", "median") not in ("median", np.median, np.nanmedian) or \
                kwargs.pop("stdfunc", "std") not in ("std", np.std, np.nanstd):
            raise NotImplementedError("remove_outliers(): only cenfunc='median' and stdfunc='std' run on the GPU kernel")
        if kwargs:
            raise TypeError("remove_outliers(): unsupported sigma_clip keyword(s) %s" % sorted(kwargs))
        lo_s = sigma if sigma_lower is None else sigma_lower
        hi_s = sigma if sigma_upper is None else sigma_upper
        col = getattr(self, column)
        data = np.array(getattr(col, "value", col), dtype=np.float64)
        mask = ~np.isfinite(data)
        it = 0
        while maxiters is None or it < maxiters:
            it += 1
            work = np.where(mask, np.nan, data)
            if np.isnan(work).all():
                break
            med, sd = engine.nanmedian_std([work])
            with np.errstate(invalid="ignore"):
                new = mask | (data < med[0] - sd[0] * lo_s) | (data > med[0] + sd[0] * hi_s)
            if new.sum() == mask.sum():
                break
            mask = new
        if return_mask:
            return self[~mask], mask
        return self[~mask]

    # ------------------------------------------------------------------ hot path: flatten
    def flatten(self, window_length=101, polyorder=2, return_trend=False, break_tolerance=5, niters=3, sigma=3,
                mask=None, **kwargs):
        """Removes the low frequency trend with a Savitzky-Golay filter (lightcurve.py:943-1078).

        Same parameters as the reference.  ``mask`` True = cadence NOT used for the fit.  The
        whole loop (sigma-clip pre-mask, gap segmentation, savgol, residual clip, interp1d) runs
        in the CUDA kernel ``lkb_flatten``; extra ``**kwargs`` for scipy's savgol_filter are not
        supported (the kernel implements the reference's own call: mode="interp", deriv=0).
        """
        if kwargs:
            raise TypeError("flatten(): unsupported savgol_filter keyword(s) %s" % sorted(kwargs))
        from . import engine
        if polyorder >= window_length:
            polyorder = window_length - 1
            log.warning("polyorder must be smaller than window_length, "
                        "using polyorder={}.".format(polyorder))
        t = np.asarray(self.time.value, dtype=np.float64)
        f = np.asarray(self.flux.value)
        out_dtype = f.dtype if f.dtype == np.float32 else np.float64
        m = None if mask is None else [np.asarray(mask, dtype=bool)]
        flat, flat_err, trend = engine.flatten([t], [f.astype(np.float64)],
                                               [np.asarray(self.flux_err.value, dtype=np.float64)], m,
                                               window_length=window_length, polyorder=polyorder,
                                               break_tolerance=break_tolerance, niters=niters, sigma=sigma)
        return self._wrap_flatten(flat[0].astype(out_dtype), flat_err[0].astype(out_dtype),
                                  trend[0].astype(out_dtype), return_trend)

    def _wrap_flatten(self, flat, flat_err, trend, return_trend):
        flatten_lc = self.copy()
        flatten_lc.flux = Quantity(flat, u.dimensionless_unscaled)
        flatten_lc.flux_err = Quantity(flat_err, u.dimensionless_unscaled)
        flatten_lc.meta["NORMALIZED"] = True
        if return_trend:
            trend_lc = self.copy()
            trend_lc.flux = Quantity(trend, self.flux.unit)
            return flatten_lc, trend_lc
        return flatten_lc

    def estimate_cdpp(self, transit_duration=13, savgol_window=101, savgol_polyorder=2, sigma=5.0):
        """Savitzky-Golay CDPP noise metric in ppm (lightcurve.py:1764-1833)."""
        if not isinstance(transit_duration, int):
            raise ValueError(
                "transit_duration must be an integer in units "
                "number of cadences, got {}.".format(transit_duration)
            )
        detrended_lc = self.flatten(window_length=savgol_window, polyorder=savgol_polyorder)
        cleaned_lc = detrended_lc.remove_outliers(sigma=sigma)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", LightkurveWarning)
            normalized_lc = cleaned_lc.normalize("ppm")
        mean = running_mean(data=np.asarray(normalized_lc.flux.value), window_size=transit_duration)
        return Quantity(np.std(mean), u.ppm)

    # ------------------------------------------------------------------ hot path: periodograms
    def to_periodogram(self, method="lombscargle", **kwargs):
        """Converts the light curve to a Periodogram (lightcurve.py:2490-2535).
        method : {'lombscargle', 'boxleastsquares', 'ls', 'bls'}"""
        supported_methods = ["ls", "bls", "lombscargle", "boxleastsquares"]
        method = validate_method(method.replace(" ", ""), supported_methods)
        if method in ["bls", "boxleastsquares"]:
            from .periodogram import BoxLeastSquaresPeriodogram
            return BoxLeastSquaresPeriodogram.from_lightcurve(lc=self, **kwargs)
        from .periodogram import LombScarglePeriodogram
        return LombScarglePeriodogram.from_lightcurve(lc=self, **kwargs)

    def to_seismology(self, **kwargs):
        """`Seismology` object for estimating numax, deltanu, radius, mass, logg (lightcurve.py:2537-2550);
        `kwargs` go to `to_periodogram`."""
        from .seismology import Seismology
        return Seismology.from_lightcurve(self, **kwargs)

    def fill_gaps(self, method="gaussian_noise"):
        """Fill gaps in time with white Gaussian noise N(mean flux, CDPP) (lightcurve.py:1329-1427; the variant for
        light curves without a cadence-number column): cadences are inserted every median time step wherever two
        consecutive times are more than 1.2 steps apart; their flux_err is interpolated.  The noise comes from
        numpy's global RNG, as in the reference."""
        lc = self.copy().remove_nans()
        tval = np.asarray(lc.time.value, dtype=np.float64)
        if len(tval) < 2:
            return lc
        dt = np.nanmedian(tval[1:] - tval[:-1])
        ntime = [tval[0]]
        for t in tval[1:]:
            prevtime = ntime[-1]
            while (t - prevtime) > 1.2 * dt:
                ntime.append(prevtime + dt)
                prevtime = ntime[-1]
            ntime.append(t)
        ntime = np.asarray(ntime, float)
        in_original = np.isin(ntime, tval)
        f = np.zeros(len(ntime))
        f[in_original] = np.asarray(lc.flux.value, dtype=np.float64)
        fe = np.zeros(len(ntime))
        fe[in_original] = np.asarray(lc.flux_err.value, dtype=np.float64)
        fe[~in_original] = np.interp(ntime[~in_original], tval, np.asarray(lc.flux_err.value, dtype=np.float64))
        if method == "gaussian_noise":
            try:
                std = float(lc.estimate_cdpp().to(lc.flux.unit).value)
            except Exception:
                std = np.nanstd(lc.flux.value)
            f[~in_original] = np.random.normal(np.nanmean(lc.flux.value), std, (~in_original).sum())
        else:
            raise NotImplementedError("No such method as {}".format(method))
        return LightCurve(time=Time(ntime, lc.time.format, lc.time.scale), flux=Quantity(f, lc.flux.unit),
                          flux_err=Quantity(fe, lc.flux_err.unit), meta=self.meta)

    def append(self, others, inplace=False):
        """Concatenate light curves in the order given (lightcurve.py:915-941)."""
        if inplace:
            raise ValueError("the `inplace` parameter is no longer supported "
                             "as of Lightkurve v2.0")
        if not hasattr(others, "__iter__"):
            others = (others,)
        lcs = [self] + list(others)
        new = self.copy()
        new.time = Time(np.concatenate([np.asarray(lc.time.value) for lc in lcs]), self.time.format, self.time.scale)
        new.flux = Quantity(np.concatenate([np.asarray(lc.flux.to(self.flux.unit).value) for lc in lcs]), self.flux.unit)
        new.flux_err = Quantity(np.concatenate([np.asarray(lc.flux_err.to(self.flux.unit).value) for lc in lcs]),
                                self.flux.unit)
        shared = set(self.__dict__.get("_columns", {}))
        for lc in lcs[1:]:
            shared &= set(lc.__dict__.get("_columns", {}))
        new._columns = {k: np.concatenate([lc._columns[k] for lc in lcs]) for k in shared}
        return new

    def to_corrector(self, method="regression", **kwargs):
        """Returns a corrector object (lightcurve.py:2732); only 'regression' is in scope."""
        method = validate_method(method, ["regression"])
        from .correctors import RegressionCorrector
        return RegressionCorrector(self, **kwargs)

    # ------------------------------------------------------------------ fold (the step after a period search)
    def fold(self, period=None, epoch_time=None, epoch_phase=0, wrap_phase=None, normalize_phase=False):
        """Returns a `FoldedLightCurve` folded on a period and epoch (lightcurve.py:1089-1214, which wraps
        astropy TimeSeries.fold): phase = ((t - epoch_time) + epoch_phase + (P - wrap)) % P - (P - wrap),
        sorted by phase; a bare float period / epoch_phase is in days."""
        t = np.asarray(self.time.value, dtype=np.float64)
        per, t0, shift, wrap, jd_warning = _fold_params(t, self.time, period, epoch_time, epoch_phase, wrap_phase,
                                                        normalize_phase)
        if jd_warning:
            warnings.warn(jd_warning, LightkurveWarning)
        rel = ((t - t0) + shift + (per - wrap)) % per - (per - wrap)
        order = np.argsort(rel, kind="stable")
        phase = rel[order] / per if normalize_phase else rel[order]
        return self._folded(t, order, phase, per, t0, epoch_time, epoch_phase, wrap_phase, normalize_phase)

    def _folded(self, t, order, phase, per, t0, epoch_time, epoch_phase, wrap_phase, normalize_phase):
        """The `FoldedLightCurve` of the cadences in `order` at the sorted `phase` that `fold` returns."""
        folded = FoldedLightCurve.__new__(FoldedLightCurve)
        folded.meta = _copy.deepcopy(self.meta)
        folded.time = Quantity(phase, u.dimensionless_unscaled if normalize_phase else u.day)
        folded.flux = Quantity(np.asarray(self.flux.value)[order], self.flux.unit, dtype=self.flux.dtype)
        folded.flux_err = Quantity(np.asarray(self.flux_err.value)[order], self.flux_err.unit, dtype=self.flux_err.dtype)
        folded.time_original = Time(t[order], self.time.format, self.time.scale)
        folded._columns = {k: v[order] for k, v in self.__dict__.get("_columns", {}).items()}
        folded.meta["PERIOD"] = Quantity(per, u.day)
        folded.meta["EPOCH_TIME"] = None if epoch_time is None else Time(t0, self.time.format, self.time.scale)
        folded.meta["EPOCH_PHASE"] = epoch_phase
        folded.meta["WRAP_PHASE"] = wrap_phase
        folded.meta["NORMALIZE_PHASE"] = normalize_phase
        return folded

    # ------------------------------------------------------------------ BLS follow-ups (host-side, cheap)
    def create_transit_mask(self, period, transit_time, duration):
        """True for in-transit cadences (lightcurve.py:2967-3037)."""
        period = np.atleast_1d(getattr(period, "value", period)).astype(float)
        duration = np.atleast_1d(getattr(duration, "value", duration)).astype(float)
        transit_time = np.atleast_1d(getattr(transit_time, "value", transit_time)).astype(float)
        t = np.asarray(self.time.value, dtype=float)
        in_transit = np.zeros(len(t), dtype=bool)
        for per, dur, t0 in zip(period, duration, transit_time):
            hp = per * 0.5
            in_transit |= np.abs((t - t0 + hp) % per - hp) < 0.5 * dur
        return in_transit


class FoldedLightCurve(LightCurve):
    """A light curve folded on a period (lightcurve.py:3166-3300): ``time`` holds the phase."""

    @property
    def phase(self):
        return self.time

    @property
    def period(self):
        return self.meta.get("PERIOD")

    @property
    def epoch_time(self):
        return self.meta.get("EPOCH_TIME")

    @property
    def cycle(self):
        """The cycle of each data point; the first one is cycle 0 whether it is complete or not
        (lightcurve.py:3213-3229).  Cycle boundaries sit half a period before `epoch_time`; without an explicit
        epoch the reference takes the smallest folded phase as the epoch - reproduced as is."""
        per = float(np.asarray(self.period.value))
        t = np.asarray(self.time_original.value, dtype=np.float64)
        ep = self.epoch_time
        if ep is None:
            ph_min = float(np.min(np.asarray(self.time.value)))
            t0 = ph_min * per if self.meta.get("NORMALIZE_PHASE") else ph_min
        else:
            t0 = float(np.asarray(ep.value))
        result = np.asarray(np.floor((t - (t0 - per / 2.0)) / per), dtype=int)
        return result - result.min()

    @property
    def odd_mask(self):
        """Boolean mask of the odd-numbered cycles (1, 3, 5, ...) (lightcurve.py:3231-3250)."""
        return self.cycle % 2 == 1

    @property
    def even_mask(self):
        """Boolean mask of the even-numbered cycles (0, 2, 4, ...)."""
        return ~self.odd_mask

    def __repr__(self):
        return "<FoldedLightCurve length={} period={}>".format(len(self), self.period)
