"""`LightCurveCollection`: /root/reference/src/lightkurve/collections.py:18-276 (list semantics)
plus the batch methods the reference lacks (SURVEY.md F6): ``to_periodogram`` and ``flatten``
over the whole collection in ONE kernel launch sequence.  Their contract is "identical to
``[lc.method(...) for lc in collection]``" - the per-light-curve preparation code is literally
the same functions (``LombScarglePeriodogram._prepare`` etc.); only the device call is batched.
"""
import logging
import math

import numpy as np

from .lightcurve import LightCurve

log = logging.getLogger(__name__)

__all__ = ["Collection", "LightCurveCollection"]


class Collection(object):
    """List-like container with numpy-style indexing (collections.py:18-142)."""

    def __init__(self, data):
        if data is not None:
            self.data = [item for item in data]
        else:
            self.data = []

    def __len__(self):
        return len(self.data)

    def __getitem__(self, index_or_mask):
        if isinstance(index_or_mask, (int, np.integer, slice)):
            res = self.data[index_or_mask]
            return type(self)(res) if isinstance(index_or_mask, slice) else res
        if all(isinstance(i, (bool, np.bool_)) for i in index_or_mask):
            if len(index_or_mask) != len(self.data):
                raise IndexError("boolean mask length does not match the collection")
            return type(self)([self.data[i] for i in np.nonzero(index_or_mask)[0]])
        return type(self)([self.data[i] for i in index_or_mask])

    def __setitem__(self, index, obj):
        self.data[index] = obj

    def append(self, obj):
        self.data.append(obj)

    def __iter__(self):
        return iter(self.data)

    def __repr__(self):
        return "{} of {} objects".format(type(self).__name__, len(self.data))


class LightCurveCollection(Collection):
    """Collection of LightCurve objects (collections.py:145-276)."""

    def __init__(self, lightcurves):
        super().__init__(lightcurves)
        for lc in self.data:
            if not isinstance(lc, LightCurve):
                raise TypeError("LightCurveCollection needs LightCurve objects")

    # ---- batched hot path (new API; == per-LC loop) -----------------------------------------
    def to_periodogram(self, method="lombscargle", **kwargs):
        """Batched ``LightCurve.to_periodogram``: returns a list of Periodogram objects."""
        from .periodogram import LombScarglePeriodogram, BoxLeastSquaresPeriodogram
        from .utils import validate_method
        from . import engine
        from . import units as u
        method = validate_method(method.replace(" ", ""), ["ls", "bls", "lombscargle", "boxleastsquares"])
        if len(self.data) == 0:
            return []
        if method in ("bls", "boxleastsquares"):
            # one engine call: the shared-grid entry when every light curve has the same grid, else per-light-curve
            # grids; light curves without usable flux_err get unit weights (bitwise the weights of dy=None)
            preps = [BoxLeastSquaresPeriodogram._prepare(lc, **dict(kwargs)) for lc in self.data]
            p0 = preps[0]
            same = all(len(p["period"]) == len(p0["period"]) and np.array_equal(p["period"], p0["period"])
                       for p in preps)
            dys = None
            if any(p["dy"] is not None for p in preps):
                dys = [np.ones(len(p["time"])) if p["dy"] is None else p["dy"] for p in preps]
            res = engine.bls_power([p["time"] for p in preps], [p["flux"] for p in preps], dys,
                                   p0["period"] if same else [p["period"] for p in preps], p0["duration"],
                                   oversample=p0["oversample"], objective=p0["objective"])
            out = []
            for b, p in enumerate(preps):
                pg = BoxLeastSquaresPeriodogram._finish(p, res, b)
                pg._dy = p["dy"]
                out.append(pg)
            return out
        preps = [LombScarglePeriodogram._prepare(lc, **dict(kwargs)) for lc in self.data]
        p0 = preps[0]
        norm, _ = LombScarglePeriodogram._norm_args(p0)
        freqs = [np.asarray(p["frequency"].to(1 / u.day).value, dtype=np.float64) for p in preps]
        scales = [LombScarglePeriodogram._norm_args(p)[1] for p in preps]
        shared_t = all(len(p["time"]) == len(p0["time"]) and np.array_equal(p["time"], p0["time"]) for p in preps)
        shared_f = all(len(f) == len(freqs[0]) and np.array_equal(f, freqs[0]) for f in freqs)
        if p0["ls_method"] in ("chi2", "fastchi2", "fastnifty_chi2"):
            fl = [np.asarray(p["lc"].flux.value) for p in preps]
            fl = [f if f.dtype == np.float32 else f.astype(np.float64) for f in fl]
            powers = engine.ls_power_chi2([p["time"] for p in preps], fl, freqs[0] if shared_f else freqs,
                                          p0["nterms"], norm, None if norm != "psd" else scales)
        elif shared_t and shared_f and len(preps) > 1:
            Y = np.stack([np.asarray(p["lc"].flux.value) for p in preps])
            if Y.dtype != np.float32:
                Y = Y.astype(np.float64)
            algo = {"direct": "simt"}.get(LombScarglePeriodogram._engine_algo(p0["ls_method"]),
                                          LombScarglePeriodogram._engine_algo(p0["ls_method"]))
            try:
                powers = engine.ls_power_shared(p0["time"], Y, freqs[0], norm, scales[0], algo=algo)
            except Exception as e:
                if algo != "nufft" or getattr(e, "status", None) != -5:          # LKB_E_UNSUPPORTED
                    raise
                powers = engine.ls_power_shared(p0["time"], Y, freqs[0], norm, scales[0], algo="auto")
        else:
            fl = [np.asarray(p["lc"].flux.value) for p in preps]
            fl = [f if f.dtype == np.float32 else f.astype(np.float64) for f in fl]
            powers = LombScarglePeriodogram._ragged_power(engine, [p["time"] for p in preps], fl,
                                                          freqs[0] if shared_f else freqs, norm,
                                                          None if norm != "psd" else scales, p0["ls_method"])
        return [LombScarglePeriodogram._finish(p, powers[b]) for b, p in enumerate(preps)]

    def find_transit_candidates(self, n_candidates=3, return_stats=False, **kwargs):
        """Search every light curve for `n_candidates` transiting planets, one after the other, in one GPU call (K3,
        K14, K10, K6; ``engine.bls_find_candidates``).  For each light curve it equals this loop, from
        ``lc = lc.remove_nans()``, repeated `n_candidates` times::

            pg = lc.to_periodogram("bls", **kwargs)
            P, D, T0 = pg.period_at_max_power, pg.duration_at_max_power, pg.transit_time_at_max_power
            # record P, D, T0 and the depth, depth error, depth_snr and power at max power
            lc = lc[~pg.get_transit_mask(period=P, duration=D, transit_time=T0)]

        `kwargs` are those of ``to_periodogram("bls")`` (duration, period, minimum_period, maximum_period,
        frequency_factor, time_unit, objective, oversample) and apply in every round; without `period` each round's
        grid follows from the survivors of the round before.  Every light curve gets `n_candidates` rounds; filter on
        ``depth_snr`` to keep the significant ones.  A box that covers every cadence removes none, so the next round
        finds it again, as the loop does.

        Returns a dict: "period", "duration", "transit_time", "depth", "depth_err", "depth_snr", "power", float64
        arrays [B, n_candidates] in each light curve's units (time_unit for period and duration, its time format for
        transit_time, its flux unit for the depths); "masked_in", one int8 array per ``lc.remove_nans()``: the round
        whose mask removed the cadence, -1 if none, so that ``lc.remove_nans()[masked_in[b] == -1]`` is the loop's
        last light curve; with `return_stats`, "stats": for each light curve a list of the `n_candidates` dicts of
        ``pg.compute_stats(P, D, T0)`` (equal to the loop's to the rounding of ``compute_stats_batch``).

        Errors are those of the loop, of the same type, for the first light curve and round at which the loop would
        raise, naming both.  Times must be finite.  At most 65 535 light curves."""
        from types import SimpleNamespace
        from . import engine
        from .periodogram import BoxLeastSquaresPeriodogram as BLS
        n_candidates = int(n_candidates)
        if not 1 <= n_candidates <= 127:
            raise ValueError("n_candidates must be in 1 .. 127, got {}".format(n_candidates))
        lcs = [lc.remove_nans() for lc in self.data]
        B = len(lcs)
        if B == 0:
            out = {k: np.zeros((0, n_candidates)) for k in engine.BLS_CANDIDATE_FIELDS}
            out["masked_in"] = []
            if return_stats:
                out["stats"] = []
            return out
        times = [np.asarray(lc.time.value, dtype=np.float64) for lc in lcs]
        for b, t in enumerate(times):
            if not np.isfinite(t).all():
                raise ValueError("light curve {} has non-finite times".format(b))
        shared = kwargs.get("period", None) is not None

        def grid(b, r, tmin, tmax, median_dt):
            return BLS._grid(tmin, tmax, median_dt, **dict(kwargs))

        res = engine.bls_find_candidates(times, [np.asarray(lc.flux.value, dtype=np.float64) for lc in lcs],
                                         [np.asarray(lc.flux_err.value, dtype=np.float64) for lc in lcs], grid,
                                         n_candidates, shared_grid=shared, return_stats=return_stats)
        if return_stats:
            owners = [SimpleNamespace(flux=lc.flux, time=lc.time) for lc in lcs]
            res["stats"] = [[BLS._k10_stats_dict(owners[b], rs["tstart"][b], res["period"][b, r],
                                                 res["transit_time"][b, r], rs, b)
                             for r, rs in enumerate(res["stats"])] for b in range(B)]
        return res

    def fill_gaps(self, method="gaussian_noise"):
        """Batched ``LightCurve.fill_gaps``: for the same ``np.random`` state, equal to
        ``LightCurveCollection([lc.fill_gaps() for lc in collection])``, and it leaves the global RNG where that loop
        leaves it.  The gap plan, the CDPP noise levels and the filled light curves come from one GPU call (K15, K6,
        K4/K11/K12; ``engine.fill_gaps_device``); the host draws the normal deviates once, in collection order.

        Times, flux_err and the flux of original cadences are bitwise the loop's.  Inserted flux is
        ``nanmean(flux) + std * z`` with `std` the CDPP of ``lkb_cdpp`` (within about 1e-8 relative of the single
        ``estimate_cdpp``) converted to the flux unit, or ``nanstd(flux)`` where ``estimate_cdpp().to(flux.unit)``
        raises; for a light curve of two or more finite cadences that happens only when the flux unit cannot be
        converted from ppm (for example electron/s).  The mean is a plain sum, so it may differ from numpy's pairwise
        one in the last bits.  Float32 flux is worked in float64.

        Raises ValueError, naming the light curve, for input the loop cannot handle: non-finite times, times that
        decrease once the NaN fluxes are removed (the loop would then mis-assign the flux), a median time step <= 0
        with some positive step (the loop would never end), and a gap of more than 2**24 median steps."""
        from . import engine
        from . import units as u
        from .units import Quantity, Time
        if method != "gaussian_noise":
            raise NotImplementedError("No such method as {}".format(method))
        if not self.data:
            return LightCurveCollection([])
        lcs = [lc.copy().remove_nans() for lc in self.data]
        times = [np.asarray(lc.time.value, dtype=np.float64) for lc in lcs]
        _check_finite_times(times)
        fluxes = [np.asarray(lc.flux.value, dtype=np.float64) for lc in lcs]
        errs = [np.asarray(lc.flux_err.value, dtype=np.float64) for lc in lcs]

        def std(cdpp_ppm):
            out = np.zeros(len(lcs))
            for b, lc in enumerate(lcs):
                if len(fluxes[b]) < 2:
                    continue
                try:
                    out[b] = float(Quantity(cdpp_ppm[b], u.ppm).to(lc.flux.unit).value)
                except Exception:                     # noqa: BLE001 - the single method's fallback
                    out[b] = np.nanstd(fluxes[b])
            return out

        tt, yy, ee = engine.fill_gaps(times, fluxes, errs, std)
        out = []
        for b, lc in enumerate(lcs):
            if len(times[b]) < 2:
                out.append(lc)
                continue
            out.append(LightCurve(time=Time(tt[b], lc.time.format, lc.time.scale), flux=Quantity(yy[b], lc.flux.unit),
                                  flux_err=Quantity(ee[b], lc.flux_err.unit), meta=self.data[b].meta))
        return LightCurveCollection(out)

    def to_seismology(self, **kwargs):
        """Batched ``LightCurve.to_seismology``: a list of `Seismology` objects whose element b, for the same
        ``np.random`` state, equals ``Seismology.from_lightcurve(lc_b, **kwargs)``, i.e. the SNR spectrum of
        ``lc.normalize().remove_nans().fill_gaps().to_periodogram(**kwargs).flatten()``.  The whole chain runs in one
        GPU call (``engine.seismology_spectra``): the raw light curves are uploaded once, normalized and cleared of
        NaN fluxes on the device, and only arrays of one value per light curve and the final spectra come back.  The
        next step is the batch estimators, e.g.::

            seis = coll.to_seismology(normalization="psd")
            numax = estimate_numax_acf2d_batch([s.periodogram for s in seis])

        `kwargs` are those of ``to_periodogram("lombscargle")`` (normalization, minimum_frequency /
        maximum_frequency, minimum_period / maximum_period, frequency / period, oversample_factor, nyquist_factor,
        freq_unit, nterms, ls_method ...).  Each light curve has its own grid, so the power comes from the exact
        direct sums (``lkb_ls_power``; ``lkb_ls_power_chi2`` for the multi-term methods "chi2", "fastchi2" and
        "fastnifty_chi2"), which agree with the single call's kernels to the Lomb-Scargle parity tolerance.  The
        normalization's median is the single ``normalize``'s K6 value and the division is IEEE fp64, so both are
        bitwise the loop's; the inserted flux follows `LightCurveCollection.fill_gaps`.  Float32 flux is worked in
        float64.

        The `from_lightcurve` info message is logged once per call; ``normalize``'s warnings are raised for every
        light curve that triggers them.  Errors: non-finite times among the kept cadences, then fill_gaps' refusals
        (ValueError), then the loop's first periodogram error, of the same type, naming the light curve.  At most
        65 535 light curves.  An empty collection returns []."""
        from . import engine
        from . import units as u
        from .lightcurve import _normalize_warnings
        from .periodogram import LombScarglePeriodogram as LS, SNRPeriodogram
        from .seismology import Seismology
        from .units import Quantity
        if not self.data:
            return []
        logging.getLogger("lightkurve_b200.seismology").info(
            "Building a Seismology object directly from a light curve "
            "uses default periodogram parameters. For further tuneability, "
            "create a periodogram object first, using `to_periodogram`.")
        B = len(self.data)
        preps = [None] * B

        def warn(med, sd):
            for b in range(B):
                _normalize_warnings(float(med[b]), float(sd[b]))

        def grid(b, median_dt, t_first, t_last, n):
            empty = np.zeros(0)
            span = (lambda: (np.median(np.diff(empty)), empty[-1], empty[0])) if n == 0 else \
                (lambda: (np.float64(median_dt), np.float64(t_first), np.float64(t_last)))
            try:
                p = LS._grid(span, **dict(kwargs))
                freq = np.asarray(p["frequency"].value, dtype=np.float64)
                if len(freq) <= 1:
                    raise ValueError("frequency and power must have a length greater than 1.")
            except Exception as e:
                raise _named(e, b) from e
            preps[b] = p
            scale = 2.0 / (n * p["oversample_factor"] * float(p["fs"].value)) if p["normalization"] == "psd" else None
            return dict(frequency=np.asarray(p["frequency"].to(1 / u.day).value, dtype=np.float64), freq=freq,
                        scale=scale, normalization=p["normalization"], nterms=p["nterms"],
                        multiterm=p["ls_method"] in ("chi2", "fastchi2", "fastnifty_chi2"))

        snr = engine.seismology_spectra([np.asarray(lc.time.value, dtype=np.float64) for lc in self.data],
                                        [np.asarray(lc.flux.value, dtype=np.float64) for lc in self.data],
                                        [np.asarray(lc.flux_err.value, dtype=np.float64) for lc in self.data], grid,
                                        on_median=warn)
        out = []
        for b, lc in enumerate(self.data):
            p = preps[b]
            pu = u.dimensionless_unscaled if p["normalization"] == "amplitude" else \
                u.dimensionless_unscaled ** 2 / p["freq_unit"]
            unit = (Quantity(np.ones(1), pu) / Quantity(np.ones(1), pu)).unit
            meta = dict(lc.copy(copy_data=False).meta)
            meta["NORMALIZED"] = True
            pg = SNRPeriodogram(p["frequency"], Quantity(snr[b], unit), nyquist=p["nyquist"],
                                targetid=meta.get("TARGETID"), label=meta.get("LABEL"), meta=meta)
            out.append(Seismology(pg))
        return out

    def flatten(self, window_length=101, polyorder=2, return_trend=False, break_tolerance=5, niters=3, sigma=3,
                mask=None):
        """Batched ``LightCurve.flatten``; `mask` is None or a list of per-LC boolean masks."""
        from . import engine
        if len(self.data) == 0:
            return LightCurveCollection([])
        if polyorder >= window_length:
            polyorder = window_length - 1
        times = [np.asarray(lc.time.value, dtype=np.float64) for lc in self.data]
        fluxes = [np.asarray(lc.flux.value, dtype=np.float64) for lc in self.data]
        errs = [np.asarray(lc.flux_err.value, dtype=np.float64) for lc in self.data]
        masks = None
        if mask is not None:
            masks = [np.zeros(len(t), bool) if m is None else np.asarray(m, dtype=bool) for t, m in zip(times, mask)]
        flat, flat_err, trend = engine.flatten(times, fluxes, errs, masks, window_length=window_length,
                                               polyorder=polyorder, break_tolerance=break_tolerance, niters=niters,
                                               sigma=sigma)
        flats, trends = [], []
        for b, lc in enumerate(self.data):
            dt = lc.flux.dtype if lc.flux.dtype == np.float32 else np.float64
            r = lc._wrap_flatten(flat[b].astype(dt), flat_err[b].astype(dt), trend[b].astype(dt), return_trend)
            if return_trend:
                flats.append(r[0])
                trends.append(r[1])
            else:
                flats.append(r)
        if return_trend:
            return LightCurveCollection(flats), LightCurveCollection(trends)
        return LightCurveCollection(flats)

    def remove_outliers(self, sigma=5.0, sigma_lower=None, sigma_upper=None, return_mask=False, column="flux",
                        maxiters=5, **kwargs):
        """Batched ``LightCurve.remove_outliers``: equal to ``[lc.remove_outliers(...) for lc in collection]``, with
        every clip round of every light curve in one GPU call (K11, ``engine.sigma_clip``).  ``maxiters=None`` clips
        until a round clips nothing.  Returns a LightCurveCollection and, with ``return_mask``, the list of boolean
        masks (True = removed).  Of astropy's further ``sigma_clip`` keywords only the defaults ``cenfunc="median"``
        and ``stdfunc="std"`` are accepted; anything else raises, as in the single-curve method."""
        from . import engine
        if kwargs.pop("cenfunc", "median") not in ("median", np.median, np.nanmedian) or \
                kwargs.pop("stdfunc", "std") not in ("std", np.std, np.nanstd):
            raise NotImplementedError("remove_outliers(): only cenfunc='median' and stdfunc='std' run on the GPU kernel")
        if kwargs:
            raise TypeError("remove_outliers(): unsupported sigma_clip keyword(s) %s" % sorted(kwargs))
        lo_s = sigma if sigma_lower is None else sigma_lower
        hi_s = sigma if sigma_upper is None else sigma_upper
        # the single-curve loop runs `while it < maxiters`: a fractional maxiters rounds up, a negative one clips nothing
        mi = -1 if maxiters is None else max(0, math.ceil(maxiters))
        cols = []
        for lc in self.data:
            col = getattr(lc, column)
            cols.append(np.array(getattr(col, "value", col), dtype=np.float64))
        masks = engine.sigma_clip(cols, float(lo_s), float(hi_s), mi)["mask"] if cols else []
        out = LightCurveCollection([lc[~m] for lc, m in zip(self.data, masks)])
        if return_mask:
            return out, [np.array(m, dtype=bool) for m in masks]
        return out

    def estimate_cdpp(self, transit_duration=13, savgol_window=101, savgol_polyorder=2, sigma=5.0):
        """Batched ``LightCurve.estimate_cdpp``: the Savitzky-Golay CDPP of every light curve in ppm, from one GPU call
        (K4 flatten, K11 remove_outliers, K12 normalize and running-mean scatter; ``engine.cdpp``) in which the
        flattened flux never leaves the device.  Returns a Quantity of shape [B].  ``transit_duration`` may also be a
        sequence of ints: the CDPP at each of them, shape [B, D], from the same call.

        Equals ``[lc.estimate_cdpp(...) for lc in collection]`` for float64 flux.  Float32 flux is worked in float64
        throughout, which equals the loop on a float64 copy; the single-curve method instead keeps float32 through
        ``normalize`` and the cumulative sum of ``running_mean``, so its result differs from this one by that float32
        rounding."""
        from . import engine
        from . import units as u
        seq = not isinstance(transit_duration, int) and np.ndim(transit_duration) == 1
        durs = list(transit_duration) if seq else [transit_duration]
        for d in durs:
            if not (isinstance(d, int) or (seq and isinstance(d, np.integer))):
                raise ValueError(
                    "transit_duration must be an integer in units "
                    "number of cadences, got {}.".format(d)
                )
        if savgol_polyorder >= savgol_window:
            savgol_polyorder = savgol_window - 1
            log.warning("polyorder must be smaller than window_length, "
                        "using polyorder={}.".format(savgol_polyorder))
        if not self.data:
            res = np.zeros((0, len(durs)))
        else:
            times = [np.asarray(lc.time.value, dtype=np.float64) for lc in self.data]
            fluxes = [np.asarray(lc.flux.value, dtype=np.float64) for lc in self.data]
            res = engine.cdpp(times, fluxes, np.asarray(durs, dtype=np.int64), savgol_window, savgol_polyorder, sigma)
        return u.Quantity(res if seq else res[:, 0], u.ppm)

    def fold(self, period=None, epoch_time=None, epoch_phase=0, wrap_phase=None, normalize_phase=False):
        """Batched ``LightCurve.fold``: equal to ``[lc.fold(...) for lc in collection]``, with the phases of every light
        curve computed and stably sorted in one GPU call (K13, ``engine.fold``).  `period`, `epoch_time`,
        `epoch_phase` and `wrap_phase` are each a scalar (float or Quantity) or a sequence of one value per light
        curve, such as a list of ``pg.period_at_max_power``.  Returns a LightCurveCollection of FoldedLightCurve
        objects.  The JD warning of `epoch_time` is raised at most once per call."""
        import warnings
        from . import engine
        from .lightcurve import _fold_params
        from .utils import LightkurveWarning
        B = len(self.data)
        if B == 0:
            return LightCurveCollection([])
        args = [_per_light_curve(v, B, name) for v, name in ((period, "period"), (epoch_time, "epoch_time"),
                                                             (epoch_phase, "epoch_phase"), (wrap_phase, "wrap_phase"))]
        times, params, jd_warning = [], [], None
        for b, lc in enumerate(self.data):
            t = np.asarray(lc.time.value, dtype=np.float64)
            p = _fold_params(t, lc.time, args[0][b], args[1][b], args[2][b], args[3][b], normalize_phase)
            jd_warning = jd_warning or p[4]
            times.append(t)
            params.append(p[:4])
        if jd_warning:
            warnings.warn(jd_warning, LightkurveWarning)
        out = [None] * B
        batch = [b for b in range(B) if params[b][0] > 0]
        for b in range(B):
            if not params[b][0] > 0:                   # numpy's remainder by a zero, negative or NaN period
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore", LightkurveWarning)
                    out[b] = self.data[b].fold(args[0][b], args[1][b], args[2][b], args[3][b], normalize_phase)
        if batch:
            per, t0, shift, wrap = (np.array([params[b][k] for b in batch], dtype=np.float64) for k in range(4))
            res = engine.fold([times[b] for b in batch], t0, shift, per, wrap, normalize=normalize_phase)
            for k, b in enumerate(batch):
                out[b] = self.data[b]._folded(times[b], res["perm"][k], res["phase"][k], params[b][0], params[b][1],
                                              args[1][b], args[2][b], args[3][b], normalize_phase)
        return LightCurveCollection(out)

    def bin(self, time_bin_size=None, time_bin_start=None, time_bin_end=None, n_bins=None, aggregate_func=None,
            bins=None, binsize=None):
        """Batched ``LightCurve.bin``: equal to ``[lc.bin(...) for lc in collection]``, with the same keywords and
        errors.  With ``aggregate_func`` None, ``np.nanmean`` or ``np.nanmedian``, every light curve is sorted and
        binned in one GPU call (K13, ``engine.bin``); the nanmean's and the errors' sums then run in a fixed order,
        so they may differ from the loop's numpy sums in the last bits.  Any other ``aggregate_func`` runs the
        per-light-curve loop.  Works on folded collections, whose time is the phase.  A zero-length light curve comes
        back as its copy; a light curve with no bin, or with bin-edge indices that do not ascend, goes through its
        own single-curve method."""
        from . import engine
        from .lightcurve import _bin_check_args, _bin_edges
        kw = dict(time_bin_size=time_bin_size, time_bin_start=time_bin_start, time_bin_end=time_bin_end,
                  n_bins=n_bins, aggregate_func=aggregate_func, bins=bins, binsize=binsize)
        agg = _bin_check_args(time_bin_size, n_bins, aggregate_func, bins, binsize)
        if agg is np.nanmean or agg is np.nanmedian:
            aggregate = "nanmean" if agg is np.nanmean else "nanmedian"
        else:
            return LightCurveCollection([lc.bin(**kw) for lc in self.data])
        out = [None] * len(self.data)
        times = [np.asarray(lc.time.value, dtype=np.float64) for lc in self.data]
        nonempty = [b for b, t in enumerate(times) if len(t)]
        for b, t in enumerate(times):
            if not len(t):
                out[b] = self.data[b].copy()
        first, last = _sorted_first_last([times[b] for b in nonempty])
        batch, starts, ends, kind = [], [], [], None
        for k, b in enumerate(nonempty):
            kind, s, e = _bin_edges(len(times[b]), first[k], last[k], time_bin_size, time_bin_start, time_bin_end,
                                    n_bins, bins, binsize)
            if len(s) == 0 or not _ascending(s):
                out[b] = self.data[b].bin(**kw)        # no bin: the single method's IndexError; unordered starts
                continue
            batch.append(b)
            starts.append(s)
            ends.append(e)
        if batch:
            errs = [np.asarray(self.data[b].flux_err.value, dtype=np.float64) for b in batch]
            res = engine.bin([times[b] for b in batch],
                             [np.asarray(self.data[b].flux.value, dtype=np.float64) for b in batch], errs, starts,
                             ends, index_edges=kind == "index", aggregate=aggregate)
            for k, b in enumerate(batch):
                out[b] = self.data[b]._binned(res["time"][k], res["flux"][k], res["flux_err"][k])
        return LightCurveCollection(out)

    def stitch(self, corrector_func=lambda x: x.normalize()):
        """Concatenate the light curves (collections.py:196-230)."""
        from .units import Quantity, Time
        lcs = [corrector_func(lc) for lc in self.data]
        first = lcs[0]
        new = first.copy()
        new.time = Time(np.concatenate([np.asarray(lc.time.value) for lc in lcs]), first.time.format, first.time.scale)
        new.flux = Quantity(np.concatenate([np.asarray(lc.flux.to(first.flux.unit).value) for lc in lcs]),
                            first.flux.unit)
        new.flux_err = Quantity(np.concatenate([np.asarray(lc.flux_err.to(first.flux.unit).value) for lc in lcs]),
                                first.flux.unit)
        return new


def _check_finite_times(times):
    for b, t in enumerate(times):
        if not np.isfinite(t).all():
            raise ValueError("light curve {} has non-finite times".format(b))


def _named(e, b):
    """`e` again, of the same type, with the light curve in front of its message."""
    try:
        return type(e)("light curve {}: {}".format(b, e))
    except Exception:                                  # an exception type that needs other arguments
        return e


def _per_light_curve(value, B, name):
    """`value` repeated for B light curves, or its B elements when it is a sequence or array of one per light curve."""
    if value is None or isinstance(value, str) or np.ndim(getattr(value, "value", value)) == 0:
        return [value] * B
    if len(value) != B:
        raise ValueError("`{}` has {} values for {} light curves".format(name, len(value), B))
    return [value[b] for b in range(B)]


def _sorted_first_last(times):
    """First and last value of each array of `times` (all non-empty) once stably sorted in numpy's order (NaN last)."""
    if not times:
        return np.zeros(0), np.zeros(0)
    cat = np.concatenate(times)
    at = np.cumsum([0] + [len(t) for t in times[:-1]])
    nan = np.add.reduceat(np.isnan(cat), at)
    with np.errstate(invalid="ignore"):
        first = np.fmin.reduceat(cat, at)
        last = np.where(nan > 0, np.nan, np.fmax.reduceat(cat, at))
    for b in np.nonzero((first == 0) | (last == 0))[0]:      # which zero, -0.0 or +0.0, comes first / last
        ts = np.sort(times[b], kind="stable")
        first[b], last[b] = ts[0], ts[-1]
    return first, last


def _ascending(s):
    """True when `s` does not decrease in numpy's order (NaN last)."""
    s = np.asarray(s)
    if s.dtype.kind != "f":
        return bool(np.all(s[1:] >= s[:-1]))
    a, b = s[:-1], s[1:]
    return not bool(np.any((b < a) | (np.isnan(a) & ~np.isnan(b))))
