"""`CBVCorrector` and `CotrendingBasisVectors`: the caller that loops `RegressionCorrector.correct` (K5) and the
Lomb-Scargle over-fitting metric (K1) inside a bounded scalar optimiser (SURVEY.md 8(f) rank 4;
/root/reference/src/lightkurve/correctors/cbvcorrector.py:45-980 and :982-1380).

Scope: everything that runs from arrays - the basis-vector container (`to_designmatrix`, `align`, `interpolate`),
`correct_gaussian_prior`, the `correct` optimiser over the regularisation `alpha`, `over_fitting_metric`,
`under_fitting_metric` (with the neighbouring light curves handed over), `correct_regressioncorrector`,
`correct_elasticnet` (scikit-learn's elastic-net coordinate descent, K8; with `correct_elasticnet_batch` for many
correctors in one call) and `correct_batch` (the alpha optimiser with both goodness metrics for many correctors, the
batch serving as its own neighbourhood; K5 + K1 + K9 per round).  Out of scope here: reading CBV FITS files /
downloading them from MAST (`load_kepler_cbvs`, `load_tess_cbvs`), the MAST neighbour search and the plots.  Basis
vectors are
therefore handed over explicitly (``CBVCorrector(lc, cbvs=[...])``, an extension of the reference signature) or
left out (``do_not_load_cbvs=True`` with an external design matrix, as in the reference's own non-remote test).
"""
import copy
import logging
import warnings

import numpy as np
from scipy.interpolate import PchipInterpolator
from scipy.optimize import minimize_scalar

from .. import units as u
from ..lightcurve import LightCurve
from ..units import Quantity, Time
from .designmatrix import DesignMatrix, DesignMatrixCollection
from .metrics import (MAST_MESSAGE, _cadence_grid, _centred, _neighbor_rows, _overfit_from_terms,
                      _require_cadenceno, overfit_metric_lombscargle, underfit_metric_neighbors)
from .optimize import minimize_bounded_lockstep
from .regressioncorrector import RegressionCorrector

log = logging.getLogger(__name__)

__all__ = ["CBVCorrector", "CotrendingBasisVectors", "ConvergenceWarning"]


class ConvergenceWarning(UserWarning):
    """The elastic-net coordinate descent stopped on `max_iter` before its duality gap reached the tolerance
    (scikit-learn's `sklearn.exceptions.ConvergenceWarning`, with the same text)."""


MESSAGE_ALPHA0 = ("With alpha=0, this algorithm does not converge well. You are advised to use the LinearRegression "
                  "estimator")
_ENET_FORWARDED = {"max_iter": 1000, "tol": 1e-4, "positive": False}
_ENET_NO_EFFECT = ("precompute", "copy_X", "warm_start", "random_state")


def _convergence_message(gap, tol, l1):
    msg = ("Objective did not converge. You might want to increase the number of iterations, check the scale of the "
           "features or consider increasing regularisation. Duality gap: {:.6e}, tolerance: {:.3e}".format(gap, tol))
    if l1 < np.finfo(np.float64).eps:
        msg += ("\nLinear regression models with a zero l1 penalization strength are more efficiently fitted using "
                "one of the solvers implemented in sklearn.linear_model.Ridge/RidgeCV instead.")
    return msg


def _elasticnet_options(kwargs):
    """ElasticNet keyword arguments -> the kernel's max_iter / tol / positive."""
    opts = dict(_ENET_FORWARDED)
    for key, value in kwargs.items():
        if key in _ENET_FORWARDED:
            opts[key] = value
        elif key == "selection":
            if value == "random":
                raise NotImplementedError("selection='random' is not available: the GPU fit is cyclic")
            if value != "cyclic":
                raise ValueError("selection must be 'cyclic' or 'random', got {!r}".format(value))
        elif key not in _ENET_NO_EFFECT:
            raise TypeError("correct_elasticnet() got an unexpected keyword argument {!r}".format(key))
    opts["positive"] = bool(opts["positive"])
    return opts


# Largest neighbour search radius (arcsec): the diagonal of a TESS camera (two CCDs wide, 24 degrees) or of one
# Kepler / K2 CCD (cbvcorrector.py:608-617)
_MAX_RADIUS = {"TESS": np.sqrt(2) * (86400 / 2.0), "Kepler": np.sqrt(2) * 4096, "K2": np.sqrt(2) * 4096}
_NOT_ENOUGH = "Not enough neighboring targets were found. under_fitting_metric failed"
# Lomb-Scargle work (cadences x bins) from which the library's `auto` takes the non-uniform FFT for one light curve
# (lkb_ls_power, ls.cu); correct_batch applies it per light curve so that the batch does not choose the family
_LS_NUFFT_MIN_WORK = 2.5e7


def _separation_arcsec(ra0, dec0, ra, dec):
    """Great-circle separation (Vincenty formula, as astropy's `SkyCoord.separation`) of degrees, in arcsec."""
    l0, b0, l1, b1 = np.radians(ra0), np.radians(dec0), np.radians(ra), np.radians(dec)
    dl = l1 - l0
    num = np.hypot(np.cos(b1) * np.sin(dl), np.cos(b0) * np.sin(b1) - np.sin(b0) * np.cos(b1) * np.cos(dl))
    den = np.sin(b0) * np.sin(b1) + np.cos(b0) * np.cos(b1) * np.cos(dl)
    return np.degrees(np.arctan2(num, den)) * 3600.0


def _sky(lc):
    ra, dec = lc.meta.get("RA"), lc.meta.get("DEC")
    if ra is None or dec is None:
        raise ValueError("selecting neighbours by radius needs meta['RA'] and meta['DEC'] (degrees) on every light "
                         "curve; pass `neighbor_index` to skip the sky geometry")
    return float(ra), float(dec)


def _own_entries(lc, pool):
    """Pool entries that are `lc` itself: the same object or the same (known) TARGETID."""
    tid = lc.meta.get("TARGETID")
    return {i for i, p in enumerate(pool) if p is lc or (tid is not None and p.meta.get("TARGETID") == tid)}


def _select_neighbors(lc, pool, exclude, radius=None, min_targets=30, max_targets=50, neighbor_index=None,
                      coords=None):
    """Indices into `pool` of the neighbours of `lc` by the reference's radius loop (cbvcorrector.py:586-637): the
    nearest `max_targets` within the radius (default 5000 arcsec for TESS, 1000 for Kepler / K2), the radius growing
    by 1.5 until `min_targets` are found or it passes the CCD diagonal.  `neighbor_index`: the candidates in order of
    preference, instead of the sky geometry."""
    mission = lc.meta.get("MISSION")
    if radius is None:
        radius = 5000 if mission == "TESS" else 1000
    if mission not in _MAX_RADIUS:
        raise Exception("Unknown mission")
    if neighbor_index is not None:
        cand = [int(i) for i in neighbor_index if int(i) not in exclude]
        if len(cand) < min_targets:
            raise Exception(_NOT_ENOUGH)
        return cand[:max_targets]
    ra0, dec0 = _sky(lc)
    if coords is None:
        coords = np.array([_sky(p) for p in pool]).reshape(-1, 2)
    others = [i for i in range(len(pool)) if i not in exclude]
    sep = _separation_arcsec(ra0, dec0, coords[others, 0], coords[others, 1])
    order = np.argsort(sep, kind="stable")
    r = radius
    while True:
        sel = [others[k] for k in order if sep[k] <= r]
        if len(sel) >= min_targets:
            return sel[:max_targets]
        if r > _MAX_RADIUS[mission]:
            raise Exception(_NOT_ENOUGH)
        r *= 1.5


def _per_item(value, n):
    """True when `value` is a list/tuple with one design matrix / mask (or None) per corrector."""
    return (isinstance(value, (list, tuple)) and len(value) == n and
            all(v is None or isinstance(v, DesignMatrix) or np.ndim(v) == 1 for v in value))


class CotrendingBasisVectors:
    """A set of cotrending basis vectors on a cadence grid (cbvcorrector.py:982-1380).

    `data`: mapping with the columns ``VECTOR_<n>`` (1-based n) and optionally ``CADENCENO`` and ``GAP``
    (defaults: 0 .. N-1 and all False); `time`: the cadence times (`Time` or array)."""

    def __init__(self, data=None, time=None, cbv_type="Generic", mission=None, band=None):
        data = {} if data is None else dict(data)
        self._vectors = {}
        n = None
        for name, col in data.items():
            if name.find("VECTOR_") > -1:
                self._vectors[int(name[7:])] = np.array(col, dtype=np.float64)
                n = len(self._vectors[int(name[7:])])
        if n is None:
            n = 0 if time is None else len(time)
        self.gap_indicators = np.array(data["GAP"], dtype=bool) if "GAP" in data else np.full(n, False)
        self.cadenceno = np.array(data["CADENCENO"]) if "CADENCENO" in data else np.arange(n)
        if time is None:
            time = np.arange(n, dtype=float)
        self.time = time if isinstance(time, Time) else Time(np.asarray(getattr(time, "value", time), dtype=float))
        if not (len(self.time) == len(self.gap_indicators) == len(self.cadenceno) == n):
            raise ValueError("all columns of a CotrendingBasisVectors object must have the same length")
        self.cbv_type, self.mission, self.band = cbv_type, mission, band

    @property
    def cbv_indices(self):
        return list(self._vectors)

    def __len__(self):
        return len(self.cadenceno)

    def __getitem__(self, key):
        if isinstance(key, str):
            if key.find("VECTOR_") > -1:
                return Quantity(self._vectors[int(key[7:])], None)
            return {"time": self.time, "GAP": self.gap_indicators, "CADENCENO": self.cadenceno}[key]
        raise TypeError("index a CotrendingBasisVectors object with a column name")

    def _like(self, vectors, time, gaps, cadenceno):
        data = {"VECTOR_{}".format(i): v for i, v in vectors.items()}
        data["GAP"], data["CADENCENO"] = gaps, cadenceno
        return self.__class__(data, time, cbv_type=self.cbv_type, mission=self.mission, band=self.band)

    def to_designmatrix(self, cbv_indices="all", name="CBVs"):
        """`DesignMatrix` whose columns are the requested basis vectors; indices that do not exist are ignored
        (cbvcorrector.py:1082-1120)."""
        if isinstance(cbv_indices, str) and not cbv_indices == "all":
            raise ValueError('cbv_indices must either be list of ints or "all"')
        if not isinstance(cbv_indices, str) and 0 in cbv_indices:
            raise ValueError("CBVs use 1-based indexing. Do not request CBV index '0'")
        if isinstance(cbv_indices, str):
            cbv_indices = self.cbv_indices
        picked = [i for i in cbv_indices if i in self._vectors]
        matrix = np.stack([self._vectors[i] for i in picked], axis=1) if picked else np.zeros((len(self), 0))
        return DesignMatrix(matrix, columns=["VECTOR_{}".format(i) for i in picked], name=name)

    def align(self, lc):
        """The basis vectors on the light curve's cadences, matched by cadence number: cadences the CBVs lack are
        inserted as NaN gaps, cadences the light curve lacks are dropped (cbvcorrector.py:1208-1307)."""
        if not isinstance(lc, LightCurve):
            raise Exception("<lc> must be a LightCurve class")
        try:
            lc_cad = np.asarray(lc.cadenceno)
        except AttributeError:
            raise Exception("align requires cadence numbers for the light curve. NO SYNCHRONIZATION OCCURRED")
        pos = {int(c): i for i, c in enumerate(self.cadenceno)}
        src = np.array([pos.get(int(c), -1) for c in lc_cad])
        have = src >= 0
        if np.count_nonzero(~have) / max(1, len(have)) > 0.5 or np.count_nonzero(have) / max(1, len(self)) < 0.5:
            log.warning("The {} CBVs do not appear to be well aligned to the "
                        'light curve. Consider using "interpolate_cbvs=True"'.format(self.cbv_type))
        vectors = {}
        for i, v in self._vectors.items():
            col = np.full(len(lc_cad), np.nan)
            col[have] = v[src[have]]
            vectors[i] = col
        gaps = np.ones(len(lc_cad), dtype=bool)
        gaps[have] = self.gap_indicators[src[have]]
        return self._like(vectors, Time(np.asarray(lc.time.value, dtype=float), lc.time.format, lc.time.scale), gaps,
                          lc_cad.copy())

    def interpolate(self, lc, extrapolate=False):
        """PCHIP interpolation of the un-gapped basis vectors to the light curve's times; values outside the CBV time
        range are extrapolated or set to zero (cbvcorrector.py:1309-1378)."""
        if not isinstance(lc, LightCurve):
            raise Exception("<lc> must be a LightCurve class")
        good = ~self.gap_indicators
        t_cbv = np.asarray(self.time.value, dtype=float)[good]
        t_lc = np.asarray(lc.time.value, dtype=float)
        if not extrapolate and (np.min(t_lc) < np.min(t_cbv) or np.max(t_lc) > np.max(t_cbv)):
            log.warning("Extrapolation of CBVs appears to be necessary. "
                        "Extrapolated values will be filled with zeros. "
                        "Recommend setting extrapolate=True")
        vectors, warned = {}, False
        for i, v in self._vectors.items():
            col = PchipInterpolator(t_cbv, v[good], extrapolate=extrapolate)(t_lc)
            if np.any(np.isnan(col)):
                col[np.isnan(col)] = 0.0
                if not warned:
                    log.warning("Some interpolated (or extrapolated) CBV values have been set to zero")
                    warned = True
            vectors[i] = col
        cad = np.asarray(lc.cadenceno) if "cadenceno" in lc.__dict__.get("_columns", {}) else np.arange(len(t_lc))
        return self._like(vectors, Time(t_lc, lc.time.format, lc.time.scale), np.full(len(t_lc), False), cad)

    def __repr__(self):
        return "CotrendingBasisVectors ({}, {} vectors, {} cadences)".format(self.cbv_type, len(self._vectors), len(self))


class CBVCorrector(RegressionCorrector):
    """Remove systematics with cotrending basis vectors under a Gaussian (L2) prior whose strength `alpha` is either
    given or optimised against the over-fitting metric (cbvcorrector.py:45-980)."""

    def __init__(self, lc, interpolate_cbvs=False, extrapolate_cbvs=False, do_not_load_cbvs=False, cbv_dir=None,
                 cbvs=None):
        if not isinstance(lc, LightCurve):
            raise Exception("<lc> must be a LightCurve class")
        assert lc.flux.unit == u.electron / u.second, "cbvCorrector expects light curve to be passed in e-/s units."
        if extrapolate_cbvs and (extrapolate_cbvs != interpolate_cbvs):
            raise Exception("interpolate_cbvs must be True if extrapolate_cbvs is True")
        lc = lc.copy().remove_nans()                         # no NaNs; the flux stays in absolute units
        super(CBVCorrector, self).__init__(lc)
        if cbvs is None and not do_not_load_cbvs:
            raise NotImplementedError(
                "loading CBV files (MAST download / FITS) is outside the scope of lightkurve_b200: pass the basis "
                "vectors with `cbvs=[CotrendingBasisVectors(...), ...]` or use `do_not_load_cbvs=True` with `ext_dm`")
        prepared = []
        for c in (cbvs or []):
            if not isinstance(c, CotrendingBasisVectors):
                raise Exception("CBVs could not be loaded. CBVCorrector must exit")
            prepared.append(c.interpolate(self.lc, extrapolate=extrapolate_cbvs) if interpolate_cbvs else c.align(self.lc))
        self.cbvs = prepared
        self.interpolated_cbvs = interpolate_cbvs
        self.extrapolated_cbvs = extrapolate_cbvs
        self.cbv_design_matrix = None
        self.extra_design_matrix = None
        self.coefficients_err = None
        self.cadence_mask = None
        self.over_fitting_score = None
        self.under_fitting_score = None
        self.alpha = None

    # ---- set-up shared by the correct_* methods (cbvcorrector.py:639-757) ----
    def _correct_initialization(self, cbv_type="SingleScale", cbv_indices="ALL", ext_dm=None):
        assert not ((cbv_type is None) ^ (cbv_indices is None)), \
            "Both cbv_type and cbv_indices must be None, or neither"
        use_cbvs = not (cbv_type is None and cbv_indices is None)
        self.extra_design_matrix = ext_dm
        if ext_dm is not None:
            assert isinstance(ext_dm, DesignMatrix), "ext_dm must be a DesignMatrix"
            if ext_dm.shape[0] != len(self.lc.flux):
                raise ValueError("ext_dm must contain the same number of cadences as lc.flux")
        self.cbv_design_matrix = []
        if use_cbvs:
            assert not isinstance(cbv_type, str) and not isinstance(cbv_indices[0], int), \
                "cbv_type and cbv_indices must be lists of strings"
            mission = self.lc.meta.get("MISSION")
            if mission in ["Kepler", "K2"]:
                assert cbv_type == ["SingleScale"], "cbv_type must be Single-Scale for Kepler and K2 missions"
            if isinstance(cbv_type, list) and len(cbv_type) != 1:
                assert mission == "TESS", "Multiple CBV types are only allowed for TESS"
            assert len(cbv_type) == len(cbv_indices), "cbv_type and cbv_indices must be the same list length"
            for kind, wanted in zip(cbv_type, cbv_indices):
                for cbvs in self.cbvs:
                    idx = cbvs.cbv_indices if (isinstance(wanted, str) and wanted == "ALL") else wanted
                    idx = np.array([i for i in idx if i in cbvs.cbv_indices])
                    if kind.find("MultiScale") >= 0:
                        if cbvs.cbv_type in kind and cbvs.band == int(kind[-1]):
                            self.cbv_design_matrix.append(cbvs.to_designmatrix(cbv_indices=idx, name=kind))
                    elif cbvs.cbv_type in kind:
                        self.cbv_design_matrix.append(cbvs.to_designmatrix(cbv_indices=idx, name=kind))
        matrices = list(self.cbv_design_matrix)
        if self.extra_design_matrix is not None:
            matrices.append(self.extra_design_matrix)
        if not matrices:
            raise ValueError("no design matrix: neither basis vectors nor `ext_dm` were given")
        matrices.append(DesignMatrix(np.ones(matrices[0].shape[0]), columns=["Constant"], name="Constant"))
        self.design_matrix_collection = DesignMatrixCollection(matrices)

    def _set_prior_width(self, sigma):
        """Same Gaussian prior width for every coefficient; None = no prior (cbvcorrector.py:759-779)."""
        if isinstance(sigma, list):
            raise Exception("separate widths is not yet implemented")
        for dm in self.design_matrix_collection:
            n = len(dm.prior_sigma)
            dm.prior_sigma = np.ones(n) * (np.inf if sigma is None else sigma)

    def correct_regressioncorrector(self, design_matrix_collection, **kwargs):
        """`RegressionCorrector.correct` of the superclass (one `lkb_regress` call)."""
        return super(CBVCorrector, self).correct(design_matrix_collection, **kwargs)

    def correct_gaussian_prior(self, cbv_type=["SingleScale"], cbv_indices=[np.arange(1, 9)], alpha=1e-20, ext_dm=None,
                               cadence_mask=None, **kwargs):
        """Fit with the L2 penalty `alpha`: prior width = median(flux_err) / sqrt(|alpha|) (cbvcorrector.py:221-292)."""
        self._correct_initialization(cbv_type=cbv_type, cbv_indices=cbv_indices, ext_dm=ext_dm)
        sigma = None if alpha == 0.0 else np.median(self.lc.flux_err.value) / np.sqrt(np.abs(alpha))
        self._set_prior_width(sigma)
        self.correct_regressioncorrector(self.design_matrix_collection, cadence_mask=cadence_mask, **kwargs)
        self.alpha = alpha
        return self.corrected_lc

    # ---- elastic net (cbvcorrector.py:294-395): scikit-learn's coordinate descent, one lkb_elasticnet call ----
    def correct_elasticnet(self, cbv_type='SingleScale', cbv_indices=np.arange(1, 9), alpha=1e-20, l1_ratio=0.01,
                           ext_dm=None, cadence_mask=None, **kwargs):
        """Fit with combined L1 and L2 penalties: the coefficients of
        ``sklearn.linear_model.ElasticNet(alpha, l1_ratio, fit_intercept=False, **kwargs).fit(X[mask], y[mask])``,
        reproduced iteration for iteration on the GPU (K8).  The model leaves out the constant column and is
        median-subtracted, so the corrected light curve keeps the flux's median.  `alpha` does not scale like the
        `alpha` of `correct_gaussian_prior`.

        Keyword arguments of ElasticNet: `max_iter`, `tol` and `positive` are honoured; `precompute`, `copy_X`,
        `warm_start` and `random_state` do not change a fresh cyclic fit and are accepted; `selection="random"` is not
        available.  A fit that stops on `max_iter` warns with ElasticNet's `ConvergenceWarning` text."""
        self._correct_initialization(cbv_type=cbv_type, cbv_indices=cbv_indices, ext_dm=ext_dm)
        CBVCorrector._run_elasticnet([self], [cadence_mask], alpha, l1_ratio, _elasticnet_options(kwargs))
        return self.corrected_lc

    @staticmethod
    def correct_elasticnet_batch(correctors, cbv_type='SingleScale', cbv_indices=np.arange(1, 9), alpha=1e-20,
                                 l1_ratio=0.01, ext_dm=None, cadence_mask=None, **kwargs):
        """`correct_elasticnet` for many correctors in as few GPU calls as possible: one call with a shared design
        matrix when every corrector's matrix is the same, one call per group of equal-shaped matrices otherwise.
        `ext_dm` and `cadence_mask` are either shared or lists with one entry per corrector.  Every corrector ends in
        the state its own `correct_elasticnet` call would leave; returns the list of corrected light curves."""
        correctors = list(correctors)
        B = len(correctors)
        ext = ext_dm if _per_item(ext_dm, B) else [ext_dm] * B
        masks = cadence_mask if _per_item(cadence_mask, B) else [cadence_mask] * B
        opts = _elasticnet_options(kwargs)
        for c, e in zip(correctors, ext):
            c._correct_initialization(cbv_type=cbv_type, cbv_indices=cbv_indices, ext_dm=e)
        CBVCorrector._run_elasticnet(correctors, masks, alpha, l1_ratio, opts)
        return [c.corrected_lc for c in correctors]

    @staticmethod
    def _run_elasticnet(correctors, masks, alpha, l1_ratio, opts):
        from .. import engine
        Xs, ys, ms = [], [], []
        for c, m in zip(correctors, masks):
            X = np.ascontiguousarray(c.design_matrix_collection.values, dtype=np.float64)
            if not np.all(np.isfinite(X)):
                raise ValueError("Input X contains NaN or infinity.")
            n = len(c.lc.flux)
            m = np.ones(n, bool) if m is None else np.asarray(m, dtype=bool)
            if m.shape != (n,):
                raise ValueError("cadence_mask must have one entry per cadence")
            Xs.append(X)
            ys.append(np.asarray(c.lc.flux.value, dtype=np.float64))
            ms.append(m)
        if alpha == 0:
            warnings.warn(MESSAGE_ALPHA0, UserWarning, stacklevel=3)
        groups = {}
        for b, X in enumerate(Xs):
            groups.setdefault(X.shape, []).append(b)
        for idx in groups.values():
            shared = all(Xs[b] is Xs[idx[0]] or np.array_equal(Xs[b], Xs[idx[0]]) for b in idx)
            X = Xs[idx[0]] if shared else np.stack([Xs[b] for b in idx])
            res = engine.elasticnet(X, np.stack([ys[b] for b in idx]), np.stack([ms[b] for b in idx]), alpha=alpha,
                                    l1_ratio=l1_ratio, **opts)
            for j, b in enumerate(idx):
                c, m = correctors[b], ms[b]
                if not res["converged"][j]:
                    n = int(np.count_nonzero(m))
                    ym = ys[b][m]
                    warnings.warn(_convergence_message(res["dual_gap"][j] * n, opts["tol"] * float(ym @ ym),
                                                       alpha * l1_ratio * n), ConvergenceWarning, stacklevel=3)
                c.coefficients = res["coefficients"][j]
                c.coefficients_err = None
                c.elasticnet_n_iter = int(res["n_iter"][j])
                c.elasticnet_dual_gap = float(res["dual_gap"][j])
                c._finish(res["model"][j])
                c.cadence_mask = m
                c.alpha = alpha

    def correct(self, cbv_type=["SingleScale"], cbv_indices=[np.arange(1, 9)], ext_dm=None, cadence_mask=None,
                alpha_bounds=[1e-4, 1e4], target_over_score=0.5, target_under_score=0.5, max_iter=100,
                neighbors=None):
        """Optimise `alpha` with a bounded scalar minimiser against the goodness metrics (cbvcorrector.py:397-501).
        The under-fitting metric needs the neighbouring light curves (`neighbors`, in place of the reference's MAST
        search); with them and `target_under_score > 0` this is `correct_batch([self], ..., neighbors=neighbors)`.
        Without them `target_under_score` must be 0."""
        if neighbors is not None and target_under_score > 0:
            CBVCorrector.correct_batch([self], cbv_type=cbv_type, cbv_indices=cbv_indices, ext_dm=ext_dm,
                                       cadence_mask=cadence_mask, alpha_bounds=alpha_bounds,
                                       target_over_score=target_over_score, target_under_score=target_under_score,
                                       max_iter=max_iter, neighbors=neighbors)
            if target_over_score > 0:
                print("Optimized Over-fitting metric: {}".format(self.over_fitting_score))
            print("Optimized Under-fitting metric: {}".format(self.under_fitting_score))
            print("Optimized Alpha: {0:2.3e}".format(self.alpha))
            return self.corrected_lc
        self._correct_initialization(cbv_type=cbv_type, cbv_indices=cbv_indices, ext_dm=ext_dm)
        if target_under_score > 0:
            raise NotImplementedError("the under-fitting metric needs a MAST search of neighbouring targets, which is "
                                      "outside the scope of lightkurve_b200: call correct(..., target_under_score=0)")
        self.optimization_params = {"alpha_bounds": alpha_bounds, "target_over_score": target_over_score,
                                    "target_under_score": target_under_score, "max_iter": max_iter,
                                    "cadence_mask": cadence_mask, "over_metric_nSamples": 1}
        result = minimize_scalar(self._goodness_metric_obj_fun, method="Bounded", bounds=alpha_bounds,
                                 options={"maxiter": max_iter, "disp": False})
        self._goodness_metric_obj_fun(result.x)            # the minimiser does not end on its best point
        if target_over_score > 0:
            self.over_fitting_score = self.over_fitting_metric(n_samples=10)
            print("Optimized Over-fitting metric: {}".format(self.over_fitting_score))
        else:
            self.over_fitting_score = -1.0
        self.under_fitting_score = -1.0
        self.alpha = result.x
        print("Optimized Alpha: {0:2.3e}".format(self.alpha))
        return self.corrected_lc

    def over_fitting_metric(self, n_samples=10):
        """`metrics.overfit_metric_lombscargle` of the original and corrected light curves on the used cadences."""
        if self.corrected_lc is None:
            log.warning("A corrected light curve does not exist, please run correct first")
            return None
        return overfit_metric_lombscargle(self.lc.copy()[self.cadence_mask], self.corrected_lc.copy()[self.cadence_mask],
                                          n_samples=n_samples)

    def under_fitting_metric(self, neighbors=None, radius=None, min_targets=30, max_targets=50, neighbor_index=None):
        """`metrics.underfit_metric_neighbors` of the corrected light curve on the used cadences, its neighbours picked
        from `neighbors` (a list or `LightCurveCollection`, in place of the reference's MAST search) by the reference's
        radius loop (cbvcorrector.py:586-637) on great-circle separations from meta["RA"], meta["DEC"] (degrees).  A
        light curve is never its own neighbour.  `neighbor_index`: indices into `neighbors` in order of preference,
        instead of the sky geometry.  `coords`: the pool's [P, 2] (RA, DEC), when the caller has them already."""
        if self.corrected_lc is None:
            raise Exception("A corrected light curve does not exist, please run correct first")
        if neighbors is None:
            raise NotImplementedError(MAST_MESSAGE)
        pool = list(neighbors)
        sel = _select_neighbors(self.lc, pool, _own_entries(self.lc, pool), radius, min_targets, max_targets,
                                neighbor_index)
        corrected = self.corrected_lc.copy()[self.cadence_mask]
        return underfit_metric_neighbors(corrected, min_targets=min_targets, max_targets=max_targets,
                                         interpolate=self.interpolated_cbvs, extrapolate=self.extrapolated_cbvs,
                                         neighbors=[pool[i] for i in sel])

    @staticmethod
    def correct_batch(correctors, cbv_type=["SingleScale"], cbv_indices=[np.arange(1, 9)], ext_dm=None,
                      cadence_mask=None, alpha_bounds=[1e-4, 1e4], target_over_score=0.5, target_under_score=0.5,
                      max_iter=100, neighbors=None, radius=None, min_targets=30, max_targets=50, neighbor_index=None):
        """`correct` for many correctors, the minimisers of all correctors run in lock step: each round fits every
        still-active corrector with its own prior width in one regression call (bitwise independent of the batch,
        LKB_REGRESS_EXACT_INVARIANT), computes their corrected and white-noise periodograms on each corrector's
        original-periodogram grid (with the kernel family the corrector's own call would take), and both goodness
        metrics in one K9 call each.  The inputs stay on the GPU across rounds.  Every corrector ends in the state its
        own `correct` would leave (`alpha`, corrected / model / diagnostic light curves, `coefficients`,
        `cadence_mask`, `over_fitting_score` at n_samples=10, `under_fitting_score`) and gains `optimization_trace`:
        one (alpha, over, under, mean_noise_power, n_positive, sum_positive) per evaluation of its objective.

        Neighbours for the under-fitting metric come from `neighbors` or, by default, from the batch's own light
        curves (the other targets of the same CCD and sector, which is what the reference's MAST search returns),
        selected per corrector as in `under_fitting_metric` (`radius`, `min_targets`, `max_targets`,
        `neighbor_index`: one index list per corrector).  Correctors built with `interpolate_cbvs=True` raise
        NotImplementedError here: their neighbours would have to be interpolated pair by pair.

        `ext_dm` and `cadence_mask` are shared or lists with one entry per corrector.  White noise: one
        ``np.random.randn(n_cadences, 1)`` per active corrector per round, in batch order, from numpy's global stream,
        then the final re-fit's draws and the ten of each final over-fitting score, corrector by corrector - a batch
        of one consumes exactly the draws of the reference's `correct`.  Returns the corrected light curves."""
        correctors = list(correctors)
        B = len(correctors)
        ext = ext_dm if _per_item(ext_dm, B) else [ext_dm] * B
        masks = cadence_mask if _per_item(cadence_mask, B) else [cadence_mask] * B
        for c, e, m in zip(correctors, ext, masks):
            # a copy per corrector: the prior widths set on the design matrices differ from corrector to corrector
            c._correct_initialization(cbv_type=cbv_type, cbv_indices=cbv_indices,
                                      ext_dm=None if e is None else copy.deepcopy(e))
            c.optimization_params = {"alpha_bounds": alpha_bounds, "target_over_score": target_over_score,
                                     "target_under_score": target_under_score, "max_iter": max_iter,
                                     "cadence_mask": m, "over_metric_nSamples": 1}
            c.optimization_trace = []
        run = _GoodnessBatch(correctors, masks, target_over_score, target_under_score)
        if target_under_score > 0:
            run.set_neighbors(neighbors, radius, min_targets, max_targets, neighbor_index)
        results = minimize_bounded_lockstep(run.evaluate, [alpha_bounds] * B, maxiter=max_iter)
        xs = np.array([r.x for r in results])
        run.evaluate(np.arange(B), xs, record=False, finish=True)   # the minimiser does not end on its best point
        for b, c in enumerate(correctors):
            c._set_prior_width(np.median(c.lc.flux_err.value) / np.sqrt(np.abs(xs[b])))
            c.over_fitting_score = c.over_fitting_metric(n_samples=10) if target_over_score > 0 else -1.0
            c.under_fitting_score = float(run.under[b]) if target_under_score > 0 else -1.0
            c.alpha = results[b].x
        return [c.corrected_lc for c in correctors]

    def _goodness_metric_obj_fun(self, alpha):
        """Penalty = -(over metric), saturating (1 % leak) above the target (cbvcorrector.py:781-854)."""
        sigma = np.median(self.lc.flux_err.value) / np.sqrt(np.abs(alpha))
        self._set_prior_width(sigma)
        self.correct_regressioncorrector(self.design_matrix_collection, cadence_mask=self.optimization_params["cadence_mask"])
        target = self.optimization_params["target_over_score"]
        over = self.over_fitting_metric(n_samples=self.optimization_params["over_metric_nSamples"]) if target > 0 else 1.0
        if target > 0 and over >= target:
            over = target + 0.01 * (over - target)
        return -(over + 1.0)

    def copy(self):
        return copy.deepcopy(self)

    def __repr__(self):
        if self.cbvs:
            kinds = ", ".join(str(c.cbv_type) for c in self.cbvs)
            return "CBVCorrector (ID: {}, CBVs: {})".format(self.lc.targetid, kinds)
        return "CBVCorrector (ID: {}, no CBVs)".format(self.lc.targetid)


def _use_device():
    """Whether correct_batch keeps its inputs on the GPU (CUDA torch tensors, device-mode engine calls)."""
    try:
        import torch
    except ImportError:
        return False
    return torch.cuda.is_available()


def _morton(ra, dec):
    """Z-order key of sky positions: targets close on the sky get close keys."""
    x = np.clip(np.asarray(ra, dtype=np.float64) / 360.0 * 65535, 0, 65535).astype(np.uint64)
    y = np.clip((np.asarray(dec, dtype=np.float64) + 90.0) / 180.0 * 65535, 0, 65535).astype(np.uint64)
    key = np.zeros_like(x)
    for bit in range(16):
        key |= ((x >> np.uint64(bit)) & np.uint64(1)) << np.uint64(2 * bit)
        key |= ((y >> np.uint64(bit)) & np.uint64(1)) << np.uint64(2 * bit + 1)
    return key


class _GoodnessBatch:
    """The objective of CBVCorrector.correct for a set of correctors, one round at a time: the regression with
    per-corrector priors, the over-fitting metric (K1 periodograms + lkb_overfit_terms) and the under-fitting metric
    (lkb_underfit_metric), as in _goodness_metric_obj_fun (cbvcorrector.py:781-854).

    The design matrices, fluxes, flux errors and cadence masks (per design-matrix shape), the original periodograms
    and the neighbour pool go to the device once and stay there; a round gathers the rows of its active correctors
    there.  Per round the models come back (the normalisation by each corrected light curve's median and the white
    noise, drawn from numpy's global stream, are host work on arrays) and the corrected rows, the noise rows and the
    under-fitting target rows go up; the power rows never leave the device.  Corrector state (light curves,
    diagnostics) is built once, at the final re-fit."""

    def __init__(self, correctors, masks, target_over, target_under):
        self.dev = _use_device()
        self.cs = correctors
        self.target_over, self.target_under = target_over, target_under
        B = len(correctors)
        self.masks, self.flux, self.fe_used, self.time_used, self.sigma0 = [], [], [], [], []
        for c, m in zip(correctors, masks):
            n = len(c.lc.flux)
            m = np.ones(n, bool) if m is None else np.asarray(m, dtype=bool)
            if m.shape != (n,):
                raise ValueError("cadence_mask must have one entry per cadence")
            self.masks.append(m)
            fe = np.asarray(c.lc.flux_err.value, dtype=np.float64)
            self.flux.append(np.asarray(c.lc.flux.value, dtype=np.float64))
            self.fe_used.append(((fe ** 2 + 0.0 ** 2) ** 0.5)[m])           # the corrected light curve's flux_err
            self.time_used.append(np.asarray(c.lc.time.value, dtype=np.float64)[m])
            self.sigma0.append(np.median(c.lc.flux_err.value))
        self.groups = []
        by_shape = {}
        for b, c in enumerate(correctors):
            X = RegressionCorrector._dense_X(c.design_matrix_collection)
            by_shape.setdefault(X.shape, []).append((b, X))
        for shape, items in by_shape.items():
            members = [b for b, _ in items]
            Xs = [X for _, X in items]
            shared = all(X is Xs[0] or np.array_equal(X, Xs[0]) for X in Xs)
            FE = np.stack([np.asarray(correctors[b].lc.flux_err.value, dtype=np.float64) for b in members])
            allnan = np.all(~np.isfinite(FE), axis=1)
            self.groups.append(dict(
                members=members, set=set(members), pos={b: j for j, b in enumerate(members)}, K=shape[1],
                shared=shared, X=self.up(Xs[0] if shared else np.stack(Xs)),
                Y=self.up(np.stack([self.flux[b] for b in members])),
                FE=None if allnan.all() else self.up(np.where(allnan[:, None], 1.0, FE)),
                CM=self.up(np.stack([self.masks[b] for b in members]).astype(np.uint8)),
                PM=np.stack([np.asarray(correctors[b].design_matrix_collection.prior_mu, dtype=np.float64)
                             for b in members])))
        self.under = np.full(B, np.nan)
        self.cta_order = None
        if target_over > 0:
            self._setup_periodograms()

    # ---- host numpy or device tensors, one code path ----
    def up(self, a):
        a = np.ascontiguousarray(a)
        if not self.dev:
            return a
        import torch
        return torch.from_numpy(a).cuda()

    def down(self, a):
        return a.cpu().numpy() if self.dev else np.asarray(a)

    def take(self, a, rows):
        """Rows `rows` (host int array, or None for all) of a resident array."""
        if rows is None or a is None:
            return a
        if self.dev:
            import torch
            return a.index_select(0, torch.from_numpy(np.asarray(rows, dtype=np.int64)).cuda())
        return np.ascontiguousarray(a[rows])

    def _setup_periodograms(self):
        """The original light curve's periodogram of each corrector, once: its grid serves every later periodogram.
        Correctors with the same grid and kernel family form one periodogram group, whose original power rows stay
        resident."""
        from ..periodogram import _PER_DAY, LombScarglePeriodogram
        self.pg, self.ls_groups = [], {}
        orig_rows = {}
        for b, (c, m) in enumerate(zip(self.cs, self.masks)):
            orig, oflux = _centred(c.lc.copy()[m])
            prep = LombScarglePeriodogram._prepare(orig)
            freq = np.asarray(prep["frequency"].to(_PER_DAY).value, dtype=np.float64)
            t = np.asarray(prep["time"], dtype=np.float64)
            # the family the corrector's own call would take (never decided from the batch)
            fam = "nufft" if len(t) * len(freq) >= _LS_NUFFT_MIN_WORK else "direct"
            key = (freq.tobytes(), fam)
            g = self.ls_groups.setdefault(key, dict(members=[], freq=freq, fam=fam))
            self.pg.append(dict(time=t, key=key, row=len(g["members"])))
            g["members"].append(b)
            orig_rows[b] = (t, oflux)
        for key, g in self.ls_groups.items():
            g["freq_dev"] = self.up(g["freq"])
            g["orig"] = self._power(g, [orig_rows[b] for b in g["members"]])

    def _power(self, g, rows):
        """float32 amplitude power [len(rows), F] of (time, flux) rows on the group's grid (device or host)."""
        from .. import engine
        times, fluxes = [r[0] for r in rows], [r[1] for r in rows]
        algos = [g["fam"], "direct"] if g["fam"] == "nufft" else ["direct"]
        for k, algo in enumerate(algos):
            try:
                if not self.dev:
                    return np.asarray(engine.ls_power_ragged(times, fluxes, g["freq"], "amplitude", None, algo=algo),
                                      dtype=np.float32)
                off = np.zeros(len(rows) + 1, np.int64)
                off[1:] = np.cumsum([len(t) for t in times])
                return engine.ls_power_ragged_device(self.up(np.concatenate(times)), self.up(np.concatenate(fluxes)),
                                                     off, g["freq_dev"], "amplitude", None, algo=algo)
            except Exception as e:
                # LKB_E_UNSUPPORTED from the non-uniform FFT (unsorted times, too few cadences): the direct sums, as
                # the library's `auto` does for a light curve that does not qualify
                if k + 1 == len(algos) or getattr(e, "status", None) != -5:
                    raise

    def set_neighbors(self, neighbors, radius, min_targets, max_targets, neighbor_index):
        cs = self.cs
        if any(c.interpolated_cbvs for c in cs):
            raise NotImplementedError("correct_batch cannot compute the under-fitting metric of correctors built with "
                                      "interpolate_cbvs=True: their neighbours would be interpolated pair by pair")
        default = neighbors is None
        pool = [c.lc for c in cs] if default else list(neighbors)
        if neighbor_index is not None and len(neighbor_index) != len(cs):
            raise ValueError("neighbor_index needs one index list per corrector")
        coords = None
        if neighbor_index is None:
            coords = np.array([_sky(p) for p in pool]).reshape(-1, 2)
        sel = []
        for b, c in enumerate(cs):
            excl = _own_entries(c.lc, pool) | ({b} if default else set())
            sel.append(_select_neighbors(c.lc, pool, excl, radius, min_targets, max_targets,
                                         None if neighbor_index is None else neighbor_index[b], coords))
        used = sorted({i for s in sel for i in s})
        for c in cs:
            _require_cadenceno(c.lc)
        for p in used:
            _require_cadenceno(pool[p])
        if coords is not None:
            # pool rows and target CTAs in sky (Z-) order: targets that share neighbours run in the same CTA wave and
            # re-read those rows from L2.  The kernel's results do not depend on the order.
            used = [used[k] for k in np.argsort(_morton(coords[used, 0], coords[used, 1]), kind="stable")]
            own = np.array([_sky(c.lc) for c in cs]).reshape(-1, 2)
            self.cta_order = np.argsort(_morton(own[:, 0], own[:, 1]), kind="stable")
        row_of = {p: r for r, p in enumerate(used)}
        self.c0, self.G = _cadence_grid([np.asarray(c.lc.cadenceno)[m] for c, m in zip(cs, self.masks)])
        self.pool = self.up(_neighbor_rows([pool[p] for p in used], None, None, self.c0, self.G))
        self.pos_on_grid = [np.asarray(c.lc.cadenceno, dtype=np.int64)[m] - self.c0 for c, m in zip(cs, self.masks)]
        self.nb = [np.array([row_of[i] for i in s], dtype=np.int32) for s in sel]

    def _centred(self, b, model):
        """The corrected light curve on its used cadences, ``remove_nans().normalize() - 1`` (metrics._centred on
        arrays): (kept cadences, centred flux, mean normalised flux_err)."""
        f = self.flux[b][self.masks[b]] - model[self.masks[b]]
        keep = ~np.isnan(f)
        if not keep.all():
            f = f[keep]
        med = np.median(f)
        with np.errstate(divide="ignore", invalid="ignore"):
            return keep, f / med - 1.0, np.nanmean(self.fe_used[b][keep] / med)

    def evaluate(self, idx, alphas, record=True, finish=False):
        from .. import engine
        idx = np.asarray(idx)
        cs = self.cs
        pos = {b: k for k, b in enumerate(idx)}
        models = {}
        # regression: every corrector its own prior width, results independent of the batch
        for g in self.groups:
            act = [b for b in idx if b in g["set"]]
            if not act:
                continue
            rows = None if len(act) == len(g["members"]) else [g["pos"][b] for b in act]
            ps = np.stack([np.ones(g["K"]) * (self.sigma0[b] / np.sqrt(np.abs(alphas[pos[b]]))) for b in act])
            pm = g["PM"] if rows is None else g["PM"][rows]
            res = engine.regress(g["X"] if g["shared"] else self.take(g["X"], rows), self.take(g["Y"], rows),
                                 self.take(g["FE"], rows), self.take(g["CM"], rows), self.up(pm), self.up(ps),
                                 exact_invariant=True)
            status = self.down(res["status"])
            if np.any(status != 0):
                raise np.linalg.LinAlgError("Singular matrix")
            model = self.down(res["model"])
            if finish:
                coeff, om = self.down(res["coefficients"]), self.down(res["outlier_mask"]).astype(bool)
            for j, b in enumerate(act):
                models[b] = model[j]
                if finish:
                    c = cs[b]
                    c.cadence_mask = self.masks[b]
                    c.outlier_mask = om[j]
                    c.coefficients = coeff[j]
                    c.coefficients_err = np.zeros(len(c.coefficients)) * np.nan
                    c._finish(model[j])
        n = len(idx)
        cen = {b: self._centred(b, models[b]) for b in idx}
        over, under = np.ones(n), np.ones(n)
        npos, spos, nmean = np.zeros(n, np.int64), np.full(n, np.nan), np.full(n, np.nan)
        if self.target_over > 0:
            noise = {}
            for b in idx:                                     # numpy's global stream, in batch order
                noise[b] = (np.random.randn(len(self.pg[b]["time"]), 1) * cen[b][2]).T[0]
            for key, g in self.ls_groups.items():
                act = [b for b in idx if self.pg[b]["key"] == key]
                if not act:
                    continue
                rows = [(self.time_used[b][cen[b][0]], cen[b][1]) for b in act] + \
                       [(self.pg[b]["time"], noise[b]) for b in act]
                pw = self._power(g, rows)
                m = len(act)
                orig = g["orig"] if m == len(g["members"]) else self.take(g["orig"], [self.pg[b]["row"] for b in act])
                terms = {name: self.down(v) for name, v in engine.overfit_terms(pw[:m], orig, pw[m:], None, 1).items()}
                for j, b in enumerate(act):
                    k = pos[b]
                    npos[k] = int(terms["n_positive"][j])
                    spos[k] = float(terms["sum_positive"][j])
                    nmean[k] = float(terms["noise_mean"][j, 0])
                    over[k] = _overfit_from_terms(npos[k], spos[k], [nmean[k]])
        if self.target_under > 0:
            order = idx if self.cta_order is None else np.array([b for b in self.cta_order if b in pos])
            T = np.full((n, self.G), np.nan)
            for r, b in enumerate(order):
                keep, cflux, _ = cen[b]
                T[r, self.pos_on_grid[b][keep]] = cflux
            off = np.zeros(n + 1, np.int64)
            off[1:] = np.cumsum([len(self.nb[b]) for b in order])
            met = self.down(engine.underfit_metric(self.pool, self.up(T), off,
                                                   np.concatenate([self.nb[b] for b in order]))["metric"])
            for r, b in enumerate(order):
                under[pos[b]] = met[r]
            self.under[idx] = under
        pen = np.empty(n)
        for k, b in enumerate(idx):
            o, un = over[k], under[k]
            if record:
                cs[b].optimization_trace.append((float(alphas[k]), float(o), float(un), float(nmean[k]), int(npos[k]),
                                                 float(spos[k])))
            if self.target_over > 0 and o >= self.target_over:
                o = self.target_over + 0.01 * (o - self.target_over)
            if self.target_under > 0 and un >= self.target_under:
                un = self.target_under + 0.01 * (un - self.target_under)
            pen[k] = -(o + un)
        return pen
