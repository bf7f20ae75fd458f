"""`CBVCorrector` and `CotrendingBasisVectors`: the caller that loops `RegressionCorrector.correct` (K5) and the
Lomb-Scargle over-fitting metric (K1) inside a bounded scalar optimiser (SURVEY.md 8(f) rank 4;
/root/reference/src/lightkurve/correctors/cbvcorrector.py:45-980 and :982-1380).

Scope: everything that runs from arrays - the basis-vector container (`to_designmatrix`, `align`, `interpolate`),
`correct_gaussian_prior`, the `correct` optimiser over the regularisation `alpha`, `over_fitting_metric`,
`correct_regressioncorrector`, and `correct_elasticnet` (scikit-learn's elastic-net coordinate descent, K8; with
`correct_elasticnet_batch` for many correctors in one call).  Out of scope here: reading CBV FITS files / downloading
them from MAST (`load_kepler_cbvs`, `load_tess_cbvs`), the under-fitting metric (it needs a MAST search of
neighbouring targets) and the plots.  Basis vectors are
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
from .metrics import overfit_metric_lombscargle
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
                alpha_bounds=[1e-4, 1e4], target_over_score=0.5, target_under_score=0.5, max_iter=100):
        """Optimise `alpha` with a bounded scalar minimiser against the goodness metrics (cbvcorrector.py:397-501).
        Only the over-fitting metric exists in this build: `target_under_score` must be 0 (the under-fitting metric
        needs neighbouring targets from MAST)."""
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

    def under_fitting_metric(self, *args, **kwargs):
        raise NotImplementedError("the under-fitting metric needs a MAST search of neighbouring targets "
                                  "(outside the scope of lightkurve_b200)")

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
