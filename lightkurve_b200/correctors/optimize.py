"""Lock-step bounded scalar minimisation for many objectives at once: a vectorised restatement of scipy's
``_minimize_scalar_bounded`` (``minimize_scalar(method="Bounded")``, Brent's method with golden-section steps), which
``CBVCorrector.correct`` runs over the regularisation strength alpha.

Each problem follows scipy's iteration exactly - the same sequence of evaluated x, the same x, fun, nfev and status -
but the objectives of all still-active problems are evaluated together, one x per problem per round, so that one
batched GPU call serves every problem of the round.  Problems that have converged leave the active set.
"""
import numpy as np
from scipy.optimize import OptimizeResult

__all__ = ["minimize_bounded_lockstep"]

_MESSAGES = {0: "Solution found.", 1: "Maximum number of function calls reached.", 2: "NaN result encountered."}


def minimize_bounded_lockstep(evaluate, bounds, xatol=1e-5, maxiter=500):
    """Minimise n scalar functions on their bounds in lock step.

    `evaluate(idx, x)` receives the indices of the problems evaluated this round (int array, ascending) and one x per
    problem, and returns their objective values.  `bounds`: [n, 2] (or one pair for all).  Returns one
    `scipy.optimize.OptimizeResult` per problem, equal to what ``minimize_scalar(f_i, method="Bounded",
    bounds=bounds[i], options={"xatol": xatol, "maxiter": maxiter})`` returns for problem i on its own."""
    bounds = np.asarray(bounds, dtype=np.float64)
    if bounds.ndim == 1:
        bounds = bounds[None, :]
    if bounds.ndim != 2 or bounds.shape[1] != 2:
        raise ValueError("bounds must have two elements.")
    if not np.all(np.isfinite(bounds)):
        raise ValueError("Optimization bounds must be finite scalars.")
    if np.any(bounds[:, 0] > bounds[:, 1]):
        raise ValueError("The lower bound exceeds the upper bound.")
    n = len(bounds)
    maxfun = maxiter
    sqrt_eps = np.sqrt(2.2e-16)
    golden_mean = 0.5 * (3.0 - np.sqrt(5.0))
    a, b = bounds[:, 0].copy(), bounds[:, 1].copy()
    fulc = a + golden_mean * (b - a)
    nfc, xf = fulc.copy(), fulc.copy()
    rat = np.zeros(n)
    e = np.zeros(n)
    fx = np.asarray(evaluate(np.arange(n), xf.copy()), dtype=np.float64).copy()
    num = np.ones(n, dtype=np.int64)
    fu = np.full(n, np.inf)
    ffulc, fnfc = fx.copy(), fx.copy()
    xm = 0.5 * (a + b)
    tol1 = sqrt_eps * np.abs(xf) + xatol / 3.0
    tol2 = 2.0 * tol1
    flag = np.zeros(n, dtype=np.int64)
    active = np.abs(xf - xm) > (tol2 - 0.5 * (b - a))
    with np.errstate(all="ignore"):
        while np.any(active):
            i = np.nonzero(active)[0]
            A, Bb, XF, FX, NFC, FNFC, FULC, FFULC = a[i], b[i], xf[i], fx[i], nfc[i], fnfc[i], fulc[i], ffulc[i]
            E, RAT, T1, T2, XM = e[i], rat[i], tol1[i], tol2[i], xm[i]
            # parabolic fit where |e| > tol1
            para = np.abs(E) > T1
            r = (XF - NFC) * (FX - FFULC)
            q = (XF - FULC) * (FX - FNFC)
            p = (XF - FULC) * q - (XF - NFC) * r
            q = 2.0 * (q - r)
            p = np.where(q > 0.0, -p, p)
            q = np.abs(q)
            r = E
            e_para = RAT
            accept = para & (np.abs(p) < np.abs(0.5 * q * r)) & (p > q * (A - XF)) & (p < q * (Bb - XF))
            rat_p = (p + 0.0) / q
            x_p = XF + rat_p
            near = ((x_p - A) < T2) | ((Bb - x_p) < T2)
            si = np.sign(XM - XF) + ((XM - XF) == 0)
            rat_p = np.where(near, T1 * si, rat_p)
            # golden-section step everywhere else
            e_gold = np.where(XF >= XM, A - XF, Bb - XF)
            E = np.where(accept, e_para, e_gold)
            RAT = np.where(accept, rat_p, golden_mean * e_gold)
            si = np.sign(RAT) + (RAT == 0)
            x = XF + si * np.maximum(np.abs(RAT), T1)
            FU = np.asarray(evaluate(i, x.copy()), dtype=np.float64)
            num[i] += 1
            better = FU <= FX
            right = x >= XF
            a[i] = np.where(better, np.where(right, XF, A), np.where(x < XF, x, A))
            b[i] = np.where(better, np.where(right, Bb, XF), np.where(x < XF, Bb, x))
            c1 = (FU <= FNFC) | (NFC == XF)
            c2 = (FU <= FFULC) | (FULC == XF) | (FULC == NFC)
            fulc[i] = np.where(better | c1, NFC, np.where(c2, x, FULC))
            ffulc[i] = np.where(better | c1, FNFC, np.where(c2, FU, FFULC))
            nfc[i] = np.where(better, XF, np.where(c1, x, NFC))
            fnfc[i] = np.where(better, FX, np.where(c1, FU, FNFC))
            xf[i] = np.where(better, x, XF)
            fx[i] = np.where(better, FU, FX)
            e[i], rat[i], fu[i] = E, RAT, FU
            xm[i] = 0.5 * (a[i] + b[i])
            tol1[i] = sqrt_eps * np.abs(xf[i]) + xatol / 3.0
            tol2[i] = 2.0 * tol1[i]
            hit = num[i] >= maxfun
            flag[i[hit]] = 1
            active[i] = ~hit & (np.abs(xf[i] - xm[i]) > (tol2[i] - 0.5 * (b[i] - a[i])))
    flag[np.isnan(xf) | np.isnan(fx) | np.isnan(fu)] = 2
    return [OptimizeResult(fun=fx[k], status=int(flag[k]), success=bool(flag[k] == 0), message=_MESSAGES[int(flag[k])],
                           x=xf[k], nfev=int(num[k]), nit=int(num[k])) for k in range(n)]
