"""Elastic-net oracle: a numpy restatement of scikit-learn 1.9's
``ElasticNet(fit_intercept=False, precompute=False, selection="cyclic").fit(X, y)``
(``linear_model/_coordinate_descent.py`` ``enet_path`` and ``_cd_fast.pyx`` ``enet_coordinate_descent`` /
``gap_enet`` / ``dual_gap_formulation_A``), which ``CBVCorrector.correct_elasticnet`` calls.

It minimises  1/2 ||y - X w||^2 + l1 ||w||_1 + l2/2 ||w||^2  with  l1 = alpha l1_ratio n,
l2 = alpha (1 - l1_ratio) n  (n = number of rows), by cyclic coordinate descent that stops on the duality gap
``gap <= tol * y.y``.  The gap is only evaluated before the first sweep, after a sweep whose largest coefficient
change is small (``d_w_max / w_max <= tol``, or ``w_max == 0``) and after the last sweep; with ``l1 > 0`` each
evaluation also runs gap-safe screening (columns proven zero at the optimum are dropped for good).

Besides the fit, ``enet_fit`` reports ``margin``: the smallest relative distance of any of the run's discrete
decisions (the two stopping tests and the screening tests) from its threshold.  A run whose margin is tiny can
legitimately stop one sweep earlier or later under a different rounding (e.g. the Gram-matrix formulation of the
GPU kernel), so tests pick fixtures whose margin is comfortably above the rounding level.

Test infrastructure only: nothing in the product imports this module."""
import numpy as np

SKLEARN_VERSION = "1.9.0"          # the release this restatement was written against

MESSAGE_CONV = ("Objective did not converge. You might want to increase the number of iterations, check the scale "
                "of the features or consider increasing regularisation.")
MESSAGE_RIDGE = ("Linear regression models with a zero l1 penalization strength are more efficiently fitted using "
                 "one of the solvers implemented in sklearn.linear_model.Ridge/RidgeCV instead.")
MESSAGE_ALPHA0 = ("With alpha=0, this algorithm does not converge well. You are advised to use the LinearRegression "
                  "estimator")


def convergence_message(gap, tol, l1):
    """Text of the ConvergenceWarning (gap and tol in the unscaled units of the coordinate descent)."""
    msg = MESSAGE_CONV + f" Duality gap: {gap:.6e}, tolerance: {tol:.3e}"
    if l1 < np.finfo(np.float64).eps:
        msg += "\n" + MESSAGE_RIDGE
    return msg


def _rel(a, b):
    return abs(a - b) / max(abs(b), 1e-300)


def _gap(X, y, w, R, l1, l2, positive):
    """(gap, X^T R - l2 w, dual norm): formulation A (l1 > 0), B (l1 = 0 < l2) or ||X^T R||^2 (both 0)."""
    w_l2 = float(w @ w) if l2 > 0 else 0.0
    R2 = float(R @ R)
    Ry = float(R @ y) if not (l1 == 0 and l2 == 0) else 0.0
    if l1 == 0:
        XtA = X.T @ R
        dn = float(XtA @ XtA)
        if l2 == 0:
            return dn, XtA, dn
        gap = R2 + 0.5 * l2 * w_l2 - Ry
        gap += 1 / (2 * l2) * dn
        return gap, XtA, dn
    XtA = X.T @ R - l2 * w
    dn = float(np.max(XtA)) if positive else float(np.max(np.abs(XtA)))
    primal = 0.5 * (R2 + l2 * w_l2) + l1 * float(np.sum(np.abs(w)))
    scale = l1 / dn if dn > l1 else 1.0
    dual = -0.5 * scale ** 2 * (R2 + l2 * w_l2) + scale * Ry
    return primal - dual, XtA, dn


def enet_fit(X, y, alpha=1.0, l1_ratio=0.5, max_iter=1000, tol=1e-4, positive=False):
    """Returns dict(coef [K], n_iter, dual_gap (= gap / n, sklearn's ``dual_gap_``), gap, tol (scaled),
    converged, l1, l2, margin)."""
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    n, K = X.shape
    l1 = alpha * l1_ratio * n
    l2 = alpha * (1.0 - l1_ratio) * n
    norm2 = np.einsum("ij,ij->j", X, X)
    w = np.zeros(K)
    R = y.copy()
    d_w_tol = tol
    tol = tol * float(y @ y)
    screening = l1 != 0
    margin = np.inf

    def note(value, threshold):
        nonlocal margin
        margin = min(margin, _rel(value, threshold))

    def screen(gap, XtA, dn, active, excluded, first):
        new = []
        for j in range(K):
            if first and norm2[j] == 0:
                w[j] = 0.0
                excluded[j] = True
                continue
            if excluded[j]:
                continue
            d_j = (1 - abs(XtA[j] / max(l1, dn))) / np.sqrt(norm2[j] + l2)
            thr = np.sqrt(2 * gap) / l1
            note(d_j, thr)
            if d_j <= thr:
                new.append(j)
                excluded[j] = False
            else:
                if w[j] != 0:
                    R[:] += w[j] * X[:, j]
                    w[j] = 0.0
                excluded[j] = True
        active[:] = new

    gap, XtA, dn = _gap(X, y, w, R, l1, l2, positive)
    note(gap, tol)
    out = dict(l1=l1, l2=l2, tol=tol)
    if gap <= tol:
        return dict(out, coef=w, n_iter=0, gap=gap, dual_gap=gap / n, converged=True, margin=margin)
    active = list(range(K))
    excluded = np.zeros(K, bool)
    if screening:
        screen(gap, XtA, dn, active, excluded, True)
    converged = False
    n_iter = 0
    for n_iter in range(max_iter):
        w_max = 0.0
        d_w_max = 0.0
        for j in active:
            if norm2[j] == 0.0:
                continue
            w_j = w[j]
            tmp = float(X[:, j] @ R) + w_j * norm2[j]
            if positive and tmp < 0:
                w[j] = 0.0
            else:
                w[j] = np.sign(tmp) * max(abs(tmp) - l1, 0.0) / (norm2[j] + l2)
            if w[j] != w_j:
                R += (w_j - w[j]) * X[:, j]
            d_w_max = max(d_w_max, abs(w[j] - w_j))
            w_max = max(w_max, abs(w[j]))
        if w_max != 0.0:
            note(d_w_max / w_max, d_w_tol)
        if w_max == 0.0 or d_w_max / w_max <= d_w_tol or n_iter == max_iter - 1:
            gap, XtA, dn = _gap(X, y, w, R, l1, l2, positive)
            note(gap, tol)
            if gap <= tol:
                converged = True
                break
            if screening:
                screen(gap, XtA, dn, active, excluded, False)
    return dict(out, coef=w, n_iter=n_iter + 1, gap=gap, dual_gap=gap / n, converged=converged, margin=margin)


def cbv_fixture(seed, N=2000, K=9, scale=1e4, kind="correlated", noise=1e-3):
    """A CBV-like design matrix [N, K] whose last column is the constant (as CBVCorrector builds it) and a flux in
    units of `scale` (e-/s when scale ~ 1e4).  kind="correlated": random-walk vectors, not orthogonal to the constant;
    kind="orthonormal": centred orthonormal vectors (what the mission's CBVs are)."""
    rng = np.random.default_rng(seed)
    if kind == "correlated":
        V = np.cumsum(rng.normal(size=(N, K - 1)), axis=0) / np.sqrt(N)
    else:
        V = np.linalg.qr(rng.normal(size=(N, K - 1)) - 0.0)[0]
        V -= V.mean(axis=0)
        V /= np.linalg.norm(V, axis=0)
    X = np.hstack([V, np.ones((N, 1))])
    w = rng.normal(size=K - 1) * np.geomspace(1.0, 1e-2, K - 1)
    y = scale * (1.0 + 0.01 * (V @ w) + noise * rng.normal(size=N))
    return X, y


def elasticnet(X, Y, cadence_mask=None, alpha=1e-20, l1_ratio=0.01, max_iter=1000, tol=1e-4, positive=False):
    """The batched contract of ``engine.elasticnet`` on the oracle: X [N, K] or [B, N, K], Y [B, N], cadence_mask
    bool [B, N] or None.  Returns dict(coefficients [B, K], model [B, N] = X[:, :-1] @ coef[:-1] minus its median
    over all cadences, n_iter [B], dual_gap [B], converged [B], gap [B], tol [B] (the last two unscaled))."""
    X = np.asarray(X, dtype=np.float64)
    Y = np.atleast_2d(np.asarray(Y, dtype=np.float64))
    B, N = Y.shape
    K = X.shape[-1]
    cm = np.ones((B, N), bool) if cadence_mask is None else np.broadcast_to(np.asarray(cadence_mask, bool), (B, N))
    out = dict(coefficients=np.empty((B, K)), model=np.empty((B, N)), n_iter=np.empty(B, np.int32),
               dual_gap=np.empty(B), converged=np.empty(B, bool), gap=np.empty(B), tol=np.empty(B),
               margin=np.empty(B))
    for b in range(B):
        Xb = X[b] if X.ndim == 3 else X
        r = enet_fit(Xb[cm[b]], Y[b][cm[b]], alpha, l1_ratio, max_iter, tol, positive)
        out["coefficients"][b] = r["coef"]
        model = Xb[:, :-1] @ r["coef"][:-1]
        out["model"][b] = model - np.median(model)
        for k in ("n_iter", "dual_gap", "converged", "gap", "tol", "margin"):
            out[k][b] = r[k]
    return out
