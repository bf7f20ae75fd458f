"""The lock-step bounded minimiser of CBVCorrector.correct_batch (lightkurve_b200/correctors/optimize.py) against
scipy.optimize.minimize_scalar(method="Bounded"): the same evaluated x, bit for bit, and the same x, fun, nfev and
status, for a batch of mixed objectives run together."""
import numpy as np
import pytest
from scipy.optimize import minimize_scalar

from lightkurve_b200.correctors.optimize import minimize_bounded_lockstep


def saturating(x):
    """CBVCorrector-like: rises to a target, then nearly flat (the 1 % leak above the target)."""
    m = 1.0 - np.exp(-x / 30.0)
    return -(0.5 + 0.01 * (m - 0.5)) if m >= 0.5 else -m


OBJECTIVES = [
    ("smooth", lambda x: (x - 2.3) ** 2 + 0.1 * np.sin(3 * x), (-5.0, 7.0)),
    ("flat", lambda x: 1.0, (0.0, 1.0)),
    ("saturating", saturating, (1e-4, 1e4)),
    ("lower boundary", lambda x: x, (1e-4, 1e4)),
    ("upper boundary", lambda x: -np.log(x), (1e-4, 1e4)),
    ("kinked", lambda x: abs(x - 1.0 / 3.0) + 1e-3 * x, (-1.0, 2.0)),
    ("quantised", lambda x: np.floor(x * 7.0) / 7.0 + (x - 3.0) ** 2, (0.0, 10.0)),
    ("degenerate bounds", lambda x: x * x, (2.0, 2.0)),
    ("nan", lambda x: np.nan if x > 4.0 else (x - 1.0) ** 2, (0.0, 10.0)),
]


def scipy_trace(f, bounds, maxiter):
    xs = []

    def g(x):
        xs.append(x)
        return f(x)
    r = minimize_scalar(g, method="Bounded", bounds=bounds, options={"maxiter": maxiter})
    return r, xs


@pytest.mark.parametrize("maxiter", [1, 3, 8, 100, 500])
def test_lockstep_matches_scipy(maxiter):
    fs = [o[1] for o in OBJECTIVES]
    bounds = [o[2] for o in OBJECTIVES]
    traces = [[] for _ in fs]
    rounds = []

    def evaluate(idx, x):
        rounds.append(len(idx))
        out = []
        for i, xi in zip(idx, x):
            traces[i].append(xi)
            out.append(fs[i](xi))
        return out

    res = minimize_bounded_lockstep(evaluate, bounds, maxiter=maxiter)
    for k, (name, f, bd) in enumerate(OBJECTIVES):
        ref, xs = scipy_trace(f, bd, maxiter)
        assert [float(v).hex() for v in traces[k]] == [float(v).hex() for v in xs], name
        assert float(res[k].x).hex() == float(ref.x).hex(), name
        assert (np.isnan(ref.fun) and np.isnan(res[k].fun)) or float(res[k].fun).hex() == float(ref.fun).hex(), name
        assert res[k].nfev == ref.nfev and res[k].status == ref.status, name
        assert res[k].success == ref.success and res[k].message == ref.message, name
    assert rounds == sorted(rounds, reverse=True)            # problems only ever leave the active set


def test_lockstep_many_random_parabolas():
    rng = np.random.default_rng(3)
    n = 200
    c, w = rng.uniform(-3, 3, n), rng.uniform(0.1, 5, n)
    bounds = np.stack([rng.uniform(-5, -1, n), rng.uniform(1, 5, n)], axis=1)

    def f(k, x):
        return w[k] * (x - c[k]) ** 2 + np.cos(x * w[k])

    def evaluate(idx, x):                 # element by element: numpy's array cos may round unlike its scalar cos
        return [f(k, xk) for k, xk in zip(idx, x)]

    res = minimize_bounded_lockstep(evaluate, bounds, maxiter=50)
    for k in range(n):
        ref = minimize_scalar(lambda x: f(k, x), method="Bounded",
                              bounds=tuple(bounds[k]), options={"maxiter": 50})
        assert res[k].x == ref.x and res[k].fun == ref.fun and res[k].nfev == ref.nfev, k


def test_lockstep_bound_errors():
    with pytest.raises(ValueError, match="lower bound exceeds"):
        minimize_bounded_lockstep(lambda i, x: x, [[2.0, 1.0]])
    with pytest.raises(ValueError, match="finite"):
        minimize_bounded_lockstep(lambda i, x: x, [[0.0, np.inf]])
