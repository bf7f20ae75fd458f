"""oracle/enet.py pinned to scikit-learn's ElasticNet(fit_intercept=False) where scikit-learn imports (and is the
release the restatement was written against): identical n_iter_, coefficients within rtol 1e-10, the same dual_gap_
and the same ConvergenceWarning."""
import warnings

import numpy as np
import pytest

from oracle import enet as oen

sklearn = pytest.importorskip("sklearn")
if sklearn.__version__ != oen.SKLEARN_VERSION:
    pytest.skip("oracle/enet.py restates scikit-learn %s, found %s" % (oen.SKLEARN_VERSION, sklearn.__version__),
                allow_module_level=True)
from sklearn.exceptions import ConvergenceWarning  # noqa: E402
from sklearn.linear_model import ElasticNet  # noqa: E402

MARGIN = 1e-9


def pick(make, seeds=range(0, 40), **kw):
    """The first seed whose stopping and screening decisions all lie further than MARGIN (relative) from their
    thresholds; a replaced seed is reported."""
    for s in seeds:
        X, y = make(s)
        r = oen.enet_fit(X, y, **kw)
        if r["margin"] > MARGIN:
            return X, y, r
        print("seed %d replaced: a decision lies %.2e (relative) from its threshold" % (s, r["margin"]))
    raise AssertionError("no seed with a clear stopping decision")


def sk_fit(X, y, alpha, l1_ratio, **kw):
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        m = ElasticNet(alpha=alpha, l1_ratio=l1_ratio, fit_intercept=False, **kw).fit(X, y)
    return m, rec


def compare(X, y, alpha, l1_ratio, **kw):
    r = oen.enet_fit(X, y, alpha=alpha, l1_ratio=l1_ratio, **kw)
    m, rec = sk_fit(X, y, alpha, l1_ratio, **kw)
    assert r["n_iter"] == m.n_iter_
    np.testing.assert_allclose(r["coef"], m.coef_, rtol=1e-10, atol=1e-10 * np.max(np.abs(m.coef_)))
    # the gap is a difference of terms of order y.y: compare it at that scale
    np.testing.assert_allclose(r["dual_gap"], m.dual_gap_, rtol=1e-6, atol=1e-12 * float(y @ y) / len(y))
    conv = [str(w.message) for w in rec if issubclass(w.category, ConvergenceWarning)]
    if r["converged"]:
        assert not conv
    else:
        assert conv == [oen.convergence_message(r["gap"], r["tol"], r["l1"])]
    return r, m


CASES = [(1e-20, 0.01), (1.0, 0.9), (1e-3, 0.5), (10.0, 1.0)]


@pytest.mark.parametrize("alpha,l1_ratio", CASES)
@pytest.mark.parametrize("kind", ["correlated", "orthonormal"])
@pytest.mark.parametrize("scale", [1.0, 1e4])
def test_oracle_matches_sklearn(alpha, l1_ratio, kind, scale):
    a = alpha * scale if alpha >= 1 else alpha              # keep the L1 cases meaningful at both flux scales
    X, y, r = pick(lambda s: oen.cbv_fixture(s, N=3000, K=9, scale=scale, kind=kind), alpha=a, l1_ratio=l1_ratio)
    compare(X, y, a, l1_ratio)


def test_defaults_stop_before_least_squares():
    """The default alpha/l1_ratio stop on the coefficient change long before the minimiser: the answer is the
    iteration's, not least squares'."""
    X, y, r = pick(lambda s: oen.cbv_fixture(s, N=20000, K=9, scale=1e4), alpha=1e-20, l1_ratio=0.01)
    compare(X, y, 1e-20, 0.01)
    ls = np.linalg.lstsq(X, y, rcond=None)[0]
    assert r["n_iter"] > 5
    assert np.max(np.abs(r["coef"] - ls) / np.max(np.abs(ls))) > 1e-8


def test_lasso_screening_removes_columns():
    X, y, _ = pick(lambda s: oen.cbv_fixture(s, N=2000, K=12, scale=1e4), alpha=30.0, l1_ratio=1.0)
    r, m = compare(X, y, 30.0, 1.0)
    assert np.count_nonzero(m.coef_ == 0) >= 2


def test_ridge_l1_ratio_zero():
    X, y, _ = pick(lambda s: oen.cbv_fixture(s, N=1500, K=7, scale=1e4), alpha=1e-2, l1_ratio=0.0)
    compare(X, y, 1e-2, 0.0)


def test_positive():
    X, y, _ = pick(lambda s: oen.cbv_fixture(s, N=1500, K=9, scale=1e4), alpha=1e-3, l1_ratio=0.5, positive=True)
    r, m = compare(X, y, 1e-3, 0.5, positive=True)
    assert np.all(m.coef_ >= 0)


def test_alpha_zero():
    X, y, _ = pick(lambda s: oen.cbv_fixture(s, N=800, K=5, scale=1.0), alpha=0.0, l1_ratio=0.5, max_iter=300)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        compare(X, y, 0.0, 0.5, max_iter=300)


def test_zero_column():
    X, y = oen.cbv_fixture(3, N=1000, K=8, scale=1e4)
    X[:, 2] = 0.0
    for a, l1r in ((1e-3, 0.5), (1e-2, 0.0)):
        r, m = compare(X, y, a, l1r)
        assert m.coef_[2] == 0.0


def test_max_iter_reached():
    X, y, _ = pick(lambda s: oen.cbv_fixture(s, N=2000, K=9, scale=1e4), alpha=1e-20, l1_ratio=0.01, max_iter=7)
    r, _ = compare(X, y, 1e-20, 0.01, max_iter=7)
    assert r["n_iter"] == 7 and not r["converged"]


def test_converged_before_first_sweep():
    X, _ = oen.cbv_fixture(1, N=500, K=4)
    r, m = compare(X, np.zeros(500), 1.0, 0.5)
    assert r["n_iter"] == 0 and m.n_iter_ == 0
