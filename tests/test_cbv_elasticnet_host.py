"""`CBVCorrector.correct_elasticnet` / `correct_elasticnet_batch` on the host: the corrector logic around the K8 call,
with `engine.elasticnet` replaced by an oracle-backed stand-in (oracle/enet.py).  On the GPU box
tests/test_gpu_enet.py runs the same logic on the kernel."""
import inspect
import types
import warnings

import numpy as np
import pytest

import lightkurve_b200 as lk
from lightkurve_b200 import units as u
from lightkurve_b200.correctors import CBVCorrector, CotrendingBasisVectors, DesignMatrix
from lightkurve_b200.correctors.cbvcorrector import ConvergenceWarning
from oracle import enet as oen


def oracle_elasticnet(X, Y, cadence_mask=None, alpha=1e-20, l1_ratio=0.01, max_iter=1000, tol=1e-4, positive=False):
    """`engine.elasticnet`'s contract on the oracle, with the refusals of lkb_elasticnet."""
    B, N = np.atleast_2d(Y).shape
    cm = None if cadence_mask is None else np.broadcast_to(np.asarray(cadence_mask, dtype=bool), (B, N))
    if alpha < 0 or not 0 <= l1_ratio <= 1 or max_iter < 1 or tol < 0:
        raise ValueError("lkb_elasticnet: parameter out of range")
    if cm is not None and not np.all(cm.any(axis=1)):
        raise ValueError("lkb_elasticnet: light curve %d has no used cadence" % int(np.argmin(cm.any(axis=1))))
    r = oen.elasticnet(X, Y, cm, alpha=alpha, l1_ratio=l1_ratio, max_iter=max_iter, tol=tol, positive=positive)
    return {k: r[k] for k in ("coefficients", "model", "n_iter", "dual_gap", "converged")}


@pytest.fixture
def engine(monkeypatch):
    from lightkurve_b200 import engine as eng
    monkeypatch.setattr(eng, "elasticnet", oracle_elasticnet)
    yield eng


def make_corrector(seed, N=600, n_cbv=8, scale=1e4):
    """A light curve in e-/s with in-test SingleScale CBVs (random walks) on the same cadences."""
    X, y = oen.cbv_fixture(seed, N=N, K=n_cbv + 1, scale=scale)
    cad = np.arange(100, 100 + N)
    lc = lk.LightCurve(time=np.arange(N) * 0.02, flux=y, flux_err=np.full(N, 3.0), cadenceno=cad,
                       flux_unit=u.electron / u.second)
    data = {"VECTOR_{}".format(i + 1): X[:, i] for i in range(n_cbv)}
    data["CADENCENO"] = cad
    cbvs = CotrendingBasisVectors(data, np.arange(N) * 0.02, cbv_type="SingleScale")
    return CBVCorrector(lc, cbvs=[cbvs]), X, y


KW = dict(cbv_type=["SingleScale"], cbv_indices=[np.arange(1, 9)])


def test_signature_and_defaults():
    sig = inspect.signature(CBVCorrector.correct_elasticnet).parameters
    assert list(sig)[:7] == ["self", "cbv_type", "cbv_indices", "alpha", "l1_ratio", "ext_dm", "cadence_mask"]
    assert sig["cbv_type"].default == "SingleScale"
    np.testing.assert_array_equal(sig["cbv_indices"].default, np.arange(1, 9))
    assert sig["alpha"].default == 1e-20 and sig["l1_ratio"].default == 0.01
    assert sig["ext_dm"].default is None and sig["cadence_mask"].default is None


def test_defaults_trip_the_list_assertion(engine):
    c, _, _ = make_corrector(0)
    with pytest.raises(AssertionError, match="must be lists of strings"):
        c.correct_elasticnet()


def test_correct_elasticnet_state(engine):
    c, X, y = make_corrector(1)
    out = c.correct_elasticnet(alpha=1.0, l1_ratio=0.9, **KW)
    r = oen.enet_fit(X, y, alpha=1.0, l1_ratio=0.9)
    np.testing.assert_array_equal(c.coefficients, r["coef"])
    model = X[:, :-1] @ r["coef"][:-1]
    np.testing.assert_allclose(c.model_lc.flux.value, model - np.median(model), rtol=0, atol=1e-9)
    assert np.all(c.model_lc.flux_err.value == 0)
    np.testing.assert_allclose(out.flux.value, y - c.model_lc.flux.value)
    np.testing.assert_allclose(out.flux_err.value, c.lc.flux_err.value)
    assert out is c.corrected_lc and c.alpha == 1.0 and np.all(c.cadence_mask)
    assert set(c.diagnostic_lightcurves) == {"SingleScale", "Constant"}
    np.testing.assert_allclose(c.diagnostic_lightcurves["SingleScale"].flux.value, model)
    np.testing.assert_allclose(c.diagnostic_lightcurves["Constant"].flux.value, r["coef"][-1])
    assert c.elasticnet_n_iter == r["n_iter"]


def test_cadence_mask_and_ext_dm(engine):
    c, X, y = make_corrector(2)
    mask = np.ones(len(y), bool)
    mask[100:180] = False
    ext = DesignMatrix(np.sin(np.arange(len(y)) / 17.0)[:, None], columns=["sin"], name="ext")
    c.correct_elasticnet(alpha=1e-3, l1_ratio=0.5, ext_dm=ext, cadence_mask=mask, **KW)
    Xf = np.hstack([X[:, :-1], ext.values, X[:, -1:]])
    r = oen.enet_fit(Xf[mask], y[mask], alpha=1e-3, l1_ratio=0.5)
    np.testing.assert_array_equal(c.coefficients, r["coef"])
    assert c.coefficients.shape == (10,)
    np.testing.assert_array_equal(c.cadence_mask, mask)
    model = Xf[:, :-1] @ r["coef"][:-1]                      # all cadences, without the constant
    np.testing.assert_allclose(c.model_lc.flux.value, model - np.median(model), atol=1e-9)
    assert set(c.diagnostic_lightcurves) == {"SingleScale", "ext", "Constant"}


def test_keyword_arguments(engine):
    c, X, y = make_corrector(3)
    c.correct_elasticnet(alpha=1e-3, l1_ratio=0.5, positive=True, max_iter=50, tol=1e-6, precompute=False,
                         copy_X=True, warm_start=True, random_state=4, selection="cyclic", **KW)
    r = oen.enet_fit(X, y, alpha=1e-3, l1_ratio=0.5, positive=True, max_iter=50, tol=1e-6)
    np.testing.assert_array_equal(c.coefficients, r["coef"])
    with pytest.raises(NotImplementedError):
        c.correct_elasticnet(selection="random", **KW)
    with pytest.raises(TypeError, match="fit_intercept"):
        c.correct_elasticnet(fit_intercept=True, **KW)
    with pytest.raises(ValueError):
        c.correct_elasticnet(l1_ratio=1.5, **KW)
    # a non-finite design matrix is refused before any fit (scikit-learn's check_array)
    Xbad = X.copy()
    Xbad[5, 2] = np.inf
    c.design_matrix_collection = types.SimpleNamespace(values=Xbad)
    with pytest.raises(ValueError, match="NaN or infinity"):
        CBVCorrector._run_elasticnet([c], [None], 1.0, 0.5, dict(max_iter=10, tol=1e-4, positive=False))


def test_warnings(engine):
    c, X, y = make_corrector(4)
    with pytest.warns(ConvergenceWarning) as rec:
        c.correct_elasticnet(max_iter=3, **KW)
    r = oen.enet_fit(X, y, alpha=1e-20, l1_ratio=0.01, max_iter=3)
    assert not r["converged"]
    msgs = [str(w.message) for w in rec if issubclass(w.category, ConvergenceWarning)]
    assert msgs == [oen.convergence_message(r["gap"], r["tol"], r["l1"])]
    assert "Ridge/RidgeCV" in msgs[0]
    assert issubclass(ConvergenceWarning, UserWarning)
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        c.correct_elasticnet(alpha=0.0, max_iter=20, **KW)
    assert any(str(w.message) == oen.MESSAGE_ALPHA0 for w in rec)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        c.correct_elasticnet(alpha=1.0, l1_ratio=0.9, **KW)          # converges: silent


def test_batch_equals_loop(engine):
    """Shared design matrix, per-corrector masks and ext_dm, and unequal lengths (one call per length)."""
    cs = [make_corrector(10 + i)[0] for i in range(3)] + [make_corrector(20, N=450)[0]]
    loop = [make_corrector(10 + i)[0] for i in range(3)] + [make_corrector(20, N=450)[0]]
    rng = np.random.default_rng(0)
    masks = [rng.random(len(c.lc.flux)) > 0.1 for c in cs]
    CBVCorrector.correct_elasticnet_batch(cs, alpha=1e-3, l1_ratio=0.5, cadence_mask=masks, **KW)
    for c, m in zip(loop, masks):
        c.correct_elasticnet(alpha=1e-3, l1_ratio=0.5, cadence_mask=m, **KW)
    for a, b in zip(cs, loop):
        np.testing.assert_allclose(a.coefficients, b.coefficients, rtol=1e-12)
        np.testing.assert_allclose(a.corrected_lc.flux.value, b.corrected_lc.flux.value, rtol=1e-12)
        np.testing.assert_array_equal(a.cadence_mask, b.cadence_mask)
        assert a.alpha == b.alpha and set(a.diagnostic_lightcurves) == set(b.diagnostic_lightcurves)
    # per-corrector ext_dm: equal lengths, different matrices -> one batched-X call
    cs = [make_corrector(30 + i)[0] for i in range(3)]
    exts = [DesignMatrix(np.cos(np.arange(600) / (5.0 + i))[:, None], name="ext") for i in range(3)]
    calls = []
    real = engine.elasticnet

    def spy(X, *a, **k):
        calls.append(np.ndim(X))
        return real(X, *a, **k)

    engine.elasticnet = spy
    CBVCorrector.correct_elasticnet_batch(cs, alpha=1.0, l1_ratio=0.9, ext_dm=exts, **KW)
    assert calls == [3]
    for i, (c, e) in enumerate(zip(cs, exts)):
        ref = make_corrector(30 + i)[0]
        ref.correct_elasticnet(alpha=1.0, l1_ratio=0.9, ext_dm=e, **KW)
        np.testing.assert_allclose(c.coefficients, ref.coefficients, rtol=1e-12)
