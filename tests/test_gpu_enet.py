"""K8 on the GPU: lkb_elasticnet and CBVCorrector.correct_elasticnet against oracle/enet.py (scikit-learn's
coordinate descent restated; scikit-learn itself where it imports)."""
import numpy as np
import pytest

from oracle import enet as oen

pytestmark = pytest.mark.gpu
MARGIN = 1e-6       # fixtures whose stopping/screening decisions lie closer than this to a threshold are replaced


@pytest.fixture(scope="module")
def engine():
    from lightkurve_b200 import engine as eng
    if eng.device_count() == 0:
        pytest.skip("needs a CUDA device")
    eng.init(0)
    return eng


def batch(B, N, K, seed, shared, kw, ragged=True):
    """B light curves (shared or per-light-curve X) with ragged masks whose oracle runs have clear decisions."""
    rng = np.random.default_rng(seed)
    X0, _ = oen.cbv_fixture(seed, N=N, K=K, scale=1e4)
    Xs, Ys, Ms, refs = [], [], [], []
    s = 0
    while len(refs) < B:
        s += 1
        Xb, y = oen.cbv_fixture(seed * 1000 + s, N=N, K=K, scale=1e4)
        if shared:
            Xb = X0
            w = rng.normal(size=K) * np.geomspace(1, 1e-2, K)
            y = 1e4 * (1 + 0.01 * (Xb[:, :-1] @ w[:-1]) + 1e-3 * rng.normal(size=N))
        m = rng.random(N) > (rng.uniform(0, 0.4) if ragged else 0.0)
        r = oen.enet_fit(Xb[m], y[m], **kw)
        if r["margin"] <= MARGIN:
            print("seed %d replaced: a decision lies %.2e (relative) from its threshold" % (s, r["margin"]))
            continue
        model = Xb[:, :-1] @ r["coef"][:-1]
        r["model"] = model - np.median(model)
        Xs.append(Xb), Ys.append(y), Ms.append(m), refs.append(r)
    X = X0 if shared else np.stack(Xs)
    return X, np.stack(Ys), np.stack(Ms), refs


def check(res, refs):
    for b, r in enumerate(refs):
        assert res["n_iter"][b] == r["n_iter"], (b, res["n_iter"][b], r["n_iter"])
        assert res["converged"][b] == r["converged"]
        np.testing.assert_allclose(res["coefficients"][b], r["coef"], rtol=1e-9,
                                   atol=1e-9 * np.max(np.abs(r["coef"])), err_msg="light curve %d" % b)
        assert np.max(np.abs(res["model"][b] - r["model"])) <= 1e-9 * np.max(np.abs(r["model"]))


@pytest.mark.parametrize("shared", [True, False])
@pytest.mark.parametrize("kw", [dict(alpha=1e-20, l1_ratio=0.01), dict(alpha=1.0, l1_ratio=0.9),
                                dict(alpha=30.0, l1_ratio=1.0), dict(alpha=1e-2, l1_ratio=0.0),
                                dict(alpha=1e-3, l1_ratio=0.5, positive=True),
                                dict(alpha=1e-20, l1_ratio=0.01, max_iter=5)])
def test_elasticnet_matches_oracle(engine, shared, kw):
    X, Y, M, refs = batch(24, 3000, 9, 11, shared, kw)
    res = engine.elasticnet(X, Y, M, **kw)
    check(res, refs)


@pytest.mark.parametrize("K", [1, 40, 165])
def test_elasticnet_sizes(engine, K):
    kw = dict(alpha=1e-3, l1_ratio=0.5, max_iter=300)
    X, Y, M, refs = batch(3, max(2000, 4 * K), K, 5 + K, True, kw)
    check(engine.elasticnet(X, Y, M, **kw), refs)


def test_elasticnet_bitwise_repeatable_and_batch_independent(engine):
    kw = dict(alpha=1.0, l1_ratio=0.9)
    X, Y, M, refs = batch(40, 2000, 9, 3, True, kw)
    a = engine.elasticnet(X, Y, M, **kw)
    b = engine.elasticnet(X, Y, M, **kw)
    for k in a:
        np.testing.assert_array_equal(a[k], b[k])
    one = engine.elasticnet(X, Y[17:18], M[17:18], **kw)
    np.testing.assert_array_equal(one["coefficients"][0], a["coefficients"][17])


def test_elasticnet_refusals(engine):
    from lightkurve_b200 import _lib
    X, Y, M, _ = batch(2, 500, 5, 1, True, dict(alpha=1.0, l1_ratio=0.5))
    for kw in (dict(alpha=-1.0), dict(l1_ratio=1.5), dict(max_iter=0), dict(tol=-1.0)):
        with pytest.raises(ValueError):
            engine.elasticnet(X, Y, M, **kw)
    M2 = M.copy()
    M2[1] = False
    with pytest.raises(ValueError, match="no used cadence"):
        engine.elasticnet(X, Y, M2)
    with pytest.raises(_lib.EngineError) as e:
        engine.elasticnet(np.ones((500, 166)), Y)
    assert e.value.status == _lib.E_UNSUPPORTED


def test_regress_unchanged_on_fixture(engine):
    """lkb_regress (whose Gram-kernel choice moved into a helper shared with lkb_elasticnet) still agrees with the
    oracle as tightly as smoke() requires."""
    from oracle import detrend as odet
    rng = np.random.default_rng(0)
    t = np.arange(0, 20, 0.02)
    X = np.vstack([np.sin(t), np.cos(t / 2), np.ones_like(t)]).T
    Y = 1 + (X @ np.array([0.01, -0.02, 0.0]))[None, :] + 1e-3 * rng.normal(size=(6, len(t)))
    rr = engine.regress(X, Y)
    for b in range(6):
        np.testing.assert_allclose(rr["coefficients"][b], odet.regress(X, Y[b])["coefficients"], rtol=1e-8, atol=1e-12)


def _corrector(seed, N=3000):
    import lightkurve_b200 as lk
    from lightkurve_b200 import units as u
    from lightkurve_b200.correctors import CBVCorrector, CotrendingBasisVectors
    X, y = oen.cbv_fixture(seed, N=N, K=9, scale=1e4)
    cad = np.arange(N)
    lc = lk.LightCurve(time=np.arange(N) * 0.02, flux=y, flux_err=np.full(N, 3.0), cadenceno=cad,
                       flux_unit=u.electron / u.second)
    data = {"VECTOR_{}".format(i + 1): X[:, i] for i in range(8)}
    data["CADENCENO"] = cad
    return CBVCorrector(lc, cbvs=[CotrendingBasisVectors(data, np.arange(N) * 0.02, cbv_type="SingleScale")]), X, y


KW = dict(cbv_type=["SingleScale"], cbv_indices=[np.arange(1, 9)])


def test_correct_elasticnet_matches_oracle_and_sklearn(engine):
    for seed, kw in ((1, dict(alpha=1e-20, l1_ratio=0.01)), (2, dict(alpha=1.0, l1_ratio=0.9))):
        c, X, y = _corrector(seed)
        r = oen.enet_fit(X, y, **kw)
        assert r["margin"] > MARGIN
        c.correct_elasticnet(**kw, **KW)
        assert c.elasticnet_n_iter == r["n_iter"]
        np.testing.assert_allclose(c.coefficients, r["coef"], rtol=1e-9, atol=1e-9 * np.max(np.abs(r["coef"])))
        try:
            from sklearn.linear_model import ElasticNet
        except ImportError:
            continue
        m = ElasticNet(fit_intercept=False, **kw).fit(X, y)
        assert m.n_iter_ == c.elasticnet_n_iter
        np.testing.assert_allclose(c.coefficients, m.coef_, rtol=1e-9, atol=1e-9 * np.max(np.abs(m.coef_)))


def test_correct_elasticnet_batch_equals_loop(engine):
    from lightkurve_b200.correctors import CBVCorrector
    cs = [_corrector(40 + i)[0] for i in range(5)]
    loop = [_corrector(40 + i)[0] for i in range(5)]
    rng = np.random.default_rng(1)
    masks = [rng.random(3000) > 0.2 for _ in cs]
    CBVCorrector.correct_elasticnet_batch(cs, alpha=1.0, l1_ratio=0.9, cadence_mask=masks, **KW)
    for c, m in zip(loop, masks):
        c.correct_elasticnet(alpha=1.0, l1_ratio=0.9, cadence_mask=m, **KW)
    for a, b in zip(cs, loop):
        np.testing.assert_allclose(a.coefficients, b.coefficients, rtol=1e-12)
        np.testing.assert_allclose(a.model_lc.flux.value, b.model_lc.flux.value, rtol=1e-12,
                                   atol=1e-12 * np.max(np.abs(b.model_lc.flux.value)))


def test_elasticnet_config4_size(engine):
    """4096 light curves x 65 000 cadences, K = 17 correlated CBVs, e-/s flux: every output finite, 16 sampled light
    curves equal the oracle."""
    B, N, K = 4096, 65000, 17
    rng = np.random.default_rng(4)
    V = np.cumsum(rng.normal(size=(N, K - 1)), axis=0) / np.sqrt(N)
    X = np.hstack([V, np.ones((N, 1))])
    W = rng.normal(size=(B, K - 1)) * np.geomspace(1, 1e-2, K - 1)
    Y = 1e4 * (1 + 0.01 * (W @ V.T)) + 3.0 * rng.normal(size=(B, N))
    kw = dict(alpha=1e-20, l1_ratio=0.01)
    res = engine.elasticnet(X, Y, **kw)
    for k in ("coefficients", "model", "dual_gap"):
        assert np.all(np.isfinite(res[k])), k
    checked = 0
    for b in rng.choice(B, 40, replace=False):
        r = oen.enet_fit(X, Y[b], **kw)
        if r["margin"] <= MARGIN:
            continue
        assert res["n_iter"][b] == r["n_iter"]
        np.testing.assert_allclose(res["coefficients"][b], r["coef"], rtol=1e-9, atol=1e-9 * np.max(np.abs(r["coef"])))
        checked += 1
        if checked == 16:
            break
    assert checked == 16
