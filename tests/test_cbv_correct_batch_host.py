"""`CBVCorrector.correct_batch`, `under_fitting_metric` and `metrics.underfit_metric_neighbors` on the host: the logic
around the K5 / K1 / K9 calls with the engine entries replaced by oracle-backed stand-ins (tests/_oracle_engine.py,
oracle/cbv.py).  On the GPU box tests/test_gpu_cbv_correct.py runs the same logic on the kernels."""
import numpy as np
import pytest

import lightkurve_b200 as lk
from lightkurve_b200 import units as u
from lightkurve_b200.correctors import CBVCorrector, CotrendingBasisVectors, DesignMatrix
from lightkurve_b200.correctors import RegressionCorrector
from lightkurve_b200.correctors import cbvcorrector as cbvmod
from lightkurve_b200.correctors import metrics as lkm
from oracle import cbv as ocbv
import _oracle_engine as oe


def oracle_regress(X, Y, flux_err=None, cadence_mask=None, prior_mu=None, prior_sigma=None, sigma=5, niters=5,
                   return_cov=False, exact_invariant=False):
    """`engine.regress` with [B, K] priors: one oracle fit per light curve."""
    Y = np.atleast_2d(Y)
    if prior_sigma is None or np.ndim(prior_sigma) == 1:
        return oe.regress(X, Y, flux_err, cadence_mask, prior_mu, prior_sigma, sigma, niters, return_cov)
    parts = []
    for b in range(len(Y)):
        pick = lambda a: None if a is None else np.broadcast_to(a, Y.shape)[b:b + 1]
        parts.append(oe.regress(X[b] if np.ndim(X) == 3 else X, Y[b:b + 1], pick(flux_err), pick(cadence_mask),
                                prior_mu[b], prior_sigma[b], sigma, niters))
    return {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}


def oracle_underfit(pool, target, nb_offsets, nb_index):
    out = [ocbv.underfit_metric(target[b], pool[nb_index[nb_offsets[b]:nb_offsets[b + 1]]])
           for b in range(len(target))]
    return dict(metric=np.array([o[0] for o in out]), n_used=np.array([o[1] for o in out], np.int32),
                c3_mean=np.array([o[2] for o in out]))


def oracle_overfit(corrected, original, noise, offsets=None, n_samples=1):
    if offsets is None:                                   # [B, F] rows on one grid
        F = corrected.shape[1]
        offsets = np.arange(len(corrected) + 1) * F
        corrected, original, noise = corrected.ravel(), original.ravel(), np.asarray(noise).ravel()
    B = len(offsets) - 1
    res = [ocbv.overfit_terms(corrected[offsets[b]:offsets[b + 1]], original[offsets[b]:offsets[b + 1]],
                              [noise[n_samples * offsets[b] + s * (offsets[b + 1] - offsets[b]):
                                     n_samples * offsets[b] + (s + 1) * (offsets[b + 1] - offsets[b])]
                               for s in range(n_samples)]) for b in range(B)]
    return dict(n_positive=np.array([r[0] for r in res], np.int32), sum_positive=np.array([r[1] for r in res]),
                noise_mean=np.array([r[2] for r in res]))


CALLS = []


@pytest.fixture
def engine(monkeypatch):
    from lightkurve_b200 import engine as eng
    CALLS.clear()

    def regress(*a, **k):
        CALLS.append(("regress", np.shape(a[0]), len(np.atleast_2d(a[1]))))
        return oracle_regress(*a, **k)
    monkeypatch.setattr(eng, "regress", regress)
    monkeypatch.setattr(eng, "ls_power_ragged", oe.ls_power_ragged)
    monkeypatch.setattr(eng, "ls_power_shared", oe.ls_power_shared)
    monkeypatch.setattr(eng, "nanmedian_std", oe.nanmedian_std)
    monkeypatch.setattr(eng, "underfit_metric", oracle_underfit)
    monkeypatch.setattr(eng, "overfit_terms", oracle_overfit)
    monkeypatch.setattr(cbvmod, "_use_device", lambda: False)     # host arrays for the stand-ins
    yield eng


def make_batch(n=36, N=240, seed=0, mission="TESS", n_cbv=4, spread_deg=0.3):
    """TESS-like light curves sharing systematic trends (the CBVs), each with its own sinusoid and noise, on the
    sky within a fraction of a degree."""
    rng = np.random.default_rng(seed)
    t = 1000.0 + np.arange(N) * (2.0 / 1440)
    cad = np.arange(5000, 5000 + N)
    x = np.linspace(-1, 1, N)
    sys = np.stack([x, x ** 2 - 1 / 3, np.sin(3 * x), np.cos(5 * x)])[:n_cbv]
    data = {"VECTOR_{}".format(i + 1): sys[i] for i in range(n_cbv)}
    data["CADENCENO"] = cad
    cbvs = CotrendingBasisVectors(data, t, cbv_type="SingleScale")
    lcs = []
    for b in range(n):
        w = rng.normal(scale=200.0, size=n_cbv)
        star = 30.0 * np.sin(2 * np.pi * t / rng.uniform(0.05, 0.2))
        flux = 1e5 + w @ sys + star + rng.normal(scale=20.0, size=N)
        lc = lk.LightCurve(time=t, flux=flux, flux_err=np.full(N, 20.0), cadenceno=cad,
                           flux_unit=u.electron / u.second)
        lc.meta.update(MISSION=mission, TARGETID=1000 + b, RA=120.0 + rng.uniform(-spread_deg, spread_deg),
                       DEC=-30.0 + rng.uniform(-spread_deg, spread_deg))
        lcs.append(lc)
    return lcs, cbvs


KW = dict(cbv_type=["SingleScale"], cbv_indices=[np.arange(1, 5)], max_iter=6, min_targets=5, max_targets=8)


def test_underfit_metric_neighbors_contract(engine):
    lcs, cbvs = make_batch(n=8)
    with pytest.raises(NotImplementedError, match="MAST"):
        lkm.underfit_metric_neighbors(lcs[0])
    with pytest.raises(lkm.MinTargetsError, match="at least 30 neighbors"):
        lkm.underfit_metric_neighbors(lcs[0], neighbors=lcs[1:])
    with pytest.raises(Exception, match="interpolate must be True"):
        lkm.underfit_metric_neighbors(lcs[0], neighbors=lcs[1:], extrapolate=True)
    # the first max_targets neighbours, aligned by cadence number; a neighbour missing cadences leaves NaN there
    short = lcs[3][10:200]
    m = lkm.underfit_metric_neighbors(lcs[0], neighbors=[lcs[1], lcs[2], short, lcs[4]], min_targets=2, max_targets=3)
    f = lambda lc: np.asarray(lc.flux.value) / np.median(np.asarray(lc.flux.value)) - 1.0
    nb = np.stack([f(lcs[1]), f(lcs[2]), np.r_[np.full(10, np.nan), f(short), np.full(40, np.nan)]])
    assert m == pytest.approx(ocbv.underfit_metric(f(lcs[0]), nb)[0], rel=1e-13)
    # a neighbour identical to the target: correlation 1
    _, _, c3 = ocbv.underfit_metric(f(lcs[0]), f(lcs[0])[None])
    assert c3 == pytest.approx(0.5)


def test_neighbor_selection(engine):
    lcs, cbvs = make_batch(n=12, spread_deg=0.2)
    c = CBVCorrector(lcs[0], cbvs=[cbvs])
    c.correct_gaussian_prior(cbv_type=["SingleScale"], cbv_indices=[np.arange(1, 5)], alpha=1.0)
    with pytest.raises(NotImplementedError, match="MAST"):
        c.under_fitting_metric()
    # never its own neighbour: the same TARGETID in the pool is skipped
    from lightkurve_b200.correctors.cbvcorrector import _own_entries, _select_neighbors, _separation_arcsec
    pool = lcs
    excl = _own_entries(c.lc, pool)
    assert excl == {0}
    got = _select_neighbors(c.lc, pool, excl, None, 4, 6)
    seps = [_separation_arcsec(lcs[0].meta["RA"], lcs[0].meta["DEC"], p.meta["RA"], p.meta["DEC"]) for p in pool]
    order = [i for i in np.argsort(seps, kind="stable") if i != 0]
    # the radius grows by 1.5 from 5000 arcsec until 4 are inside, then the nearest 6 inside that radius are kept
    r = 5000.0
    while sum(seps[i] <= r for i in order) < 4:
        r *= 1.5
    assert got == [i for i in order if seps[i] <= r][:6]
    # the metric through the corrector equals the module function on the selected neighbours
    m = c.under_fitting_metric(neighbors=pool, min_targets=4, max_targets=6)
    assert m == lkm.underfit_metric_neighbors(c.corrected_lc, neighbors=[pool[i] for i in got], min_targets=4,
                                              max_targets=6)
    # neighbor_index skips the geometry (and still drops the light curve itself)
    assert _select_neighbors(c.lc, pool, excl, None, 2, 3, neighbor_index=[0, 5, 4, 7, 9]) == [5, 4, 7]
    with pytest.raises(Exception, match="Not enough neighboring targets"):
        _select_neighbors(c.lc, pool, excl, None, 20, 30)
    with pytest.raises(Exception, match="Not enough neighboring targets"):
        _select_neighbors(c.lc, pool, excl, None, 5, 6, neighbor_index=[0, 1, 2])
    # Kepler / K2 start at 1000 arcsec and stop at one CCD diagonal; other missions are refused
    kep = lk.LightCurve(time=lcs[0].time.value, flux=np.ones(240), flux_err=np.ones(240))
    kep.meta.update(MISSION="Kepler", RA=120.0, DEC=-30.0)
    far = []
    for k, d in enumerate([0.25, 0.4, 0.6, 2.5]):          # 900", 1440", 2160", 9000" away
        x = lk.LightCurve(time=lcs[0].time.value, flux=np.ones(240), flux_err=np.ones(240))
        x.meta.update(MISSION="Kepler", RA=120.0, DEC=-30.0 + d)
        far.append(x)
    assert _select_neighbors(kep, far, set(), None, 1, 5) == [0]
    assert _select_neighbors(kep, far, set(), None, 3, 5) == [0, 1, 2]            # 1000 -> 1500 -> 2250
    with pytest.raises(Exception, match="Not enough neighboring targets"):
        _select_neighbors(kep, far, set(), None, 4, 5)    # the last radius tried, 7594", is past sqrt(2) 4096"
    kep.meta["MISSION"] = "Other"
    with pytest.raises(Exception, match="Unknown mission"):
        _select_neighbors(kep, far, set(), None, 1, 5)


def test_correct_without_neighbors_is_unchanged(engine):
    lcs, cbvs = make_batch(n=2)
    c = CBVCorrector(lcs[0], cbvs=[cbvs])
    with pytest.raises(NotImplementedError, match="target_under_score=0"):
        c.correct(cbv_type=["SingleScale"], cbv_indices=[np.arange(1, 5)])
    c.correct(cbv_type=["SingleScale"], cbv_indices=[np.arange(1, 5)], target_under_score=0, max_iter=4)
    assert c.under_fitting_score == -1.0 and not hasattr(c, "optimization_trace")


def check_state(c, alpha_bounds=(1e-4, 1e4)):
    assert alpha_bounds[0] <= c.alpha <= alpha_bounds[1]
    assert c.corrected_lc is not None and c.model_lc is not None
    assert set(c.diagnostic_lightcurves) == {dm.name for dm in c.design_matrix_collection}
    sigma = np.median(c.lc.flux_err.value) / np.sqrt(abs(c.alpha))
    for dm in c.design_matrix_collection:
        np.testing.assert_array_equal(dm.prior_sigma, np.ones(dm.shape[1]) * sigma)
    # the final state is the fit at alpha
    ref = oracle_regress(RegressionCorrector._dense_X(c.design_matrix_collection), np.asarray(c.lc.flux.value)[None],
                         np.asarray(c.lc.flux_err.value)[None], c.cadence_mask[None],
                         np.asarray(c.design_matrix_collection.prior_mu)[None],
                         np.asarray(c.design_matrix_collection.prior_sigma)[None])
    np.testing.assert_array_equal(c.coefficients, ref["coefficients"][0])
    np.testing.assert_array_equal(c.corrected_lc.flux.value, c.lc.flux.value - ref["model"][0])


def test_correct_batch_state_and_trace(engine):
    lcs, cbvs = make_batch(n=10)
    cs = [CBVCorrector(lc, cbvs=[cbvs]) for lc in lcs]
    np.random.seed(7)
    out = CBVCorrector.correct_batch(cs, **KW)
    assert len(out) == 10
    for b, c in enumerate(cs):
        check_state(c)
        assert 0 < len(c.optimization_trace) <= KW["max_iter"]
        assert 0 <= c.over_fitting_score <= 1 and 0 <= c.under_fitting_score <= 1
        # the last traced under metric at the final alpha is the one the corrector keeps
        a, over, under, mnp, npos, spos = c.optimization_trace[-1]
        assert np.isfinite(mnp) and npos >= 0 and np.isfinite(spos)
        assert over == pytest.approx(ocbv.overfit_metric(npos, spos, [mnp]), rel=1e-15)
    # the final under-fitting score equals the metric through the corrector's own method
    c = cs[3]
    assert c.under_fitting_score == c.under_fitting_metric(neighbors=lcs, min_targets=5, max_targets=8)


def same_trace(c1, c2):
    """Bitwise equal traces (NaN where a metric is off)."""
    np.testing.assert_array_equal(np.array(c1.optimization_trace, float), np.array(c2.optimization_trace, float))


def test_batch_of_one_equals_its_part(engine):
    """Over-fitting metric off (no noise draws): every corrector's alpha and trace in the batch equal its own
    correct_batch([c], neighbors=batch) call, and do not change under permutation."""
    lcs, cbvs = make_batch(n=8, seed=3)
    kw = dict(KW, target_over_score=0.0, target_under_score=0.9, min_targets=4, max_targets=5)
    cs = [CBVCorrector(lc, cbvs=[cbvs]) for lc in lcs]
    CBVCorrector.correct_batch(cs, **kw)
    one = CBVCorrector(lcs[5], cbvs=[cbvs])
    CBVCorrector.correct_batch([one], neighbors=lcs, **kw)
    assert one.alpha == cs[5].alpha
    same_trace(one, cs[5])
    np.testing.assert_array_equal(one.corrected_lc.flux.value, cs[5].corrected_lc.flux.value)
    perm = [3, 7, 0, 5, 1, 6, 2, 4]
    ps = [CBVCorrector(lcs[i], cbvs=[cbvs]) for i in perm]
    CBVCorrector.correct_batch(ps, **kw)
    for j, i in enumerate(perm):
        assert ps[j].alpha == cs[i].alpha
        same_trace(ps[j], cs[i])


def test_correct_with_neighbors_is_a_batch_of_one(engine):
    lcs, cbvs = make_batch(n=33, seed=6, spread_deg=0.05)
    kw = dict(cbv_type=KW["cbv_type"], cbv_indices=KW["cbv_indices"], max_iter=5, target_over_score=0.0,
              target_under_score=0.9)
    single = CBVCorrector(lcs[0], cbvs=[cbvs])
    single.correct(neighbors=lcs, **kw)                      # default min_targets=30, max_targets=50
    one = CBVCorrector(lcs[0], cbvs=[cbvs])
    CBVCorrector.correct_batch([one], neighbors=lcs, **kw)
    assert single.alpha == one.alpha and 0 < single.under_fitting_score <= 1
    same_trace(single, one)


def test_grouping_and_per_corrector_inputs(engine):
    lcs, cbvs = make_batch(n=8, seed=4)
    N = 240
    extra = [None] * 4 + [DesignMatrix(np.random.default_rng(1).normal(size=(N, 1)), name="extra")] * 4
    mask = np.ones(N, bool)
    mask[50:70] = False
    cs = [CBVCorrector(lc, cbvs=[cbvs]) for lc in lcs]
    CBVCorrector.correct_batch(cs, ext_dm=extra, cadence_mask=[None] * 4 + [mask] * 4,
                               **dict(KW, target_over_score=0.0, min_targets=4, max_targets=6, max_iter=3))
    shapes = {s for name, s, _ in CALLS}
    assert shapes == {(N, 5), (N, 6)}                     # two design-matrix shapes, one call per shape and round
    assert max(n for _, _, n in CALLS) == 4
    assert np.array_equal(cs[6].cadence_mask, mask) and cs[1].cadence_mask.all()
    for c in cs:
        check_state(c)


def test_interpolated_cbvs_refused(engine):
    lcs, cbvs = make_batch(n=6)
    cs = [CBVCorrector(lc, cbvs=[cbvs], interpolate_cbvs=True) for lc in lcs]
    with pytest.raises(NotImplementedError, match="interpolate_cbvs=True"):
        CBVCorrector.correct_batch(cs, **dict(KW, min_targets=3))


def test_noise_draws_in_batch_order(engine):
    """One randn(n, 1) per active corrector per round in batch order, then the final re-fit's and ten per final
    score: a batch of one draws exactly what the reference's correct() draws."""
    lcs, cbvs = make_batch(n=6, seed=5)
    cs = [CBVCorrector(lc, cbvs=[cbvs]) for lc in lcs]
    np.random.seed(11)
    CBVCorrector.correct_batch(cs, **dict(KW, min_targets=3, max_targets=4))
    draws = sum(len(c.optimization_trace) for c in cs) + len(cs) * (1 + 10)
    after = np.random.randn()
    np.random.seed(11)
    np.random.randn(draws * 240)
    assert np.random.randn() == after


# ---- every traced metric, recomputed independently --------------------------------------------------------------
def record_rounds(monkeypatch):
    """Record the correctors evaluated in each traced round and every white-noise draw, in order."""
    calls, draws = [], []
    real_eval = cbvmod._GoodnessBatch.evaluate
    real_randn = np.random.randn

    def evaluate(self, idx, alphas, record=True, finish=False):
        if record:
            calls.append([int(b) for b in idx])
        return real_eval(self, idx, alphas, record, finish)

    def randn(*shape):
        x = real_randn(*shape)
        draws.append(x.copy())
        return x
    monkeypatch.setattr(cbvmod._GoodnessBatch, "evaluate", evaluate)
    monkeypatch.setattr(np.random, "randn", randn)
    return calls, draws


def recheck_trace(cs, pool, calls, draws, picks, rtol=1e-5, nbin_tol=3, default_pool=True, min_targets=30,
                  max_targets=50):
    """Trace entries `picks` [(corrector, entry)] against oracle/cbv.py on a fit redone by the oracle at the traced
    alpha, the oracle's Lomb-Scargle (fp64 direct sums, rounded to fp32 as the periodograms store them) and the same
    noise draw."""
    from collections import defaultdict
    from lightkurve_b200.correctors.cbvcorrector import _own_entries, _select_neighbors
    from lightkurve_b200.periodogram import _PER_DAY, LombScarglePeriodogram
    from oracle import detrend as odet
    from oracle import ls as ols
    seen, jobs = defaultdict(int), []
    for k, b in enumerate(b for call in calls for b in call):
        if (b, seen[b]) in picks:
            jobs.append((b, seen[b], draws[k][:, 0]))
        seen[b] += 1
    assert len(jobs) == len(picks)
    cen = lambda v: v / np.median(v) - 1.0
    for b, j, z in jobs:
        c = cs[b]
        alpha, over, under, mnp, npos, spos = c.optimization_trace[j]
        m = c.cadence_mask
        X = RegressionCorrector._dense_X(c.design_matrix_collection)
        y, fe = np.asarray(c.lc.flux.value, float), np.asarray(c.lc.flux_err.value, float)
        t = np.asarray(c.lc.time.value, float)[m]
        K = X.shape[1]
        r = odet.regress(X, y, fe, m, np.zeros(K), np.full(K, np.median(fe) / np.sqrt(abs(alpha))))
        f = (y - r["model"])[m]
        corrected = cen(f)
        if c.optimization_params["target_over_score"] > 0:
            freq = np.asarray(LombScarglePeriodogram._prepare(c.lc.copy()[m].normalize())["frequency"].to(_PER_DAY)
                              .value, dtype=np.float64)
            amp = lambda v: (np.sqrt(np.maximum(ols.ls_slow_psd(t, v, freq), 0)) * np.sqrt(4.0 / len(v))).astype(
                np.float32)
            n_o, s_o, (m_o,) = ocbv.overfit_terms(amp(corrected), amp(cen(y[m])),
                                                  [amp(z * np.mean(fe[m] / np.median(f)))])
            assert abs(npos - n_o) <= nbin_tol, (b, j, npos, n_o)
            assert spos == pytest.approx(s_o, rel=rtol) and mnp == pytest.approx(m_o, rel=rtol), (b, j)
            assert over == pytest.approx(ocbv.overfit_metric(n_o, s_o, [m_o]), rel=rtol, abs=rtol), (b, j)
        if c.optimization_params["target_under_score"] > 0:
            excl = _own_entries(c.lc, pool) | ({b} if default_pool else set())
            nb = _select_neighbors(c.lc, pool, excl, None, min_targets, max_targets)
            rows = np.stack([cen(np.asarray(pool[i].flux.value, float))[m] for i in nb])
            assert under == pytest.approx(ocbv.underfit_metric(corrected, rows)[0], rel=rtol), (b, j)


def test_traced_metrics_against_the_oracle(engine, monkeypatch):
    lcs, cbvs = make_batch(n=10, seed=8)
    cs = [CBVCorrector(lc, cbvs=[cbvs]) for lc in lcs]
    calls, draws = record_rounds(monkeypatch)
    np.random.seed(3)
    CBVCorrector.correct_batch(cs, **KW)
    picks = {(0, 0), (3, 2), (7, len(cs[7].optimization_trace) - 1), (9, 4)}
    recheck_trace(cs, lcs, calls, draws, picks, rtol=1e-9, nbin_tol=0, min_targets=5, max_targets=8)
