"""K11/K12 on the GPU: LightCurveCollection.estimate_cdpp / remove_outliers against the per-light-curve loop on a ragged
collection that takes both the shared-memory and the streaming path, the reference's known answers, the clip cases of
tests/_cdpp_cases.py against the oracle, device mode against host mode, and batch invariance."""
import os
import sys

import numpy as np
import pytest
from numpy.testing import assert_almost_equal

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _cdpp_cases as C  # noqa: E402
import _cdpp_oracle as O  # noqa: E402

import lightkurve_b200 as lk  # noqa: E402

pytestmark = pytest.mark.gpu


def collection(seed=31, n=240):
    """Kepler-like (30-minute cadence, up to 65 000 cadences) and TESS-like (2-minute, up to a sector) light curves
    with transits, flares, NaN runs and gaps; a few just around the shared-memory capacity."""
    rng = np.random.default_rng(seed)
    kinds = ["plain", "transit", "flares", "nans", "gaps", "everything"]
    lens = list(np.round(10 ** rng.uniform(np.log10(500), np.log10(20016), n - 12)).astype(int))
    lens += [C.RES_CAP - 1, C.RES_CAP, C.RES_CAP + 1, 8191, 8192, 40, 25000, 30000, 48000, 65000, 4400, 65000]
    lcs = []
    for b, m in enumerate(lens):
        kepler = m > C.RES_CAP or b % 5 == 0
        t, f = C.light_curve(rng, int(m), 10 ** rng.uniform(1, 3), kinds[b % len(kinds)],
                             cadence=(30.0 if kepler else 2.0) / 1440)
        lcs.append(lk.LightCurve(time=t, flux=f, flux_err=np.full(int(m), 1e-4)))
    return lk.LightCurveCollection(lcs)


@pytest.fixture(scope="module")
def coll(engine):
    return collection()


def loop_steps_exact(lc, durations):
    """estimate_cdpp of one light curve through its own steps (flatten, remove_outliers, normalize("ppm") - the
    single-curve methods, on the GPU) with the running means taken by an extended-precision cumulative sum: the loop
    without the rounding of its float64 cumsum of values near 1e6 ppm."""
    v = lc.flatten().remove_outliers(sigma=5.0).normalize("ppm").flux.value
    c = np.cumsum(np.insert(np.asarray(v, np.longdouble), 0, 0))
    out = []
    for d in durations:
        w = min(d, len(v))
        out.append(float(np.std((c[w:] - c[:-w]) / w)) if len(v) else np.nan)
    return out


def test_estimate_cdpp_equals_the_loop(coll):
    """To rtol 1e-9 against the loop's steps with an exact running mean, and to 5e-9 against the loop itself: the
    float64 cumsum of running_mean over up to 65 000 values near 1e6 ppm rounds by up to ~2e-9 of the CDPP on its
    own for the quietest light curves here (the centred sums of K12 stay within ~1e-11 of extended precision)."""
    durs = [13, 1, 30]
    got = coll.estimate_cdpp(transit_duration=durs).value
    assert got.shape == (len(coll), 3)
    loop = np.array([[lc.estimate_cdpp(transit_duration=d).value for d in durs] for lc in coll])
    exact = np.array([loop_steps_exact(lc, durs) for lc in coll])
    np.testing.assert_allclose(got, exact, rtol=1e-9, atol=0)
    np.testing.assert_allclose(got, loop, rtol=5e-9, atol=0)
    np.testing.assert_array_equal(coll.estimate_cdpp().value, got[:, 0])
    with np.errstate(invalid="ignore"):
        print("worst relative difference: %.3g to the loop, %.3g to its exact running mean"
              % (np.nanmax(np.abs(got / loop - 1)), np.nanmax(np.abs(got / exact - 1))))


@pytest.mark.parametrize("kw", [dict(), dict(sigma=3.0, maxiters=None), dict(sigma_lower=2.0, sigma_upper=np.inf),
                                dict(maxiters=1), dict(column="flux_err")])
def test_remove_outliers_masks_equal_the_loop(coll, kw):
    out, masks = coll.remove_outliers(return_mask=True, **kw)
    for lc, o, m in zip(coll, out, masks):
        ref_lc, ref_m = lc.remove_outliers(return_mask=True, **kw)
        assert np.array_equal(m, ref_m)
        assert np.array_equal(o.flux.value, ref_lc.flux.value, equal_nan=True)


def test_reference_known_answers(engine):
    """tests/test_gpu_shim.py::test_cdpp of the reference, on a collection."""
    flat = lk.LightCurve(time=np.arange(10000), flux=np.ones(10000))
    np.random.seed(1)
    noisy = lk.LightCurve(time=np.arange(10000), flux=np.random.normal(loc=1, scale=100e-6, size=10000),
                          flux_err=np.zeros(10000) + 100e-6)
    got = lk.LightCurveCollection([flat, noisy]).estimate_cdpp(transit_duration=1).value
    assert_almost_equal(got[0], 0)
    assert_almost_equal(got[1], 100, decimal=-0.5)
    with pytest.raises(ValueError):
        lk.LightCurveCollection([noisy]).estimate_cdpp(1.5)
    with pytest.raises(ValueError):
        lk.LightCurveCollection([noisy]).estimate_cdpp([1, 0])


CASES = C.clip_cases()


def test_clip_cases_match_the_oracle(engine):
    for name, x, sl, su, mi in CASES:
        r = engine.sigma_clip([x], sl, su, mi)
        ref = O.sigma_clip_mask(x, sigma_lower=sl, sigma_upper=su, maxiters=mi)
        assert np.array_equal(r["mask"][0], ref), "%s: %d cadences differ" % (name, np.count_nonzero(r["mask"][0] != ref))
        kept = x[~ref]
        assert r["n_kept"][0] == len(kept), name
        if len(kept):
            assert r["center"][0] == np.median(kept), name
            np.testing.assert_allclose(r["std"][0], np.std(kept), rtol=1e-12, err_msg=name)
    # the cases with the same parameters in one call: each light curve as on its own
    same = [c[1] for c in CASES if (c[2], c[3], c[4]) == (3.0, 3.0, 5)]
    r = engine.sigma_clip(same, 3.0, 3.0, 5)
    for b, x in enumerate(same):
        assert np.array_equal(r["mask"][b], O.sigma_clip_mask(x, 3.0))


def test_cdpp_matches_the_oracle(engine):
    rng = np.random.default_rng(8)
    lcs = [C.light_curve(rng, n, ppm, kind) for n, ppm, kind in
           [(3000, 300, "everything"), (18000, 60, "transit"), (C.RES_CAP + 500, 100, "nans"), (65000, 40, "gaps")]]
    got = engine.cdpp([t for t, _ in lcs], [f for _, f in lcs], [13, 2, 500])
    for b, (t, f) in enumerate(lcs):
        for d, dur in enumerate((13, 2, 500)):
            np.testing.assert_allclose(got[b, d], O.cdpp(t, f, dur), rtol=1e-6)


def test_device_mode_equals_host_mode_and_batch_invariance(engine, coll):
    import torch
    times = [np.asarray(lc.time.value, np.float64) for lc in coll]
    fluxes = [np.asarray(lc.flux.value, np.float64) for lc in coll]
    off = np.r_[0, np.cumsum([len(t) for t in times])]
    durs = [13, 7]
    host = engine.cdpp(times, fluxes, durs)
    td = torch.tensor(np.concatenate(times), device="cuda")
    fd = torch.tensor(np.concatenate(fluxes), device="cuda")
    dev = engine.cdpp(td, fd, durs, offsets=off)
    torch.cuda.synchronize()
    assert np.array_equal(dev.cpu().numpy(), host, equal_nan=True)
    hc = engine.sigma_clip(fluxes, 4.0, 2.0, None)
    dc = engine.sigma_clip(fd, 4.0, 2.0, None, offsets=off)
    torch.cuda.synchronize()
    assert np.array_equal(dc["mask"].cpu().numpy().astype(bool), np.concatenate(hc["mask"]))
    for k in ("center", "std", "n_kept"):
        assert np.array_equal(dc[k].cpu().numpy(), hc[k], equal_nan=True), k
    # permuted, and every sixth light curve alone with different neighbours: bitwise the same
    perm = np.random.default_rng(2).permutation(len(times))
    p = engine.cdpp([times[i] for i in perm], [fluxes[i] for i in perm], durs)
    assert np.array_equal(p, host[perm], equal_nan=True)
    sub = list(range(0, len(times), 6))
    s = engine.cdpp([times[i] for i in sub], [fluxes[i] for i in sub], durs)
    assert np.array_equal(s, host[sub], equal_nan=True)
