"""Pins the LS / BLS oracle against REAL astropy when it is importable (it is not in the build container nor on the GPU
box of this run: SURVEY.md 8c - every test here then skips, and DESIGN.md keeps saying "parity unpinned" for the power
values).  On any machine with astropy >= 5 this file turns that statement around: run
    python -m pytest tests/test_oracle_vs_astropy.py -q
and, to freeze golden vectors from real astropy next to the oracle's own, tests/golden/make_golden.py --astropy."""
import numpy as np
import pytest

astropy = pytest.importorskip("astropy", reason="astropy is not installed here (no network, not in the wheelhouse)")

from astropy.timeseries import BoxLeastSquares, LombScargle  # noqa: E402

from oracle import bls as obls, ls as ols  # noqa: E402


def _lc(seed, n=800):
    rng = np.random.default_rng(seed)
    t = np.sort(rng.uniform(0, 40, n)) + 2457000.0
    y = 1 + 0.01 * np.sin(2 * np.pi * (t - t[0]) / 3.3) + 2e-3 * rng.normal(size=n)
    return t, y


@pytest.mark.parametrize("seed", [1, 2])
def test_ls_slow_matches_astropy(seed):
    """lightkurve's call: LombScargle(t, y, nterms=1, normalization="psd").power(f, method="slow")
    (/root/reference/src/lightkurve/periodogram.py:961-964)."""
    t, y = _lc(seed)
    f = np.linspace(0.01, 5, 700)
    ref = LombScargle(t, y, nterms=1, normalization="psd").power(f, method="slow")
    np.testing.assert_allclose(ols.ls_slow_psd(t, y, f), np.asarray(ref), rtol=1e-9, atol=1e-14)


def test_ls_fast_matches_astropy():
    t, y = _lc(3)
    df = 1.0 / (5 * (t[-1] - t[0]))
    f = df * (1 + np.arange(2000))
    ref = LombScargle(t, y, nterms=1, normalization="psd").power(f, method="fast")
    np.testing.assert_allclose(ols.ls_fast_psd(t, y, f[0], df, len(f)), np.asarray(ref), rtol=1e-8, atol=1e-14)


@pytest.mark.parametrize("nterms", [1, 2, 3])
def test_ls_chi2_matches_astropy(nterms):
    t, y = _lc(4)
    f = np.linspace(0.05, 3, 300)
    ref = LombScargle(t, y, nterms=nterms, normalization="psd").power(f, method="chi2")
    np.testing.assert_allclose(ols.ls_chi2_psd(t, y, f, nterms), np.asarray(ref), rtol=1e-8, atol=1e-14)


def test_bls_matches_astropy_bit_exact_bins():
    rng = np.random.default_rng(5)
    t = np.arange(0, 27, 1 / 48.0)
    y = 1 + 5e-4 * rng.normal(size=len(t))
    y[np.abs((t - 0.7 + 1.5) % 3.0 - 1.5) < 0.06] -= 3e-3
    dy = np.full(len(t), 5e-4)
    dur = [0.05, 0.1, 0.2]
    model = BoxLeastSquares(t, y, dy)
    per = model.autoperiod(dur, minimum_period=0.5, maximum_period=9.0, frequency_factor=10)
    np.testing.assert_array_equal(per, obls.autoperiod(t, dur, 0.5, 9.0, frequency_factor=10))
    ref = model.power(per, dur)                              # method="fast", objective="likelihood", oversample=10
    got = obls.bls_power_c(t, y, dy, per, dur)
    for k, rk in (("power", "power"), ("depth", "depth"), ("depth_err", "depth_err"), ("duration", "duration"),
                  ("transit_time", "transit_time"), ("depth_snr", "depth_snr"), ("log_likelihood", "log_likelihood")):
        np.testing.assert_allclose(got[k], np.asarray(getattr(ref, rk)), rtol=1e-12, atol=1e-14, err_msg=k)


@pytest.mark.parametrize("case", ["normal_flares", "deep_dips"])
def test_sigma_clip_mask_matches_astropy(case):
    """oracle.detrend.sigma_clip_mask (and rg_clip_kernel, which tests/test_regress_clip_emulated.py pins to it) keeps
    a value masked once a round has clipped it.  If astropy's final mask were instead "outside the LAST round's
    bounds", the two would differ where a value clipped early lies inside the final bounds: one-sided deep dips move
    the median between rounds, which is where that shows."""
    from astropy.stats import sigma_clip

    from oracle import detrend as odet
    rng = np.random.default_rng(11)
    x = rng.normal(size=20000)
    if case == "normal_flares":
        x[rng.choice(20000, 200, replace=False)] += rng.exponential(6.0, 200)
    else:
        for s in rng.choice(19960, 60, replace=False):
            x[s:s + 30] -= np.exp(rng.uniform(np.log(2.0), np.log(80.0)))
    x[::997] = np.nan
    for sigma in (3.0, 5.0):
        ref = np.ma.getmaskarray(sigma_clip(x, sigma=sigma, maxiters=5))
        np.testing.assert_array_equal(odet.sigma_clip_mask(x, sigma), ref)
