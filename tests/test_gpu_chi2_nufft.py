"""Multi-term (nterms 1..4) Lomb-Scargle through the non-uniform FFT on the GPU: parity with the fp64 oracle, the
`auto` selection rule and its refusals, independence of a light curve's row from its neighbours, the collection-level
shim, and the worst bins of one GPU's share of config 5."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ls as ols  # noqa: E402

pytestmark = pytest.mark.gpu
COND_MAX = 1e6          # bins whose oracle normal matrix is worse conditioned than this are not compared


@pytest.fixture(scope="module")
def engine():
    from lightkurve_b200 import engine as eng
    eng.init(0)
    return eng


def _batch(seed, ns, span=25.0):
    """ragged light curves: irregular times, non-sinusoidal signals of very different strengths, noise"""
    rng = np.random.default_rng(seed)
    times, fluxes = [], []
    for b, n in enumerate(ns):
        t = 1300.0 + np.sort(rng.uniform(0, span * rng.uniform(0.5, 1.0), n))
        ph = 2 * np.pi * rng.uniform(0.2, 5.0) * t + rng.uniform(0, 2 * np.pi)
        a = 10 ** rng.uniform(-4, -2)
        y = 1 + a * (np.sin(ph) + 0.5 * np.cos(2 * ph + 0.3) + 0.25 * np.sin(3 * ph + 1.1)) \
            + 10 ** rng.uniform(-4, -3) * rng.normal(size=n)
        times.append(t)
        fluxes.append(y.astype(np.float32))
    return times, fluxes


def _grid(times, F, k0=1):
    df = 1.0 / (5.0 * max(t[-1] - t[0] for t in times))
    return df * (k0 + np.arange(F))


def _oracle_amplitude(t, y, freq, nterms):
    """amplitude spectrum from astropy's lombscargle_chi2 math (fp64) and the condition number of each bin's normal
    matrix"""
    y = np.asarray(y, np.float64)
    p = ols.ls_chi2_psd(t, y, freq, nterms)
    tr = t - t[0]
    cond = np.empty(len(freq))
    for i0 in range(0, len(freq), 64):
        ph = 2 * np.pi * freq[i0:i0 + 64, None] * tr[None, :]
        cols = [np.ones_like(ph)]
        for j in range(1, nterms + 1):
            cols += [np.sin(j * ph), np.cos(j * ph)]
        X = np.stack(cols, axis=-1)
        cond[i0:i0 + 64] = np.linalg.cond(np.einsum("fnm,fnk->fmk", X, X))
    return np.sqrt(p) * np.sqrt(4.0 / len(t)), cond


@pytest.mark.parametrize("nterms", [1, 2, 3, 4])
def test_nufft_parity_with_the_oracle(engine, nterms):
    times, fluxes = _batch(40 + nterms, [1500, 400, 900, 120, 2200])
    freq = _grid(times, 5000)
    out = np.asarray(engine.ls_power_chi2(times, fluxes, freq, nterms, "amplitude", algo="nufft"))
    assert engine.ls_last_algo() == "nufft"
    worst, n_bad = 0.0, 0
    for b in range(len(times)):
        ref, cond = _oracle_amplitude(times[b], fluxes[b], freq, nterms)
        good = cond <= COND_MAX
        n_bad += int((~good).sum())
        ex = np.abs(out[b][good] - ref[good]) / (1e-5 * ref[good].max() + 1e-4 * ref[good])
        worst = max(worst, float(ex.max()))
        assert not np.any(np.isinf(out[b]))
    print("nterms %d: worst excess %.3f, %d ill-conditioned bins" % (nterms, worst, n_bad))
    assert worst <= 1.0
    assert n_bad <= out.size // 100


def test_auto_selection_and_refusals(engine):
    # large job on one regular grid: the NUFFT family
    times, fluxes = _batch(3, [2000] * 256)
    freq = _grid(times, 20000)
    engine.ls_power_chi2(times, fluxes, freq, 2, "amplitude")
    assert engine.ls_last_algo() == "nufft"
    engine.ls_power_chi2(times[:16], fluxes[:16], freq, 4, "amplitude")
    assert engine.ls_last_algo() == "nufft"
    # config 1 (1 light curve, 1000 cadences, 2497 bins): the direct kernel
    t1, f1 = _batch(4, [1000])
    engine.ls_power_chi2(t1, f1, _grid(t1, 2497), 2, "amplitude")
    assert engine.ls_last_algo() == "simt"
    # ineligible inputs: `auto` runs the direct kernel, an explicit NUFFT request fails with LKB_E_UNSUPPORTED
    times, fluxes = _batch(5, [3000] * 16)
    freq = _grid(times, 20000)
    t_unsorted = [t.copy() for t in times]
    t_unsorted[3][[10, 11]] = t_unsorted[3][[11, 10]]
    irregular = np.geomspace(freq[0], freq[-1], len(freq))
    cases = {
        "irregular grid": lambda algo: engine.ls_power_chi2(times, fluxes, irregular, 2, "amplitude", algo=algo),
        "per-light-curve grids": lambda algo: engine.ls_power_chi2(times, fluxes, [freq] * len(times), 2, "amplitude",
                                                                   algo=algo),
        "theta": lambda algo: engine.ls_power_chi2(times[:2], fluxes[:2], freq, 2, "amplitude", return_theta=True,
                                                   algo=algo),
        "unsorted times": lambda algo: engine.ls_power_chi2(t_unsorted, fluxes, freq, 2, "amplitude", algo=algo),
    }
    for name, call in cases.items():
        with pytest.raises(Exception) as ei:
            call("nufft")
        assert getattr(ei.value, "status", None) == -5, name
        call("auto")
        assert engine.ls_last_algo() == "simt", name


def test_rows_do_not_depend_on_the_neighbours(engine):
    times, fluxes = _batch(8, [3000, 800, 120, 2500, 60, 1700, 900, 2200])
    freq = _grid(times, 20000)
    out = np.asarray(engine.ls_power_chi2(times, fluxes, freq, 3, "amplitude", algo="nufft"))
    perm = np.random.default_rng(1).permutation(len(times))
    out_p = np.asarray(engine.ls_power_chi2([times[i] for i in perm], [fluxes[i] for i in perm], freq, 3, "amplitude",
                                            algo="nufft"))
    np.testing.assert_array_equal(out_p, out[perm])


def test_collection_fastchi2_above_the_threshold(engine):
    from lightkurve_b200 import LightCurve, LightCurveCollection
    times, fluxes = _batch(9, list(np.random.default_rng(9).integers(1000, 3000, 64)))
    freq = _grid(times, 10000)
    lcs = LightCurveCollection([LightCurve(time=t, flux=f.astype(np.float64), flux_err=np.full(len(t), 1e-3))
                                for t, f in zip(times, fluxes)])
    pgs = lcs.to_periodogram(ls_method="fastchi2", nterms=3, frequency=freq)
    assert engine.ls_last_algo() == "nufft"
    worst = 0.0
    for b, pg in enumerate(pgs):
        ref = np.asarray(engine.ls_power_chi2([times[b]], [fluxes[b].astype(np.float64)], freq, 3, "amplitude",
                                              algo="direct"))[0].astype(np.float64)
        got = np.asarray(pg.power.value, dtype=np.float64)
        worst = max(worst, float((np.abs(got - ref) / (1e-5 * ref.max() + 1e-4 * ref)).max()))
    print("collection fastchi2 nterms 3 vs direct: worst excess %.3f" % worst)
    assert worst <= 1.0


@pytest.mark.parametrize("nterms", [2, 4])
def test_config5_share_worst_bins_chi2(engine, nterms):
    """One GPU's share of BASELINE configs[4] (2048 ragged light curves, 20 000 bins): NUFFT and direct sums on every
    (light curve, bin) pair; the pairs where they disagree most, plus random ones, go to the fp64 oracle."""
    from bench import make_c5_workload
    times, fluxes, freq = make_c5_workload(1005, B=2048, F=20000)
    B, F = len(times), len(freq)
    out_n = np.asarray(engine.ls_power_chi2(times, fluxes, freq, nterms, "amplitude", algo="nufft"))
    assert engine.ls_last_algo() == "nufft"
    out_d = np.asarray(engine.ls_power_chi2(times, fluxes, freq, nterms, "amplitude", algo="direct"))
    assert out_n.shape == (B, F) and not np.isinf(out_n).any()
    d = np.abs(out_d - out_n) / (1e-5 * np.nanmax(out_n, axis=1, keepdims=True) + 1e-4 * out_n)
    d[~np.isfinite(d)] = np.inf
    rng = np.random.default_rng(5)
    flat = np.unique(np.concatenate([np.argpartition(d.ravel(), -600)[-600:], rng.choice(B * F, 300, replace=False)]))
    del d
    bb, kk = np.unravel_index(flat, (B, F))
    ref, cond = np.empty(len(flat)), np.empty(len(flat))
    for b in np.unique(bb):
        sel = bb == b
        ref[sel], cond[sel] = _oracle_amplitude(times[b], fluxes[b], freq[kk[sel]], nterms)
    # bins whose normal matrix has condition number > COND_MAX (the lowest rows at nterms >= 3: f * baseline ~ 0.07,
    # condition number ~ 1e16) are not compared; there the fp64 sums of either family can give a power just below
    # zero, i.e. a NaN amplitude, and only finite-or-NaN is required.  The row peaks ignore those NaNs.
    good = cond <= COND_MAX
    assert not np.isinf(out_n[bb, kk]).any()
    pmax = np.nanmax(out_d, axis=1)[bb]
    tol = 1e-5 * np.maximum(pmax, ref) + 1e-4 * ref
    ex = np.abs(out_n[bb, kk] - ref) / tol
    worst = float(ex[good].max())
    print("config-5 share, nterms %d: worst NUFFT excess %.3f over %d pairs (%d ill-conditioned, not compared; %d NaN "
          "amplitudes among them)" % (nterms, worst, int(good.sum()), int((~good).sum()),
                                      int(np.isnan(out_n[bb, kk][~good]).sum())))
    assert worst <= 1.0
