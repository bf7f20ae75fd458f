"""Multi-term Lomb-Scargle (K1c, lkb_ls_power_chi2_ex, nterms 1..4) on every kernel path, cadence count, grid shape and
NUFFT transform size, against the fp64 oracle (tests/_chi2_cases.py: astropy lombscargle_chi2 restated, with the
condition number of every bin's normal matrix).

Paths:
  direct  ls_chi2_kernel<NT> (ls.cu): fp64 sums, one warp per (light curve, bin), 8 bins per block (LS_WARPS), the light
          curve staged through shared memory in tiles of 1024 cadences by bulk copies.  The reference of the other LS
          tests (test_gpu_ls_paths.py, test_gpu_chi2_nufft.py), so it is held to the fp64 formulation's own accuracy:
          |X - X_oracle| <= 1e-9 max X + 1e-7 X (fp32 output) on EVERY bin with condition number <= 1e6.
  NUFFT   ls_nufft_chi2_ragged_launch (ls_nufft.cu): v2 transforms of 2^p / 2^p2 cells, p = max(fine_log2(n (k0 + F)), 14),
          p2 = max(fine_log2(2 n (k0 + F)), 14); held to 1e-5 max A + 1e-4 A (amplitude) against the direct kernel on
          EVERY bin and against the oracle on the worst 500 + 200 random.
Worse-conditioned bins are only required to be finite or NaN.  Every case prints its worst excess and the path / plan
it ran."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _chi2_cases as C  # noqa: E402

from oracle import ls as ols  # noqa: E402

pytestmark = pytest.mark.gpu
NORMS = ("amplitude", "psd", "psd_raw")


def _direct(engine, times, fluxes, freq, nterms, norm="psd_raw", scale=None, **kw):
    out = engine.ls_power_chi2(times, fluxes, freq, nterms, norm, norm_scale=scale, algo="direct", **kw)
    assert engine.ls_last_algo() == "simt"
    return out


def _check_direct(name, out, times, fluxes, freqs, nterms, norm="psd_raw", scale=None, skip_short=True):
    """`out` (rows per light curve) against the oracle on every bin, TOL_DIRECT.  Light curves with fewer cadences
    than parameters (the estimator is undefined) are only required to have no +-inf; an empty one must be all NaN."""
    M = 2 * nterms + 1
    worst, where, n_bad = 0.0, None, 0
    for b in range(len(times)):
        n = len(times[b])
        fr = freqs[b] if isinstance(freqs, list) else freqs
        o = np.asarray(out[b], np.float64)
        assert not np.isinf(o).any(), (name, b)
        if n == 0:
            assert np.isnan(o).all(), (name, "empty light curve")
            continue
        if n < M and skip_short:
            continue
        P, cond = C.oracle(times[b], fluxes[b], fr, nterms)
        ref = C.normalise(P, norm, n, 1.0 if scale is None else scale[b])
        ex, k, bad = C.excess(o, ref, cond, C.TOL_DIRECT)      # (a NaN on a well-conditioned bin is an infinite excess)
        n_bad += bad
        if ex > worst:
            worst, where = ex, (b, k)
    print("%-70s direct: worst excess %.3g at (lc, bin) %s; %d ill-conditioned bins" % (name, worst, where, n_bad))
    if worst > 1.0:
        b, k = where
        fr = freqs[b] if isinstance(freqs, list) else freqs
        pl, _ = C.oracle_longdouble(times[b], fluxes[b], fr[k], nterms)
        print("   arbiter (long double) at that bin: psd_raw %.17g" % pl)
    assert worst <= 1.0, (name, worst, where)
    return worst


# ====================================================================================== direct kernel
def _ns(nterms):
    M = 2 * nterms + 1
    return sorted({1, 2, 2 * nterms, M, 8, 1023, 1024, 1025, 2048, 2049, 65000})


@pytest.mark.parametrize("nterms", [1, 2, 3, 4])
def test_direct_cadence_counts(engine, nterms):
    """Cadence counts at the edges of the 1024-cadence tiles and of the estimator (n < 2 nterms + 1), an empty light
    curve among them; F = 43 irregular bins (5 full blocks of LS_WARPS and a partial one)."""
    rng = np.random.default_rng(nterms)
    ns = _ns(nterms)
    ns.insert(3, 0)
    times = [C.irregular_times(rng, n, 27.0) for n in ns]
    fluxes = [C.signal(rng, t, rng.uniform(0.3, 3.0), 3e-3) if len(t) else np.zeros(0) for t in times]
    freq = np.sort(rng.uniform(0.05, 30.0, 5 * C.LS_WARPS + 3))
    out = _direct(engine, times, fluxes, freq, nterms)
    _check_direct("cadence counts %s, nterms %d" % (ns, nterms), out, times, fluxes, freq, nterms)
    M = 2 * nterms + 1
    for b, n in enumerate(ns):
        if 0 < n < M:
            o = out[b].astype(np.float64)
            print("   n = %d < %d parameters: %d NaN, %d finite bins, finite range [%.3g, %.3g]; 0.5 sum(yc^2) = %.3g"
                  % (n, M, np.isnan(o).sum(), np.isfinite(o).sum(), np.nanmin(o) if np.isfinite(o).any() else 0,
                     np.nanmax(o) if np.isfinite(o).any() else 0,
                     0.5 * np.sum((fluxes[b] - fluxes[b].mean()) ** 2)))


@pytest.mark.parametrize("nterms", [1, 2, 3, 4])
def test_direct_grids_dtypes_and_normalisations(engine, nterms):
    """Shared regular grids of F = 1, LS_WARPS - 1, LS_WARPS + 1 and 61 bins from f = 0 (that bin is exactly singular:
    NaN, as the oracle's LinAlgError); float32 and float64 flux, one of them in e-/s around 1e5, one constant (power 0);
    amplitude, psd with a per-light-curve scale, psd_raw."""
    rng = np.random.default_rng(10 + nterms)
    ns = (300, 1500, 1024, 3001, 777)
    times = [C.irregular_times(rng, n, rng.uniform(10.0, 30.0)) for n in ns]
    fluxes = [C.signal(rng, times[0], 1.1, 1e-2), C.signal(rng, times[1], 0.37, 1e-4),
              C.signal(rng, times[2], 2.9, 300.0, 30.0, mean=1e5), np.full(ns[3], 1.25),
              C.signal(rng, times[4], 0.8, 3e-3)]
    scale = rng.uniform(0.5, 2.0, len(ns))
    grids = {"F=1": np.array([1.37]), "F=%d" % (C.LS_WARPS - 1): 0.2 + 0.31 * np.arange(C.LS_WARPS - 1),
             "F=%d" % (C.LS_WARPS + 1): 0.05 + 0.4 * np.arange(C.LS_WARPS + 1),
             "F=61 from f=0": 0.045 * np.arange(61)}
    for gname, freq in grids.items():
        for dt in (np.float32, np.float64):
            fl = [f.astype(dt) for f in fluxes]
            for norm in NORMS:
                sc = scale if norm == "psd" else None
                out = _direct(engine, times, fl, freq, nterms, norm, sc)
                _check_direct("%s, %s, %s, nterms %d" % (gname, dt.__name__, norm, nterms), out, times, fl, freq,
                              nterms, norm, sc)
                assert np.all((out[3] == 0) | np.isnan(out[3])), "constant flux must have power 0"
                if freq[0] == 0.0:
                    assert np.isnan(out[:, 0]).all()
    # per-light-curve grids of different lengths, one of a single bin, regular and irregular ones
    pl = [np.array([0.91]), 0.1 + 0.2 * np.arange(C.LS_WARPS + 1), np.sort(rng.uniform(0.02, 12.0, 37)),
          0.03 * (1 + np.arange(130)), 0.5 + 0.01 * np.arange(C.LS_WARPS - 1)]
    out = _direct(engine, times, fluxes, pl, nterms, "psd", scale)
    _check_direct("per-light-curve grids of 1..130 bins, psd, nterms %d" % nterms, out, times, fluxes, pl, nterms,
                  "psd", scale)


@pytest.mark.parametrize("nterms", [1, 2, 3, 4])
def test_direct_kepler_four_years(engine, nterms):
    """4 years of 30-min cadences (70 000 points with gaps) up to 24 / d: phases of 3.5e4 cycles, harmonics to 1.4e5."""
    rng = np.random.default_rng(20 + nterms)
    t = 120.0 + np.arange(70128) * (30.0 / 1440.0)
    keep = np.ones(len(t), bool)
    for c in rng.choice(len(t) - 2000, 8, replace=False):
        keep[c:c + int(rng.integers(200, 1500))] = False
    t = t[keep] + 1e-4 * rng.normal(size=keep.sum())
    y = C.signal(rng, t, 3.3, 2e-4, 5e-4)
    freq = np.concatenate([np.sort(rng.uniform(0.002, 24.0, 40)), 23.9 + 0.1 / 24 * np.arange(24)])
    out = _direct(engine, [t], [y], freq, nterms, "amplitude")
    _check_direct("Kepler 4 yr, %d cadences, to 24 / d, nterms %d" % (len(t), nterms), out, [t], [y], freq, nterms,
                  "amplitude")


def test_direct_largest_batch(engine):
    """B = 65535 light curves of 6 cadences (the grid's y extent); 65536 is refused."""
    rng = np.random.default_rng(30)
    B = 65535
    times = [C.irregular_times(rng, 6, 3.0) for _ in range(B)]
    fluxes = [1 + 1e-2 * rng.normal(size=6) for _ in range(B)]
    freq = np.array([0.7, 1.9])
    out = _direct(engine, times, fluxes, freq, 2)
    assert out.shape == (B, 2)
    pick = sorted(set(rng.choice(B, 60, replace=False)) | {0, B - 1})
    _check_direct("B = 65535 x 6 cadences, nterms 2 (%d checked)" % len(pick), out[pick], [times[i] for i in pick],
                  [fluxes[i] for i in pick], freq, 2)
    with pytest.raises(ValueError):
        engine.ls_power_chi2(times + times[:1], fluxes + fluxes[:1], freq, 2, "psd_raw", algo="direct")


@pytest.mark.parametrize("nterms", [1, 2, 3, 4])
def test_direct_theta(engine, nterms):
    """theta [offset, sin 1, cos 1, ...] of every well-conditioned bin against lstsq on the oracle's design matrix
    (1e-9 of the bin's largest coefficient), per-light-curve grids in the [foff[b]:foff[b+1]] layout (each light curve's
    block equal to its own one-light-curve call), NaN theta on the singular f = 0 bin."""
    rng = np.random.default_rng(40 + nterms)
    ns = (700, 2049, 130)
    times = [C.irregular_times(rng, n, rng.uniform(8.0, 25.0)) for n in ns]
    fluxes = [C.signal(rng, t, rng.uniform(0.3, 3.0), a) for t, a in zip(times, (1e-2, 3e-4, 2e-3))]
    grids = [0.02 * np.arange(50), np.array([1.23]), np.sort(rng.uniform(0.05, 9.0, 23))]
    out, theta = _direct(engine, times, fluxes, grids, nterms, return_theta=True)
    _check_direct("theta call, per-light-curve grids, nterms %d" % nterms, out, times, fluxes, grids, nterms)
    M = 2 * nterms + 1
    worst = 0.0
    for b in range(len(ns)):
        assert theta[b].shape == (len(grids[b]), M)
        ob, tb = _direct(engine, [times[b]], [fluxes[b]], [grids[b]], nterms, return_theta=True)
        assert np.array_equal(ob[0], out[b], equal_nan=True) and np.array_equal(tb[0], theta[b], equal_nan=True)
        _, cond = C.oracle(times[b], fluxes[b], grids[b], nterms)
        yc = np.asarray(fluxes[b], np.float64) - np.mean(fluxes[b])
        for k, f in enumerate(grids[b]):
            if f == 0.0:
                assert np.isnan(theta[b][k]).all() and np.isnan(out[b][k])
                continue
            if cond[k] > C.COND_MAX:
                continue
            X = ols.design_matrix(times[b] - times[b][0], f, True, nterms)
            ref = np.linalg.lstsq(X, yc, rcond=None)[0]
            worst = max(worst, float(np.max(np.abs(theta[b][k] - ref)) / (1e-9 * np.max(np.abs(ref)))))
    print("theta, nterms %d: worst excess %.3g (1e-9 of the largest coefficient)" % (nterms, worst))
    assert worst <= 1.0


# ====================================================================================== NUFFT family
def _kmax_for(nterms, p, at_power_of_two):
    """k0 + F whose flux grid is 2^p cells at this nterms: just above 2^(p-3) harmonic modes, or the most that fit."""
    return (2 ** (p - 2)) // nterms if at_power_of_two else (2 ** (p - 3)) // nterms + 1


def _nufft_batch(seed, kmax, ns=(1500, 900, 2000), k0=1):
    rng = np.random.default_rng(seed)
    times = [C.irregular_times(rng, n, rng.uniform(20.0, 30.0)) for n in ns]
    df = 1.0 / (5.0 * max(t[-1] - t[0] for t in times))
    freq = df * (k0 + np.arange(kmax - k0))
    fluxes = [C.signal(rng, t, freq[int(rng.integers(len(freq) // 8, len(freq)))] / 3, 10 ** rng.uniform(-3.5, -2))
              .astype(np.float32) for t in times]
    return times, fluxes, freq


def _nufft_vs_direct(engine, name, times, fluxes, freq, nterms, plan=None, **kw):
    out = np.asarray(engine.ls_power_chi2(times, fluxes, freq, nterms, "amplitude", algo="nufft", **kw))
    assert engine.ls_last_algo() == "nufft"
    got_plan = engine.ls_last_nufft_plan()
    if plan is not None:
        assert got_plan == plan, (got_plan, plan)
    ref = np.asarray(_direct(engine, times, fluxes, freq, nterms, "amplitude"))
    C.compare_to_reference("%s, nterms %d, plan %s" % (name, nterms, got_plan[1:]), out, ref, times, fluxes, freq,
                           nterms)
    return out


@pytest.mark.parametrize("nterms", [1, 2, 3, 4])
@pytest.mark.parametrize("p", list(range(14, 23)))
@pytest.mark.parametrize("at_power_of_two", [False, True])
def test_nufft_every_transform_size(engine, nterms, p, at_power_of_two):
    kmax = _kmax_for(nterms, p, at_power_of_two)
    times, fluxes, freq = _nufft_batch(100 * p + 10 * nterms + at_power_of_two, kmax)
    plan = C.chi2_plan(nterms, kmax)
    assert plan == ("v2", p, p + 1)
    _nufft_vs_direct(engine, "v2 k0+F=%d" % kmax, times, fluxes, freq, nterms, plan)


@pytest.mark.parametrize("nterms", [1, 2, 3, 4])
@pytest.mark.parametrize("kmax", [64, 1044, 2048])
def test_nufft_small_grids(engine, nterms, kmax):
    """Grids whose harmonics need fewer than 2^14 cells take the smallest v2 grid (they used to be refused)."""
    times, fluxes, freq = _nufft_batch(kmax + nterms, kmax)
    plan = C.chi2_plan(nterms, kmax)
    assert plan[1] == max(14, C.fine_log2(nterms * kmax))
    _nufft_vs_direct(engine, "small grid k0+F=%d" % kmax, times, fluxes, freq, nterms, plan)


@pytest.mark.parametrize("nterms", [1, 2, 3, 4])
def test_nufft_beyond_the_v2_range(engine, nterms):
    """The first k0 + F whose window grid needs 2^24 cells: algo="nufft" is refused (-5), `auto` runs the direct
    kernel."""
    kmax = 2 ** 20 // nterms + 1
    assert C.fine_log2(2 * nterms * kmax) == 24 and C.fine_log2(2 * nterms * (kmax - 1)) == 23
    times, fluxes, freq = _nufft_batch(7 + nterms, kmax, ns=(300, 200, 400))
    with pytest.raises(Exception) as ei:
        engine.ls_power_chi2(times, fluxes, freq, nterms, "amplitude", algo="nufft")
    assert getattr(ei.value, "status", None) == -5
    out = engine.ls_power_chi2(times, fluxes, freq, nterms, "amplitude")
    assert engine.ls_last_algo() == "simt"
    ref = _direct(engine, times, fluxes, freq, nterms, "amplitude")
    assert np.array_equal(out, ref, equal_nan=True)
    ks = np.sort(np.random.default_rng(nterms).choice(len(freq), 300, replace=False))
    _check_direct("auto beyond the v2 range, k0+F=%d (300 bins)" % kmax, out[:, ks], times, fluxes, freq[ks], nterms,
                  "amplitude")


@pytest.mark.parametrize("nterms", [1, 2, 3, 4])
def test_nufft_regular_cadence_to_nyquist(engine, nterms):
    """A 2-min cadence without gaps on a grid up to its Nyquist frequency: the harmonics of the last bins reach the
    sampling rate, where the finish recomputes the nearly coherent bins in fp64."""
    rng = np.random.default_rng(50 + nterms)
    times = [C.cadence_times(rng, n, gap=0.0) for n in (3000, 1800, 2500)]
    fluxes = [C.signal(rng, t, rng.uniform(3.0, 30.0), a).astype(np.float32) for t, a in zip(times, (3e-3, 1e-4, 1e-3))]
    df = 1.0 / (5.0 * max(t[-1] - t[0] for t in times))
    freq = df * (1 + np.arange(int(360.0 / df)))
    _nufft_vs_direct(engine, "2-min cadence to Nyquist", times, fluxes, freq, nterms, C.chi2_plan(nterms, 1 + len(freq)))


@pytest.mark.parametrize("nterms,f_line", [(2, 300.0), (4, 300.0), (2, 150.0)])
def test_nufft_loud_line_above_the_band(engine, nterms, f_line):
    """A loud line (8e-3) above the band and only noise (2e-4) in it, regular 2-min cadence."""
    rng = np.random.default_rng(int(f_line) + nterms)
    times = [C.cadence_times(rng, 3000, gap=0.0) for _ in range(2)]
    fluxes = [C.hostile(rng, t, f_line).astype(np.float32) for t in times]
    df = 1.0 / (5.0 * max(t[-1] - t[0] for t in times))
    freq = df * (1 + np.arange(int(60.0 / df)))
    _nufft_vs_direct(engine, "loud line at %g / d above a band to 60 / d" % f_line, times, fluxes, freq, nterms)


def test_nufft_groups_of_one(engine, monkeypatch):
    """A fine-grid budget of 0.5 MB: every light curve is its own group; an odd batch."""
    monkeypatch.setenv("LKB_NUFFT_RAGGED_MB", "0.5")
    times, fluxes, freq = _nufft_batch(61, 3001, ns=(900, 300, 1500, 8, 1200))
    _nufft_vs_direct(engine, "groups of one, B = 5, one light curve of 8 cadences", times, fluxes, freq, 3)


@pytest.mark.parametrize("nterms", [2, 4])
def test_nufft_eight_and_seven_cadences(engine, nterms):
    """8 cadences are eligible; 7 are refused (-5) and `auto` runs the direct kernel for the whole call."""
    times, fluxes, freq = _nufft_batch(70 + nterms, 20001, ns=(2000, 8, 1500))
    _nufft_vs_direct(engine, "a light curve of 8 cadences", times, fluxes, freq, nterms)
    times[1], fluxes[1] = times[1][:7], fluxes[1][:7]
    with pytest.raises(Exception) as ei:
        engine.ls_power_chi2(times, fluxes, freq, nterms, "amplitude", algo="nufft")
    assert getattr(ei.value, "status", None) == -5
    out = engine.ls_power_chi2(times, fluxes, freq, nterms, "amplitude")
    assert engine.ls_last_algo() == "simt"
    assert np.array_equal(out, _direct(engine, times, fluxes, freq, nterms, "amplitude"), equal_nan=True)


# ====================================================================================== invariance
@pytest.mark.parametrize("family", ["direct", "nufft"])
def test_permutation_and_device_mode_are_bitwise(engine, family):
    """A batch permutation permutes the rows bitwise; device mode through the C ABI (torch device pointers; for the
    NUFFT family this reads the grid back to the host to recognise it as regular) is bitwise equal to host mode."""
    import torch
    from lightkurve_b200 import _lib as L
    nterms = 3
    times, fluxes, freq = _nufft_batch(80, 5001, ns=(3000, 800, 120, 2500, 60, 1700))
    B, F, M = len(times), len(freq), 2 * nterms + 1
    kw = dict(return_theta=True) if family == "direct" else {}
    host = engine.ls_power_chi2(times, fluxes, freq, nterms, "amplitude", algo=family, **kw)
    assert engine.ls_last_algo() == {"direct": "simt"}.get(family, family)
    out, theta = host if family == "direct" else (host, None)
    perm = np.random.default_rng(1).permutation(B)
    hp = engine.ls_power_chi2([times[i] for i in perm], [fluxes[i] for i in perm], freq, nterms, "amplitude",
                              algo=family, **kw)
    op = hp[0] if family == "direct" else hp
    assert np.array_equal(op, out[perm], equal_nan=True)
    if theta is not None:
        assert np.array_equal(hp[1], theta[perm], equal_nan=True)
    lib = L.load()
    offs = np.concatenate([[0], np.cumsum([len(t) for t in times])]).astype(np.int64)
    t_d = torch.from_numpy(np.concatenate(times)).cuda()
    y_d = torch.from_numpy(np.concatenate(fluxes)).cuda()
    f_d = torch.from_numpy(freq).cuda()
    o_d = torch.full((B, F), -1.0, dtype=torch.float32, device="cuda")
    th_d = torch.full((B, F, M), -1.0, dtype=torch.float64, device="cuda") if theta is not None else None
    algo = {"direct": L.LS_ALGO_SIMT, "nufft": L.LS_ALGO_NUFFT}[family]
    L.check(lib.lkb_ls_power_chi2_ex(L.ptr(t_d), L.ptr(y_d), L.DTYPE_F32, L.ptr(offs), B, L.ptr(f_d), None, F, nterms,
                                     L.LS_NORM_AMPLITUDE, None, L.ptr(o_d), L.ptr(th_d), L.MEM_DEVICE,
                                     torch.cuda.current_stream().cuda_stream, algo))
    torch.cuda.synchronize()
    assert engine.ls_last_algo() == {"direct": "simt"}.get(family, family)
    assert np.array_equal(o_d.cpu().numpy(), out, equal_nan=True), family + ": device mode differs from host mode"
    if theta is not None:
        assert np.array_equal(th_d.cpu().numpy(), theta, equal_nan=True)
    print("%s: permutation and device mode bitwise equal (B = %d, F = %d)" % (family, B, F))


# ====================================================================================== shim
@pytest.mark.parametrize("nterms", [2, 3, 4])
def test_shim_periodogram_and_model(engine, nterms):
    """LightCurve.to_periodogram(ls_method="fastchi2" / "chi2", nterms) against the oracle on every bin; pg.model() at
    the peak and at an explicit frequency against oracle.ls.ls_model, at times inside and outside the fitted range."""
    from lightkurve_b200 import LightCurve
    rng = np.random.default_rng(90 + nterms)
    t = C.irregular_times(rng, 1200, 20.0)
    y = C.signal(rng, t, 0.83, 5e-3, 3e-4)
    lc = LightCurve(time=t, flux=y, flux_err=np.full(len(t), 3e-4))
    freq = np.linspace(0.05, 6.0, 1500)
    tv = np.concatenate([t[0] - 7.3 + 3 * np.arange(3), t[::97], t[-1] + 11.1 + 2 * np.arange(3)])
    for method in ("fastchi2", "chi2"):
        pg = lc.to_periodogram(ls_method=method, nterms=nterms, frequency=freq)
        assert pg.nterms == nterms
        got = np.asarray(pg.power.value, np.float64)
        P, cond = C.oracle(t, y, freq, nterms)
        ex, _, _ = C.excess(got, C.normalise(P, "amplitude", len(t)), cond, C.TOL_DIRECT)
        worst_m = 0.0
        for f in (None, 1.7 * 0.83):
            m = pg.model(tv, f)
            fb = float(pg.frequency_at_max_power.value) if f is None else f
            ref = ols.ls_model(t, y, fb, tv, nterms)
            ref = ref / np.median(ref)
            worst_m = max(worst_m, float(np.max(np.abs(np.asarray(m.flux.value) - ref)) / (1e-10 * np.max(np.abs(ref)))))
        print("shim %s nterms %d (path %s): power worst excess %.3g, model worst excess %.3g (1e-10 of the flux)"
              % (method, nterms, engine.ls_last_algo(), ex, worst_m))
        assert ex <= 1.0 and worst_m <= 1.0


def test_shim_collection_with_own_grids(engine):
    """LightCurveCollection.to_periodogram(nterms=3) with each light curve's default grid (the grids differ, so the
    collection takes per-light-curve grids) against the oracle on every bin."""
    from lightkurve_b200 import LightCurve, LightCurveCollection
    rng = np.random.default_rng(95)
    lcs, data = [], []
    for n, span in ((300, 10.0), (450, 13.0), (200, 6.5)):
        t = C.irregular_times(rng, n, span)
        y = C.signal(rng, t, rng.uniform(0.5, 2.0), 3e-3, 3e-4)
        lcs.append(LightCurve(time=t, flux=y, flux_err=np.full(n, 3e-4)))
        data.append((t, y))
    pgs = LightCurveCollection(lcs).to_periodogram(ls_method="fastchi2", nterms=3)
    assert len({len(pg.frequency) for pg in pgs}) > 1
    worst = 0.0
    for pg, (t, y) in zip(pgs, data):
        fr = np.asarray(pg.frequency.value, np.float64)
        P, cond = C.oracle(t, y, fr, 3)
        worst = max(worst, C.excess(np.asarray(pg.power.value), C.normalise(P, "amplitude", len(t)), cond,
                                    C.TOL_DIRECT)[0])
    print("collection, nterms 3, own grids: worst excess %.3g" % worst)
    assert worst <= 1.0
