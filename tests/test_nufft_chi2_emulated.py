"""The multi-term (nterms 1..4) Lomb-Scargle path of lightkurve_b200/csrc/ls_nufft.cu - spread, v2 transforms of the
flux and of unit strengths sized for the harmonics, per-bin fp64 normal-equation solve, direct low rows, the fp64
recompute of nearly coherent bins, grouping - executed on the CPU through tests/native/cuda_emu.h and compared with
the fp64 oracle (astropy lombscargle_chi2, tests/_chi2_cases.py) on every bin.

Every case asserts the fine grids it ran ("v2", p, p2) and the path counters of LKB_CHI2_OBSERVE it was written for:
  coherent  bins recomputed in fp64 because a harmonic's window sum is nearly coherent (|C_j + i S_j| >= 0.25 N)
  low       (light curve, bin) pairs with f * baseline <= 2, direct fp64 sums; exactly those pairs
  groups    groups of light curves through the fine-grid buffers (LKB_NUFFT_RAGGED_MB)
and prints them with its worst excess."""
import ctypes
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _chi2_cases as C  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
c_vp, c_i64, c_int, c_dbl = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_double
CUDA_INC = "/usr/local/cuda/include"
NORMS = {0: "psd_raw", 1: "psd", 2: "amplitude"}
LS_LOWF_CYCLES = 2.0


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    out = str(tmp_path_factory.mktemp("emu") / "libnufft_chi2_emu.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-pthread", "-I" + CUDA_INC, "-Wno-attributes", "-shared", "-fPIC",
                           "-Wl,-Bsymbolic", "-o", out, os.path.join(HERE, "native", "nufft_chi2_emu_driver.cpp")])
    lib = ctypes.CDLL(out)
    ragged = [c_vp, c_vp, c_vp, c_vp, c_int, c_i64, c_i64, c_vp, c_vp, c_i64, c_dbl, c_dbl, c_int, c_vp, c_vp]
    lib.emu_nufft_ragged.argtypes = ragged
    lib.emu_nufft_chi2_ragged.argtypes = ragged + [c_int]
    lib.emu_last_error.restype = ctypes.c_char_p
    lib.emu_chi2_paths.argtypes = [c_vp]
    lib.emu_last_nufft_plan.argtypes = [c_vp]
    assert lib.emu_chi2_path_count() == 3
    return lib


def _run(emu, bt, F, f0, df, normalization, scale, nterms):
    """(status, power [B, F], counters {coherent, low, groups}, plan) of one emulated call."""
    power = np.full((bt["B"], F), -1.0, np.float32)
    args = [bt["tt"].ctypes.data, bt["yy"].ctypes.data, bt["off"].ctypes.data, bt["poff"].ctypes.data, bt["B"],
            bt["ptotal"], bt["nmax"], bt["span"].ctypes.data, bt["ysum"].ctypes.data, F, f0, df, normalization,
            scale.ctypes.data, power.ctypes.data]
    emu.emu_chi2_reset_paths()
    rc = emu.emu_nufft_chi2_ragged(*args, nterms) if nterms else emu.emu_nufft_ragged(*args)
    cnt = np.zeros(3, np.int64)
    emu.emu_chi2_paths(cnt.ctypes.data)
    plan = np.zeros(3, np.int32)
    emu.emu_last_nufft_plan(plan.ctypes.data)
    return rc, power, dict(coherent=int(cnt[0]), low=int(cnt[1]), groups=int(cnt[2])), \
        ("v2" if plan[0] == 1 else "round-1", int(plan[1]), int(plan[2]))


def _low_pairs(bt, F, f0, df):
    """(light curve, bin) pairs the low-row kernel must take: f * span <= 2, in the kernel's fp64 arithmetic."""
    fr = f0 + np.arange(F, dtype=np.float64) * df
    return int(sum(np.count_nonzero(~(fr * s > LS_LOWF_CYCLES)) for s in bt["span"]))


def _check(name, bt, power, F, f0, df, nterms, normalization, scale, cnt, plan, limit=1.0):
    """Every bin of every light curve against the oracle (condition-number rule, TOL_NUFFT); returns the worst excess."""
    freq = f0 + df * np.arange(F)
    worst, n_bad = 0.0, 0
    for b in range(bt["B"]):
        n = len(bt["times"][b])
        P, cond = C.oracle(bt["times"][b], bt["fluxes"][b], freq, nterms)
        ref = C.normalise(P, NORMS[normalization], n, scale[b])
        ex, _, bad = C.excess(power[b], ref, cond, C.TOL_NUFFT)
        worst, n_bad = max(worst, ex), n_bad + bad
    print("%-52s plan %s, counters %s: worst excess %.3g, %d ill-conditioned bins" % (name, plan[1:], cnt, worst, n_bad))
    assert worst <= limit, (name, worst)
    assert n_bad <= power.size // 20
    return worst


@pytest.mark.parametrize("nterms", [1, 2, 3, 4])
@pytest.mark.parametrize("kind,k0,normalization,ragged_mb", [
    ("irregular", 1, 2, None),        # amplitude, one group
    ("tess", 3, 1, "0.5"),            # 2-min cadence with a gap, psd scaled, a fine-grid budget that forces groups
    ("irregular", 3, 0, "0.5"),       # raw psd, groups
])
def test_chi2_nufft_matches_the_oracle(emu, monkeypatch, nterms, kind, k0, normalization, ragged_mb):
    """Light curves of different lengths in one batch; 3500 bins (fine grids of 2^14 .. 2^17 cells: the v2 transform);
    the first rows of every light curve are low rows (f * baseline <= 2, direct sums).  The 2-min cadence reaches its
    sampling alias (720 / d) with the harmonics and takes the coherent recompute there.  (So do a few bins of the
    37-cadence irregular light curve: a random window sum exceeds 0.25 N with probability ~exp(-N / 16).)"""
    if ragged_mb:
        monkeypatch.setenv("LKB_NUFFT_RAGGED_MB", ragged_mb)
    bt = C.layout(*C.batch(kind, [400, 90, 260, 37], 100 * nterms + k0))
    F = 3500
    df = 1.0 / (5.0 * bt["span"].max())
    f0 = k0 * df
    scale = np.random.default_rng(7).uniform(0.5, 2.0, bt["B"])
    rc, power, cnt, plan = _run(emu, bt, F, f0, df, normalization, scale, nterms)
    assert rc == 0, emu.emu_last_error()
    assert plan == C.chi2_plan(nterms, k0 + F)
    assert cnt["low"] == _low_pairs(bt, F, f0, df) > 0
    assert (cnt["groups"] > 1) if ragged_mb else (cnt["groups"] == 1)
    if kind == "tess":
        assert cnt["coherent"] > 0
    _check("nterms %d %s k0=%d" % (nterms, kind, k0), bt, power, F, f0, df, nterms, normalization, scale, cnt, plan)


def _sized_batch(seed, kmax, ns=(300, 420, 360)):
    """Irregular light curves and the grid f_k = (k0 + k) df, k0 = 1, k0 + F = kmax, df = 1 / (5 baseline)."""
    bt = C.layout(*C.batch("irregular", list(ns), seed))
    df = 1.0 / (5.0 * bt["span"].max())
    return bt, kmax - 1, df, df


def _kmax_for(nterms, p, at_power_of_two):
    """k0 + F whose flux grid is 2^p cells at this nterms: just above 2^(p-3) harmonics, or the most that fit 2^p."""
    return (2 ** (p - 2)) // nterms if at_power_of_two else (2 ** (p - 3)) // nterms + 1


@pytest.mark.parametrize("nterms", [1, 2, 3, 4])
@pytest.mark.parametrize("p", [14, 15, 16, 17])
@pytest.mark.parametrize("at_power_of_two", [False, True])
def test_chi2_nufft_every_small_transform_size(emu, nterms, p, at_power_of_two):
    kmax = _kmax_for(nterms, p, at_power_of_two)
    bt, F, f0, df = _sized_batch(1000 * p + 10 * nterms + at_power_of_two, kmax)
    scale = np.ones(bt["B"])
    rc, power, cnt, plan = _run(emu, bt, F, f0, df, 2, scale, nterms)
    assert rc == 0, emu.emu_last_error()
    assert plan == C.chi2_plan(nterms, kmax) == ("v2", p, p + 1)
    assert cnt["low"] == _low_pairs(bt, F, f0, df) and cnt["coherent"] == 0 and cnt["groups"] == 1
    _check("nterms %d k0+F=%d" % (nterms, kmax), bt, power, F, f0, df, nterms, 2, scale, cnt, plan)


@pytest.mark.parametrize("nterms", [1, 2, 3, 4])
@pytest.mark.parametrize("kmax", [64, 1044, 2048])
def test_chi2_nufft_small_grids_take_the_smallest_v2_grid(emu, nterms, kmax):
    """Grids whose harmonics need fewer than 2^14 cells run on the 2^14-cell v2 grid (they used to be refused)."""
    bt, F, f0, df = _sized_batch(kmax + nterms, kmax)
    scale = np.ones(bt["B"])
    rc, power, cnt, plan = _run(emu, bt, F, f0, df, 2, scale, nterms)
    assert rc == 0, emu.emu_last_error()
    assert plan == C.chi2_plan(nterms, kmax)
    assert plan[1] == max(14, C.fine_log2(nterms * kmax)) and plan[2] == max(14, C.fine_log2(2 * nterms * kmax))
    assert cnt["low"] == _low_pairs(bt, F, f0, df) and cnt["coherent"] == 0
    _check("small grid nterms %d k0+F=%d" % (nterms, kmax), bt, power, F, f0, df, nterms, 2, scale, cnt, plan)


@pytest.mark.parametrize("nterms", [1, 2, 3, 4])
def test_chi2_nufft_grid_from_zero(emu, nterms):
    """k0 = 0: the f = 0 row is exactly singular (the sine columns vanish) - NaN, as in the oracle; the rest as usual."""
    bt, _, _, df = _sized_batch(50 + nterms, 2000)
    F = 2000
    scale = np.ones(bt["B"])
    rc, power, cnt, plan = _run(emu, bt, F, 0.0, df, 0, scale, nterms)
    assert rc == 0, emu.emu_last_error()
    assert plan == C.chi2_plan(nterms, F) and cnt["low"] == _low_pairs(bt, F, 0.0, df)
    assert np.isnan(power[:, 0]).all()
    P0 = [C.oracle(bt["times"][b], bt["fluxes"][b], [0.0], nterms)[0][0] for b in range(bt["B"])]
    assert np.isnan(P0).all()
    _check("k0=0 nterms %d" % nterms, bt, power, F, 0.0, df, nterms, 0, scale, cnt, plan)


@pytest.mark.parametrize("nterms", [1, 2, 3, 4])
def test_chi2_nufft_regular_cadence_to_nyquist(emu, nterms):
    """A 2-min cadence without gaps on a grid up to its Nyquist frequency (360 / d): harmonic 2 of the last bins sits
    on the sampling rate.  Those bins are recomputed in fp64; the rest of the row is the fp32 transforms'."""
    rng = np.random.default_rng(60 + nterms)
    times = [C.cadence_times(rng, n, gap=0.0) for n in (1500, 700)]
    fluxes = [C.signal(rng, t, rng.uniform(3.0, 30.0), a) for t, a in zip(times, (3e-3, 1e-4))]
    bt = C.layout(times, fluxes)
    df = 1.0 / (5.0 * bt["span"].max())
    F = int(360.0 / df)
    scale = np.ones(bt["B"])
    rc, power, cnt, plan = _run(emu, bt, F, df, df, 2, scale, nterms)
    assert rc == 0, emu.emu_last_error()
    assert plan == C.chi2_plan(nterms, 1 + F)
    assert cnt["coherent"] > 0 and cnt["low"] == _low_pairs(bt, F, df, df)
    _check("2-min cadence to Nyquist, nterms %d" % nterms, bt, power, F, df, df, nterms, 2, scale, cnt, plan)


def test_chi2_nufft_at_one_term_agrees_with_the_single_term_path(emu):
    bt = C.layout(*C.batch("irregular", [300, 77, 512, 150, 40], 5))
    F = 3500
    df = 1.0 / (5.0 * bt["span"].max())
    scale = np.ones(bt["B"])
    rc, p1, _, _ = _run(emu, bt, F, df, df, 1, scale, 1)
    assert rc == 0, emu.emu_last_error()
    rc, p0, _, _ = _run(emu, bt, F, df, df, 1, scale, 0)
    assert rc == 0, emu.emu_last_error()
    ex = np.abs(p1 - p0) / (1e-5 * p0.max(axis=1, keepdims=True) + 1e-4 * p0)
    assert ex.max() <= 1.0, ex.max()


def test_chi2_nufft_refuses_ineligible_light_curves(emu):
    bt = C.layout(*C.batch("irregular", [300, 120], 11))
    F = 3500
    df = 1.0 / (5.0 * bt["span"].max())
    scale = np.ones(bt["B"])
    tt = bt["tt"].copy()
    bt["tt"][[5, 6]] = bt["tt"][[6, 5]]                         # unsorted times
    rc, _, _, _ = _run(emu, bt, F, df, df, 2, scale, 2)
    assert rc == -5 and b"unsorted" in emu.emu_last_error()
    bt["tt"] = tt
    df_long = 1.5 / bt["span"].max()                            # df * baseline > 1
    rc, _, _, _ = _run(emu, bt, F, df_long, df_long, 2, scale, 2)
    assert rc == -5 and b"baseline" in emu.emu_last_error()
    rc, _, _, _ = _run(emu, bt, F, 1.5 * df, df, 2, scale, 2)   # f0 not a multiple of df
    assert rc == -5
    kmax = 2 ** 20 // 2 + 1                                     # nterms 2: the window grid would need 2^24 cells
    rc, _, _, _ = _run(emu, bt, kmax - 1, df, df / 2e4, 2, scale, 2)
    assert rc == -5 and b"outside the v2" in emu.emu_last_error()


def test_oracle_restatement_matches_oracle_ls():
    """tests/_chi2_cases.py:oracle (many bins at once) is oracle.ls.ls_chi2_psd, and the extended-precision restatement
    agrees with both."""
    from oracle import ls as ols
    rng = np.random.default_rng(1)
    for nterms in (1, 2, 3, 4):
        t = C.irregular_times(rng, 300, 20.0)
        y = C.signal(rng, t, 1.3, 1e-2, 1e-3)
        f = np.concatenate([[0.0], np.sort(rng.uniform(0.01, 30.0, 100))])
        P, cond, th = C.oracle(t, y, f, nterms, theta=True)
        Q = ols.ls_chi2_psd(t - t[0], y, f, nterms)
        good = cond <= C.COND_MAX
        assert np.isnan(P[0]) and np.isnan(Q[0]) and np.isnan(th[0]).all() and not good[0]
        assert np.max(np.abs(P[good] - Q[good])) <= 1e-11 * Q[good].max()
        pl, sl = C.oracle_longdouble(t, y, f[7], nterms)
        assert abs(pl - P[7]) <= 1e-12 * P[7] and np.max(np.abs(sl - th[7])) <= 1e-12 * np.abs(sl).max()
