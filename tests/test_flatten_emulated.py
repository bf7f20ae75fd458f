"""The K4 v2 kernel (lightkurve_b200/csrc/flatten_v2.cuh: bitmask bookkeeping, sliding-moment Savitzky-Golay, moment
edges, one final interpolation) executed on the CPU through tests/native/cuda_emu.h and compared with the reference's
own flatten body on the real scipy (oracle/detrend.py).  Leaves only hardware-side behaviour to the GPU tests."""
import ctypes
import os
import shutil
import subprocess
from fractions import Fraction

import numpy as np
import pytest
import scipy.signal

from oracle import detrend as odet
from test_gpu_flatten_paths import F2_MAXN, plan

HERE = os.path.dirname(os.path.abspath(__file__))
CUDA_INC = "/usr/local/cuda/include"
c_vp, c_int, c_dbl = ctypes.c_void_p, ctypes.c_int, ctypes.c_double


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    out = str(tmp_path_factory.mktemp("emu") / "libflatten_emu.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-pthread", "-I" + CUDA_INC, "-Wno-attributes", "-shared", "-fPIC", "-Wl,-Bsymbolic",
                           "-o", out, os.path.join(HERE, "native", "flatten_emu_driver.cpp")])
    return _bind(ctypes.CDLL(out))


def _bind(lib):
    lib.emu_flatten_plan.argtypes = [c_int, c_int, ctypes.c_int64, c_vp, c_vp]
    lib.emu_flatten2.argtypes = [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_dbl, c_int, c_dbl, c_vp, c_vp, c_int,
                                 c_vp, c_vp, c_vp, c_vp]
    return lib


def _coef(w, p):
    """What flatten.cu::savgol_ginv hands to the kernel: the inverse normal matrix on u = (k - c) / c and the even
    centre-tap coefficients in units of j^s."""
    c = 0.5 * (w - 1)
    sc = c if c > 0 else 1.0
    u = (np.arange(w) - c) / sc
    V = u[:, None] ** np.arange(p + 1)[None, :]
    Ginv = np.linalg.inv(V.T @ V)
    A = np.zeros(3)
    A[0] = Ginv[0, 0]
    if p + 1 > 2:
        A[1] = Ginv[0, 2] / sc ** 2
    if p + 1 > 4:
        A[2] = Ginv[0, 4] / sc ** 4
    return np.ascontiguousarray(A), np.ascontiguousarray(Ginv)


def _run(emu, times, fluxes, errs, masks, w, p, bt, niters, sigma, tile_out=None):
    B = len(times)
    off = np.zeros(B + 1, np.int64)
    np.cumsum([len(t) for t in times], out=off[1:])
    t = np.ascontiguousarray(np.concatenate(times))
    f = np.ascontiguousarray(np.concatenate(fluxes))
    fe = np.ascontiguousarray(np.concatenate(errs))
    ex = None if masks is None else np.ascontiguousarray(np.concatenate(masks).astype(np.uint8))
    A, Ginv = _coef(w, p)
    flat, flat_err, trend = (np.full(len(t), -7.0) for _ in range(3))
    status = np.full(B, -1, np.int32)
    emu.emu_flatten2(t.ctypes.data, f.ctypes.data, fe.ctypes.data, None if ex is None else ex.ctypes.data, off.ctypes.data, B,
                     w, p, np.nan if bt is None else float(bt), niters, float(sigma), A.ctypes.data, Ginv.ctypes.data,
                     tile_out or 0, flat.ctypes.data, flat_err.ctypes.data, trend.ctypes.data, status.ctypes.data)
    sp = lambda a: [a[off[b]:off[b + 1]] for b in range(B)]
    return sp(flat), sp(flat_err), sp(trend), status


def _lc(rng, n, gaps=2, outliers=10, nans=0, dt=0.0204336):
    keep = np.ones(int(n * 1.3), bool)
    for _ in range(gaps):
        g0 = int(rng.integers(0, len(keep) - 60))
        keep[g0:g0 + int(rng.integers(8, 50))] = False
    idx = np.flatnonzero(keep)[:n]
    t = 131.5 + idx * dt
    f = 1 + 5e-3 * np.sin(2 * np.pi * (t - t[0]) / 7.3) + 2e-3 * np.cos(2 * np.pi * (t - t[0]) / 1.9) + 3e-4 * rng.normal(size=n)
    f[rng.choice(n, outliers, replace=False)] += 8 * 3e-4 * rng.choice([-1, 1], outliers)
    if nans:
        f[rng.choice(n, nans, replace=False)] = np.nan
    fe = 3e-4 * rng.uniform(0.8, 1.2, n)
    return t, f, fe


@pytest.mark.parametrize("w,p,bt,niters,sigma,nans,tile", [
    (101, 2, 5, 3, 3, 0, None),        # reference defaults
    (401, 2, 5, 3, 3, 4, None),        # config-4 window, NaNs in the flux
    (101, 3, 5, 2, 2.5, 0, 300),       # several tiles per segment
    (51, 1, 5, 3, 3, 0, None),         # boxcar-with-slope (NM = 1)
    (75, 4, 5, 3, 3, 0, None),         # fourth-order moments (NM = 5)
    (101, 2, None, 3, 3, 0, None),     # break_tolerance=None: one segment whatever the gaps
    (301, 2, 5, 3, 3, 0, None),        # window longer than some segments: median fallback
])
def test_flatten_v2_kernel_on_the_emulator(emu, w, p, bt, niters, sigma, nans, tile):
    rng = np.random.default_rng(100 + w + p)
    lcs = [_lc(rng, n, gaps=g, nans=nans) for n, g in ((1500, 2), (700, 3), (2300, 1))]
    if w == 301:
        # a light curve whose middle segment (between two large gaps) is shorter than the window
        t, f, fe = lcs[1]
        t = t.copy()
        t[250:] += 3.0
        t[400:] += 3.0
        lcs[1] = (t, f, fe)
    times, fluxes, errs = (list(x) for x in zip(*lcs))
    flat, flat_err, trend, status = _run(emu, times, fluxes, errs, None, w, p, bt, niters, sigma, tile)
    assert (status == 0).all(), status
    for b in range(len(times)):
        rf, re_, rt = odet.flatten(times[b], fluxes[b], errs[b], window_length=w, polyorder=p, break_tolerance=bt,
                                   niters=niters, sigma=sigma)
        np.testing.assert_allclose(trend[b], rt, rtol=1e-9)
        np.testing.assert_allclose(flat[b], rf, rtol=1e-9, equal_nan=True)
        np.testing.assert_allclose(flat_err[b], re_, rtol=1e-9, equal_nan=True)


@pytest.fixture(scope="module")
def emu_bad_bracket(tmp_path_factory):
    """The same translation unit with the test hook that hands the dt median a STALE bracket from the second iteration
    on: the restart path of block_nanmedian_fast (fresh sample, observer reset)."""
    if shutil.which("g++") is None or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    out = str(tmp_path_factory.mktemp("emu") / "libflatten_emu_bad.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-pthread", "-I" + CUDA_INC, "-Wno-attributes", "-shared", "-fPIC",
                           "-Wl,-Bsymbolic", "-DLKB_FS_TEST_BAD_BRACKET", "-o", out,
                           os.path.join(HERE, "native", "flatten_emu_driver.cpp")])
    return _bind(ctypes.CDLL(out))


def test_flatten_v2_stale_bracket_restarts_on_the_emulator(emu_bad_bracket):
    rng = np.random.default_rng(32)
    t1, f1, fe1 = _lc(rng, 9000, gaps=3, outliers=40)
    flat, flat_err, trend, status = _run(emu_bad_bracket, [t1], [f1], [fe1], None, 201, 2, 5, 3, 3)
    assert (status == 0).all(), status
    rf, _, rt = odet.flatten(t1, f1, fe1, window_length=201)
    np.testing.assert_allclose(trend[0], rt, rtol=1e-9)
    np.testing.assert_allclose(flat[0], rf, rtol=1e-9)


def test_flatten_v2_sampling_select_on_the_emulator(emu):
    """Light curves long enough (>= 8192 cadences) for the two-pass sampling median (select.cuh block_nanmedian_fast):
    regular cadence (every dt within rounding of one value: the equal-to-pivot branches) and jittered cadence (many
    distinct dt: the candidate buffer); three iterations, so the dt median's bracket is carried over twice."""
    rng = np.random.default_rng(31)
    t1, f1, fe1 = _lc(rng, 9000, gaps=3, outliers=40)
    t2, f2, fe2 = _lc(rng, 9500, gaps=2, outliers=30)
    t2 = np.sort(t2 + rng.uniform(-2e-3, 2e-3, len(t2)))
    flat, flat_err, trend, status = _run(emu, [t1, t2], [f1, f2], [fe1, fe2], None, 201, 2, 5, 3, 3)
    assert (status == 0).all(), status
    for b, (t, f, fe) in enumerate(((t1, f1, fe1), (t2, f2, fe2))):
        rf, _, rt = odet.flatten(t, f, fe, window_length=201)
        np.testing.assert_allclose(trend[b], rt, rtol=1e-9)
        np.testing.assert_allclose(flat[b], rf, rtol=1e-9)


def test_flatten_v2_mask_and_failure_on_the_emulator(emu):
    """An exclude mask (lightkurve's mask=True cadences), and a light curve with fewer than two usable cadences (NaN
    trend, status 1) next to a healthy one."""
    rng = np.random.default_rng(9)
    t, f, fe = _lc(rng, 1200)
    mask = np.zeros(len(t), bool)
    mask[300:420] = True                                   # e.g. a transit the user wants left out of the fit
    f2 = f.copy()
    f2[300:420] -= 5e-3
    tb, fb, feb = t[:40].copy(), np.full(40, np.nan), fe[:40].copy()
    fb[7] = 1.0
    flat, flat_err, trend, status = _run(emu, [t, tb], [f2, fb], [fe, feb], [mask, np.zeros(40, bool)], 101, 2, 5, 3, 3)
    assert list(status) == [0, 1]
    rf, _, rt = odet.flatten(t, f2, fe, window_length=101, mask=mask)
    np.testing.assert_allclose(trend[0], rt, rtol=1e-9)
    np.testing.assert_allclose(flat[0], rf, rtol=1e-9)
    assert np.isnan(trend[1]).all() and np.isnan(flat[1]).all()


def test_plan_restated_in_python_matches_flatten_plan_h(emu):
    """tests/test_gpu_flatten_paths.py::plan (the GPU tests' expected paths) against flatten_plan.h itself."""
    routes = {0: "v2", 1: "polyorder", 2: "tile", 3: "length"}
    tile, direct = c_int(), c_int()
    for w in list(range(1, 300, 2)) + list(range(301, 8192, 34)) + [1509, 1511, 2601, 2603, 3967, 3969, 8191]:
        for p in range(min(w, 13)):
            for nmax in (1000, F2_MAXN, F2_MAXN + 1):
                r = emu.emu_flatten_plan(w, p, nmax, ctypes.byref(tile), ctypes.byref(direct))
                assert (routes[r], tile.value, bool(direct.value)) == tuple(plan(w, p, nmax)[i] for i in (0, 2, 3)), (w, p, nmax)


def _exact_rows(w, p, rows):
    """Rows i of the least-squares projection onto degree-p polynomials over w equispaced points, exact (rational)."""
    xs = [k - w // 2 for k in range(w)]
    q = p + 1
    M = [[Fraction(sum(x ** (r + s) for x in xs)) for s in range(q)] + [Fraction(int(r == s)) for s in range(q)]
         for r in range(q)]
    for c in range(q):                                                # Gauss-Jordan: M = [G | I] -> [I | G^-1]
        piv = next(r for r in range(c, q) if M[r][c] != 0)
        M[c], M[piv] = M[piv], M[c]
        M[c] = [v / M[c][c] for v in M[c]]
        for r in range(q):
            if r != c and M[r][c] != 0:
                M[r] = [a - M[r][c] * b for a, b in zip(M[r], M[c])]
    gi = [row[q:] for row in M]
    out = []
    for i in rows:
        a = [sum(xs[i] ** r * gi[r][s] for r in range(q)) for s in range(q)]
        out.append([float(sum(a[s] * x ** s for s in range(q))) for x in xs])
    return np.array(out)


@pytest.mark.parametrize("w,p", [(5, 2), (7, 4), (21, 5), (101, 2), (201, 5), (1001, 5), (51, 12), (401, 12), (13, 12)])
def test_savgol_lsq_matches_exact_taps(w, p):
    """oracle.detrend.savgol_lsq (the GPU tests' reference filter) against exact rational least squares: centre taps
    and edge rows to 1e-13 of sum |tap| max |x|; and against scipy.signal.savgol_filter where scipy's own taps are
    accurate (polyorder <= 3)."""
    half = w // 2
    rows = [half, 0, half - 1]
    exact = _exact_rows(w, p, rows)
    rng = np.random.default_rng(w + p)
    x = rng.normal(size=3 * w)
    y = odet.savgol_lsq(x, w, p)
    tol = lambda taps: 1e-13 * np.abs(taps).sum() * np.abs(x).max()
    np.testing.assert_allclose(y[half:len(x) - half], np.convolve(x, exact[0][::-1], mode="valid"), rtol=0,
                               atol=tol(exact[0]))
    np.testing.assert_allclose(y[0], exact[1] @ x[:w], rtol=0, atol=tol(exact[1]))
    np.testing.assert_allclose(y[half - 1], exact[2] @ x[:w], rtol=0, atol=tol(exact[2]))
    if p <= 3:
        np.testing.assert_allclose(y, scipy.signal.savgol_filter(x, w, p), rtol=0, atol=1e-12 * np.abs(x).max())


# (window, polyorder) of the short windows and of polyorder 4-5, the cases whose interior the sliding moments of
# flatten_v2.cuh got wrong by up to 8e-8 before the direct taps (flatten_plan.h)
SHORT_AND_QUARTIC = [(5, 3), (7, 2), (9, 2), (11, 2), (15, 2), (15, 3), (21, 2), (25, 3), (31, 2), (7, 4), (7, 5), (9, 4),
                     (11, 5), (21, 4), (41, 5), (75, 4), (101, 4), (101, 5), (201, 5), (401, 5), (1001, 5), (3, 1),
                     (1001, 1)]


@pytest.mark.parametrize("w,p", SHORT_AND_QUARTIC, ids=["w%d-p%d" % c for c in SHORT_AND_QUARTIC])
def test_flatten_v2_short_windows_and_quartic_on_the_emulator(emu, w, p):
    """flatten.cu's plan (tile and interior method) on 3000 + 1200 cadences with gaps and outliers, flux ~1 or in
    e-/s, against the reference flatten body with the well-conditioned filter (scipy's own taps are off by up to 1e-6
    at polyorder 5 and long windows): trend, flat and flat_err to rtol 1e-9."""
    rng = np.random.default_rng(7 * w + p)
    lcs = [_lc(rng, n) for n in (3000, 1200)]
    if (w + p) % 2:
        lcs = [(t, 1e5 * f, 1e5 * fe) for t, f, fe in lcs]
    times, fluxes, errs = (list(x) for x in zip(*lcs))
    flat, flat_err, trend, status = _run(emu, times, fluxes, errs, None, w, p, 5, 3, 3)
    assert (status == 0).all(), status
    for b in range(len(times)):
        rf, re_, rt = odet.flatten(times[b], fluxes[b], errs[b], window_length=w, polyorder=p, savgol=odet.savgol_lsq)
        np.testing.assert_allclose(trend[b], rt, rtol=1e-9)
        np.testing.assert_allclose(flat[b], rf, rtol=1e-9, equal_nan=True)
        np.testing.assert_allclose(flat_err[b], re_, rtol=1e-9, equal_nan=True)
