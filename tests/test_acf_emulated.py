"""The K7 windowed-autocorrelation kernels and their launcher (lightkurve_b200/csrc/acf.cuh) executed on the CPU
through tests/native/cuda_emu.h and compared with np.correlate, the call they replace in the seismology estimators
(autocorrelate: y = window - nanmean(window), np.correlate(y, y, "full")[n-1:], metric = (sum |acf| - 1) / n)."""
import ctypes
import os
import shutil
import subprocess
import warnings

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
CUDA_INC = "/usr/local/cuda/include"
c_vp, c_int = ctypes.c_void_p, ctypes.c_int
ACF_TL = 1152                     # lags per CTA (acf.cuh ACF_TL)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    out = str(tmp_path_factory.mktemp("emu") / "libacf_emu.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-pthread", "-I" + CUDA_INC, "-Wno-attributes", "-shared", "-fPIC",
                           "-Wl,-Bsymbolic", "-o", out, os.path.join(HERE, "native", "acf_emu_driver.cpp")])
    lib = ctypes.CDLL(out)
    lib.emu_acf_windows.argtypes = [c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_int]
    lib.emu_acf_windows.restype = c_int
    lib.emu_last_error.restype = ctypes.c_char_p
    lib.emu_launches.restype = ctypes.c_int64
    return lib


def run(emu, series, starts, lengths, want_acf=True, mem=0):
    """Same arguments as engine.acf_windows; returns (status, metrics, acfs)."""
    B = len(series)
    x = np.ascontiguousarray(np.concatenate([np.asarray(s, np.float64) for s in series]) if B else np.zeros(0))
    xo = np.zeros(B + 1, np.int64)
    np.cumsum([len(s) for s in series], out=xo[1:])
    wo = np.zeros(B + 1, np.int64)
    np.cumsum([len(s) for s in starts], out=wo[1:])
    ws = np.ascontiguousarray(np.concatenate([np.asarray(s, np.int64) for s in starts]) if B else np.zeros(0, np.int64))
    wl = np.ascontiguousarray(lengths, dtype=np.int64)
    W = int(wo[-1])
    metric = np.full(max(W, 1), -7.0)
    nl = sum(len(s) * int(n) for s, n in zip(starts, lengths))
    acf = np.full(max(nl, 1), -7.0) if want_acf else None
    st = emu.emu_acf_windows(x.ctypes.data, xo.ctypes.data, B, wo.ctypes.data, ws.ctypes.data, wl.ctypes.data,
                             metric.ctypes.data, None if acf is None else acf.ctypes.data, mem)
    metrics, acfs, a0 = [], [], 0
    for b in range(B):
        metrics.append(metric[wo[b]:wo[b + 1]])
        k, n = len(starts[b]), int(lengths[b])
        if want_acf:
            acfs.append(acf[a0:a0 + k * n].reshape(k, n))
        a0 += k * n
    return st, metrics, acfs


def ref_acf(x, start, n):
    sel = np.array(x[start:start + n], dtype=np.float64)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        sel -= np.nanmean(sel)
    acf = np.correlate(sel, sel, mode="full")[n - 1:]
    return acf, (np.sum(np.abs(acf)) - 1) / len(acf)


def check(series, starts, lengths, metrics, acfs):
    for b, x in enumerate(series):
        for k, s in enumerate(starts[b]):
            ra, rm = ref_acf(x, int(s), int(lengths[b]))
            got = acfs[b][k]
            np.testing.assert_array_equal(np.isnan(got), np.isnan(ra))
            ok = ~np.isnan(ra)
            if ok.any():
                scale = abs(ra[0]) if not np.isnan(ra[0]) else np.nanmax(np.abs(ra))
                assert np.max(np.abs(got[ok] - ra[ok])) <= 1e-12 * scale, (b, k)
            np.testing.assert_allclose(metrics[b][k], rm, rtol=1e-10, equal_nan=True)


@pytest.mark.parametrize("n", [1, 2, 63, 64, 65, 1000, ACF_TL + 517])
def test_acf_lengths_on_the_emulator(emu, n):
    rng = np.random.default_rng(n)
    F = n + 300
    x = 1 + rng.exponential(size=F)
    starts = [np.array(sorted({0, F - n, int(rng.integers(0, F - n + 1))}), np.int64)]
    st, m, a = run(emu, [x], starts, [n])
    assert st == 0, emu.emu_last_error()
    check([x], starts, [n], m, a)


def test_acf_ragged_batch_on_the_emulator(emu):
    """Several series with different lengths, window counts and window lengths (one without windows); host-mode
    staging and device pointers agree bitwise, and the metric alone equals the metric computed with the acf."""
    rng = np.random.default_rng(7)
    lengths = [40, 301, 1, 130, 7]
    Fs = [500, 900, 20, 130, 60]
    counts = [5, 3, 4, 1, 0]
    series = [rng.gamma(2.0, size=F) for F in Fs]
    starts = [np.sort(rng.integers(0, F - n + 1, size=c)).astype(np.int64) for F, n, c in zip(Fs, lengths, counts)]
    st, m, a = run(emu, series, starts, lengths)
    assert st == 0, emu.emu_last_error()
    check(series, starts, lengths, m, a)
    st, m2, a2 = run(emu, series, starts, lengths, mem=1)
    assert st == 0
    for b in range(len(series)):
        np.testing.assert_array_equal(m2[b], m[b])
        np.testing.assert_array_equal(a2[b], a[b])
    st, m3, _ = run(emu, series, starts, lengths, want_acf=False)
    assert st == 0
    for b in range(len(series)):
        np.testing.assert_array_equal(m3[b], m[b])
    # one series alone gives bitwise the batch's results
    st, m4, a4 = run(emu, [series[1]], [starts[1]], [lengths[1]])
    np.testing.assert_array_equal(m4[0], m[1])
    np.testing.assert_array_equal(a4[0], a[1])


def test_acf_nan_windows_on_the_emulator(emu):
    """One NaN: metric NaN and the acf NaN exactly at numpy's lags (k + L < n or k >= L); an all-NaN window."""
    rng = np.random.default_rng(3)
    n = 200
    x = rng.normal(size=900) + 3
    x[250] = np.nan                         # window at 100: k = 150 -> lags 0..50 from i = k, lags 0..150 from i + L = k
    x[700:700 + n] = np.nan
    starts = [np.array([100, 700, 420], np.int64)]
    st, m, a = run(emu, [x], starts, [n])
    assert st == 0, emu.emu_last_error()
    assert np.isnan(m[0][0]) and np.isnan(m[0][1]) and not np.isnan(m[0][2])
    assert not np.isnan(a[0][0]).all() and np.isnan(a[0][1]).all()
    check([x], starts, [n], m, a)
    # a NaN at the window's first bin poisons every lag; at the last bin too
    y = rng.normal(size=300)
    y[100] = np.nan
    st, m, a = run(emu, [y], [np.array([100, 100 - 63 + 1], np.int64)], [63])
    check([y], [np.array([100, 100 - 63 + 1])], [63], m, a)
    assert np.isnan(a[0]).all()


def test_acf_refusals_on_the_emulator(emu):
    x = np.ones(100)
    for starts, lengths in (([np.array([-1])], [10]), ([np.array([91])], [10]), ([np.array([0])], [0]),
                            ([np.array([0])], [101])):
        st, _, _ = run(emu, [x], starts, lengths)
        assert st == -1, (starts, lengths)
    st, _, _ = run(emu, [], [], [])
    assert st == 0
