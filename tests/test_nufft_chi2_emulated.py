"""The multi-term (nterms 1..4) Lomb-Scargle path of lightkurve_b200/csrc/ls_nufft.cu - spread, v2 transforms of the
flux and of unit strengths sized for the harmonics, per-bin fp64 normal-equation solve, direct low rows, grouping -
executed on the CPU through tests/native/cuda_emu.h and compared with the fp64 oracle (astropy lombscargle_chi2)."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import ls as ols

HERE = os.path.dirname(os.path.abspath(__file__))
c_vp, c_i64, c_int, c_dbl = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_double
CUDA_INC = "/usr/local/cuda/include"
COND_MAX = 1e6          # bins whose oracle normal matrix is worse conditioned than this are not compared


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
    return lib


def _times(kind, n, rng):
    if kind == "irregular":
        return np.sort(rng.uniform(0, 25.0 * rng.uniform(0.4, 1.0), n))
    # TESS-like: 2-minute cadence from a random start, one data gap of a fifth of the span
    t = 2000.0 + rng.uniform(0, 1) + np.arange(int(n * 1.25)) * (2.0 / 1440.0)
    g0 = int(rng.integers(n // 8, n // 2))
    return np.delete(t, np.arange(g0, g0 + len(t) - n))


def _batch(kind, ns, seed):
    """light curves (non-sinusoidal signals of very different strengths + noise) in the K1 prologue's layout"""
    rng = np.random.default_rng(seed)
    B = len(ns)
    off = np.zeros(B + 1, np.int64)
    poff = np.zeros(B + 1, np.int64)
    for b, n in enumerate(ns):
        off[b + 1] = off[b] + n
        poff[b + 1] = poff[b] + ((n + 3) // 4) * 4
    ptotal = int(poff[-1])
    tt, yy = np.zeros(ptotal + 4), np.zeros(ptotal + 4, np.float32)
    times, fluxes, span, ysum = [], [], np.zeros(B), np.zeros(B)
    for b, n in enumerate(ns):
        t = _times(kind, n, rng)
        f1 = rng.uniform(0.3, 3.0) if kind == "irregular" else rng.uniform(3.0, 30.0)
        ph = 2 * np.pi * f1 * (t - t[0]) + rng.uniform(0, 2 * np.pi)
        a = [1e-2, 1e-3, 3e-3, 1e-4, 5e-3][b % 5]
        y = 1 + a * (np.sin(ph) + 0.5 * np.cos(2 * ph + 0.3) + 0.25 * np.sin(3 * ph + 1.1)) \
            + 10 ** rng.uniform(-4, -3) * rng.normal(size=n)
        times.append(t)
        fluxes.append(y)
        tr = t - t[0]
        yc = (y - y.mean()).astype(np.float32)
        tt[poff[b]:poff[b] + n] = tr
        yy[poff[b]:poff[b] + n] = yc
        span[b] = tr.max()
        ysum[b] = yc.astype(np.float64).sum()
    return dict(B=B, off=off, poff=poff, ptotal=ptotal, tt=tt, yy=yy, times=times, fluxes=fluxes, span=span, ysum=ysum,
                nmax=max(ns))


def _run(emu, bt, F, f0, df, normalization, scale, nterms):
    power = np.full((bt["B"], F), -1.0, np.float32)
    args = [bt["tt"].ctypes.data, bt["yy"].ctypes.data, bt["off"].ctypes.data, bt["poff"].ctypes.data, bt["B"],
            bt["ptotal"], bt["nmax"], bt["span"].ctypes.data, bt["ysum"].ctypes.data, F, f0, df, normalization,
            scale.ctypes.data, power.ctypes.data]
    rc = emu.emu_nufft_chi2_ragged(*args, nterms) if nterms else emu.emu_nufft_ragged(*args)
    return rc, power


def _oracle(t, y, freq, nterms):
    """fp64 power (astropy lombscargle_chi2, psd) and the condition number of every bin's normal matrix"""
    p = ols.ls_chi2_psd(t, y, freq, nterms)
    tr = t - t[0]
    cond = np.empty(len(freq))
    for i0 in range(0, len(freq), 256):
        ph = 2 * np.pi * freq[i0:i0 + 256, None] * tr[None, :]
        cols = [np.ones_like(ph)]
        for j in range(1, nterms + 1):
            cols += [np.sin(j * ph), np.cos(j * ph)]
        X = np.stack(cols, axis=-1)
        cond[i0:i0 + 256] = np.linalg.cond(np.einsum("fnm,fnk->fmk", X, X))
    return p, cond


def _normalised(p, n, normalization, scale):
    if normalization == 2:
        return np.sqrt(p) * np.sqrt(4.0 / n)
    return p * scale if normalization == 1 else p


@pytest.mark.parametrize("nterms", [1, 2, 3, 4])
@pytest.mark.parametrize("kind,k0,normalization,ragged_mb", [
    ("irregular", 1, 2, None),        # amplitude, one group
    ("tess", 3, 1, "0.5"),            # 2-min cadence with a gap, psd scaled, a fine-grid budget that forces groups
    ("irregular", 3, 0, "0.5"),       # raw psd, groups
])
def test_chi2_nufft_matches_the_oracle(emu, monkeypatch, nterms, kind, k0, normalization, ragged_mb):
    """Light curves of different lengths in one batch; 3500 bins (fine grids of 2^14 .. 2^17 cells: the v2 transform);
    the first rows of every light curve are low rows (f * baseline <= 2, direct sums)."""
    if ragged_mb:
        monkeypatch.setenv("LKB_NUFFT_RAGGED_MB", ragged_mb)
    bt = _batch(kind, [400, 90, 260, 37], 100 * nterms + k0)
    F = 3500
    df = 1.0 / (5.0 * bt["span"].max())
    f0 = k0 * df
    freq = f0 + df * np.arange(F)
    scale = np.random.default_rng(7).uniform(0.5, 2.0, bt["B"])
    rc, power = _run(emu, bt, F, f0, df, normalization, scale, nterms)
    assert rc == 0, emu.emu_last_error()
    assert np.any(freq * bt["span"].min() <= 2.0)             # low rows were exercised
    for b in range(bt["B"]):
        n = len(bt["times"][b])
        p, cond = _oracle(bt["times"][b], bt["fluxes"][b], freq, nterms)
        ref = _normalised(p, n, normalization, scale[b])
        good = cond <= COND_MAX
        got = power[b].astype(np.float64)
        ex = np.abs(got[good] - ref[good]) / (1e-5 * ref[good].max() + 1e-4 * ref[good])
        bad = int((~good).sum())
        print("nterms %d %s lc %d: worst excess %.3f at bin %d; %d ill-conditioned bins"
              % (nterms, kind, b, ex.max(), int(np.flatnonzero(good)[np.argmax(ex)]), bad))
        assert ex.max() <= 1.0, (b, ex.max())
        assert bad <= F // 20
        assert not np.any(np.isinf(got[~good]))


def test_chi2_nufft_at_one_term_agrees_with_the_single_term_path(emu):
    bt = _batch("irregular", [300, 77, 512, 150, 40], 5)
    F = 3500
    df = 1.0 / (5.0 * bt["span"].max())
    scale = np.ones(bt["B"])
    rc, p1 = _run(emu, bt, F, df, df, 1, scale, 1)
    assert rc == 0, emu.emu_last_error()
    rc, p0 = _run(emu, bt, F, df, df, 1, scale, 0)
    assert rc == 0, emu.emu_last_error()
    ex = np.abs(p1 - p0) / (1e-5 * p0.max(axis=1, keepdims=True) + 1e-4 * p0)
    assert ex.max() <= 1.0, ex.max()


def test_chi2_nufft_refuses_ineligible_light_curves(emu):
    bt = _batch("irregular", [300, 120], 11)
    F = 3500
    df = 1.0 / (5.0 * bt["span"].max())
    scale = np.ones(bt["B"])
    tt = bt["tt"].copy()
    bt["tt"][[5, 6]] = bt["tt"][[6, 5]]                         # unsorted times
    rc, _ = _run(emu, bt, F, df, df, 2, scale, 2)
    assert rc == -5 and b"unsorted" in emu.emu_last_error()
    bt["tt"] = tt
    df_long = 1.5 / bt["span"].max()                            # df * baseline > 1
    rc, _ = _run(emu, bt, F, df_long, df_long, 2, scale, 2)
    assert rc == -5 and b"baseline" in emu.emu_last_error()
    rc, _ = _run(emu, bt, F, 1.5 * df, df, 2, scale, 2)         # f0 not a multiple of df
    assert rc == -5
