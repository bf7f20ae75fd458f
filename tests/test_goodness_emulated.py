"""The K9 goodness-metric kernels (lightkurve_b200/csrc/goodness.cuh) executed on the CPU through
tests/native/cuda_emu.h and compared with oracle/cbv.py, the numpy restatement of lightkurve's metrics.  Also pins
oracle/cbv.py itself to hand-computed cases of the reference formulas."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import cbv as ocbv

HERE = os.path.dirname(os.path.abspath(__file__))
CUDA_INC = "/usr/local/cuda/include"
c_vp, c_int, c_i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    out = str(tmp_path_factory.mktemp("emu") / "libgoodness_emu.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-pthread", "-I" + CUDA_INC, "-Wno-attributes", "-shared", "-fPIC",
                           "-Wl,-Bsymbolic", "-o", out, os.path.join(HERE, "native", "goodness_emu_driver.cpp")])
    lib = ctypes.CDLL(out)
    lib.emu_underfit.argtypes = [c_vp, c_int, c_vp, c_int, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp]
    lib.emu_underfit.restype = c_int
    lib.emu_overfit.argtypes = [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp]
    lib.emu_overfit.restype = c_int
    lib.emu_last_error.restype = ctypes.c_char_p
    return lib


def emu_underfit(emu, pool, target, nbs):
    pool = np.ascontiguousarray(pool, np.float64)
    target = np.ascontiguousarray(np.atleast_2d(target), np.float64)
    off = np.zeros(len(nbs) + 1, np.int64)
    off[1:] = np.cumsum([len(n) for n in nbs])
    idx = np.ascontiguousarray(np.concatenate([np.asarray(n, np.int32) for n in nbs]) if off[-1] else
                               np.zeros(1, np.int32))
    B, G = target.shape
    metric, n_used, c3 = np.full(B, -7.0), np.full(B, -7, np.int32), np.full(B, -7.0)
    st = emu.emu_underfit(pool.ctypes.data, len(pool), target.ctypes.data, B, G, off.ctypes.data, idx.ctypes.data,
                          metric.ctypes.data, n_used.ctypes.data, c3.ctypes.data)
    assert st == 0, emu.emu_last_error()
    return metric, n_used, c3


def check_underfit(emu, pool, target, nbs):
    metric, n_used, c3 = emu_underfit(emu, pool, target, nbs)
    for b, nb in enumerate(nbs):
        m, n, c = ocbv.underfit_metric(target[b], pool[list(nb)])
        assert n_used[b] == n, b
        np.testing.assert_allclose(c3[b], c, rtol=1e-12, atol=1e-300, err_msg="target %d" % b)
        np.testing.assert_allclose(metric[b], m, rtol=1e-12, err_msg="target %d" % b)
    return metric, n_used, c3


def systematics_pool(rng, P, G, n_sys=3, nan_frac=0.02):
    """P light curves sharing a few systematic trends with individual weights, plus white noise and NaN gaps."""
    t = np.linspace(0, 1, G)
    sys = np.stack([np.sin(2 * np.pi * (k + 1) * t + k) for k in range(n_sys)])
    pool = rng.normal(size=(P, n_sys)) @ sys * 1e-3 + rng.normal(scale=1e-3, size=(P, G))
    pool[rng.random((P, G)) < nan_frac] = np.nan
    return pool


@pytest.mark.parametrize("M", [1, 2, 7, 31, 32, 33, 64])
def test_underfit_neighbour_counts(emu, M):
    rng = np.random.default_rng(M)
    G = 700
    pool = systematics_pool(rng, 80, G)
    target = systematics_pool(rng, 3, G)
    nbs = [rng.choice(80, M, replace=False) for _ in range(3)]
    check_underfit(emu, pool, target, nbs)


def test_underfit_nan_union_and_zero_rms(emu):
    """Cadences dropped when ANY neighbour is NaN; a neighbour that is zero on the surviving cadences (RMS 0 -> inf)
    contributes correlation 0 and still counts in the mean; a constant target likewise."""
    rng = np.random.default_rng(5)
    G = 517                                          # not a multiple of 32 or of 128
    pool = systematics_pool(rng, 12, G, nan_frac=0.0)
    pool[0, 10:60] = np.nan
    pool[1, 200:230] = np.nan
    pool[2] = 0.0
    pool[3, ::2] = np.nan
    pool[3, 1::2] = 0.0                              # zero wherever it is present
    target = systematics_pool(rng, 3, G, nan_frac=0.05)
    target[2] = 0.0
    nbs = [[0, 1, 2, 4, 5], [3, 6, 7], [0, 2, 8, 9]]
    metric, n_used, _ = check_underfit(emu, pool, target, nbs)
    assert n_used[0] == int(np.sum(~np.isnan(target[0]) & ~np.isnan(pool[0]) & ~np.isnan(pool[1])))
    assert n_used[1] == int(np.sum(~np.isnan(target[1]) & ~np.isnan(pool[3])))


def test_underfit_overlapping_neighbour_sets(emu):
    """Targets whose neighbour lists overlap (and repeat pool rows in different orders) on a longer grid."""
    rng = np.random.default_rng(11)
    G = 3000
    pool = systematics_pool(rng, 40, G)
    target = pool[:6] + rng.normal(scale=1e-4, size=(6, G))
    nbs = [np.r_[np.arange(b + 1, b + 21)] for b in range(6)]
    nbs[3] = nbs[3][::-1]
    check_underfit(emu, pool, target, nbs)
    # a target's result does not depend on the other targets of the call
    one, n1, c1 = emu_underfit(emu, pool, target[4:5], nbs[4:5])
    allm, alln, allc = emu_underfit(emu, pool, target, nbs)
    assert one[0] == allm[4] and n1[0] == alln[4] and c1[0] == allc[4]


def test_underfit_no_cadence_left(emu):
    pool = np.full((2, 50), np.nan)
    target = np.ones((1, 50))
    metric, n_used, c3 = check_underfit(emu, pool, target, [[0, 1]])
    assert n_used[0] == 0 and c3[0] == 0.0 and metric[0] == 1.0


def test_oracle_underfit_hand_cases():
    """oracle/cbv.py against the reference formulas worked by hand."""
    rng = np.random.default_rng(0)
    x = rng.normal(size=400)
    # a neighbour identical to the target: correlation 1, mean of (1^3, 0) = 0.5
    m, n, c3 = ocbv.underfit_metric(x, x[None, :])
    assert n == 400 and c3 == pytest.approx(0.5, rel=1e-15)
    wgn = 0.0007 + 0.8083 * 400 ** -0.5023
    assert m == pytest.approx(2.0 / (1 + np.exp(np.log(2 / 0.95 - 1) / wgn * 0.5)), rel=1e-14)
    # anti-correlated neighbour: |c|^3 = 1 as well
    assert ocbv.underfit_metric(x, -x[None, :])[2] == pytest.approx(0.5, rel=1e-15)
    # orthogonal neighbour: c = 0 -> metric = 1
    y = np.r_[np.ones(200), -np.ones(200)]
    z = np.r_[np.ones(100), -np.ones(100), np.ones(100), -np.ones(100)]
    assert ocbv.underfit_metric(y, z[None, :])[0] == 1.0
    # two neighbours with c = 1 and c = 1 / sqrt(2): (1 + 2^-1.5 + 0) / 3
    a = np.r_[np.ones(2), -np.ones(2)]
    b = np.r_[np.ones(1), np.zeros(1), -np.ones(1), np.zeros(1)] * np.sqrt(2)
    _, _, c3 = ocbv.underfit_metric(a, np.stack([a, b]))
    assert c3 == pytest.approx((1 + (1 / np.sqrt(2)) ** 3) / 3, rel=1e-14)


def test_oracle_overfit_hand_cases():
    n, s, means = ocbv.overfit_terms([1.0, 2.0, np.nan, 5.0], [0.5, 3.0, 1.0, 1.0], [[1.0, np.nan, 3.0]])
    assert n == 2 and s == 4.5 and means == [2.0]
    assert ocbv.overfit_metric(n, s, means) == pytest.approx(2.0 / (1 + np.exp(4.5 / (2 * 2.0))))
    assert ocbv.overfit_metric(0, 0.0, [1.0]) == 1.0
    assert ocbv.overfit_metric(3, 1.0, [0.0]) == 0.0
    assert ocbv.objective(0.7, 0.9, 0.5, 0.8) == pytest.approx(-(0.5 + 0.002 + 0.8 + 0.001))
    assert ocbv.objective(0.3, 0.2, 0.5, 0.0) == pytest.approx(-1.3)


def emu_overfit(emu, corr, orig, noise, off, S):
    corr, orig = np.ascontiguousarray(corr, np.float32), np.ascontiguousarray(orig, np.float32)
    noise = np.ascontiguousarray(noise, np.float32) if S else np.zeros(1, np.float32)
    off = np.ascontiguousarray(off, np.int64)
    B = len(off) - 1
    npos, spos, nmean = np.full(B, -7, np.int32), np.full(B, -7.0), np.full(max(1, B * S), -7.0)
    st = emu.emu_overfit(corr.ctypes.data, orig.ctypes.data, noise.ctypes.data, off.ctypes.data, B, S,
                         npos.ctypes.data, spos.ctypes.data, nmean.ctypes.data)
    assert st == 0, emu.emu_last_error()
    return npos, spos, nmean[:B * S].reshape(B, S)


@pytest.mark.parametrize("S", [0, 1, 3])
def test_overfit_terms_on_the_emulator(emu, S):
    rng = np.random.default_rng(S)
    lens = [1, 37, 256, 257, 3001]
    off = np.r_[0, np.cumsum(lens)]
    corr = rng.random(off[-1]).astype(np.float32)
    orig = rng.random(off[-1]).astype(np.float32)
    corr[::17] = np.nan
    orig[5::23] = np.nan
    noise = rng.random(S * off[-1]).astype(np.float32)
    noise[::13] = np.nan
    npos, spos, nmean = emu_overfit(emu, corr, orig, noise, off, S)
    for b, n in enumerate(lens):
        rows = [noise[S * off[b] + s * n: S * off[b] + (s + 1) * n] for s in range(S)]
        n_o, s_o, m_o = ocbv.overfit_terms(corr[off[b]:off[b + 1]], orig[off[b]:off[b + 1]], rows)
        assert npos[b] == n_o, b
        np.testing.assert_allclose(spos[b], s_o, rtol=1e-12, atol=0)
        np.testing.assert_allclose(nmean[b], m_o, rtol=1e-12)
