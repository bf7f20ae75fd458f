"""The regression sigma clip and final model (lightkurve_b200/csrc/regress_clip.cuh: rg_clip_kernel, rg_final_kernel)
executed on the CPU through tests/native/cuda_emu.h, at the light-curve lengths where the clip's median takes the
sampling select (N >= 8192) and one below, against oracle/detrend.py:
  outlier mask   identical to sigma_clip_mask(np.where(used, y - X w, nan), sigma)
  final model    X w - median(X w) within 1e-12 max|X w| (the same coefficients)
The clip strikes values out inside the median's partition pass, gathers the standard deviation's sums in that pass
(shifted by the bracket's lower value) and carries the bracket from round to round; the cases below need all five
rounds, tie the residuals, hide most cadences, or hide all of them.  With model_ready = 1 the kernels read X w from the
workspace (as regress() leaves it after rg_model_mma_kernel); with 0 they compute it (rg_model_rows), from a shared or
a per-light-curve design matrix."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import detrend as odet

HERE = os.path.dirname(os.path.abspath(__file__))
CUDA_INC = "/usr/local/cuda/include"
c_vp, c_int, c_dbl, c_i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_int64


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    out = str(tmp_path_factory.mktemp("emu") / "libclip_emu.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-pthread", "-I" + CUDA_INC, "-Wno-attributes", "-shared", "-fPIC",
                           "-Wl,-Bsymbolic", "-o", out, os.path.join(HERE, "native", "clip_emu_driver.cpp")])
    lib = ctypes.CDLL(out)
    lib.emu_clip_final.argtypes = [c_vp, c_int, c_vp, c_vp, c_int, c_i64, c_int, c_vp, c_dbl, c_int, c_vp, c_vp, c_vp]
    lib.emu_clip_final.restype = c_int
    return lib


def run(emu, X, Y, used, W, sigma, model_ready):
    B, N = Y.shape
    K = X.shape[-1]
    X = np.ascontiguousarray(X, np.float64)
    Y = np.ascontiguousarray(Y, np.float64)
    W = np.ascontiguousarray(W, np.float64)
    u8 = np.ascontiguousarray(used, np.uint8)
    xw = np.ascontiguousarray(np.einsum("...nk,bk->bn", X, W) if X.ndim == 2 else np.einsum("bnk,bk->bn", X, W))
    om = np.full((B, N), 7, np.uint8)
    model = np.full((B, N), -7.0)
    emu.emu_clip_final(X.ctypes.data, int(X.ndim == 3), Y.ctypes.data, u8.ctypes.data, B, N, K, W.ctypes.data,
                       float(sigma), int(model_ready), xw.ctypes.data, om.ctypes.data, model.ctypes.data)
    return om.astype(bool), model, xw


def clip_rounds(data, sigma):
    """Rounds of oracle.detrend.sigma_clip_mask that changed the mask (the kernel must run all of them)."""
    return [np.count_nonzero(odet.sigma_clip_mask(data, sigma, maxiters=k) != odet.sigma_clip_mask(data, sigma, k - 1))
            for k in range(1, 6)]


def light_curve(kind, rng, N, K, sigma):
    """(coefficients, residuals, used) of one light curve of the given kind: an offset of 1e4 (flux in e-/s) and
    residual noise of scale 1."""
    w = rng.normal(size=K) * 50.0
    w[0] = 1e4
    used = np.ones(N, bool)
    r = rng.normal(size=N)
    if kind == "dips":
        # transit-like dips on 5 % of the cadences, of log-uniform depths: each clip exposes the next shallower ones.
        # Redrawn until the oracle changes its mask in each of the five rounds.
        for _ in range(20):
            r = rng.normal(size=N)
            for s in rng.choice(N - 40, N // 600, replace=False):
                r[s:s + 30] -= np.exp(rng.uniform(np.log(2.0), np.log(80.0)))
            if all(clip_rounds(r, sigma)):
                break
    elif kind == "flares":
        k = rng.choice(N, N // 100, replace=False)
        r[k] += rng.exponential(6.0, len(k))
    elif kind == "quantised":
        # integer residuals (many ties at the median and at the clip bounds' neighbours) on an exactly integer model
        w = rng.integers(-20, 20, K).astype(np.float64)
        r = np.round(2.0 * rng.normal(size=N))
        r[rng.choice(N, N // 50, replace=False)] += 15.0
    elif kind == "sparse":
        used = rng.random(N) < 0.05
        r[rng.choice(N, N // 200, replace=False)] -= 9.0
    elif kind == "none":
        used = np.zeros(N, bool)
    elif kind == "cadence_mask":
        used = rng.random(N) > 0.1
        r[rng.choice(N, N // 100, replace=False)] += 8.0
    return w, r, used


KINDS = ["quantised", "dips", "flares", "sparse", "none", "cadence_mask"]     # (the first one's X is the shared one)


def design(rng, N, K, quantised=False):
    t = np.linspace(0.0, 1.0, N)
    cols = [np.ones(N)] + [np.sin(2 * np.pi * (k + 1) * t + rng.uniform(0, 6)) * 10 ** rng.uniform(-1, 1)
                           for k in range(K - 1)]
    X = np.stack(cols, axis=1)
    return np.round(4 * X) if quantised else X


@pytest.mark.parametrize("N,K,sigma,model_ready,x_batched,kinds", [
    (8191, 4, 3.0, 1, False, KINDS[:5]),  # below the sampling threshold: radix-select median, two-pass std
    (8192, 5, 5.0, 0, True, KINDS[:3]),   # the first length that samples; X w from per-light-curve design matrices
    (65000, 4, 3.0, 1, False, KINDS),     # a Kepler light curve, X w from the workspace
    (65000, 5, 5.0, 1, False, KINDS[1:3]),
])
def test_clip_and_final_model(emu, N, K, sigma, model_ready, x_batched, kinds):
    """(model_ready = 0 computes X w one warp per cadence: slow on the emulator, so it runs at the smaller length.)"""
    rng = np.random.default_rng(N + 10 * K)
    Xs, Ws, Ys, Us = [], [], [], []
    for kind in kinds:
        X = design(rng, N, K, quantised=(kind == "quantised"))
        w, r, used = light_curve(kind, rng, N, K, sigma)
        y = X @ w + r
        Xs.append(X), Ws.append(w), Ys.append(y), Us.append(used)
    X = np.stack(Xs) if x_batched else Xs[0]
    if not x_batched:              # one shared design matrix: rebuild every flux on it
        for b in range(len(kinds)):
            Ys[b] = Ys[b] - Xs[b] @ Ws[b] + X @ Ws[b]
    W, Y, U = np.stack(Ws), np.stack(Ys), np.stack(Us)
    om, model, xw = run(emu, X, Y, U, W, sigma, model_ready)
    for b, kind in enumerate(kinds):
        res = np.where(U[b], Y[b] - xw[b], np.nan)
        ref = odet.sigma_clip_mask(res, sigma)
        assert np.array_equal(om[b], ref), "%s: %d cadences differ (%d clipped by the oracle)" % (
            kind, np.count_nonzero(om[b] != ref), np.count_nonzero(ref & U[b]))
        ref_model = xw[b] - np.median(xw[b])
        np.testing.assert_allclose(model[b], ref_model, rtol=0, atol=1e-12 * np.max(np.abs(xw[b])), err_msg=kind)
        if kind == "dips":
            assert all(clip_rounds(res, sigma)), "the dips case must need all five clip rounds"
        if kind == "none":
            assert om[b].all()
        if kind == "quantised":
            assert np.all(res[U[b]] == np.round(res[U[b]]))            # the residuals really are integers


def test_singular_fit_and_all_clipped(emu):
    """NaN coefficients (a singular fit): every residual is NaN, so every cadence is masked, and the final model is NaN
    (np.median propagates it), next to a healthy light curve that must be unaffected."""
    rng = np.random.default_rng(3)
    N, K = 1000, 3
    X = design(rng, N, K)
    W = np.stack([np.full(K, np.nan), np.array([1e4, 3.0, -2.0])])
    Y = (X @ np.nan_to_num(W).T).T + rng.normal(size=(2, N))
    Y[1, ::97] += 12.0
    U = np.ones((2, N), bool)
    for model_ready in (0, 1):
        om, model, xw = run(emu, X, Y, U, W, 3.0, model_ready)
        assert om[0].all() and np.isnan(model[0]).all()
        assert np.array_equal(om[1], odet.sigma_clip_mask(Y[1] - xw[1], 3.0))
        np.testing.assert_allclose(model[1], xw[1] - np.median(xw[1]), rtol=0, atol=1e-12 * np.abs(xw[1]).max())
