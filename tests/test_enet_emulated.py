"""The K8 elastic-net kernel (lightkurve_b200/csrc/enet.cuh, enet_cd_kernel and its launcher) executed on the CPU
through tests/native/cuda_emu.h, on Gram matrices built here in numpy, and compared with oracle/enet.py (scikit-learn's
coordinate descent restated on X): identical n_iter and convergence flag, coefficients within rtol 1e-9.

The kernel iterates on the Gram matrix while the oracle iterates on X, so the two round differently.  A fixture whose
stopping or screening decision lies within 1e-6 (relative) of its threshold could then legitimately stop a sweep
earlier or later; such seeds are replaced (and reported), as in tests/test_enet_oracle.py."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import enet as oen

HERE = os.path.dirname(os.path.abspath(__file__))
CUDA_INC = "/usr/local/cuda/include"
c_vp, c_int, c_dbl = ctypes.c_void_p, ctypes.c_int, ctypes.c_double
MARGIN = 1e-6


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    out = str(tmp_path_factory.mktemp("emu") / "libenet_emu.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-pthread", "-I" + CUDA_INC, "-Wno-attributes", "-shared", "-fPIC",
                           "-Wl,-Bsymbolic", "-o", out, os.path.join(HERE, "native", "enet_emu_driver.cpp")])
    lib = ctypes.CDLL(out)
    lib.emu_enet_cd.argtypes = [c_vp, c_vp, c_int, c_int, c_dbl, c_dbl, c_int, c_dbl, c_int, c_vp, c_vp, c_vp, c_vp]
    lib.emu_enet_cd.restype = c_int
    lib.emu_last_error.restype = ctypes.c_char_p
    lib.emu_warps_per_cta.argtypes = [c_int]
    return lib


def gram_of(Xs, ys, masks):
    """[B, K+1, K+1] with the upper triangle of [X | y]^T [X | y] over the masked rows and NaN below the diagonal
    (the kernel must read the upper triangle only), and the used-cadence counts."""
    B, K = len(Xs), Xs[0].shape[1]
    G = np.empty((B, K + 1, K + 1))
    for b in range(B):
        A = np.hstack([Xs[b], ys[b][:, None]])[masks[b]]
        M = A.T @ A
        M[np.tril_indices(K + 1, -1)] = np.nan
        G[b] = M
    return G, np.array([int(m.sum()) for m in masks], np.int32)


def run(emu, Xs, ys, masks=None, alpha=1e-20, l1_ratio=0.01, max_iter=1000, tol=1e-4, positive=False):
    masks = [np.ones(len(y), bool) for y in ys] if masks is None else masks
    G, cnt = gram_of(Xs, ys, masks)
    B, K = len(Xs), Xs[0].shape[1]
    coeff = np.full((B, K), -7.0)
    n_iter = np.full(B, -7, np.int32)
    gap = np.full(B, -7.0)
    conv = np.full(B, 7, np.uint8)
    st = emu.emu_enet_cd(G.ctypes.data, cnt.ctypes.data, B, K, alpha, l1_ratio, max_iter, tol, int(positive),
                         coeff.ctypes.data, n_iter.ctypes.data, gap.ctypes.data, conv.ctypes.data)
    assert st == 0, emu.emu_last_error()
    return coeff, n_iter, gap, conv.astype(bool)


def fixtures(n, make, seeds, **kw):
    """n (X, y, oracle result) whose decisions all clear MARGIN."""
    out = []
    for s in seeds:
        X, y = make(s)
        r = oen.enet_fit(X, y, **kw)
        if r["margin"] > MARGIN:
            out.append((X, y, r))
            if len(out) == n:
                return out
        else:
            print("seed %d replaced: a decision lies %.2e (relative) from its threshold" % (s, r["margin"]))
    raise AssertionError("not enough seeds with clear decisions")


def check(emu, fx, **kw):
    Xs, ys, rs = [f[0] for f in fx], [f[1] for f in fx], [f[2] for f in fx]
    coeff, n_iter, gap, conv = run(emu, Xs, ys, **kw)
    for b, r in enumerate(rs):
        assert n_iter[b] == r["n_iter"], (b, n_iter[b], r["n_iter"])
        assert conv[b] == r["converged"], b
        scale = max(np.max(np.abs(r["coef"])), 1e-300)
        np.testing.assert_allclose(coeff[b], r["coef"], rtol=1e-9, atol=1e-9 * scale, err_msg="light curve %d" % b)
        yy = float(ys[b] @ ys[b])
        np.testing.assert_allclose(gap[b], r["dual_gap"], rtol=1e-6, atol=1e-10 * yy / len(ys[b]))
    return coeff, n_iter


@pytest.mark.parametrize("K", [1, 2, 5, 17, 33, 64])
def test_enet_sizes_on_the_emulator(emu, K):
    kw = dict(alpha=1e-20, l1_ratio=0.01)
    fx = fixtures(3, lambda s: oen.cbv_fixture(100 * K + s, N=max(400, 4 * K), K=K, scale=1e4), range(40), **kw)
    check(emu, fx, **kw)


def test_enet_k165_on_the_emulator(emu):
    """The largest K: one light curve per CTA, 220 KB of shared memory."""
    assert emu.emu_warps_per_cta(165) == 1
    kw = dict(alpha=1e-3, l1_ratio=0.5, max_iter=40)
    fx = fixtures(1, lambda s: oen.cbv_fixture(s, N=600, K=165, scale=1e4, kind="orthonormal"), range(20), **kw)
    check(emu, fx, **kw)


def test_enet_many_light_curves_per_cta(emu):
    """K = 9 packs eight light curves per CTA: eleven light curves fill one CTA and part of the next, with ragged
    masks, and each one's results equal its own single-light-curve run bitwise."""
    assert emu.emu_warps_per_cta(9) == 8
    kw = dict(alpha=1.0, l1_ratio=0.9)

    def masked(s):
        X, y = oen.cbv_fixture(s, N=700, K=9, scale=1e4)
        m = np.random.default_rng(1000 + s).random(700) > 0.05 * (s % 11)
        return X, y, m

    Xs, ys, masks, rs = [], [], [], []
    for s in range(60):
        X, y, m = masked(s)
        r = oen.enet_fit(X[m], y[m], **kw)
        if r["margin"] <= MARGIN:
            print("seed %d replaced: a decision lies %.2e (relative) from its threshold" % (s, r["margin"]))
            continue
        Xs.append(X), ys.append(y), masks.append(m), rs.append(r)
        if len(rs) == 11:
            break
    coeff, n_iter, _, conv = run(emu, Xs, ys, masks, **kw)
    for b, r in enumerate(rs):
        assert n_iter[b] == r["n_iter"] and conv[b] == r["converged"], b
        np.testing.assert_allclose(coeff[b], r["coef"], rtol=1e-9, atol=1e-9 * np.max(np.abs(r["coef"])))
    c1, n1, _, _ = run(emu, [Xs[9]], [ys[9]], [masks[9]], **kw)
    np.testing.assert_array_equal(c1[0], coeff[9])
    assert n1[0] == n_iter[9]


def test_enet_screening_on_the_emulator(emu):
    kw = dict(alpha=30.0, l1_ratio=1.0)
    fx = fixtures(3, lambda s: oen.cbv_fixture(s, N=800, K=12, scale=1e4), range(40), **kw)
    coeff, _ = check(emu, fx, **kw)
    assert np.count_nonzero(coeff == 0) >= 3


@pytest.mark.parametrize("case", ["positive", "alpha0", "ridge", "max_iter"])
def test_enet_options_on_the_emulator(emu, case):
    kw = {"positive": dict(alpha=1e-3, l1_ratio=0.5, positive=True),
          "alpha0": dict(alpha=0.0, l1_ratio=0.5, max_iter=200),
          "ridge": dict(alpha=1e-2, l1_ratio=0.0),
          "max_iter": dict(alpha=1e-20, l1_ratio=0.01, max_iter=6)}[case]
    scale = 1.0 if case == "alpha0" else 1e4
    fx = fixtures(3, lambda s: oen.cbv_fixture(s, N=600, K=7, scale=scale), range(40), **kw)
    coeff, n_iter = check(emu, fx, **kw)
    if case == "positive":
        assert np.all(coeff >= 0)
    if case == "max_iter":
        assert np.all(n_iter == 6)


def test_enet_zero_column_and_zero_flux_on_the_emulator(emu):
    X, y = oen.cbv_fixture(3, N=500, K=8, scale=1e4)
    X[:, 2] = 0.0
    for kw in (dict(alpha=1e-3, l1_ratio=0.5), dict(alpha=1e-2, l1_ratio=0.0), dict(alpha=1e-20, l1_ratio=0.01)):
        r = oen.enet_fit(X, y, **kw)
        assert r["margin"] > MARGIN
        coeff, n_iter = check(emu, [(X, y, r)], **kw)
        assert coeff[0, 2] == 0.0
    # zero flux: the gap is zero before the first sweep
    r = oen.enet_fit(X, np.zeros(500), alpha=1.0, l1_ratio=0.5)
    coeff, n_iter = check(emu, [(X, np.zeros(500), r)], alpha=1.0, l1_ratio=0.5)
    assert n_iter[0] == 0 and np.all(coeff == 0)
