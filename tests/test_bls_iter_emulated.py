"""K14 (bls_best_kernel, transit_count_kernel and transit_compact_kernel of lightkurve_b200/csrc/bls_iter.cuh) executed
on the CPU through tests/native/cuda_emu.h:
  bls_best   against np.nanargmax: NaNs, exact ties, all-NaN segments (index -1, NaN outputs), one-period grids, CSR
             and shared grids, segment lengths on both sides of the CTA's 256 threads; the period is 1 / (1 / p)
  compact    against numpy's lc[~get_transit_mask]: fewer than half, more than half and exactly half the cadences in
             transit, a box covering every cadence (nothing removed) and none; the survivors in order with their
             original indices, masked_in, the first / smallest / largest surviving time, the flux_err flag and the
             weights it selects, and np.diff of the surviving times."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
CUDA_INC = "/usr/local/cuda/include"
c_vp, c_int, c_i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    out = str(tmp_path_factory.mktemp("emu") / "libbls_iter_emu.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-pthread", "-I" + CUDA_INC,
                           "-Wno-attributes", "-shared", "-fPIC", "-Wl,-Bsymbolic", "-o", out,
                           os.path.join(HERE, "native", "bls_iter_emu_driver.cpp")])
    lib = ctypes.CDLL(out)
    lib.emu_bls_best.argtypes = [c_vp, c_vp, c_vp, c_int, c_i64, c_vp, c_vp]
    lib.emu_bls_best.restype = None
    lib.emu_transit_compact.argtypes = [c_vp] * 5 + [c_int, c_vp, c_vp, c_int] + [c_vp] * 12
    lib.emu_transit_compact.restype = None
    return lib


def _p(x):
    return None if x is None else x.ctypes.data


def _csr(arrays, dtype=np.float64):
    off = np.zeros(len(arrays) + 1, np.int64)
    off[1:] = np.cumsum([len(a) for a in arrays])
    return np.ascontiguousarray(np.concatenate([np.asarray(a, dtype) for a in arrays])), off


def run_best(emu, powers, shared):
    """powers: per light curve; shared: all the same length, laid out [B, P] with one grid."""
    rng = np.random.default_rng(len(powers))
    B = len(powers)
    if shared:
        P = len(powers[0])
        period = np.ascontiguousarray(rng.uniform(0.5, 9.0, P))
        fields = [np.ascontiguousarray(np.stack(powers))] + [np.ascontiguousarray(rng.normal(size=(B, P)))
                                                             for _ in range(5)]
        pofs = None
        seg = [slice(b * P, (b + 1) * P) for b in range(B)]
        per_of = [period] * B
    else:
        pw, pofs = _csr(powers)
        P = int(pofs[-1])
        period = np.ascontiguousarray(rng.uniform(0.5, 9.0, P))
        fields = [pw] + [np.ascontiguousarray(rng.normal(size=P)) for _ in range(5)]
        seg = [slice(pofs[b], pofs[b + 1]) for b in range(B)]
        per_of = [period[s] for s in seg]
    ptrs = (c_vp * 6)(*[f.ctypes.data for f in fields])
    out = np.full((7, B), -7.0)
    index = np.full(B, -7, np.int64)
    emu.emu_bls_best(ptrs, _p(period), _p(pofs), B, P, _p(out), _p(index))
    flat = [f.reshape(-1) for f in fields]
    for b, pw_b in enumerate(powers):
        if np.all(np.isnan(pw_b)):
            assert index[b] == -1 and np.all(np.isnan(out[:, b]))
            continue
        k = int(np.nanargmax(pw_b))
        assert index[b] == k, b
        assert out[0, b] == 1.0 / (1.0 / per_of[b][k])
        # the fields in the ABI's output order: duration, transit_time, depth, depth_err, depth_snr, power
        for j, f in zip(range(1, 6), (3, 4, 1, 2, 5)):
            assert out[j, b] == flat[f][seg[b]][k]
        assert out[6, b] == pw_b[k]


def _powers(rng):
    ps = []
    for n in (1, 2, 31, 255, 256, 257, 600, 1000):
        p = rng.normal(size=n)
        ps.append(p)
        q = p.copy()
        q[rng.choice(n, max(1, n // 3), replace=False)] = np.nan
        ps.append(q)
        ps.append(np.full(n, np.nan))
        t = np.round(rng.uniform(0, 3, n))            # exact ties: the first index wins
        ps.append(t)
    return ps


def test_best_csr(emu):
    run_best(emu, _powers(np.random.default_rng(1)), shared=False)


@pytest.mark.parametrize("P", [1, 7, 256, 513])
def test_best_shared(emu, P):
    rng = np.random.default_rng(P)
    ps = [rng.normal(size=P), np.full(P, np.nan), np.round(rng.uniform(0, 2, P)), rng.normal(size=P)]
    ps[3][::2] = np.nan
    run_best(emu, ps, shared=True)


# ---------------------------------------------------------------------------------------------------------- compact
def _case(rng, n, kind):
    t = 10.0 + np.sort(rng.uniform(0, 5, n))
    y = 1 + 1e-3 * rng.normal(size=n)
    dy = np.full(n, 1e-3)
    m_in = np.zeros(n, bool)
    if kind == "few":
        m_in[rng.choice(n, n // 5, replace=False)] = True
    elif kind == "many":
        m_in[rng.choice(n, n - n // 5, replace=False)] = True
    elif kind == "half":
        m_in[rng.choice(n, n // 2, replace=False)] = True
    elif kind == "all":
        m_in[:] = True
    dy[np.flatnonzero(m_in)[:2]] = np.nan             # NaN errors in transit only
    n_in = int(m_in.sum())
    y_in = np.nan if n_in == 0 else 0.99 + 1e-4 * rng.normal()
    y_out = np.nan if n_in == n else 1.0 + 1e-4 * rng.normal()
    if kind == "half_equal":                          # exactly half, both levels equal: nothing removed
        m_in[rng.choice(n, n // 2, replace=False)] = True
        n_in, y_in, y_out = int(m_in.sum()), 1.0, 1.0
    return t, y, dy, m_in, n_in, y_in, y_out


def _mask(m_in, n_in, y_in, y_out):
    """get_transit_mask_batch's rule."""
    n = len(m_in)
    med = y_out if 2 * n_in < n else (y_in if 2 * n_in > n else np.mean([y_in, y_out]))
    return np.where(m_in, y_in != med, y_out != med)


KINDS = ["few", "many", "half", "all", "none", "half_equal"]


@pytest.mark.parametrize("n", [1, 2, 8, 255, 256, 257, 700])
def test_compact(emu, n):
    rng = np.random.default_rng(n)
    cases = [_case(rng, n + (k % 2 if n > 2 else 0), kind) for k, kind in enumerate(KINDS)]
    B = len(cases)
    # this round's light curves are subsets of their originals: index = every other original cadence
    orig_n = [2 * len(c[0]) for c in cases]
    orig_off = np.zeros(B + 1, np.int64)
    orig_off[1:] = np.cumsum(orig_n)
    idx, off = _csr([np.arange(len(c[0])) * 2 + 1 for c in cases], np.int32)
    t, _ = _csr([c[0] for c in cases])
    y, _ = _csr([c[1] for c in cases])
    dy, _ = _csr([c[2] for c in cases])
    m_in, _ = _csr([c[3] for c in cases], np.uint8)
    stats = np.zeros((B, 15))
    for b, c in enumerate(cases):
        stats[b, 12], stats[b, 13], stats[b, 14] = c[5], c[6], c[4]
    masked = np.full(int(orig_off[-1]), -1, np.int8)
    N = max(int(off[-1]), 1)
    outs = [np.full(N, -7.0) for _ in range(4)]
    idx_out = np.full(N, -7, np.int32)
    noff, doff = np.zeros(B + 1, np.int64), np.zeros(B + 1, np.int64)
    tinfo, fin, dt = np.full((B, 3), -7.0), np.full(B, 7, np.uint8), np.full(N, -7.0)
    emu.emu_transit_compact(_p(t), _p(y), _p(dy), _p(idx), _p(off), B, _p(m_in), _p(stats), 2, _p(orig_off),
                            _p(masked), *[_p(o) for o in outs], _p(idx_out), _p(noff), _p(doff), _p(tinfo), _p(fin),
                            _p(dt))
    for b, (tb, yb, dyb, mb, n_in, y_in, y_out) in enumerate(cases):
        mask = _mask(mb, n_in, y_in, y_out)
        keep = ~mask
        s = slice(noff[b], noff[b + 1])
        assert noff[b + 1] - noff[b] == keep.sum(), (b, KINDS[b])
        np.testing.assert_array_equal(outs[0][s], tb[keep])
        np.testing.assert_array_equal(outs[1][s], yb[keep])
        np.testing.assert_array_equal(outs[2][s], dyb[keep])
        finite = bool(np.isfinite(dyb[keep]).all())
        assert fin[b] == finite
        np.testing.assert_array_equal(outs[3][s], dyb[keep] if finite else np.ones(keep.sum()))
        orig_idx = np.arange(len(tb)) * 2 + 1
        np.testing.assert_array_equal(idx_out[s], orig_idx[keep])
        mo = masked[orig_off[b]:orig_off[b + 1]]
        want = np.full(orig_n[b], -1, np.int8)
        want[orig_idx[mask]] = 2
        np.testing.assert_array_equal(mo, want)
        if keep.any():
            assert (tinfo[b, 0], tinfo[b, 1], tinfo[b, 2]) == (tb[keep][0], np.min(tb[keep]), np.max(tb[keep]))
        else:
            assert np.all(np.isnan(tinfo[b]))
        np.testing.assert_array_equal(dt[doff[b]:doff[b + 1]], np.diff(tb[keep]))
    if n >= 8:
        assert noff[4] - noff[3] == len(cases[3][0]), "a box covering every cadence removes nothing"
