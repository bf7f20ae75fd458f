"""K11 (batched sigma clip) and K12 (CDPP finish) of lightkurve_b200/csrc/clip.cuh executed on the CPU through
tests/native/cuda_emu.h, against tests/_cdpp_oracle.py (on oracle/detrend.py):
  clip mask      identical to sigma_clip_mask(x, sigma_lower=, sigma_upper=, maxiters=) on every case of
                 tests/_cdpp_cases.py (flares, one-sided deep dips, NaN/inf, asymmetric and infinite sigmas, maxiters
                 0, 1, 5 and until converged, ties, a constant light curve, 0, 1 and 2 finite values, and light curves
                 past the shared-memory capacity that stream from global memory)
  centre / std   np.median / np.std of the kept values; n_kept their count
  CDPP           cdpp_of_flat (remove_outliers, normalize("ppm"), the cumsum running_mean, np.std) to rtol 1e-6, fed
                 the oracle's flattened flux
and bitwise independence of a light curve's outputs from its neighbours, its position and where it works (shared or
global memory)."""
import ctypes
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _cdpp_cases as C  # noqa: E402
import _cdpp_oracle as O  # noqa: E402

from oracle import detrend as odet  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
CUDA_INC = "/usr/local/cuda/include"
c_vp, c_int, c_dbl, c_i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_int64


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    out = str(tmp_path_factory.mktemp("emu") / "libclip_cdpp_emu.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-pthread", "-I" + CUDA_INC,
                           "-Wno-attributes", "-shared", "-fPIC", "-Wl,-Bsymbolic", "-o", out,
                           os.path.join(HERE, "native", "clip_cdpp_emu_driver.cpp")])
    lib = ctypes.CDLL(out)
    lib.emu_clip_cdpp.argtypes = [c_vp, c_vp, c_int, c_dbl, c_dbl, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_vp,
                                  c_i64]
    lib.emu_clip_cdpp.restype = c_int
    assert lib.emu_cl_res_cap() == C.RES_CAP
    return lib


def run(emu, xs, sigma_lower=3.0, sigma_upper=3.0, maxiters=5, durations=None, res_cap=-1):
    """dict(mask (list of bool), center, std, n_kept, cdpp [B, D] or None, streamed) of one emulated launch."""
    B = len(xs)
    off = np.zeros(B + 1, np.int64)
    off[1:] = np.cumsum([len(x) for x in xs])
    x = np.ascontiguousarray(np.concatenate([np.asarray(v, np.float64) for v in xs]) if B else np.zeros(0))
    mask = np.full(max(int(off[-1]), 1), 7, np.uint8)
    center, sd, nk = np.full(B, -7.0), np.full(B, -7.0), np.full(B, -7, np.int64)
    dur = None if durations is None else np.ascontiguousarray(durations, np.int32)
    D = 0 if dur is None else len(dur)
    cd = np.full((B, max(D, 1)), -7.0)
    streamed = emu.emu_clip_cdpp(x.ctypes.data, off.ctypes.data, B, float(sigma_lower), float(sigma_upper),
                                 -1 if maxiters is None else int(maxiters), mask.ctypes.data, center.ctypes.data,
                                 sd.ctypes.data, nk.ctypes.data, None if dur is None else dur.ctypes.data, D,
                                 cd.ctypes.data, int(res_cap))
    return dict(mask=[mask[off[b]:off[b + 1]].astype(bool) for b in range(B)], center=center, std=sd, n_kept=nk,
                cdpp=cd[:, :D] if D else None, streamed=bool(streamed))


CASES = C.clip_cases()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_clip_matches_oracle(emu, case):
    name, x, sl, su, mi = case
    r = run(emu, [x], sl, su, mi)
    ref = O.sigma_clip_mask(x, sigma_lower=sl, sigma_upper=su, maxiters=mi)
    assert np.array_equal(r["mask"][0], ref), "%s: %d cadences differ (%d masked by the oracle)" % (
        name, np.count_nonzero(r["mask"][0] != ref), np.count_nonzero(ref))
    assert r["streamed"] == (len(x) > C.RES_CAP)
    kept = x[~ref]
    assert r["n_kept"][0] == len(kept)
    if len(kept):
        assert r["center"][0] == np.median(kept)
        np.testing.assert_allclose(r["std"][0], np.std(kept), rtol=1e-12, atol=1e-300)
    else:
        assert np.isnan(r["center"][0]) and np.isnan(r["std"][0])
    if name == "deep_dips":                       # every one of the five rounds changes the mask
        rounds = [np.count_nonzero(O.sigma_clip_mask(x, 3.0, k) != O.sigma_clip_mask(x, 3.0, k - 1))
                  for k in range(1, 6)]
        assert all(rounds), rounds
    if name == "deep_dips_converged":             # and it needs more than five to converge
        assert not np.array_equal(ref, O.sigma_clip_mask(x, 3.0, 5))
    if name == "two_finite":                      # both values lie exactly on the bounds (0.75 -+ 1.75): both kept
        assert r["n_kept"][0] == 2


def _flat_cases():
    rng = np.random.default_rng(77)
    specs = [(3000, 300, "everything"), (18000, 60, "transit"), (9000, 1000, "flares"), (C.RES_CAP + 500, 100, "nans"),
             (65000, 40, "gaps")]
    flats = []
    for n, ppm, kind in specs:
        t, f = C.light_curve(rng, n, ppm, kind)
        flats.append(odet.flatten(t, f)[0])
    flats.append(flats[0][:10])                   # fewer kept cadences than the duration: the window shrinks
    one = np.full(40, np.nan)
    one[3] = 1.0001
    flats.append(one)                             # one kept cadence: 0
    flats.append(np.full(25, np.nan))             # none: NaN
    flats.append(np.zeros(0))
    return flats


DURATIONS = [13, 1, 2, 30, 500, 100000]


def test_cdpp_matches_oracle(emu):
    flats = _flat_cases()
    r = run(emu, flats, 5.0, 5.0, 5, DURATIONS)
    assert r["streamed"]
    for b, flat in enumerate(flats):
        assert np.array_equal(r["mask"][b], O.sigma_clip_mask(flat, 5.0)), b
        for d, dur in enumerate(DURATIONS):
            ref = O.cdpp_of_flat(flat, dur, 5.0)
            got = r["cdpp"][b, d]
            if np.isnan(ref):
                assert np.isnan(got), (b, dur)
            else:
                np.testing.assert_allclose(got, ref, rtol=1e-6, atol=0, err_msg="light curve %d, duration %d" % (b, dur))
    # ten kept cadences: durations of 10 or more shrink to one window (0), durations 1 and 2 do not
    np.testing.assert_array_equal(r["cdpp"][-4] > 0, [False, True, True, False, False, False])
    assert np.all(r["cdpp"][-3] == 0.0)            # one kept cadence
    assert np.all(np.isnan(r["cdpp"][-2])) and np.all(np.isnan(r["cdpp"][-1]))   # none kept, no cadence


def _same(a, b, i, j):
    assert np.array_equal(a["mask"][i], b["mask"][j])
    for k in ("center", "std", "n_kept"):
        assert np.array_equal(a[k][i], b[k][j], equal_nan=True), k
    if a["cdpp"] is not None:
        assert np.array_equal(a["cdpp"][i], b["cdpp"][j], equal_nan=True)


def test_batch_position_neighbours_and_memory(emu):
    """Each light curve's outputs are bitwise those of its own launch, in any order, with any neighbours, whether it
    works in shared memory or in global memory (res_cap 0: all stream)."""
    xs = [c[1] for c in CASES if c[2] == 3.0 and c[3] == 3.0 and c[4] == 5]
    flats = _flat_cases()
    xs = xs + flats[:3] + flats[-4:]
    base = run(emu, xs, durations=DURATIONS)
    perm = np.random.default_rng(5).permutation(len(xs))
    shuffled = run(emu, [xs[p] for p in perm], durations=DURATIONS)
    streamed = run(emu, xs, durations=DURATIONS, res_cap=0)
    assert streamed["streamed"]
    for j, p in enumerate(perm):
        _same(base, shuffled, p, j)
    for i in range(len(xs)):
        _same(base, streamed, i, i)
    for i in (0, 3, len(xs) - 1):
        _same(base, run(emu, [xs[i]], durations=DURATIONS), i, 0)
