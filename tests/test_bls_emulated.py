"""K3 Box Least Squares - the whole translation unit lightkurve_b200/csrc/bls.cu: prologue, lookup tables, launch
planning, the cadence and boundary paths, shared-memory and global histograms - executed on the CPU through
tests/native/cuda_emu.h and compared with the C restatement of astropy's bls.c (oracle/bls_c.c) at every oversample.

The fixtures are exact-arithmetic ones (tests/_bls_cases.py): every sum is exact in fp64, so the bins and all seven
outputs must equal bls_power_c bit for bit, ties included, with no tie allowance.  Every case asserts the kernel paths
it was written to reach (LKB_BLS_OBSERVE counters) and prints them with the number of exact ties it checked
(`pytest -s` or `-rP` shows them)."""
import ctypes
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _bls_cases as C  # noqa: E402

from oracle import bls as obls  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
CUDA_INC = "/usr/local/cuda/include"
PATHS = ("cadence", "boundary", "ghist", "wrap3", "slow_div", "exact_walk")    # enum BlsPath in bls.cu
c_vp, c_int, c_i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64


def build_emulator(out_dir):
    """g++ build of tests/native/bls_emu_driver.cpp; returns the loaded library (None without g++ / CUDA headers)."""
    if shutil.which("g++") is None or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        return None
    out = os.path.join(str(out_dir), "libbls_emu.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-pthread", "-ffp-contract=off", "-I" + CUDA_INC,
                           "-Wno-attributes", "-shared", "-fPIC", "-Wl,-Bsymbolic", "-o", out,
                           os.path.join(HERE, "native", "bls_emu_driver.cpp")])
    lib = ctypes.CDLL(out)
    lib.emu_bls_power.argtypes = [c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_i64, c_vp, c_int, c_int, c_int] + [c_vp] * 8
    lib.emu_bls_power.restype = c_int
    lib.emu_bls_bin_index.argtypes = [c_vp, c_i64, ctypes.c_double, ctypes.c_double, ctypes.c_double, c_vp]
    lib.emu_bls_bin_index.restype = c_int
    lib.emu_bls_paths.argtypes = [c_vp]
    lib.emu_bls_set_table_budget.argtypes = [c_i64]
    lib.emu_launches.restype = c_i64
    lib.emu_last_error.restype = ctypes.c_char_p
    assert lib.emu_bls_path_count() == len(PATHS)
    return lib


def _p(a):
    return None if a is None else a.ctypes.data


def emu_power(lib, ts, ys, dys, period, duration, oversample=10, objective="likelihood"):
    """lkb_bls_power_ex through the emulator.  period: one shared grid, or a list of per-light-curve grids.
    Returns (per-light-curve result dicts with "bins", path counters)."""
    B = len(ts)
    off = np.concatenate([[0], np.cumsum([len(a) for a in ts])]).astype(np.int64)
    t = np.ascontiguousarray(np.concatenate(ts), dtype=np.float64)
    y = np.ascontiguousarray(np.concatenate(ys), dtype=np.float64)
    dy = None
    if dys is not None:
        dy = np.ascontiguousarray(np.concatenate([np.ones(len(a)) if e is None else e for a, e in zip(ts, dys)]))
    per_lc = isinstance(period, list)
    if per_lc:
        grids = [np.asarray(g, dtype=np.float64) for g in period]
        per = np.ascontiguousarray(np.concatenate(grids))
        pofs = np.concatenate([[0], np.cumsum([len(g) for g in grids])]).astype(np.int64)
        shape = (len(per),)
    else:
        per = np.ascontiguousarray(period, dtype=np.float64)
        pofs = None
        shape = (B, len(per))
    dur = np.ascontiguousarray(duration, dtype=np.float64)
    outs = [np.full(shape, 7.0) for _ in range(7)]
    bins = np.full(shape + (2,), 7, dtype=np.int32)
    lib.emu_bls_reset_paths()
    rc = lib.emu_bls_power(_p(t), _p(y), _p(dy), _p(off), B, _p(per), _p(pofs), len(per), _p(dur), len(dur),
                           int(oversample), 1 if objective == "snr" else 0, *[_p(o) for o in outs], _p(bins))
    if rc != 0:
        raise RuntimeError("emu_bls_power: %d %s" % (rc, lib.emu_last_error().decode()))
    cnt = np.zeros(len(PATHS), dtype=np.int64)
    lib.emu_bls_paths(_p(cnt))
    res = []
    for b in range(B):
        sl = slice(pofs[b], pofs[b + 1]) if per_lc else b
        r = {k: o[sl] for k, o in zip(C.FIELDS, outs)}
        r["bins"] = bins[sl]
        res.append(r)
    return res, dict(zip(PATHS, cnt.tolist()))


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = build_emulator(tmp_path_factory.mktemp("bls_emu"))
    if lib is None:
        pytest.skip("needs g++ and the CUDA headers")
    return lib


def check_all(res, ts, ys, dys, grids, duration, oversample, objective, label):
    """Every non-empty light curve bitwise equal to bls_power_c; prints and returns the exact ties checked."""
    tied_periods = tied_boxes = 0
    for b, (t, y) in enumerate(zip(ts, ys)):
        dy = None if dys is None else dys[b]
        g = grids[b] if isinstance(grids, list) else grids
        if len(t) == 0:
            assert np.all(np.isnan(res[b]["power"])) and np.all(res[b]["bins"] == -1)
            continue
        tp, tb = C.assert_exact(res[b], t, y, dy, g, duration, oversample, objective, "%s lc %d" % (label, b))
        tied_periods += tp
        tied_boxes += tb
    return tied_periods, tied_boxes


def report(label, cnt, ties=None):
    msg = "%s: paths %s" % (label, " ".join("%s=%d" % kv for kv in cnt.items()))
    if ties is not None:
        msg += "; exact ties checked bitwise: %d periods (%d boxes)" % ties
    print(msg)


# ---- the matrix: oversample x objective x path, with histogram placement and grid layout rotating ----------------
OVERSAMPLES = (1, 2, 3, 10, 40)
PATH_ENV = {"cadence": "1e31", "boundary": "0", "auto": None}
HIST_ENV = {"smem": ("1000000000", None), "global": ("0", None), "global_tiny_cap": ("0", "1")}


def set_env(monkeypatch, path, hist):
    for k, v in (("LKB_BLS_MIN_DENSITY", PATH_ENV[path]), ("LKB_BLS_GHIST_BINS", HIST_ENV[hist][0]),
                 ("LKB_BLS_HIST_CAP_MB", HIST_ENV[hist][1])):
        if v is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, v)


@pytest.mark.parametrize("objective", ["likelihood", "snr"])
@pytest.mark.parametrize("path", list(PATH_ENV))
@pytest.mark.parametrize("oversample", OVERSAMPLES)
def test_matrix_bitwise(emu, monkeypatch, oversample, path, objective):
    """Each (oversample, path) meets every histogram placement over the two objectives and both grid layouts over
    neighbouring oversamples: hist = (path + objective) mod 3, layout = (oversample index + objective) mod 2."""
    pi, oi, si = list(PATH_ENV).index(path), ("likelihood", "snr").index(objective), OVERSAMPLES.index(oversample)
    hist = list(HIST_ENV)[(pi + oi) % 3]
    csr = (si + oi) % 2 == 1
    set_env(monkeypatch, path, hist)
    cases = C.matrix_batch()
    names, ts, ys, dys = zip(*cases)
    grid = C.matrix_grid()
    grids = [grid[b % 3::1 + b % 2] for b in range(len(ts))] if csr else grid
    res, cnt = emu_power(emu, list(ts), list(ys), list(dys), grids, C.DUR, oversample, objective)
    ties = check_all(res, ts, ys, dys, grids, C.DUR, oversample, objective, "matrix")
    label = "oversample=%d %s %s %s %s" % (oversample, objective, path, hist, "csr" if csr else "shared")
    report(label, cnt, ties)
    total = sum(len(grids[b]) if csr else len(grid) for b in range(len(ts)))
    assert cnt["cadence"] + cnt["boundary"] == total
    if path == "cadence":
        assert cnt["boundary"] == 0
    if path == "boundary" and oversample > 1:
        assert cnt["boundary"] > 0           # sorted light curves with K1 + 1 >= 33 (every period from 0.4 d on)
    if path == "boundary" and oversample == 1:
        assert cnt["boundary"] > 0 and cnt["cadence"] > 0      # both sides of the K1 + 1 >= 33 gate
    assert cnt["ghist"] == (0 if hist == "smem" else total)
    assert cnt["wrap3"] > 0 or path == "boundary"
    assert ties[0] > 0                        # the constant light curve alone ties at every period


# ---- edges ---------------------------------------------------------------------------------------------------------
def test_no_box_qualifies_and_empty_light_curve(emu, monkeypatch):
    """One or two cadences, all cadences at one time (no box has ivar_in and ivar_out both >= DBL_EPSILON: power
    -inf, bins -1, the C code's zeros and transit time t_ref) and an empty light curve inside the batch (NaN)."""
    rng = np.random.default_rng(1)
    ts = [np.array([C.T0 + 0.5]), C.T0 + np.array([0.25, 3.0]), np.zeros(0), np.full(40, C.T0 + 2.0),
          C.dyadic_times(rng, 60, 6.0)]
    ys = [np.array([3 / 64.0]), np.array([1 / 64.0, -2 / 64.0]), np.zeros(0),
          rng.integers(-4, 5, 40) / 64.0, C.dyadic_flux(rng, ts[4], 1.5)]
    grid = C.matrix_grid(16)
    for path in ("cadence", "boundary"):
        set_env(monkeypatch, path, "smem")
        for oversample in (1, 10):
            res, cnt = emu_power(emu, ts, ys, None, grid, C.DUR, oversample)
            ties = check_all(res, ts, ys, None, grid, C.DUR, oversample, "likelihood", "edge")
            report("no box / empty, %s, oversample=%d" % (path, oversample), cnt, ties)
            for b in (0, 3):
                assert np.all(res[b]["power"] == -np.inf) and np.all(res[b]["bins"] == -1)
            assert np.all(np.isnan(res[2]["power"])) and np.all(np.isnan(res[2]["transit_time"]))
            # the empty light curve writes its outputs but takes no path
            assert cnt["cadence"] + cnt["boundary"] == 4 * len(grid)


@pytest.mark.parametrize("n", [1023, 1024, 1025, 2049])
def test_lengths_around_the_tile(emu, monkeypatch, n):
    """Light curves of BLS_TILE +- 1 and 2 tiles + 1 cadences on the cadence path (tile staging, the last partial warp
    of a tile) and on the boundary path."""
    rng = np.random.default_rng(n)
    t = C.dyadic_times(rng, n, 40.0)
    y = C.dyadic_flux(rng, t, 2.75)
    dy = C.pow2_errors(rng, n)
    grid = np.linspace(0.5, 6.0, 9)
    for path in ("cadence", "boundary"):
        set_env(monkeypatch, path, "smem")
        res, cnt = emu_power(emu, [t], [y], [dy], grid, C.DUR, 10)
        ties = check_all(res, [t], [y], [dy], grid, C.DUR, 10, "likelihood", "n=%d" % n)
        report("n=%d %s" % (n, path), cnt, ties)
        assert cnt[path] == len(grid)


def test_oversample_above_32_and_periods_on_bin_edges(emu, monkeypatch):
    """oversample 33, 40 and 64 (the wrap-pad loop takes a second lane pass) and periods that are exact multiples
    of the bin width, on data whose cadences are also multiples of it."""
    rng = np.random.default_rng(5)
    t = C.T0 + np.sort(rng.choice(6 * 1024, 700, replace=False)) / 1024.0
    y = C.dyadic_flux(rng, t, 1.25)
    for oversample in (33, 40, 64):
        grid = np.concatenate([C.bin_multiple_periods(oversample), [0.75, 1.5, 2.5]])
        for path in ("cadence", "boundary"):
            set_env(monkeypatch, path, "global")
            res, cnt = emu_power(emu, [t], [y], None, grid, C.DUR, oversample)
            ties = check_all(res, [t], [y], None, grid, C.DUR, oversample, "likelihood", "os>32")
            report("oversample=%d %s, periods on bin multiples" % (oversample, path), cnt, ties)
            assert cnt["ghist"] == len(grid)


def test_boundary_gate_k1_32_33_34(emu, monkeypatch):
    """Dense data whose K1 + 1 = ceil(P / bin) + 1 is 32, 33 and 34: the boundary path is refused at 32 and taken
    from 33 on (LKB_BLS_MIN_DENSITY=0), and every side equals the C code."""
    t = C.T0 + np.arange(2000) / 256.0                               # 5.6-min cadence, 7.8 d
    rng = np.random.default_rng(6)
    y = C.dyadic_flux(rng, t, 0.40625, duration=0.0625)
    set_env(monkeypatch, "boundary", "smem")
    for oversample in (2, 10):
        bd = C.DUR.min() / oversample
        for k1p1, path in ((32, "cadence"), (33, "boundary"), (34, "boundary")):
            per = (k1p1 - 1.5) * bd                                  # ceil(per / bd) = k1p1 - 1
            dur = [d for d in C.DUR if d < per] or [C.DUR.min()]
            grid = np.array([per])
            res, cnt = emu_power(emu, [t], [y], None, grid, dur, oversample)
            ties = check_all(res, [t], [y], None, grid, dur, oversample, "likelihood", "gate")
            report("K1+1=%d oversample=%d" % (k1p1, oversample), cnt, ties)
            assert cnt[path] == 1, (k1p1, cnt)


def test_cadences_on_bin_edges(emu, monkeypatch):
    """The t_adv construction of test_bls_dense_sampling_boundary_path: cadences every quarter bin, so whole families
    of them sit on bin edges; the cadence path takes the slow division and the boundary path the exact walk."""
    bd = 0.005
    t_adv = 1325.0 + np.arange(3000) * (bd / 4)
    rng = np.random.default_rng(7)
    y = rng.integers(-6, 7, len(t_adv)) / 64.0
    duration = np.array([0.05, 0.1])
    grid = np.array([0.3314, 0.335 + 1e-13, 0.5, 1.0, 0.4 + bd / 3, 2.5])
    seen = {}
    for path in ("cadence", "boundary"):
        set_env(monkeypatch, path, "smem")
        res, cnt = emu_power(emu, [t_adv], [y], None, grid, duration, 10)
        # t_adv is not dyadic (0.005 / 4): the sums are not exact, so the values are held to the oracle's rounding
        # (the order differs) and the bins to the oracle's except at its own mathematical ties
        ref = obls.bls_power_c(t_adv, y, None, grid, duration, oversample=10, return_bins=True)
        same = np.all(res[0]["bins"] == ref["bins"], axis=1)
        for p in np.flatnonzero(~same):
            n, d = res[0]["bins"][p]
            o = obls.objective_at(t_adv, y, None, grid[p], duration, int(n), int(d))
            assert abs(o - ref["power"][p]) <= 1e-10 * abs(ref["power"][p])
        for k in ("power", "depth", "depth_err", "depth_snr", "log_likelihood"):
            np.testing.assert_allclose(res[0][k], ref[k], rtol=1e-10, atol=1e-14, err_msg=k)
        report("cadences on bin edges, %s (tie-broken periods %d)" % (path, (~same).sum()), cnt)
        seen[path] = cnt
    assert seen["cadence"]["slow_div"] > 0
    assert seen["boundary"]["exact_walk"] > 0
    # and the index rule itself, bitwise
    tr = t_adv - t_adv.min()
    for per in grid:
        got = np.zeros(len(tr), dtype=np.int32)
        assert emu.emu_bls_bin_index(_p(tr), len(tr), 0.0, per, bd, _p(got)) == 0
        np.testing.assert_array_equal(got, obls.bin_index_c(tr, 0.0, per, bd))


def test_three_or_more_wraps_per_warp(emu, monkeypatch):
    """Sparse data at short periods: a warp's 32 cadences cross two or more period wraps (npieces > 2)."""
    rng = np.random.default_rng(8)
    t = C.dyadic_times(rng, 300, 60.0)
    y = C.dyadic_flux(rng, t, 0.875, duration=0.0625)
    grid = np.linspace(0.3, 0.9, 12)
    set_env(monkeypatch, "auto", "smem")
    for oversample in (3, 40):
        res, cnt = emu_power(emu, [t], [y], None, grid, C.DUR, oversample, "snr")
        ties = check_all(res, [t], [y], None, grid, C.DUR, oversample, "snr", "wraps")
        report("wraps, oversample=%d" % oversample, cnt, ties)
        assert cnt["wrap3"] > 0 and cnt["cadence"] == len(grid)


def test_table_groups(emu, monkeypatch):
    """Per-light-curve grids with a table budget small enough that the boundary-path tables form several groups:
    every light curve still equals the C code and its own one-light-curve call."""
    cases = C.matrix_batch(seed=3)
    names, ts, ys, dys = zip(*cases)
    grids = [C.matrix_grid(8, 0.5 + 0.1 * b, 3.0) for b in range(len(ts))]
    set_env(monkeypatch, "boundary", "smem")
    l0 = emu.emu_launches()
    emu_power(emu, list(ts), list(ys), list(dys), grids, C.DUR, 3)
    one_group = emu.emu_launches() - l0
    emu.emu_bls_set_table_budget(8000)     # each light curve's table has ~6 000 entries: one group per light curve
    try:
        l0 = emu.emu_launches()
        res, cnt = emu_power(emu, list(ts), list(ys), list(dys), grids, C.DUR, 3)
        launches = emu.emu_launches() - l0
        ties = check_all(res, ts, ys, dys, grids, C.DUR, 3, "likelihood", "table groups")
        report("table groups (%d launch checks)" % launches, cnt, ties)
        assert cnt["boundary"] > 0
        for b in range(len(ts)):
            one, _ = emu_power(emu, [ts[b]], [ys[b]], [dys[b]], [grids[b]], C.DUR, 3)
            for k in C.FIELDS + ("bins",):
                np.testing.assert_array_equal(C.bits(res[b][k]), C.bits(one[0][k]), err_msg="%s %s" % (names[b], k))
    finally:
        emu.emu_bls_set_table_budget(1 << 28)
    # one launch check per table group's searches (plus the prologue and the first tables): three groups or more
    assert launches - one_group >= 2, (launches, one_group)


def test_batch_and_permutation_invariance(emu, monkeypatch):
    """Each light curve's batched result is bitwise its one-light-curve result and its result in a permuted batch,
    on a shared grid and on per-light-curve grids."""
    set_env(monkeypatch, "auto", "smem")
    cases = C.matrix_batch(seed=4)
    names, ts, ys, dys = zip(*cases)
    ts, ys, dys = list(ts), list(ys), list(dys)
    ts.insert(2, np.zeros(0)); ys.insert(2, np.zeros(0)); dys.insert(2, None)
    grid = C.matrix_grid(12)
    grids = [grid[b % 2::1 + b % 3] for b in range(len(ts))]
    perm = np.random.default_rng(0).permutation(len(ts))
    for g in (grid, grids):
        full, _ = emu_power(emu, ts, ys, dys, g, C.DUR, 2)
        pg = [g[i] for i in perm] if isinstance(g, list) else g
        permuted, _ = emu_power(emu, [ts[i] for i in perm], [ys[i] for i in perm], [dys[i] for i in perm], pg, C.DUR, 2)
        for b in range(len(ts)):
            gb = [g[b]] if isinstance(g, list) else g
            one, _ = emu_power(emu, [ts[b]], [ys[b]], [dys[b]], gb, C.DUR, 2)
            j = int(np.flatnonzero(perm == b)[0])
            for k in C.FIELDS + ("bins",):
                np.testing.assert_array_equal(C.bits(full[b][k]), C.bits(one[0][k]), err_msg="batch %d %s" % (b, k))
                np.testing.assert_array_equal(C.bits(permuted[j][k]), C.bits(one[0][k]), err_msg="perm %d %s" % (b, k))
