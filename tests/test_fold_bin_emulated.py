"""K13 (fold_kernel and bin_kernel of lightkurve_b200/csrc/foldbin.cuh) executed on the CPU through
tests/native/cuda_emu.h, against the single-curve methods LightCurve.fold and LightCurve.bin:
  fold   the permutation equals np.argsort(rel, kind="stable") and the phases are bitwise those of LightCurve.fold, on
         unsorted and duplicate times, a period that divides the cadence step (many equal phases), wrap_phase 0 and P
         (where numpy's remainder gives +0.0 for an exact multiple and plain fmod gives -0.0), normalize_phase,
         negative and fractional epoch phases, NaN and inf times, and lengths 0, 1, 2 and either side of the
         shared-memory cap (given to the driver, so that both placements run)
  bin    every mode of LightCurve.bin (time_bin_size, n_bins with empty trailing bins, time_bin_start before the first
         cadence and time_bin_end, bins=int, bins=<indices>, binsize) on unsorted times, cadences on an interior edge
         and on the closed last edge, NaN and inf flux, all-NaN and partly finite errors, bins of one cadence, and
         nanmedian with odd and even counts: the bin centres are bitwise equal, the counts and the NaN pattern exact,
         the medians ==, and the means and errors within n 2^-52 mean|x| of the loop (n the bin's count)
and bitwise independence of a light curve's outputs from its neighbours, its position and where it sorts."""
import ctypes
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lightkurve_b200 import LightCurve  # noqa: E402
from lightkurve_b200.lightcurve import _bin_edges, _fold_params  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
CUDA_INC = "/usr/local/cuda/include"
c_vp, c_int, c_i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64
EPS = 2.0 ** -52


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    out = str(tmp_path_factory.mktemp("emu") / "libfold_bin_emu.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-pthread", "-I" + CUDA_INC,
                           "-Wno-attributes", "-shared", "-fPIC", "-Wl,-Bsymbolic", "-o", out,
                           os.path.join(HERE, "native", "fold_bin_emu_driver.cpp")])
    lib = ctypes.CDLL(out)
    lib.emu_fold.argtypes = [c_vp, c_vp, c_int, c_vp, c_int, c_vp, c_vp, c_i64]
    lib.emu_fold.restype = c_int
    lib.emu_bin.argtypes = [c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp,
                            c_vp, c_i64]
    lib.emu_bin.restype = c_int
    return lib


def _csr(arrays, dtype=np.float64):
    off = np.zeros(len(arrays) + 1, np.int64)
    off[1:] = np.cumsum([len(a) for a in arrays])
    cat = np.concatenate([np.asarray(a, dtype) for a in arrays]) if len(arrays) else np.zeros(0, dtype)
    return np.ascontiguousarray(cat, dtype), off


def _p(x):
    return None if x is None else x.ctypes.data


# ------------------------------------------------------------------------------------------------------------ fold
def run_fold(emu, times, pars, normalize, res_cap=-1):
    """(phases, perms, sorted in global memory) of one emulated launch; pars: (t0, shift, period, wrap) per curve."""
    t, off = _csr(times)
    par = np.ascontiguousarray(np.asarray(pars, np.float64).reshape(-1))
    n = max(int(off[-1]), 1)
    phase, perm = np.full(n, -7.0), np.full(n, -7, np.int32)
    g = emu.emu_fold(_p(t), _p(off), len(times), _p(par), int(normalize), _p(phase), _p(perm), int(res_cap))
    return ([phase[off[b]:off[b + 1]] for b in range(len(times))], [perm[off[b]:off[b + 1]] for b in range(len(times))],
            bool(g))


def _fold_cases():
    rng = np.random.default_rng(13)
    base = 1000.0 + np.arange(300) * 0.0208333
    cases = [("unsorted", rng.permutation(base + rng.normal(0, 1e-3, 300)), dict(period=0.731)),
             ("unsorted_epoch", rng.permutation(base), dict(period=1.37, epoch_time=1000.2)),
             ("duplicates_step_multiple", np.repeat(np.arange(40) * 0.5, 3), dict(period=0.25)),
             ("duplicates_wrap_P", np.repeat(np.arange(40) * 0.5, 3), dict(period=0.25, wrap_phase=0.25)),
             ("duplicates_wrap_0", np.repeat(np.arange(40) * 0.5, 3), dict(period=0.25, wrap_phase=0.0)),
             ("negative_multiples_wrap_P", np.arange(-20, 20) * 0.75, dict(period=0.75, epoch_time=0.0,
                                                                          wrap_phase=0.75)),
             ("normalize", base, dict(period=0.9, normalize_phase=True)),
             ("normalize_wrap_1", base, dict(period=0.5, normalize_phase=True, wrap_phase=1.0)),
             ("normalize_wrap_0", base, dict(period=0.5, normalize_phase=True, wrap_phase=0.0)),
             ("negative_epoch_phase", base, dict(period=1.1, epoch_phase=-0.37)),
             ("fractional_epoch_phase_normalized", base, dict(period=1.1, epoch_phase=2.61, normalize_phase=True)),
             ("nan_inf", np.r_[base[:50], np.nan, np.inf, -np.inf, base[50:60], np.nan], dict(period=0.3,
                                                                                             epoch_time=1000.0)),
             ("length_0", np.zeros(0), dict(period=0.3, epoch_time=1.0)),
             ("length_1", np.array([5.0]), dict(period=0.3)),
             ("length_2", np.array([5.3, 5.0]), dict(period=0.3))]
    for n in (63, 64, 65):
        cases.append(("cap_%d" % n, rng.permutation(base[:n]), dict(period=0.173)))
    return cases


FOLD_CASES = _fold_cases()


def _fold_ref(t, kw):
    """(phase, order, pars) of LightCurve.fold; the flux is the cadence index, so the folded flux is the order."""
    lc = LightCurve(time=t, flux=np.arange(len(t), dtype=float))
    kw = dict(kw)
    kw.setdefault("epoch_time", None)
    folded = lc.fold(**kw)
    per, t0, shift, wrap, _ = _fold_params(np.asarray(t, np.float64), lc.time, kw["period"], kw["epoch_time"],
                                           kw.get("epoch_phase", 0), kw.get("wrap_phase"), kw.get("normalize_phase",
                                                                                                 False))
    return np.asarray(folded.time.value), np.asarray(folded.flux.value).astype(np.int64), (t0, shift, per, wrap)


def _bits(x):
    return np.asarray(x, np.float64).view(np.int64)


@pytest.mark.parametrize("res_cap", [-1, 64], ids=["shared", "cap64"])
def test_fold_matches_single_method(emu, res_cap):
    times = [c[1] for c in FOLD_CASES]
    refs = [_fold_ref(t, c[2]) for t, c in zip(times, FOLD_CASES)]
    # one launch per normalize setting, every case of that setting batched
    for norm in (False, True):
        sel = [i for i, c in enumerate(FOLD_CASES) if bool(c[2].get("normalize_phase", False)) == norm]
        ph, pm, g = run_fold(emu, [times[i] for i in sel], [refs[i][2] for i in sel], norm, res_cap)
        assert g == (res_cap == 64)
        for k, i in enumerate(sel):
            name, t, _ = FOLD_CASES[i]
            assert np.array_equal(pm[k], refs[i][1]), name
            assert np.array_equal(_bits(ph[k]), _bits(refs[i][0])), name
    wrapP = FOLD_CASES[[c[0] for c in FOLD_CASES].index("negative_multiples_wrap_P")]
    ph = _fold_ref(wrapP[1], wrapP[2])[0]
    assert np.count_nonzero(ph == 0) >= 10 and not np.any(np.signbit(ph[ph == 0]))   # all +0.0, as numpy gives


def test_fold_either_side_of_the_library_cap(emu):
    rng = np.random.default_rng(3)
    cap = emu.emu_fold_cap()
    times = [rng.permutation(np.arange(n) * 0.0013888) for n in (cap, cap + 1)]
    pars = [_fold_ref(t, dict(period=0.61))[2] for t in times]
    ph, pm, g = run_fold(emu, times, pars, False)
    assert g
    for t, p, m in zip(times, ph, pm):
        phase, order, _ = _fold_ref(t, dict(period=0.61))
        assert np.array_equal(m, order) and np.array_equal(_bits(p), _bits(phase))


# ------------------------------------------------------------------------------------------------------------- bin
def run_bin(emu, times, fluxes, errs, edges, agg, res_cap=-1):
    """dict(time, flux, flux_err, count, status, streamed) of one emulated launch; edges: (kind, starts, ends) each."""
    t, off = _csr(times)
    f, _ = _csr(fluxes)
    fe = None if errs is None else _csr(errs)[0]
    index = edges[0][0] == "index" if edges else False
    dt = np.int32 if index else np.float64
    s, boff = _csr([e[1] for e in edges], dt)
    e, _ = _csr([e[2] for e in edges], dt)
    nb = max(int(boff[-1]), 1)
    centre, flux, err = np.full(nb, -7.0), np.full(nb, -7.0), np.full(nb, -7.0)
    count, status = np.full(nb, -7, np.int32), np.full(len(times), -7, np.int32)
    g = emu.emu_bin(_p(t), _p(f), _p(fe), _p(off), len(times), _p(boff), None if index else _p(s),
                    None if index else _p(e), _p(s) if index else None, _p(e) if index else None,
                    1 if agg is np.nanmedian else 0, _p(centre), _p(flux), _p(err), _p(count), _p(status),
                    int(res_cap))
    sl = [slice(boff[b], boff[b + 1]) for b in range(len(times))]
    return dict(time=[centre[x] for x in sl], flux=[flux[x] for x in sl], flux_err=[err[x] for x in sl],
                count=[count[x] for x in sl], status=status, streamed=bool(g))


def _edges(t, kw):
    ts = np.sort(np.asarray(t, np.float64), kind="stable")
    return _bin_edges(len(ts), ts[0], ts[-1], kw.get("time_bin_size"), kw.get("time_bin_start"),
                      kw.get("time_bin_end"), kw.get("n_bins"), kw.get("bins"), kw.get("binsize"))


def _bin_ref(t, f, fe, kw, agg):
    """(binned light curve, counts, per-bin flux values, per-bin error values) of LightCurve.bin."""
    lc = LightCurve(time=t, flux=f, flux_err=fe)
    out = lc.bin(aggregate_func=agg, **kw)
    kind, starts, ends = _edges(t, kw)
    order = np.argsort(t, kind="stable")
    ts, fs = np.asarray(t, np.float64)[order], np.asarray(f, np.float64)[order]
    es = np.asarray(lc.flux_err.value, np.float64)[order]
    if kind == "index":
        starts, ends = ts[starts], ts[ends]
    nb = len(starts)
    which = np.searchsorted(starts, ts, side="right") - 1
    inside = (which >= 0) & ((ts < ends[np.clip(which, 0, nb - 1)]) | ((which == nb - 1) & (ts <= ends[-1])))
    counts = np.bincount(which[inside], minlength=nb)
    return out, counts, [fs[inside & (which == j)] for j in range(nb)], [es[inside & (which == j)] for j in range(nb)]


def _check_bin(name, got, b, ref):
    out, counts, fvals, evals = ref
    assert np.array_equal(_bits(got["time"][b]), _bits(out.time.value)), name
    assert np.array_equal(got["count"][b], counts), name
    for key, want in (("flux", np.asarray(out.flux.value)), ("flux_err", np.asarray(out.flux_err.value))):
        have = got[key][b]
        assert np.array_equal(np.isnan(have), np.isnan(want)), (name, key)
        for j in np.nonzero(~np.isnan(want))[0]:
            x = fvals[j] if key == "flux" or not np.any(np.isfinite(evals[j])) else evals[j]   # errors or nanstd
            x = x[np.isfinite(x)]
            scale = np.mean(np.abs(x)) if len(x) else 0.0
            tol = 4 * counts[j] * EPS * scale
            assert have[j] == want[j] or abs(have[j] - want[j]) <= tol, (name, key, j, have[j], want[j], tol)


def _bin_inputs():
    rng = np.random.default_rng(21)
    n = 700
    t = rng.permutation(np.arange(n) * 0.02)                              # unsorted; 0.02 * k lands on edges
    f = 1 + 1e-3 * rng.standard_normal(n)
    f[rng.choice(n, 25, replace=False)] = np.nan
    f[rng.choice(n, 3, replace=False)] = np.inf
    fe = np.full(n, 2e-4)
    fe[rng.choice(n, 60, replace=False)] = np.nan
    fe[rng.choice(n, 2, replace=False)] = np.inf
    t2 = np.repeat(np.arange(90) * 0.1, 2)                               # duplicates, many cadences on edges
    f2 = rng.standard_normal(len(t2))
    inputs = [("unsorted_nan_inf_errors", t, f, fe),
              ("all_nan_errors", t, f, np.full(n, np.nan)),
              ("duplicates_on_edges", t2, f2, np.full(len(t2), np.nan)),
              ("all_nan_flux_bins", t, np.where(t < 3.0, np.nan, f), fe),
              ("one_cadence", np.array([4.0]), np.array([2.0]), np.array([0.1])),
              ("two_cadences", np.array([4.5, 4.0]), np.array([2.0, 3.0]), np.array([np.nan, np.nan]))]
    return inputs


BIN_MODES = [("time_bin_size", dict(time_bin_size=0.13)),
             ("time_bin_size_edges", dict(time_bin_size=0.1)),
             ("default_size", dict()),
             ("n_bins_trailing_empty", dict(time_bin_size=0.2, n_bins=200)),
             ("start_before_first_and_end", dict(time_bin_size=0.3, time_bin_start=-1.05, time_bin_end=9.0)),
             ("bins_int", dict(bins=37)),
             ("bins_int_1", dict(bins=1)),
             ("bins_indices", dict(bins=[0, 3, 4, 5, 50, -1])),
             ("binsize", dict(binsize=7)),
             ("binsize_1", dict(binsize=1))]


@pytest.mark.parametrize("agg", [np.nanmean, np.nanmedian], ids=["nanmean", "nanmedian"])
@pytest.mark.parametrize("mode", BIN_MODES, ids=[m[0] for m in BIN_MODES])
def test_bin_matches_single_method(emu, mode, agg):
    name, kw = mode
    inputs = [x for x in _bin_inputs() if not (x[0] in ("one_cadence", "two_cadences") and "bins" in kw
                                                  and np.size(kw["bins"]) > 1)]
    edges = [_edges(x[1], kw) for x in inputs]
    refs = [_bin_ref(x[1], x[2], x[3], kw, agg) for x in inputs]
    for res_cap in (-1, 100):
        got = run_bin(emu, [x[1] for x in inputs], [x[2] for x in inputs], [x[3] for x in inputs], edges, agg,
                      res_cap)
        assert np.all(got["status"] == 0)
        assert got["streamed"] == (res_cap == 100)
        for b, x in enumerate(inputs):
            _check_bin("%s/%s" % (name, x[0]), got, b, refs[b])


def test_bin_cases_reach_their_edges(emu):
    """The inputs hold what the docstring lists: cadences on an interior and on the closed last edge, bins of one
    cadence, empty trailing bins and nanmedians of odd and even counts."""
    t2 = _bin_inputs()[2][1]
    _, counts, fv, _ = _bin_ref(t2, np.ones(len(t2)), np.ones(len(t2)), dict(time_bin_size=0.1), np.nanmedian)
    assert np.all(counts[:-1] == 2) and counts[-1] == 4    # pairs on interior edges; the closed last edge takes two
    t = _bin_inputs()[0][1]
    _, counts, fv, _ = _bin_ref(t, np.ones(len(t)), np.ones(len(t)), dict(binsize=1), np.nanmedian)
    assert np.any(counts == 1)
    _, counts, _, _ = _bin_ref(t, np.ones(len(t)), np.ones(len(t)), dict(time_bin_size=0.2, n_bins=200),
                               np.nanmedian)
    assert counts[-1] == 0 and counts[0] > 0
    _, _, fv, _ = _bin_ref(*_bin_inputs()[0][1:], dict(time_bin_size=0.13), np.nanmedian)
    nn = [np.count_nonzero(~np.isnan(v)) for v in fv]
    assert any(c % 2 for c in nn) and any(c and not c % 2 for c in nn)


def test_bin_rejects_bad_edges(emu):
    t = np.arange(10.0)
    f = np.ones(10)
    got = run_bin(emu, [t, t, t], [f, f, f], None,
                  [("index", np.array([0, 5]), np.array([5, 9])), ("index", np.array([0, 5]), np.array([5, 10])),
                   ("index", np.array([5, 2]), np.array([2, 9]))], np.nanmean)
    assert list(got["status"]) == [0, 2, 1]
    got = run_bin(emu, [t, t], [f, f], None, [("time", np.array([0.0, np.nan]), np.array([1.0, 2.0])),
                                              ("time", np.array([np.nan, 0.0]), np.array([1.0, 2.0]))], np.nanmean)
    assert list(got["status"]) == [0, 1]


# ------------------------------------------------------------------------------------------------------ invariance
def _same(a, b, i, j):
    for k in ("time", "flux", "flux_err"):
        assert np.array_equal(_bits(a[k][i]), _bits(b[k][j])), k
    assert np.array_equal(a["count"][i], b["count"][j])


@pytest.mark.parametrize("agg", [np.nanmean, np.nanmedian], ids=["nanmean", "nanmedian"])
def test_batch_position_neighbours_and_memory(emu, agg):
    """Each light curve's outputs are bitwise those of its own launch, in any order, with any neighbours, whether it
    sorts in shared memory or in global memory (res_cap 0: all in global memory)."""
    inputs = _bin_inputs()
    kw = dict(time_bin_size=0.13)
    edges = [_edges(x[1], kw) for x in inputs]
    args = ([x[1] for x in inputs], [x[2] for x in inputs], [x[3] for x in inputs])
    base = run_bin(emu, *args, edges, agg)
    perm = np.random.default_rng(5).permutation(len(inputs))
    shuffled = run_bin(emu, *[[a[p] for p in perm] for a in args], [edges[p] for p in perm], agg)
    glob = run_bin(emu, *args, edges, agg, res_cap=0)
    assert glob["streamed"]
    for j, p in enumerate(perm):
        _same(base, shuffled, p, j)
    for i in range(len(inputs)):
        _same(base, glob, i, i)
    for i in (0, 3, len(inputs) - 1):
        _same(base, run_bin(emu, [args[0][i]], [args[1][i]], [args[2][i]], [edges[i]], agg), i, 0)

    times = [c[1] for c in FOLD_CASES if not c[2].get("normalize_phase")]
    pars = [_fold_ref(c[1], c[2])[2] for c in FOLD_CASES if not c[2].get("normalize_phase")]
    fb = run_fold(emu, times, pars, False)
    fg = run_fold(emu, times, pars, False, res_cap=0)
    fr = run_fold(emu, times[::-1], pars[::-1], False)
    for i in range(len(times)):
        assert np.array_equal(_bits(fb[0][i]), _bits(fg[0][i])) and np.array_equal(fb[1][i], fg[1][i])
        k = len(times) - 1 - i
        assert np.array_equal(_bits(fb[0][i]), _bits(fr[0][k])) and np.array_equal(fb[1][i], fr[1][k])
