"""K3 Box Least Squares on the H100 on every kernel path and at every oversample, against the C restatement of
astropy's bls.c (oracle/bls_c.c), and against the same translation unit run on the CPU emulator.

* Exact-arithmetic fixtures (tests/_bls_cases.py, every sum exact in fp64): bins and all seven outputs bitwise equal to
  bls_power_c, ties included, on the oversample x objective x path x histogram matrix and the edges of
  tests/test_bls_emulated.py at GPU sizes.
* An oversample sweep {1, 2, 3, 5, 10, 20, 40} x both objectives on the dense fixture of
  test_gpu_engine.py::test_bls_dense_sampling_boundary_path, a sparse 30-min light curve and a 4-year Kepler
  long-cadence light curve (periods to 700 d: global histograms and long boundary walks), held to assert_bls_close;
  the tie-broken count of every case is printed.
* Where g++ and the CUDA headers exist, the emulator build of bls.cu: both sides are IEEE fp64 without contraction
  and sum in the same order, so the GPU must equal it bitwise, on dyadic and on non-dyadic data."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _bls_cases as C  # noqa: E402

from oracle import bls as obls  # noqa: E402

pytestmark = pytest.mark.gpu

OVERSAMPLES = (1, 2, 3, 10, 40)
PATH_ENV = {"cadence": "1e31", "boundary": "0", "auto": None}
# (a 16 MiB cap: the largest chunk of one light curve here needs 8 MiB, and the batch is then launched in groups)
HIST_ENV = {"smem": ("1000000000", None), "global": ("0", None), "global_tiny_cap": ("0", "16")}


def set_env(monkeypatch, path, hist):
    for k, v in (("LKB_BLS_MIN_DENSITY", PATH_ENV[path]), ("LKB_BLS_GHIST_BINS", HIST_ENV[hist][0]),
                 ("LKB_BLS_HIST_CAP_MB", HIST_ENV[hist][1])):
        if v is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, v)


def gpu_power(engine, ts, ys, dys, period, duration, oversample, objective="likelihood"):
    """engine.bls_power as a list of per-light-curve result dicts (shared grid or per-light-curve grids)."""
    dys = None if dys is None or all(d is None for d in dys) else [np.ones(len(t)) if d is None else d
                                                                    for t, d in zip(ts, dys)]
    r = engine.bls_power(list(ts), list(ys), dys, period, duration, oversample=oversample, objective=objective,
                         return_bins=True)
    return [{k: r[k][b] for k in C.FIELDS + ("bins",)} for b in range(len(ts))]


def check_exact(res, ts, ys, dys, grids, duration, oversample, objective, label, count_ties=True):
    tied = 0
    for b, (t, y) in enumerate(zip(ts, ys)):
        g = grids[b] if isinstance(grids, list) else grids
        if len(t) == 0:
            assert np.all(np.isnan(res[b]["power"])) and np.all(res[b]["bins"] == -1)
            continue
        tied += C.assert_exact(res[b], t, y, None if dys is None else dys[b], g, duration, oversample, objective,
                               "%s lc %d" % (label, b), count_ties)[0]
    if count_ties:
        print("%s: exact ties checked bitwise in %d periods" % (label, tied))
    return tied


@pytest.mark.parametrize("objective", ["likelihood", "snr"])
@pytest.mark.parametrize("path", list(PATH_ENV))
@pytest.mark.parametrize("oversample", OVERSAMPLES)
def test_matrix_bitwise(engine, monkeypatch, oversample, path, objective):
    """Every histogram placement and both grid layouts for each (oversample, path, objective), at 4x the emulator's
    cadence counts and spans."""
    cases = C.matrix_batch(scale=4, seed=10)
    names, ts, ys, dys = zip(*cases)
    grid = C.matrix_grid(300, 0.4, 12.0)
    for hist in HIST_ENV:
        set_env(monkeypatch, path, hist)
        for csr in (False, True):
            grids = [grid[b % 3::1 + b % 2] for b in range(len(ts))] if csr else grid
            res = gpu_power(engine, ts, ys, dys, grids, C.DUR, oversample, objective)
            first = hist == "smem" and not csr          # the ties are those of the inputs: counted once
            tied = check_exact(res, ts, ys, dys, grids, C.DUR, oversample, objective,
                               "oversample=%d %s %s %s %s" % (oversample, objective, path, hist, "csr" if csr else "shared"),
                               count_ties=first)
            assert tied > 0 or not first


def test_edges_bitwise(engine, monkeypatch):
    """No box qualifies (one, two, all-equal cadences), an empty light curve inside the batch, lengths around
    BLS_TILE, unsorted times, oversample > 32 with periods on bin multiples, and the K1 + 1 = 32 / 33 / 34 gate."""
    rng = np.random.default_rng(20)
    ts = [np.array([C.T0 + 0.5]), C.T0 + np.array([0.25, 3.0]), np.zeros(0), np.full(40, C.T0 + 2.0)]
    ys = [np.array([3 / 64.0]), np.array([1 / 64.0, -2 / 64.0]), np.zeros(0), rng.integers(-4, 5, 40) / 64.0]
    for n in (1023, 1024, 1025, 2049, 4097):
        t = C.dyadic_times(rng, n, 40.0)
        ts.append(t)
        ys.append(C.dyadic_flux(rng, t, 2.75))
    ts.append(rng.permutation(ts[-1]))
    ys.append(C.dyadic_flux(rng, ts[-1], 1.5))
    dys = [None if b % 2 else C.pow2_errors(rng, len(t)) for b, t in enumerate(ts)]
    for path in ("cadence", "boundary", "auto"):
        for hist in ("smem", "global"):
            set_env(monkeypatch, path, hist)
            for oversample in (1, 10, 33, 64):
                grid = np.concatenate([np.linspace(0.5, 6.0, 40), C.bin_multiple_periods(oversample)])
                res = gpu_power(engine, ts, ys, dys, grid, C.DUR, oversample)
                check_exact(res, ts, ys, dys, grid, C.DUR, oversample, "likelihood",
                            "edges %s %s oversample=%d" % (path, hist, oversample))
                for b in (0, 3):                     # one cadence; all cadences at one time
                    assert np.all(res[b]["power"] == -np.inf)
    # both sides of the boundary gate, forced on
    set_env(monkeypatch, "boundary", "smem")
    t = C.T0 + np.arange(8000) / 256.0
    y = C.dyadic_flux(rng, t, 0.40625, duration=0.0625)
    for oversample in (2, 10):
        bd = C.DUR.min() / oversample
        for k1p1 in (32, 33, 34):
            per = np.array([(k1p1 - 1.5) * bd])
            dur = [d for d in C.DUR if d < per[0]] or [C.DUR.min()]
            res = gpu_power(engine, [t], [y], None, per, dur, oversample)
            check_exact(res, [t], [y], None, per, dur, oversample, "likelihood", "gate K1+1=%d" % k1p1)


# ---- the oversample sweep on non-dyadic light curves ---------------------------------------------------------------
def dense_fixture():
    """test_gpu_engine.py::test_bls_dense_sampling_boundary_path's light curves and periods."""
    rng = np.random.default_rng(35)
    lcs, dys = [], []
    for n_keep, p_true in ((9000, 2.17), (7000, 0.9), (3000, 4.4)):
        grid = 1325.0 + np.arange(10000) / 720.0
        grid = np.concatenate([grid[:4200], grid[4900:]])
        keep = np.sort(rng.choice(len(grid), n_keep, replace=False))
        t = grid[keep] + rng.uniform(-2e-4, 2e-4, n_keep)
        t.sort()
        y = 1 + 5e-4 * rng.normal(size=n_keep)
        y[np.abs((t - 1326.0 + 0.5 * p_true) % p_true - 0.5 * p_true) < 0.06] -= 3e-3
        lcs.append((t, y))
        dys.append(5e-4 * rng.uniform(0.8, 1.2, n_keep))
    t_adv = 1325.0 + np.arange(9000) * (0.005 / 4)
    lcs.append((t_adv, 1 + 5e-4 * rng.normal(size=len(t_adv))))
    dys.append(np.full(len(t_adv), 5e-4))
    duration = np.linspace(0.05, 0.33, 10)
    period = np.concatenate([obls.autoperiod(lcs[0][0], duration, 0.3314, 9.26, frequency_factor=10),
                             [0.3314, 0.335 + 1e-13, 0.5, 1.0, 0.4 + 0.005 / 3, 2.5, 13.0]])
    return [l[0] for l in lcs], [l[1] for l in lcs], dys, period, duration, [0.02, 0.02, 0.02, 0.5]


def sparse_fixture():
    """30-min cadence with gaps and an injected transit, 80 d."""
    rng = np.random.default_rng(36)
    t = 2000.0 + np.arange(0, 80, 1.0 / 48)
    t = t[rng.random(len(t)) < 0.85]
    y = 1 + 4e-4 * rng.normal(size=len(t))
    y[np.abs((t - 2001.3 + 3.7) % 7.4 - 3.7) < 0.08] -= 2e-3
    dy = 4e-4 * rng.uniform(0.8, 1.2, len(t))
    duration = np.array([0.05, 0.1, 0.2, 0.3])
    period = obls.autoperiod(t, duration, 0.5, 30.0, frequency_factor=3)
    return [t], [y], [dy], period, duration, [0.02]


def kepler_fixture():
    """A 4-year Kepler long-cadence light curve: ~65 000 cadences over 1 470 d, periods to 700 d."""
    rng = np.random.default_rng(37)
    t = 120.5 + np.arange(0, 1470.0, 29.4244 / 1440)
    t = t[rng.random(len(t)) < 0.9]
    y = 1 + 1e-4 * rng.normal(size=len(t))
    y[np.abs((t - 170.2 + 0.5 * 289.9) % 289.9 - 0.5 * 289.9) < 0.2] -= 5e-4
    dy = 1e-4 * rng.uniform(0.9, 1.1, len(t))
    duration = np.array([0.1, 0.2, 0.4])
    period = np.geomspace(1.0, 700.0, 160)
    return [t], [y], [dy], period, duration, [0.02]


@pytest.mark.parametrize("objective", ["likelihood", "snr"])
@pytest.mark.parametrize("oversample", [1, 2, 3, 5, 10, 20, 40])
@pytest.mark.parametrize("fixture", ["dense", "sparse30", "kepler4yr"])
def test_oversample_sweep(engine, fixture, oversample, objective):
    ts, ys, dys, period, duration, tied_frac = {"dense": dense_fixture, "sparse30": sparse_fixture,
                                                "kepler4yr": kepler_fixture}[fixture]()
    res = gpu_power(engine, ts, ys, dys, period, duration, oversample, objective)
    broken = []
    for b, (t, y) in enumerate(zip(ts, ys)):
        ref = obls.bls_power_c(t, y, dys[b], period, duration, oversample=oversample, objective=objective,
                               return_bins=True)
        broken.append(C.assert_bls_close(res[b], ref, t, y, dys[b], period, duration, oversample, objective,
                                         max_tied_frac=tied_frac[b]))
    print("%s oversample=%d %s: tie-broken periods per light curve %s of %d" % (fixture, oversample, objective,
                                                                               broken, len(period)))


# ---- GPU == emulator ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    from test_bls_emulated import build_emulator
    lib = build_emulator(tmp_path_factory.mktemp("bls_emu_gpu"))
    if lib is None:
        pytest.skip("needs g++ and the CUDA headers")
    return lib


def test_gpu_equals_emulator_bitwise(engine, emu, monkeypatch):
    from test_bls_emulated import emu_power
    cases = C.matrix_batch(seed=30)
    names, ts, ys, dys = map(list, zip(*cases))
    rng = np.random.default_rng(31)
    t = np.sort(rng.uniform(1400.0, 1406.0, 900))                     # non-dyadic: sums round, in the same order
    ts.append(t)
    ys.append(1 + 1e-3 * rng.normal(size=len(t)))
    dys.append(1e-3 * rng.uniform(0.8, 1.2, len(t)))
    grid = C.matrix_grid(24)
    grids = [grid[b % 3::1 + b % 2] for b in range(len(ts))]
    for path, hist, oversample, objective in (("cadence", "smem", 10, "likelihood"), ("boundary", "global", 3, "snr"),
                                              ("auto", "global_tiny_cap", 40, "likelihood"),
                                              ("boundary", "smem", 1, "likelihood")):
        set_env(monkeypatch, path, hist)
        for g in (grid, grids):
            got = gpu_power(engine, ts, ys, dys, g, C.DUR, oversample, objective)
            ref, cnt = emu_power(emu, ts, ys, dys, g, C.DUR, oversample, objective)
            for b in range(len(ts)):
                for k in C.FIELDS + ("bins",):
                    np.testing.assert_array_equal(C.bits(got[b][k]), C.bits(ref[b][k]),
                                                  err_msg="%s %s %d lc %d %s" % (path, hist, oversample, b, k))
            print("GPU == emulator: %s %s oversample=%d %s, emulator paths %s" % (path, hist, oversample, objective, cnt))
