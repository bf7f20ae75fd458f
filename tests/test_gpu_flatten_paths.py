"""K4 (LightCurve.flatten: lkb_flatten) on every kernel path flatten.cu chooses, against oracle.detrend.flatten on
EVERY light curve of every batch.

Which path a call takes follows from the window, the polyorder and the longest light curve (flatten_plan.h, restated
once below as `plan`):
  "v2-moments"  streaming kernel (flatten_v2.cuh), interior from sliding moments: NM = 1 (polyorder 0-1) always;
                NM = 3 / 5 (polyorder 2-3 / 4-5) where the predicted rounding of the moments,
                eps T (T / 2 half)^(NM - 1) with T = tile_out + 2 half, is at most F2_MOMENT_TOL = 2e-10
  "v2-direct"   streaming kernel, interior from the direct dot product of the centre taps (the short windows)
  "v1"          FIR kernel (flatten.cu): polyorder > 5, a tile of fewer than 128 outputs (long windows), or some light
                curve longer than F2_MAXN = 131072 cadences (then the whole batch runs on v1)
  "v1-rerun"    FIR kernel after the streaming kernel found more than 1022 gap cuts in some light curve
engine.flatten_last_path() reports the path that ran, and every case asserts it.

Reference: the reference's flatten body (oracle/detrend.py) with savgol=savgol_lsq, the Savitzky-Golay filter from a
well-conditioned least-squares basis.  scipy.signal.savgol_filter builds its taps from the unscaled Vandermonde matrix
of the window offsets: at polyorder 5 its taps are off by 1e-8 relative at window 201 and 1e-6 at 1001, and at
polyorder 12 they are wrong altogether (tests/test_flatten_emulated.py pins savgol_lsq against exact rational taps and
against scipy where scipy is accurate).  Tolerance: trend, flat and flat_err to rtol 1e-9 on every path.

Left out: window = polyorder + 1.  There the filter is the identity, the residuals are rounding noise (~1e-16) and
the clip threshold is sigma * std + 1e-14, so which cadences the reference keeps is decided by rounding."""
import numpy as np
import pytest

from oracle import detrend as odet

pytestmark = pytest.mark.gpu

F2_MAXN = 131072
F2_MOMENT_TOL = 2e-10
RTOL = 1e-9
DT = 0.0204336


def plan(w, p, nmax):
    """flatten_plan.h: (route, NM, tile_out, direct); route "v2" or the reason for v1."""
    half = w // 2
    nm = 1 if p <= 1 else 3 if p <= 3 else 5
    tile = min(2048, 65536 // (8 * nm) - 2 * half - 1, 4094 - 2 * half)
    if nm == 5:
        tile = min(tile, max(128, 10 * half))
    route = "polyorder" if p > 5 else "tile" if tile < 128 else "length" if nmax > F2_MAXN else "v2"
    T = tile + 2.0 * half
    direct = nm > 1 and np.finfo(float).eps * T * (T / (2.0 * half)) ** (nm - 1) > F2_MOMENT_TOL
    return route, nm, tile, bool(direct)


def expected_path(w, p, nmax, overflow=False):
    route, _, _, direct = plan(w, p, nmax)
    if route != "v2":
        return "v1"
    if overflow:
        return "v1-rerun"
    return "v2-direct" if direct else "v2-moments"


def longest_v2_window(p):
    return max(w for w in range(3, 8192, 2) if plan(w, p, 1000)[0] == "v2")


# ---------------------------------------------------------------------------------------------------- light curves
def lc(rng, n, gaps=2, outliers=None, nans=0, eps=False, errs=True, jitter=0.0, t=None):
    """A Kepler-like light curve of n cadences: gaps, outliers, NaNs; flux normalised (~1, noise 3e-4) or in e-/s
    (1e5 offset, noise 30); flux_err per cadence or None."""
    if t is None:
        keep = np.ones(int(n * 1.3) + 200, bool)
        for _ in range(gaps):
            g0 = int(rng.integers(0, len(keep) - 60))
            keep[g0:g0 + int(rng.integers(8, 50))] = False
        t = 131.5 + np.flatnonzero(keep)[:n] * DT
        if jitter:
            t = t + rng.uniform(-jitter, jitter, n) * DT
    n = len(t)
    off, noise = (1e5, 30.0) if eps else (1.0, 3e-4)
    x = t - (t[0] if n else 0.0)
    f = off * (1 + 5e-3 * np.sin(2 * np.pi * x / 7.3) + 2e-3 * np.cos(2 * np.pi * x / 1.9)) + noise * rng.normal(size=n)
    k = min(n, max(1, n // 300)) if outliers is None else outliers
    if k:
        f[rng.choice(n, k, replace=False)] += 8 * noise * rng.choice([-1, 1], k)
    if nans:
        f[rng.choice(n, nans, replace=False)] = np.nan
    fe = noise * rng.uniform(0.8, 1.2, n) if errs else None
    return t, f, fe


def segments_lc(rng, lengths, gap=10):
    """Segments of the given numbers of cadences separated by gaps of `gap` cadence steps."""
    idx, start = [], 0
    for L in lengths:
        idx.append(start + np.arange(L))
        start += L + gap
    return lc(rng, 0, t=131.5 + np.concatenate(idx) * DT, outliers=0)


def check(engine, lcs, w, p, path, masks=None, bt=5, niters=3, sigma=3, nan_lcs=()):
    """Runs the batch, asserts the path, compares every light curve with the reference; the light curves in
    `nan_lcs` (fewer than two usable cadences: the reference's interp1d raises) must come back all NaN."""
    times = [l[0] for l in lcs]
    fluxes = [l[1] for l in lcs]
    errs = [l[2] for l in lcs]
    no_err = any(e is None for e in errs)
    flat, flat_err, trend = engine.flatten(times, fluxes, None if no_err else errs, masks, window_length=w,
                                           polyorder=p, break_tolerance=bt, niters=niters, sigma=sigma)
    assert engine.flatten_last_path() == path
    worst = 0.0
    for b in range(len(lcs)):
        if b in nan_lcs:
            assert np.isnan(trend[b]).all() and np.isnan(flat[b]).all() and np.isnan(flat_err[b]).all(), b
            continue
        if len(times[b]) == 0:
            assert len(trend[b]) == len(flat[b]) == len(flat_err[b]) == 0
            continue
        rf, rfe, rt = odet.flatten(times[b], fluxes[b], None if no_err else errs[b], window_length=w, polyorder=p,
                                   break_tolerance=bt, niters=niters, sigma=sigma,
                                   mask=None if masks is None else masks[b], savgol=odet.savgol_lsq)
        msg = "w=%d p=%d light curve %d (n=%d)" % (w, p, b, len(times[b]))
        np.testing.assert_allclose(trend[b], rt, rtol=RTOL, equal_nan=True, err_msg="trend " + msg)
        np.testing.assert_allclose(flat[b], rf, rtol=RTOL, equal_nan=True, err_msg="flat " + msg)
        np.testing.assert_allclose(flat_err[b], rfe, rtol=RTOL, equal_nan=True, err_msg="flat_err " + msg)
        if no_err:
            assert np.isnan(flat_err[b]).all()
        ok = np.isfinite(rt) & (rt != 0)
        if ok.any():
            worst = max(worst, float(np.max(np.abs(trend[b][ok] - rt[ok]) / np.abs(rt[ok]))))
    return worst


# ---------------------------------------------------------------------------------------------------- case table
WINDOWS = (3, 5, 7, 9, 11, 15, 21, 31, 51, 101, 201, 401, 1001)
SWEEP = [(w, p) for p in range(6) for w in WINDOWS + (longest_v2_window(p),) if w > p + 1]
SWEEP_N = (3000, 1200)
# (id, window, polyorder, longest light curve, expected path): the v2 / v1 edge of each NM, the largest window
EDGES = [
    ("nm1-last-v2", 3967, 1, 12000, "v2-moments"), ("nm1-first-v1", 3969, 1, 12000, "v1"),
    ("nm3-last-v2", 2601, 2, 8000, "v2-moments"), ("nm3-first-v1", 2603, 3, 8000, "v1"),
    ("nm5-last-v2", 1509, 5, 5000, "v2-moments"), ("nm5-first-v1", 1511, 4, 5000, "v1"),
    ("w8191", 8191, 2, 20000, "v1"),
]
HIGH_P = [(w, p) for p in range(6, 13) for w in (25, 51, 401) if w > p + 1]


def test_case_table_matches_the_selection_rules():
    for w, p in SWEEP:
        assert plan(w, p, max(SWEEP_N))[0] == "v2"
    for cid, w, p, n, path in EDGES:
        assert expected_path(w, p, n) == path, cid
    assert [longest_v2_window(p) for p in (0, 2, 4)] == [3967, 2601, 1509]
    for w, p in HIGH_P:
        assert plan(w, p, 3000)[0] == "polyorder"
    assert plan(101, 2, F2_MAXN) == ("v2", 3, 2048, True) and plan(101, 2, F2_MAXN + 1)[0] == "length"
    # the sweep reaches both interior methods of NM = 3 and 5, and the bench leg (401, 2) stays on moments at 2048
    paths = {(plan(w, p, 3000)[1], expected_path(w, p, 3000)) for w, p in SWEEP}
    assert {(3, "v2-direct"), (3, "v2-moments"), (5, "v2-direct"), (5, "v2-moments"), (1, "v2-moments")} <= paths
    assert plan(401, 2, 65000) == ("v2", 3, 2048, False)


@pytest.mark.parametrize("w,p", SWEEP, ids=["w%d-p%d" % c for c in SWEEP])
def test_window_polyorder_sweep(engine, w, p):
    rng = np.random.default_rng(1000 * p + w)
    lcs = [lc(rng, n) for n in SWEEP_N]
    check(engine, lcs, w, p, expected_path(w, p, max(SWEEP_N)))


@pytest.mark.parametrize("cid,w,p,n,path", EDGES, ids=[c[0] for c in EDGES])
def test_tile_edges_and_longest_window(engine, cid, w, p, n, path):
    rng = np.random.default_rng(w + p)
    check(engine, [lc(rng, n, eps=(p % 2 == 1)), lc(rng, n // 2 + 7)], w, p, path)


def test_window_above_8191_is_rejected(engine):
    rng = np.random.default_rng(3)
    t, f, fe = lc(rng, 20000)
    with pytest.raises(ValueError):
        engine.flatten([t], [f], [fe], None, window_length=8193, polyorder=2)


@pytest.mark.parametrize("w,p", HIGH_P, ids=["w%d-p%d" % c for c in HIGH_P])
def test_high_polyorder_on_v1(engine, w, p):
    rng = np.random.default_rng(50 * p + w)
    check(engine, [lc(rng, 3000), lc(rng, 1300, eps=True)], w, p, "v1")


def test_lengths_at_the_v2_limit(engine):
    """n = F2_MAXN runs v2; the same batch plus one light curve of F2_MAXN + 1 cadences runs v1 as a whole."""
    rng = np.random.default_rng(131)
    base = [lc(rng, F2_MAXN, gaps=6, eps=True), lc(rng, 3000)]
    check(engine, base, 101, 2, expected_path(101, 2, F2_MAXN))
    check(engine, base + [lc(rng, F2_MAXN + 1, gaps=4)], 101, 2, "v1")


@pytest.mark.parametrize("w,p", [(101, 2), (401, 2), (51, 4), (41, 1)], ids=["w101-p2", "w401-p2", "w51-p4", "w41-p1"])
def test_kept_counts_around_the_tile_and_the_sampling_median(engine, w, p):
    """Light curves whose kept counts (first iteration: no gaps, no outliers) are tile_out - 1, tile_out,
    tile_out + 1 and 2 tile_out, and 8191 / 8192 cadences (below / at the sampling median's threshold 4 * 2048)."""
    tile = plan(w, p, 8192)[2]
    rng = np.random.default_rng(tile + w)
    lcs = [lc(rng, n, gaps=0, outliers=0) for n in (tile - 1, tile, tile + 1, 2 * tile, 8191, 8192)]
    check(engine, lcs, w, p, expected_path(w, p, 8192))


def test_sampling_median_under_stress(engine):
    """n >= 8192 (two-pass sampling median of select.cuh): regular cadence (every dt equal to rounding), jittered
    cadence (many distinct dts), heavy NaN flux (the kept count falls between iterations), an exclude mask; then
    niters = 5 (the dt median's bracket carried four times)."""
    rng = np.random.default_rng(8192)
    lcs = [lc(rng, 9000, gaps=0), lc(rng, 12000, jitter=0.3), lc(rng, 20000, nans=6000, eps=True), lc(rng, 16384)]
    masks = [np.zeros(len(l[0]), bool) for l in lcs]
    masks[3][rng.choice(16384, 3000, replace=False)] = True
    masks[3][5000:5400] = True
    for niters in (3, 5):
        check(engine, lcs, 201, 2, expected_path(201, 2, 20000), masks=masks, niters=niters)


def test_gap_segmentation_edges(engine):
    """Segments of exactly w kept cadences (filtered), w - 1 (median fallback) and fewer than break_tolerance
    (median fallback although w fits)."""
    rng = np.random.default_rng(77)
    w = 21
    lcs = [segments_lc(rng, [600, w, 400, w - 1, 300]), segments_lc(rng, [500, 4, 500, 3, 800]), lc(rng, 2000)]
    check(engine, lcs, w, 2, expected_path(w, 2, 2000), niters=1)
    check(engine, lcs[1:], 3, 1, "v2-moments", bt=5, niters=1)
    check(engine, lcs, w, 2, expected_path(w, 2, 2000))


def test_gap_cut_limit(engine):
    """1023 segments of 8 cadences (1022 cuts) stay on v2; 1024 segments (1023 cuts) re-run on v1."""
    rng = np.random.default_rng(1022)
    ok = segments_lc(rng, [8] * 1023)
    over = segments_lc(rng, [8] * 1024)
    other = lc(rng, 3000)
    check(engine, [ok, other], 5, 2, expected_path(5, 2, 8184), niters=1)
    check(engine, [over, other], 5, 2, "v1-rerun", niters=1)


def test_many_cut_candidates_few_cuts(engine):
    """More than 1024 dts above break_tolerance times the sampling median's lower bracket value but below
    break_tolerance times the median (the kernel's candidate list overflows and it re-reads the time stamps), plus a
    few real cuts.  dts: 18900 uniform in [0.5, 1.5] DT, 1100 of 5.1 DT, 20 of 8 DT: median ~1.06 DT, lower bracket
    (sample rank 1024 - 64 of 2048) ~1.00 DT, so 5.1 DT is a candidate (> 5.0) and not a cut (< 5.3)."""
    rng = np.random.default_rng(1024)
    dts = np.concatenate([rng.uniform(0.5, 1.5, 18900), np.full(1100, 5.1), np.full(20, 8.0)]) * DT
    t = 131.5 + np.concatenate([[0.0], np.cumsum(rng.permutation(dts))])
    check(engine, [lc(rng, 0, t=t), lc(rng, 3000)], 101, 2, expected_path(101, 2, len(t)))


@pytest.mark.parametrize("w,p", [(101, 2), (9, 4), (401, 2)], ids=["w101-p2", "w9-p4", "w401-p2"])
def test_flux_units_errors_and_degenerate_light_curves(engine, w, p):
    """e-/s flux next to normalised flux; n = 0, 1, 2, fewer than two usable cadences (NaN trend) and w > n (median
    fallback) in the same batch as healthy light curves; then the batch without flux errors (flat_err all NaN)."""
    rng = np.random.default_rng(w * 10 + p)
    few = lc(rng, 50)
    few[1][:] = np.nan
    few[1][7] = 1.0
    lcs = [lc(rng, 4000, eps=True), lc(rng, 0, t=np.zeros(0)), lc(rng, 0, t=np.array([131.5]), outliers=0),
           lc(rng, 0, t=131.5 + np.arange(2) * DT, outliers=0), few, lc(rng, w - 2, gaps=0, outliers=0), lc(rng, 3000)]
    check(engine, lcs, w, p, expected_path(w, p, 4000), nan_lcs=(2, 4))
    check(engine, [(t, f, None) for t, f, _ in lcs], w, p, expected_path(w, p, 4000), nan_lcs=(2, 4))
