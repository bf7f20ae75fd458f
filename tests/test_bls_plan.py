"""The K3 launch planner (lightkurve_b200/csrc/bls_plan.h) built with g++ and checked on the host: every
(light curve, period) is searched exactly once, each CTA covers the periods a one-light-curve call gives it,
the launch count of a batch does not grow with the batch, the boundary-path tables are budgeted per group, and a
shared grid is planned chunk by chunk as the shared-grid entry always did."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
c_vp, c_int, c_i64, c_dbl = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_double

WARPS, TILE = 8, 1024
FIXED_SMEM = (3 * TILE + 2 + 2 * WARPS * 32) * 8
SMEM_CAP, SMEM_SM = 200 * 1024, 227 * 1024
DEFAULT_CAP = 12 << 30


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    out = str(tmp_path_factory.mktemp("blsplan") / "libbls_plan.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-o", out,
                           os.path.join(HERE, "native", "bls_plan_driver.cpp")])
    lib = ctypes.CDLL(out)
    lib.emu_bls_plan.argtypes = [c_vp, c_vp, c_i64, c_int, c_dbl, c_int, c_int, c_i64, c_vp, c_vp, c_vp]
    lib.emu_bls_plan.restype = c_int
    lib.emu_bls_plan_get.argtypes = [c_vp, c_vp]
    lib.emu_bls_plan_get.restype = None
    lib.emu_bls_table_groups.argtypes = [c_vp, c_vp, c_int, c_dbl, c_int, c_int, c_i64, c_vp, c_vp]
    lib.emu_bls_table_groups.restype = c_int
    lib.emu_last_error.restype = ctypes.c_char_p
    return lib


def plan(lib, grids, shared=False, bin_duration=0.005, oversample=10, ghist_bins=-1, hist_cap=0):
    """grids: one array (shared=True, with len(grids) ignored: pass (grid, B)) or a list of per-LC grids."""
    if shared:
        grid, B = grids
        per = np.ascontiguousarray(grid, dtype=np.float64)
        pofs = None
    else:
        B = len(grids)
        per = np.ascontiguousarray(np.concatenate(grids), dtype=np.float64)
        pofs = np.zeros(B + 1, np.int64)
        np.cumsum([len(g) for g in grids], out=pofs[1:])
    n_cta, n_launch, gb = c_i64(), c_i64(), c_i64()
    st = lib.emu_bls_plan(per.ctypes.data, None if pofs is None else pofs.ctypes.data, len(per), B, bin_duration,
                          oversample, ghist_bins, hist_cap, ctypes.byref(n_cta), ctypes.byref(n_launch),
                          ctypes.byref(gb))
    if st != 0:
        raise RuntimeError(lib.emu_last_error().decode())
    cta = np.zeros((n_cta.value, 3), np.int64)
    launch = np.zeros((n_launch.value, 6), np.int64)
    lib.emu_bls_plan_get(cta.ctypes.data, launch.ctypes.data)
    return cta, launch, gb.value, pofs


def chunks_today(per, bin_duration, oversample, ghist_bins=-1):
    """The chunking of the shared-grid entry before the planner existed, restated: (p0, p1, stride, W, ghist, smem)."""
    out, p0, P = [], 0, len(per)
    nb = (np.ceil(per / bin_duration)).astype(np.int64) + oversample
    while p0 < P:
        lo = hi = int(nb[p0])
        p1 = p0 + 1
        while p1 < P:
            a, b = min(lo, int(nb[p1])), max(hi, int(nb[p1]))
            if b > a + a // 4 + 64:
                break
            lo, hi = a, b
            p1 += 1
        stride = (hi + 1 + 3) // 4 * 4
        W = WARPS
        while W > 1 and FIXED_SMEM + W * 16 * stride > SMEM_CAP:
            W >>= 1
        smem = FIXED_SMEM + W * 16 * stride
        if (stride > ghist_bins) if ghist_bins >= 0 else 4 * (smem + 1024) > SMEM_SM:
            smem = SMEM_CAP + 1
        ghist = smem > SMEM_CAP
        if ghist:
            W, smem = WARPS, FIXED_SMEM
        out.append((p0, p1, stride, W, int(ghist), smem))
        p0 = p1
    return out


def lk_grid(rng, baseline=None, dt=None, durations=(0.05, 0.10, 0.15, 0.20, 0.25, 0.33), frequency_factor=10):
    """lightkurve's default BLS period grid for a light curve of the given baseline and cadence."""
    baseline = rng.uniform(20, 28) if baseline is None else baseline
    dt = 2.0 / 1440 if dt is None else dt
    pmin = max(4 * dt, max(durations) + dt)
    pmax = baseline / 3.0
    df = frequency_factor * min(durations) / baseline ** 2
    nf = 1 + int(np.round((1 / pmin - 1 / pmax) / df))
    return 1.0 / (1 / pmin - df * np.arange(nf))


def check_plan(cta, launch, pofs, grids, bin_duration, oversample, ghist_bins=-1, hist_cap=DEFAULT_CAP):
    B = len(grids)
    P = int(pofs[-1])
    # every (light curve, period) exactly once, and only periods of the light curve's own grid
    hits = np.zeros(P, np.int64)
    for p, b, n in cta:
        assert 1 <= n <= WARPS
        assert pofs[b] <= p and p + n <= pofs[b + 1]
        hits[p:p + n] += 1
    assert np.all(hits == 1)
    # launches partition the CTA list; each launch is uniform in W and placement and sized for its CTAs
    assert launch[0, 0] == 0 and launch[-1, 1] == len(cta)
    assert np.all(launch[1:, 0] == launch[:-1, 1])
    for c0, c1, W, stride, ghist, smem in launch:
        assert c1 > c0
        assert np.all(cta[c0:c1, 2] <= W)
        if ghist:
            assert smem == FIXED_SMEM and W == WARPS
            assert (c1 - c0) * W * 16 * stride <= max(hist_cap, W * 16 * stride)
        else:
            assert smem == FIXED_SMEM + W * 16 * stride and smem <= SMEM_CAP
    # each CTA's periods are those of the one-light-curve plan of its grid, with the same W, placement and a
    # stride at least that light curve's chunk stride
    cta_launch = np.repeat(np.arange(len(launch)), launch[:, 1] - launch[:, 0])
    for b in range(B):
        mine = cta[:, 1] == b
        got = {(int(p - pofs[b]), int(n)): launch[cta_launch[i]] for i, (p, _, n) in zip(np.flatnonzero(mine),
                                                                                          cta[mine])}
        want = {}
        for p0, p1, stride, W, ghist, smem in chunks_today(grids[b], bin_duration, oversample, ghist_bins):
            for p in range(p0, p1, W):
                want[(p, min(W, p1 - p))] = (stride, W, ghist)
        assert set(got) == set(want), "light curve %d: CTA periods differ from its one-light-curve plan" % b
        for k, (stride, W, ghist) in want.items():
            ln = got[k]
            assert ln[2] == W and ln[4] == ghist and ln[3] >= stride


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_ragged_plan_matches_one_light_curve_plans(lib, seed):
    rng = np.random.default_rng(seed)
    grids = [lk_grid(rng, dt=rng.choice([2.0 / 1440, 10.0 / 1440, 30.0 / 1440])) for _ in range(12)]
    grids.append(np.array([0.7]))                                   # one-period grid
    grids.append(np.sort(rng.uniform(0.4, 12.0, 500)))             # unsorted-free random grid
    grids.append(np.sort(rng.uniform(0.4, 12.0, 300))[::-1].copy())  # descending
    grids.append(rng.permutation(lk_grid(rng)))                     # unsorted
    order = rng.permutation(len(grids))
    grids = [grids[i] for i in order]
    cta, launch, gb, pofs = plan(lib, grids)
    assert np.any(launch[:, 4] == 1) and np.any(launch[:, 4] == 0)   # both histogram placements occur
    check_plan(cta, launch, pofs, grids, 0.005, 10)


def test_global_histograms_and_tiny_cap(lib):
    rng = np.random.default_rng(5)
    grids = [lk_grid(rng) for _ in range(6)] + [np.linspace(2.0, 13.0, 40)]
    cap = 8 << 20
    cta, launch, gb, pofs = plan(lib, grids, ghist_bins=0, hist_cap=cap)
    assert np.all(launch[:, 4] == 1)
    assert gb <= cap
    check_plan(cta, launch, pofs, grids, 0.005, 10, ghist_bins=0, hist_cap=cap)
    # a chunk whose histograms do not fit the cap for one light curve is refused, as a one-light-curve call refuses it
    with pytest.raises(RuntimeError, match="histogram workspace per light curve"):
        plan(lib, grids, ghist_bins=0, hist_cap=1 << 14)
    with pytest.raises(RuntimeError, match="histogram workspace per light curve"):
        plan(lib, grids[:1], ghist_bins=0, hist_cap=1 << 14)


def test_launch_count_does_not_grow_with_batch(lib):
    rng = np.random.default_rng(7)
    base = [lk_grid(rng, dt=rng.choice([2.0 / 1440, 10.0 / 1440])) for _ in range(8)]
    counts = []
    for reps in (1, 4, 16):
        grids = [g for _ in range(reps) for g in base]
        cta, launch, gb, pofs = plan(lib, grids)
        counts.append(len(launch))
        if reps == 4:
            check_plan(cta, launch, pofs, grids, 0.005, 10)
    assert counts[0] == counts[1] == counts[2], counts
    # and far fewer launches than chunks
    n_chunks = sum(len(chunks_today(g, 0.005, 10)) for g in base) * 16
    assert counts[-1] < n_chunks / 20


@pytest.mark.parametrize("ghist_bins,cap", [(-1, 0), (0, 8 << 20), (100, 0)])
def test_shared_plan_equals_todays_chunking(lib, ghist_bins, cap):
    rng = np.random.default_rng(11)
    grid = 1.0 / np.linspace(1 / 0.3314, 1 / 9.26, 3000)
    B = 5
    cta, launch, gb, _ = plan(lib, (grid, B), shared=True, ghist_bins=ghist_bins, hist_cap=cap)
    hist_cap = cap if cap else DEFAULT_CAP
    want_cta, want_launch = [], []
    for p0, p1, stride, W, ghist, smem in chunks_today(grid, 0.005, 10, ghist_bins):
        gx = (p1 - p0 + W - 1) // W
        b_group = min(B, max(1, hist_cap // (gx * W * 16 * stride))) if ghist else B
        for bb in range(0, B, b_group):
            c0 = len(want_cta)
            for b in range(bb, min(B, bb + b_group)):
                for x in range(gx):
                    p = p0 + x * W
                    want_cta.append((p, b, min(W, p1 - p)))
            want_launch.append((c0, len(want_cta), W, stride, ghist, smem))
    np.testing.assert_array_equal(cta, np.array(want_cta))
    np.testing.assert_array_equal(launch, np.array(want_launch))
    del rng


def table_groups(lib, n, x_max, inv_delta, shared, budget, enabled=True):
    B = len(n)
    n = np.ascontiguousarray(n, np.int64)
    x_max = np.ascontiguousarray(x_max, np.float64)
    groups = np.zeros((max(B, 1), 3), np.int64)
    to = np.zeros(B + 1, np.int64)
    k = lib.emu_bls_table_groups(n.ctypes.data, x_max.ctypes.data, B, inv_delta, int(enabled), int(shared), budget,
                                 groups.ctypes.data, to.ctypes.data)
    return groups[:k], to


def one_lc_has_table(n, x_max, inv_delta):
    cells = x_max * inv_delta
    return n > 0 and cells >= 0 and cells <= 6.0e7


@pytest.mark.parametrize("budget", [1 << 28, 200_000, 1])
def test_table_groups_budget(lib, budget):
    rng = np.random.default_rng(3)
    B = 300
    n = rng.integers(0, 20000, B)
    n[rng.choice(B, 10, replace=False)] = 0                         # empty light curves
    x_max = rng.uniform(1, 27.8, B)
    x_max[rng.choice(B, 5, replace=False)] = 1e6                    # too long a baseline for a table
    inv_delta = 8 / 0.005
    groups, to = table_groups(lib, n, x_max, inv_delta, False, budget)
    assert groups[0, 0] == 0 and groups[-1, 1] == B and np.all(groups[1:, 0] == groups[:-1, 1])
    for b0, b1, table in groups:
        entries = to[b1] - to[b0]
        assert entries <= budget or b1 - b0 == 1
        for b in range(b0, b1):
            if not one_lc_has_table(n[b], x_max[b], inv_delta):
                if n[b] > 0:
                    assert b1 - b0 == 1 and not table            # a light curve without a table: a group of its own
            else:
                assert table and to[b + 1] - to[b] == int(x_max[b] * inv_delta) + 3
    # a batch that fits one budget is one group
    g1, _ = table_groups(lib, n[:20], np.minimum(x_max[:20], 27.8), inv_delta, False, 1 << 28)
    assert len(g1) == 1


def test_table_groups_shared_rule_unchanged(lib):
    inv_delta = 8 / 0.005
    n = np.array([100, 0, 5000])
    g, to = table_groups(lib, n, np.array([10.0, 0.0, 27.0]), inv_delta, True, 1 << 28)
    assert g.tolist() == [[0, 3, 1]] and to[-1] == int(10 * inv_delta) + 3 + int(27 * inv_delta) + 3
    g, to = table_groups(lib, n, np.array([10.0, 0.0, 1e6]), inv_delta, True, 1 << 28)   # one light curve too long
    assert g.tolist() == [[0, 3, 0]]
    g, _ = table_groups(lib, n, np.array([10.0, 0.0, 27.0]), inv_delta, True, 1000)     # batch over budget
    assert g.tolist() == [[0, 3, 0]]
    g, _ = table_groups(lib, n, np.array([10.0, 0.0, 27.0]), inv_delta, False, 1 << 28, enabled=False)
    assert g.tolist() == [[0, 3, 0]]
