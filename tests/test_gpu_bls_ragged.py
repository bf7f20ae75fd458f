"""Box Least Squares over light curves with their own period grids (lkb_bls_power_ex with period_offsets) on the
GPU: parity with the oracle on every light curve, bitwise equality with one-light-curve lkb_bls_power calls, and the
batch-level invariances (permutation, global histograms with a tiny workspace cap, shared grid as CSR, device mode)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import bls as obls

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
FIELDS = ("power", "depth", "depth_err", "duration", "transit_time", "depth_snr", "log_likelihood", "bins")
DUR = [0.05, 0.1, 0.2]


def assert_bls_close(got, ref, t, y, dy, period, duration, objective="likelihood", max_tied_frac=0.02):
    """The tolerances and tie rule of test_gpu_engine.assert_bls_close: the winning box equals the oracle's except
    at the oracle's own mathematical ties; values rtol 1e-9; duration / transit_time where the boxes coincide."""
    same = np.all(got["bins"] == ref["bins"], axis=1)
    for p_idx in np.flatnonzero(~same):
        n, dur = got["bins"][p_idx]
        o = obls.objective_at(t, y, dy, period[p_idx], duration, int(n), int(dur), objective=objective)
        assert abs(o - ref["power"][p_idx]) <= 1e-10 * abs(ref["power"][p_idx]), "period %d not tied" % p_idx
    assert (~same).mean() <= max_tied_frac, "too many tie-broken periods: %d" % (~same).sum()
    for k in ("power", "depth", "depth_err", "depth_snr", "log_likelihood"):
        np.testing.assert_allclose(got[k], ref[k], rtol=1e-9, atol=1e-12, err_msg=k)
    for k in ("duration", "transit_time"):
        np.testing.assert_allclose(got[k][same], ref[k][same], rtol=1e-12, atol=1e-9, err_msg=k)


def transit_flux(rng, t, depth=3e-3):
    per, dur = rng.uniform(1.2, 6), rng.uniform(0.06, 0.2)
    y = 1 + 5e-4 * rng.standard_normal(len(t))
    y[np.abs((t - t.min() - 0.4 + 0.5 * per) % per - 0.5 * per) < 0.5 * dur] -= depth
    return y


def ragged_batch(seed=0, small=False):
    """Light curves that reach every path: dense 2-min (boundary path), sparse 30-min (cadence path), unsorted
    times, an empty light curve, a one-period grid and long periods (global histograms)."""
    rng = np.random.default_rng(seed)
    ts, grids = [], []
    span = 12.0 if small else 27.0
    t = 1325 + np.arange(0, span, 2.0 / 1440)
    ts.append(t[rng.random(len(t)) < 0.95])                                      # dense, boundary path
    grids.append(obls.autoperiod(ts[-1], DUR, 0.4, span / 2.5, frequency_factor=30 if small else 3))
    t = 1400 + np.arange(0, span * 0.8, 2.0 / 1440)
    ts.append(t[rng.random(len(t)) < 0.8])                                       # dense, shorter baseline
    grids.append(obls.autoperiod(ts[-1], DUR, 0.3, span / 3, frequency_factor=30 if small else 3))
    t = np.sort(rng.uniform(1500, 1500 + span, 400))                             # sparse: cadence path
    ts.append(t)
    grids.append(obls.autoperiod(t, DUR, 0.5, span / 2, frequency_factor=30 if small else 2))
    t = 1600 + np.arange(0, span, 10.0 / 1440)
    ts.append(rng.permutation(t))                                                # unsorted times
    grids.append(obls.autoperiod(t, DUR, 0.45, span / 3, frequency_factor=30 if small else 2))
    ts.append(np.zeros(0))                                                       # empty light curve
    grids.append(np.linspace(0.5, 3.0, 37))
    t = 1700 + np.arange(0, span, 2.0 / 1440)
    ts.append(t)
    grids.append(np.array([1.37]))                                               # one-period grid
    t = 1800 + np.arange(0, span, 5.0 / 1440)
    ts.append(t)
    grids.append(np.linspace(span / 3.0, span / 2.05, 20 if small else 300))      # long periods: global histograms
    ys = [transit_flux(rng, t) if len(t) else np.zeros(0) for t in ts]
    dys = [np.full(len(t), 5e-4) * rng.uniform(0.8, 1.2, len(t)) for t in ts]
    return ts, ys, dys, grids


def one_by_one(engine, ts, ys, dys, grids, objective="likelihood"):
    return [engine.bls_power([t], [y], None if dys is None else [dy], g, DUR, objective=objective, return_bins=True)
            for t, y, dy, g in zip(ts, ys, dys if dys is not None else [None] * len(ts), grids)]


def assert_bitwise(ragged, singles):
    for b, s in enumerate(singles):
        for k in FIELDS:
            np.testing.assert_array_equal(ragged[k][b], s[k][0], err_msg="light curve %d, %s" % (b, k))
        np.testing.assert_array_equal(ragged["period"][b], s["period"])


@pytest.mark.parametrize("objective", ["likelihood", "snr"])
@pytest.mark.parametrize("with_dy", [True, False])
def test_ragged_parity_and_bitwise(engine, objective, with_dy):
    ts, ys, dys, grids = ragged_batch(1)
    dys = dys if with_dy else None
    l0 = engine.launch_count()
    res = engine.bls_power(ts, ys, dys, grids, DUR, objective=objective, return_bins=True)
    assert engine.launch_count() - l0 < 40
    for b, (t, y, g) in enumerate(zip(ts, ys, grids)):
        dy = None if dys is None else dys[b]
        got = {k: res[k][b] for k in FIELDS}
        if len(t) == 0:
            assert np.all(np.isnan(got["power"])) and np.all(got["bins"] == -1)
            continue
        ref = obls.bls_power_c(t, y, dy, g, DUR, objective=objective, return_bins=True)
        assert_bls_close(got, ref, t, y, dy, g, DUR, objective=objective)
    assert_bitwise(res, one_by_one(engine, ts, ys, dys, grids, objective))


def test_unit_dy_is_bitwise_no_dy(engine):
    ts, ys, dys, grids = ragged_batch(2)
    a = engine.bls_power(ts, ys, None, grids, DUR, return_bins=True)
    b = engine.bls_power(ts, ys, [np.ones(len(t)) for t in ts], grids, DUR, return_bins=True)
    for k in FIELDS:
        for x, z in zip(a[k], b[k]):
            np.testing.assert_array_equal(x, z)


def test_permuted_batch(engine):
    ts, ys, dys, grids = ragged_batch(3)
    res = engine.bls_power(ts, ys, dys, grids, DUR, return_bins=True)
    perm = np.random.default_rng(0).permutation(len(ts))
    rp = engine.bls_power([ts[i] for i in perm], [ys[i] for i in perm], [dys[i] for i in perm],
                          [grids[i] for i in perm], DUR, return_bins=True)
    for j, i in enumerate(perm):
        for k in FIELDS:
            np.testing.assert_array_equal(rp[k][j], res[k][i])


def test_shared_grid_as_csr_and_device_mode(engine):
    import torch
    from lightkurve_b200 import _lib as L
    ts, ys, dys, _ = ragged_batch(4)
    grid = np.linspace(0.5, 4.0, 1500)
    shared = engine.bls_power(ts, ys, dys, grid, DUR, return_bins=True)
    csr = engine.bls_power(ts, ys, dys, [grid] * len(ts), DUR, return_bins=True)
    for k in FIELDS:
        np.testing.assert_array_equal(np.stack(csr[k]), shared[k])
    # device-pointer mode of the ragged entry equals its host mode
    grids = [grid[:700], grid[300:], grid[::3], grid[5:6], grid[::-2], grid[100:900], grid]
    host = engine.bls_power(ts, ys, dys, grids, DUR, return_bins=True)
    t, off = engine._csr(ts)
    y, _ = engine._csr(ys)
    dy, _ = engine._csr(dys)
    per, pofs = engine._csr(grids)
    dev = torch.device("cuda:0")
    td, yd, dyd, pd, dd = (torch.from_numpy(a).to(dev) for a in (t, y, dy, per, np.asarray(DUR, np.float64)))
    P = int(pofs[-1])
    outs = [torch.empty(P, dtype=torch.float64, device=dev) for _ in range(7)]
    bins = torch.empty((P, 2), dtype=torch.int32, device=dev)
    L.check(L.load().lkb_bls_power_ex(L.ptr(td), L.ptr(yd), L.ptr(dyd), L.ptr(off), len(ts), L.ptr(pd), L.ptr(pofs),
                                      P, L.ptr(dd), len(DUR), 10, L.BLS_LIKELIHOOD, *[L.ptr(o) for o in outs],
                                      L.ptr(bins), L.MEM_DEVICE, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    for k, o in zip(FIELDS[:7], outs):
        np.testing.assert_array_equal(o.cpu().numpy(), np.concatenate(host[k]), err_msg=k)
    np.testing.assert_array_equal(bins.cpu().numpy(), np.concatenate(host["bins"]))


def test_global_histograms_tiny_cap_subprocess(engine, tmp_path):
    """LKB_BLS_GHIST_BINS=0 (every chunk in global histograms) with a 1 MiB workspace cap gives the same results.
    The histogram placement is read once per process, so the variant runs in a child process."""
    ts, ys, dys, grids = ragged_batch(5, small=True)
    res = engine.bls_power(ts, ys, dys, grids, DUR, return_bins=True)
    np.savez(tmp_path / "in.npz", *[a for quad in zip(ts, ys, dys, grids) for a in quad])
    code = ("import sys, numpy as np; sys.path.insert(0, %r)\n"
            "from lightkurve_b200 import engine\n"
            "engine.init(0)\n"
            "z = np.load(%r); a = [z['arr_%%d' %% i] for i in range(len(z.files))]\n"
            "ts, ys, dys, gs = a[0::4], a[1::4], a[2::4], a[3::4]\n"
            "r = engine.bls_power(ts, ys, dys, gs, %r, return_bins=True)\n"
            "np.savez(%r, **{k: np.concatenate(v) for k, v in r.items()})\n"
            % (ROOT, str(tmp_path / "in.npz"), DUR, str(tmp_path / "out.npz")))
    env = dict(os.environ, LKB_BLS_GHIST_BINS="0", LKB_BLS_HIST_CAP_MB="1")
    subprocess.check_call([sys.executable, "-c", code], env=env, timeout=600)
    out = np.load(tmp_path / "out.npz")
    for k in FIELDS:
        np.testing.assert_array_equal(out[k], np.concatenate(res[k]), err_msg=k)


def test_refusals(engine):
    ts, ys, dys, grids = ragged_batch(6, small=True)
    bad = list(grids)
    bad[2] = np.array([0.5, np.nan, 1.0])
    with pytest.raises(ValueError, match="light curve 2"):
        engine.bls_power(ts, ys, dys, bad, DUR)
    bad = list(grids)
    bad[3] = np.zeros(0)
    with pytest.raises(ValueError, match="light curve 3 has an empty period grid"):
        engine.bls_power(ts, ys, dys, bad, DUR)
    bad = list(grids)
    bad[1] = np.array([0.15, 1.0])                   # shorter than the longest duration for light curve 1 only
    with pytest.raises(ValueError, match="^The maximum transit duration must be shorter than the minimum period$"):
        engine.bls_power(ts, ys, dys, bad, DUR)
    from lightkurve_b200 import _lib as L
    t, off = engine._csr(ts)
    y, _ = engine._csr(ys)
    per, pofs = engine._csr(grids)
    pofs_bad = pofs.copy()
    pofs_bad[3], pofs_bad[4] = pofs[4], pofs[3]
    P = int(pofs[-1])
    outs = [np.empty(P) for _ in range(7)]
    st = L.load().lkb_bls_power_ex(L.ptr(t), L.ptr(y), None, L.ptr(off), len(ts), L.ptr(per), L.ptr(pofs_bad), P,
                                   L.ptr(np.asarray(DUR, np.float64)), len(DUR), 10, 0, *[L.ptr(o) for o in outs],
                                   None, L.MEM_HOST, None)
    assert st == L.E_ARG and b"light curve 3" in L.load().lkb_last_error()


def test_collection_batched_equals_loop(engine):
    import lightkurve_b200 as lk
    ts, ys, dys, _ = ragged_batch(7)
    lcs = []
    for b, (t, y, dy) in enumerate(zip(ts, ys, dys)):
        if len(t) == 0:
            continue
        o = np.argsort(t)
        lcs.append(lk.LightCurve(time=t[o], flux=y[o], flux_err=dy[o] if b % 2 else np.full(len(t), np.nan)))
    l0 = engine.launch_count()
    pgs = lk.LightCurveCollection(lcs).to_periodogram("bls", duration=DUR, frequency_factor=5)
    batched_launches = engine.launch_count() - l0
    loop = [lc.to_periodogram("bls", duration=DUR, frequency_factor=5) for lc in lcs]
    assert batched_launches < engine.launch_count() - l0 - batched_launches
    for a, b in zip(pgs, loop):
        np.testing.assert_array_equal(a.period.value, b.period.value)
        for k in a._BLS_result:
            np.testing.assert_array_equal(a._BLS_result[k], b._BLS_result[k])
        assert (a._dy is None) == (b._dy is None)


def test_fullsize_c5(engine):
    """All 16 384 config-5 light curves with their default grids in one call (several boundary-path table groups)."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import bench_bls_ragged as bb
    times, fluxes, errs = bb.make_c5_bls(B=16384)
    grids = [bb.default_grid(t) for t in times]
    res = engine.bls_power(times, fluxes, errs, grids, bb.DURATIONS, return_bins=True)
    rng = np.random.default_rng(11)
    pick = rng.choice(len(times), 16, replace=False)
    for b in pick:
        s = engine.bls_power([times[b]], [fluxes[b]], [errs[b]], grids[b], bb.DURATIONS, return_bins=True)
        for k in FIELDS:
            np.testing.assert_array_equal(res[k][b], s[k][0], err_msg="light curve %d, %s" % (b, k))
    for b in pick[:2]:
        sub = np.sort(rng.choice(len(grids[b]), min(2000, len(grids[b])), replace=False))
        ref = obls.bls_power_c(times[b], fluxes[b], errs[b], grids[b][sub], bb.DURATIONS, return_bins=True)
        got = {k: res[k][b][sub] for k in FIELDS}
        assert_bls_close(got, ref, times[b], fluxes[b], errs[b], grids[b][sub], bb.DURATIONS)
