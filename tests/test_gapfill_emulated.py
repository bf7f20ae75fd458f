"""K15 (gap_steps_kernel, gap_plan_kernel and gap_fill_kernel of lightkurve_b200/csrc/gapfill.cuh) executed on the CPU
through tests/native/cuda_emu.h, against the loop of LightCurve.fill_gaps written out in numpy (the same statements):
times, inserted positions and flux_err bitwise, inserted flux bitwise mean + std * z for given mean, std and z.
Cases: no gap, a one-cadence gap, a step of exactly 1.2 dt, a gap of more than 1 000 cadences, duplicate times, NaN
errors next to a gap, equal errors on both sides, lengths 0, 1 and 2, light curves longer than one CTA tile; the
reject flags; outputs independent of a light curve's position and neighbours."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
CUDA_INC = "/usr/local/cuda/include"
c_vp, c_int = ctypes.c_void_p, ctypes.c_int


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    out = str(tmp_path_factory.mktemp("emu") / "libgapfill_emu.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-pthread", "-I" + CUDA_INC,
                           "-Wno-attributes", "-shared", "-fPIC", "-Wl,-Bsymbolic", "-o", out,
                           os.path.join(HERE, "native", "gapfill_emu_driver.cpp")])
    lib = ctypes.CDLL(out)
    lib.emu_gap_steps.argtypes = [c_vp, c_vp, c_vp, c_int, c_vp, c_vp]
    lib.emu_gap_plan.argtypes = [c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp]
    lib.emu_gap_fill.argtypes = [c_vp] * 5 + [c_int] + [c_vp] * 7
    for f in (lib.emu_gap_steps, lib.emu_gap_plan, lib.emu_gap_fill):
        f.restype = None
    return lib


def _p(x):
    return x.ctypes.data


def loop(t, fe):
    """LightCurve.fill_gaps' statements for NaN-free sorted input, without the noise: (times, in_original, flux_err,
    number inserted)."""
    if len(t) < 2:
        return t.copy(), None, fe.copy(), 0
    dt = np.nanmedian(t[1:] - t[:-1])
    ntime = [t[0]]
    for x in t[1:]:
        prev = ntime[-1]
        while (x - prev) > 1.2 * dt:
            ntime.append(prev + dt)
            prev = ntime[-1]
        ntime.append(x)
    ntime = np.asarray(ntime, float)
    ino = np.isin(ntime, t)
    e = np.zeros(len(ntime))
    e[ino] = fe
    e[~ino] = np.interp(ntime[~ino], t, fe)
    k = int((~ino).sum())
    return ntime, ino, e, k


def run(emu, times, fluxes, errs, stds, zs):
    B = len(times)
    off = np.zeros(B + 1, np.int64)
    off[1:] = np.cumsum([len(t) for t in times])
    def cat(arrays):
        x = np.concatenate([np.asarray(a, np.float64) for a in arrays])
        return np.ascontiguousarray(x) if len(x) else np.zeros(1)

    t, y, e = cat(times), cat(fluxes), cat(errs)
    doff = np.zeros(B + 1, np.int64)
    doff[1:] = np.cumsum([max(len(x) - 1, 0) for x in times])
    steps = np.zeros(max(int(doff[-1]), 1))
    flags = np.zeros(B, np.int32)
    emu.emu_gap_steps(_p(t), _p(off), _p(doff), B, _p(steps), _p(flags))
    dt = np.array([np.median(steps[doff[b]:doff[b + 1]]) if doff[b + 1] > doff[b] else np.nan for b in range(B)])
    n_ins, mean = np.zeros(B, np.int64), np.zeros(B)
    emu.emu_gap_plan(_p(t), _p(y), _p(off), B, _p(dt), _p(n_ins), _p(mean), _p(flags))
    noff = off.copy()
    noff[1:] += np.cumsum(n_ins)
    z = np.ascontiguousarray(np.concatenate([zs[b][:n_ins[b]] for b in range(B)]) if n_ins.sum() else np.zeros(1))
    std = np.ascontiguousarray(stds, dtype=np.float64)
    n = max(int(noff[-1]), 1)
    to, yo, eo = np.zeros(n), np.zeros(n), np.zeros(n)
    emu.emu_gap_fill(_p(t), _p(y), _p(e), _p(off), _p(noff), B, _p(dt), _p(mean), _p(std), _p(z), _p(to), _p(yo),
                     _p(eo))
    sl = [slice(noff[b], noff[b + 1]) for b in range(B)]
    return [to[s] for s in sl], [yo[s] for s in sl], [eo[s] for s in sl], mean, flags, dt, steps[:doff[-1]]


def cases():
    dt = 1765.5 / 86400.0
    t = 100.0 + np.arange(40) * dt
    e = np.linspace(1e-4, 2e-4, 40)
    e2 = e.copy()
    e2[19] = np.nan
    e3 = e.copy()
    e3[21] = e3[19]
    rng = np.random.default_rng(1)
    # steps of 0.25 (exact) and a last step of exactly 1.2 * 0.25: the median step is 0.25 bitwise
    edge = np.append(-5.0 + 0.25 * np.arange(21), 1.2 * 0.25)
    assert edge[-1] - edge[-2] == 1.2 * np.median(np.diff(edge))
    long_t = 10.0 + np.arange(3000) * dt
    long_t = np.concatenate([long_t[:1000], long_t[1720:]])
    out = [
        (t, e),
        (np.delete(t, 20), np.delete(e, 20)),
        (edge, e[:len(edge)]),                       # last step exactly 1.2 dt: no insert
        (np.append(edge[:-1], np.nextafter(edge[-1], 1.0)), e[:len(edge)]),     # one ulp more: one insert
        (np.concatenate([t[:10], t[10:] + 1200 * dt]), e),
        (np.concatenate([t[:5], t[4:39]]), e),
        (np.delete(t, 20), np.delete(e2, 20)),
        (np.delete(t, 20), np.delete(e3, 20)),
        (t[:0], e[:0]), (t[:1], e[:1]), (t[:2], e[:2]),
        (np.sort(rng.uniform(0, 30, 700)), rng.uniform(1, 2, 700)),
        (long_t, rng.uniform(1, 2, len(long_t))),
    ]
    return out


def test_fill_equals_the_loop(emu):
    cs = cases()
    rng = np.random.default_rng(5)
    times = [c[0] for c in cs]
    errs = [c[1] for c in cs]
    fluxes = [rng.normal(1, 1e-3, len(c[0])) for c in cs]
    stds = rng.uniform(1e-4, 1e-3, len(cs))
    zs = [rng.normal(size=5000) for _ in cs]
    to, yo, eo, mean, flags, dt, _ = run(emu, times, fluxes, errs, stds, zs)
    assert not np.any(flags & 5)
    for b in range(len(cs)):
        nt, ino, ne, k = loop(times[b], errs[b])
        np.testing.assert_array_equal(to[b], nt, err_msg="time %d" % b)
        np.testing.assert_array_equal(eo[b], ne, err_msg="flux_err %d" % b)
        if ino is None:
            np.testing.assert_array_equal(yo[b], fluxes[b])
            continue
        np.testing.assert_array_equal(yo[b][ino], fluxes[b])
        np.testing.assert_array_equal(yo[b][~ino], mean[b] + stds[b] * zs[b][:k])
        np.testing.assert_allclose(mean[b], np.mean(fluxes[b]), rtol=1e-14)
    assert len(to[4]) - len(times[4]) > 1000
    assert len(to[2]) == len(times[2])
    assert len(to[3]) == len(times[3]) + 1


def test_position_and_neighbour_invariance(emu):
    cs = cases()
    rng = np.random.default_rng(8)
    fl = [rng.normal(1, 1e-3, len(c[0])) for c in cs]
    zs = [rng.normal(size=5000) for _ in cs]
    stds = rng.uniform(1e-4, 1e-3, len(cs))
    full = run(emu, [c[0] for c in cs], fl, [c[1] for c in cs], stds, zs)
    perm = rng.permutation(len(cs))
    pm = run(emu, [cs[i][0] for i in perm], [fl[i] for i in perm], [cs[i][1] for i in perm], stds[perm],
             [zs[i] for i in perm])
    for k, i in enumerate(perm):
        for a in range(3):
            np.testing.assert_array_equal(pm[a][k], full[a][i])
        one = run(emu, [cs[i][0]], [fl[i]], [cs[i][1]], stds[i:i + 1], [zs[i]])
        for a in range(3):
            np.testing.assert_array_equal(one[a][0], full[a][i])


def test_reject_flags(emu):
    t = np.arange(10.0)
    res = run(emu, [t[::-1].copy(), np.array([0.0, 0, 0, 0, 1]), t, np.array([0.0, 1, 2, 1e9])],
              [np.ones(10), np.ones(5), np.ones(10), np.ones(4)], [np.ones(10), np.ones(5), np.ones(10), np.ones(4)],
              np.ones(4), [np.zeros(1)] * 4)
    flags, dt = res[4], res[5]
    assert flags[0] & 1 and not flags[2] & 1
    assert flags[1] & 2 and dt[1] == 0
    assert flags[2] == 2
    assert flags[3] & 4
