"""Lomb-Scargle (K1 / K1n ragged, K2 / K2n shared grid) on every kernel path and NUFFT transform size, against the fp64
reference on EVERY bin.

Which path a call takes:
  shared grid (lkb_ls_power_shared)
    "nufft"    regular grid f_k = (k0 + k) df, df * baseline <= 1, ascending times; `auto` when B N F >= 2.5e7.  The v2
               transform (nufft_v2.cuh, one real transform per light curve) on a flux grid of 2^p cells,
               p = max(fine_grid_log2(k0 + F), 14) (2^p >= 4 (k0 + F)), so p = 14 .. 23: the column kernel is
               instantiated for PA = p - 10 = 4 .. 13, in float2 and in double2 (the precision escalation pass).
               The window terms come from one transform of unit strengths on 2^p2 cells, p2 = fine_grid_log2(2 (k0 + F)).
    "tcgen05"  wgmma contraction (ls_tc.cu): B >= 64, N >= 256, F >= 128
    "simt"     CUDA-core contraction (ls_shared_simt_kernel)
  ragged batch (lkb_ls_power)
    "nufft"    one shared regular grid, >= 8 cadences and a non-zero baseline per light curve; flux grid 2^p and window
               grid 2^(p + 1) cells, both in the v2 range (k0 + F <= 2^20); else `auto` runs the direct kernel and
               algo="nufft" fails with LKB_E_UNSUPPORTED (-5)
    "direct"   ls_direct_kernel<REGULAR>: fixed-point phases when every light curve's grid is regular, fp64 phases
               otherwise; TMA tiles of 768 / 1536 cadences, 4 bins per warp, 32 bins per block (LS_FPB)
engine.ls_last_algo() and engine.ls_last_nufft_plan() report the path that ran, and every case asserts it.

Reference: the fp64 direct sums (engine.ls_power_chi2 with nterms = 1 and algo="direct", ls_chi2_kernel<1>) on every
(light curve, bin); the 500 (light curve, bin) pairs where the path under test disagrees with it most, plus 200 random
pairs, go to the fp64 oracle (oracle.ls.ls_slow_psd).  Tolerance, in units of which the worst excess is printed:
  "tol"       1e-5 max(A_b) + 1e-4 A  on the amplitude spectrum A (2e-5 max P + 2e-4 P on a power spectrum)
  "tol_data"  the same with the floor 1e-5 max(max A_b, sqrt(2) std(y_b)): relative to the light curve's own
              variability, for fp32 sums over data whose variability lies outside the frequency grid
The NUFFT family is held to "tol" at 1x; "tol_data" is used only where a case says its inputs are hostile."""
import numpy as np
import pytest

from oracle import ls as ols

pytestmark = pytest.mark.gpu

N_WORST, N_RANDOM = 500, 200
V2_P_MIN = 14
DT = 0.0204336


def fine_log2(kmax):
    """nufft_core.h fine_grid_log2 at upsampling 2: the smallest p with 2^p >= 4 kmax."""
    p = 4
    while (1 << p) < 4 * kmax:
        p += 1
    return p


def shared_plan(kmax):
    return ("v2", max(fine_log2(kmax), V2_P_MIN), fine_log2(2 * kmax))


def ragged_plan(kmax):
    p = max(fine_log2(kmax), V2_P_MIN)
    return ("v2", p, p + 1)


# ------------------------------------------------------------------------------------------------------ inputs
def regular_times(rng, n, gaps=4):
    """A near-regular cadence of n samples with a few gaps (a spacecraft light curve)."""
    keep = np.ones(n + 60 * gaps, bool)
    for c in rng.choice(len(keep) - 60, gaps, replace=False):
        keep[c:c + int(rng.integers(10, 50))] = False
    idx = np.flatnonzero(keep)[:n]
    return 131.5 + idx * DT


def random_times(rng, n, span):
    t = np.sort(rng.uniform(0.0, span, n))
    return 131.5 + t


def flux(rng, t, f_line, amp=None, noise=None):
    amp = 10 ** rng.uniform(-3.5, -2) if amp is None else amp
    noise = 10 ** rng.uniform(-4, -3) if noise is None else noise
    return 1 + amp * np.sin(2 * np.pi * f_line * t + rng.uniform(0, 6.3)) + noise * rng.normal(size=len(t))


def hostile(rng, t, f_above):
    """A loud line above the frequency grid and only noise in band: the case the escalation pass exists for.  Its flux
    excursion is ~450x its in-band peak amplitude at 6000 cadences, above the escalation threshold of 250x.  (At
    ~2000x, noise 5e-5, even the double-precision pass cannot meet the stated tolerance: its input is the centred
    flux rounded to fp32, and that rounding alone reaches 2.3x the in-band peak's tolerance for some noise draws.)"""
    return 1 + 8e-3 * np.sin(2 * np.pi * f_above * t + 0.4) + 2e-4 * rng.normal(size=len(t))


# ------------------------------------------------------------------------------------------------------ checks
def _norm(P, norm, n, scale):
    if norm == "amplitude":
        return np.sqrt(np.maximum(P, 0.0)) * np.sqrt(4.0 / n)          # (fp64 sums can leave -1e-20 for a zero power)
    return P * scale if norm == "psd" else P


def _tol(ref, amax, norm, floor=None):
    k = 1.0 if norm == "amplitude" else 2.0
    m = amax if floor is None else np.maximum(amax, floor)
    return k * (1e-5 * m + 1e-4 * ref)


def reference(engine, times, fluxes, freq):
    """fp64 direct sums, psd_raw: [B, F] (shared grid) or a list of rows (per-light-curve grids)."""
    return engine.ls_power_chi2(times, fluxes, freq, 1, "psd_raw", algo="direct")


def compare(engine, name, out, ref_raw, times, fluxes, freqs, norm="amplitude", scale=1.0, data_floor=(), skip=(),
            limit=1.0):
    """out / ref_raw: rows per light curve; freqs: one grid or one per light curve.  Light curves in `data_floor` are
    held to tol_data, those in `skip` are not compared.  Returns the worst excess (stated tolerance)."""
    B = len(times)
    rows = [b for b in range(B) if b not in skip]
    fr = [freqs[b] if isinstance(freqs, list) else freqs for b in range(B)]
    y64 = [np.asarray(f, np.float64) for f in fluxes]
    refs, floors = {}, {}
    worst_full = 0.0
    cand = []
    rng = np.random.default_rng(17)
    for b in rows:
        r = _norm(np.asarray(ref_raw[b], np.float64), norm, len(times[b]), scale)
        o = np.asarray(out[b], np.float64)
        ok = np.isfinite(r)
        assert np.array_equal(np.isnan(o), ~ok), (name, b, "NaN bins differ from the reference")
        amax = float(np.max(r[ok])) if ok.any() else 0.0
        fl = None
        if b in data_floor:
            s = np.sqrt(2.0) * np.std(y64[b])
            fl = s if norm == "amplitude" else s * s * len(times[b]) / 4.0 * (scale if norm == "psd" else 1.0)
        floors[b] = fl
        refs[b] = (r, amax)
        ex = np.zeros(len(r))
        ex[ok] = np.abs(o[ok] - r[ok]) / _tol(r[ok], amax, norm, fl)
        worst_full = max(worst_full, float(ex.max()) if len(ex) else 0.0)
        kk = np.flatnonzero(ok)
        if len(kk):
            top = kk[np.argsort(ex[kk])[-N_WORST:]]
            cand += [(float(ex[k]), b, int(k)) for k in top]
    cand.sort(reverse=True)
    picks = {(b, k) for _, b, k in cand[:N_WORST]}
    finite = {b: np.flatnonzero(np.isfinite(refs[b][0])) for b in rows}
    live = [b for b in rows if len(finite[b])]
    for _ in range(N_RANDOM if live else 0):
        b = live[int(rng.integers(len(live)))]
        picks.add((b, int(finite[b][int(rng.integers(len(finite[b])))])))
    worst_oracle, worst_ref = 0.0, 0.0
    for b in sorted({b for b, _ in picks}):
        ks = np.array(sorted(k for bb, k in picks if bb == b))
        o = _norm(ols.ls_slow_psd(times[b], y64[b], fr[b][ks]), norm, len(times[b]), scale)
        r, amax = refs[b]
        tol = _tol(o, amax, norm, floors[b])
        worst_oracle = max(worst_oracle, float(np.max(np.abs(np.asarray(out[b], np.float64)[ks] - o) / tol)))
        worst_ref = max(worst_ref, float(np.max(np.abs(r[ks] - o) / _tol(o, amax, norm))))
    print("%-58s worst excess: all bins vs fp64 kernel %.3g, picked bins vs oracle %.3g (reference itself %.2g)"
          % (name, worst_full, worst_oracle, worst_ref))
    assert worst_ref < 0.05, (name, "the fp64 reference disagrees with the oracle", worst_ref)
    assert worst_full <= limit and worst_oracle <= limit, (name, worst_full, worst_oracle)
    return worst_full


def rows_of(a):
    return [np.asarray(r) for r in a]


def expect_unsupported(call):
    with pytest.raises(Exception) as ei:
        call()
    assert getattr(ei.value, "status", None) == -5, ei.value


# ============================================================================ shared grid, NUFFT v2 at every PA
SHARED_V2 = [(p, kmax) for p in range(14, 24) for kmax in (2 ** (p - 3) + 1, 2 ** (p - 2))]


def shared_v2_batch(seed, kmax, B=4, N=6000):
    """Regular cadence; the grid's top sits at 0.3 / dt so that a line at 0.42 / dt is above the grid and below the
    Nyquist frequency (the largest grids are oversampled up to 1200x for that).  The first bin is at f T >= 0.5: below,
    the normal equations of the floating-mean fit cancel so badly that even fp64 sums are no reference.  Light curve 0
    is hostile (that line, and only noise in band)."""
    rng = np.random.default_rng(seed)
    t = regular_times(rng, N, gaps=0)
    T = t[-1] - t[0]
    os_ = max(1.0, kmax * DT / (0.3 * T))
    df = 1.0 / (os_ * T)
    k0 = max(1, int(np.ceil(0.5 * os_)))
    F = kmax - k0
    freq = df * (k0 + np.arange(F))
    Y = [hostile(rng, t, 0.42 / DT)] + [flux(rng, t, freq[int(rng.integers(F // 8, F))]) for _ in range(B - 1)]
    return t, np.stack(Y), freq


@pytest.mark.parametrize("p,kmax", SHARED_V2)
def test_shared_nufft_v2_every_transform_size(engine, monkeypatch, p, kmax):
    import torch
    t, Y, freq = shared_v2_batch(100 + p, kmax)
    B, N = Y.shape
    Y32 = Y.astype(np.float32)
    times, fluxes = [t] * B, list(Y32)
    ref = reference(engine, times, fluxes, freq)
    name = "shared v2 p=%d k0+F=%d" % (p, kmax)
    # escalation off: the float2 kernels alone (the hostile light curve against its data-relative floor)
    monkeypatch.setenv("LKB_NUFFT_ESCALATE", "0")
    off = engine.ls_power_shared(t, Y32, freq, "amplitude", algo="nufft")
    assert engine.ls_last_algo() == "nufft" and engine.ls_last_nufft_plan() == shared_plan(kmax) == ("v2", p, p + 1)
    assert engine.ls_last_escalated() == 0
    compare(engine, name + " escalation off", rows_of(off), ref, times, fluxes, freq, data_floor=(0,))
    # every light curve listed: the double2 list kernels at this PA
    monkeypatch.setenv("LKB_NUFFT_ESCALATE", "1e-6")
    full = engine.ls_power_shared(t, Y32, freq, "amplitude", algo="nufft")
    assert engine.ls_last_escalated() == B
    compare(engine, name + " all escalated", rows_of(full), ref, times, fluxes, freq)
    # default threshold: exactly the hostile light curve is escalated
    monkeypatch.delenv("LKB_NUFFT_ESCALATE")
    dflt = engine.ls_power_shared(t, Y32, freq, "amplitude", algo="nufft")
    assert engine.ls_last_escalated() == 1
    assert not np.array_equal(dflt[0], off[0]) and np.array_equal(dflt[1:], off[1:])
    compare(engine, name + " default", rows_of(dflt), ref, times, fluxes, freq)
    # bitwise: batch permutation, device mode
    perm = np.random.default_rng(p).permutation(B)
    out_p = engine.ls_power_shared(t, np.ascontiguousarray(Y32[perm]), freq, "amplitude", algo="nufft")
    assert np.array_equal(out_p, dflt[perm]), name + ": a light curve's row depends on its neighbours"
    dev = engine.ls_power_shared(torch.from_numpy(t).cuda(), torch.from_numpy(Y32).cuda(), torch.from_numpy(freq).cuda(),
                                 "amplitude", algo="nufft")
    torch.cuda.synchronize()
    assert np.array_equal(dev.cpu().numpy(), dflt), name + ": device mode differs from host mode"


def test_shared_nufft_escalation_in_several_rounds(engine, monkeypatch):
    """40 light curves all listed, at most 16 per round: three rounds through the same double2 buffers.  Random
    cadences: on a strictly regular cadence a grid reaching 1 / dt has a bin where every cadence has the same phase,
    where the estimator is 0 / 0."""
    monkeypatch.setenv("LKB_NUFFT_ESCALATE", "1e-6")
    monkeypatch.setenv("LKB_NUFFT_ESCALATE_CAP", "16")
    rng = np.random.default_rng(4)
    t = random_times(rng, 1200, 30.0)
    kmax = 2 ** 13
    df = 1.0 / (5.0 * (t[-1] - t[0]))
    freq = df * (1 + np.arange(kmax - 1))
    Y32 = np.stack([flux(rng, t, freq[int(rng.integers(100, kmax - 1))]) for _ in range(40)]).astype(np.float32)
    ref = reference(engine, [t] * 40, list(Y32), freq)
    out = engine.ls_power_shared(t, Y32, freq, "amplitude", algo="nufft")
    assert engine.ls_last_nufft_plan() == shared_plan(kmax) and engine.ls_last_escalated() == 40
    compare(engine, "shared v2 p=15, 40 escalated in rounds of 16", rows_of(out), ref, [t] * 40, list(Y32), freq)


# ============================================ shared grid, the small grids (k0 + F <= 2048) that were pair-packed
@pytest.mark.parametrize("p_fine", [9, 10, 11, 12, 13])
def test_shared_small_grids_take_v2(engine, p_fine):
    kmax = 2 ** (p_fine - 2)
    rng = np.random.default_rng(p_fine)
    t = random_times(rng, 1500, 30.0)
    df = 1.0 / (5.0 * (t[-1] - t[0]))
    freq = df * (1 + np.arange(kmax - 1))
    amps = [3e-2, 1e-4, 1e-2, 3e-4, 1e-3, 3e-2, 1e-4]             # loud and quiet light curves side by side
    Y32 = np.stack([flux(rng, t, freq[int(rng.integers(0, len(freq)))], amp=a, noise=1e-4) for a in amps]).astype(np.float32)
    B = len(amps)
    out = engine.ls_power_shared(t, Y32, freq, "amplitude", algo="nufft")
    assert engine.ls_last_nufft_plan() == shared_plan(kmax) == ("v2", 14, p_fine + 1)
    compare(engine, "shared small grid k0+F=%d" % kmax, rows_of(out), reference(engine, [t] * B, list(Y32), freq),
            [t] * B, list(Y32), freq)
    perm = np.random.default_rng(1).permutation(B)
    assert np.array_equal(engine.ls_power_shared(t, np.ascontiguousarray(Y32[perm]), freq, "amplitude", algo="nufft"), out[perm])


def test_shared_small_grid_auto(engine):
    """`auto` takes the NUFFT from B N F >= 2.5e7, also on a small grid."""
    rng = np.random.default_rng(8)
    t = random_times(rng, 2000, 30.0)
    df = 1.0 / (5.0 * (t[-1] - t[0]))
    freq = df * (1 + np.arange(256))
    Y32 = np.stack([flux(rng, t, freq[int(rng.integers(0, 256))]) for _ in range(64)]).astype(np.float32)
    out = engine.ls_power_shared(t, Y32, freq, "amplitude")
    assert engine.ls_last_algo() == "nufft" and engine.ls_last_nufft_plan() == shared_plan(257)
    compare(engine, "shared auto, 64 x 2000 x 256", rows_of(out), reference(engine, [t] * 64, list(Y32), freq), [t] * 64,
            list(Y32), freq)


def test_shared_small_grid_partner_pair(engine, monkeypatch):
    """A quiet light curve (noise 1e-4, one 3e-3 outlier) next to a loud one (3e-2 line at bin F / 2): the pair-packed
    round-1 transform left the quiet one 1.2x / 1.9x over the tolerance next to the partner's line, depending on the
    order.  Now its row is bitwise the same in either order and alone."""
    monkeypatch.setenv("LKB_NUFFT_ESCALATE", "0")
    rng = np.random.default_rng(3)
    N, F = 6000, 1000
    t = random_times(rng, N, 30.0)
    df = 1.0 / (5.0 * (t[-1] - t[0]))
    freq = df * (1 + np.arange(F))
    quiet = 1 + 1e-4 * rng.normal(size=N)
    quiet[N // 3] += 3e-3
    loud = 1 + 3e-2 * np.sin(2 * np.pi * freq[F // 2] * t + 0.3) + 1e-7 * rng.normal(size=N)
    Y32 = np.stack([quiet, loud]).astype(np.float32)
    a = engine.ls_power_shared(t, Y32, freq, "amplitude", algo="nufft")
    assert engine.ls_last_nufft_plan() == ("v2", 14, 13)
    b = engine.ls_power_shared(t, np.ascontiguousarray(Y32[::-1]), freq, "amplitude", algo="nufft")
    alone = engine.ls_power_shared(t, Y32[:1], freq, "amplitude", algo="nufft")
    assert np.array_equal(a[0], b[1]) and np.array_equal(a[0], alone[0]) and np.array_equal(a[1], b[0])
    compare(engine, "shared partner pair (quiet, loud)", rows_of(a), reference(engine, [t, t], list(Y32), freq), [t, t],
            list(Y32), freq)


@pytest.mark.parametrize("kmax", [2049, 2 ** 16, 2 ** 18])
def test_shared_pipeline_equals_one_shot(engine, monkeypatch, kmax):
    """Host mode with 513 light curves: chunks of 64, 64, 128, 256 and a last chunk of 1, on two streams."""
    rng = np.random.default_rng(kmax)
    t = random_times(rng, 300, 30.0)
    df = 1.0 / (5.0 * (t[-1] - t[0]))
    freq = df * (1 + np.arange(kmax - 1))
    Y32 = (1 + 1e-3 * np.sin(2 * np.pi * freq[kmax // 3] * t)[None, :]
           + 10 ** rng.uniform(-4, -3, (513, 1)) * rng.normal(size=(513, len(t)))).astype(np.float32)
    a = engine.ls_power_shared(t, Y32, freq, "amplitude", algo="nufft")
    assert engine.ls_last_nufft_plan() == shared_plan(kmax)
    monkeypatch.setenv("LKB_LS_NO_PIPELINE", "1")
    b = engine.ls_power_shared(t, Y32, freq, "amplitude", algo="nufft")
    assert np.array_equal(a, b)
    sub = [0, 63, 64, 255, 256, 511, 512]
    compare(engine, "shared pipelined, 513 light curves, k0+F=%d" % kmax, rows_of(a[sub]),
            reference(engine, [t] * len(sub), list(Y32[sub]), freq), [t] * len(sub), list(Y32[sub]), freq)


# ======================================================================= grid edges, both NUFFT entries
EDGES = {                                  # (k0, F, oversample)
    "k0=0 (f = 0 row)": (0, 500, 5.0),
    "k0=20 (no low rows)": (20, 500, 5.0),
    "all low rows": (1, 9, 5.0),
    "first bin at f T = 2": (10, 500, 5.0),
    "oversample 1 (wrap-around)": (1, 700, 1.0),
}


def _scale(N, os_, df):
    return 2.0 / (N * os_ * df)


@pytest.mark.parametrize("edge", list(EDGES))
def test_nufft_grid_edges(engine, edge):
    k0, F, os_ = EDGES[edge]
    rng = np.random.default_rng(len(edge))
    # shared entry
    t = random_times(rng, 800, 25.0)
    T = t[-1] - t[0]
    df = 1.0 / (os_ * T)
    freq = df * (k0 + np.arange(F))
    Y = np.stack([flux(rng, t, freq[min(F - 1, 3 * F // 4)]) for _ in range(3)])
    c = 1 if k0 == 0 else 0          # f = 0: the estimator is 0 / 0 (NaN where the oracle's is, left out of the sweep)
    for dt in (np.float32, np.float64):
        Yd = Y.astype(dt)
        ref = reference(engine, [t] * 3, list(Yd), freq[c:])
        for norm in ("amplitude", "psd", "psd_raw"):
            sc = _scale(len(t), os_, df)
            out = engine.ls_power_shared(t, Yd, freq, norm, norm_scale=sc if norm == "psd" else None, algo="nufft")
            assert engine.ls_last_nufft_plan() == shared_plan(k0 + F)
            if c:
                nan0 = np.array([np.isnan(ols.ls_slow_psd(t, Yd[b].astype(np.float64), freq[:1]))[0] for b in range(3)])
                assert np.isnan(out[nan0, 0]).all()
            compare(engine, "shared %s, %s, %s" % (edge, dt.__name__, norm), rows_of(out[:, c:]), ref, [t] * 3, list(Yd),
                    freq[c:], norm=norm, scale=sc)
    # ragged entry: own times per light curve, df * baseline <= 1 for the longest
    times = [random_times(rng, n, s) for n, s in ((900, 25.0), (400, 18.0), (1300, 22.0))]
    df = 1.0 / (os_ * max(x[-1] - x[0] for x in times))
    freq = df * (k0 + np.arange(F))
    fl = [flux(rng, x, freq[min(F - 1, F // 2)]) for x in times]
    for dt in (np.float32, np.float64):
        fd = [f.astype(dt) for f in fl]
        ref = reference(engine, times, fd, freq[c:])
        for norm in ("amplitude", "psd", "psd_raw"):
            sc = 1.7
            out = engine.ls_power_ragged(times, fd, freq, norm, norm_scale=sc if norm == "psd" else None, algo="nufft")
            assert engine.ls_last_algo() == "nufft" and engine.ls_last_nufft_plan() == ragged_plan(k0 + F)
            if c:
                nan0 = np.array([np.isnan(ols.ls_slow_psd(times[b], fd[b].astype(np.float64), freq[:1]))[0] for b in range(3)])
                assert np.isnan(out[nan0, 0]).all()
            compare(engine, "ragged %s, %s, %s" % (edge, dt.__name__, norm), rows_of(out[:, c:]), ref, times, fd,
                    freq[c:], norm=norm, scale=sc)


# ================================================================================= ragged NUFFT, every size
RAGGED_V2 = [2048, 2049] + [2 ** (p - 2) for p in range(15, 23)]


def ragged_batch(seed, kmax, ns=(1500, 900, 2000), k0=1):
    rng = np.random.default_rng(seed)
    times = [random_times(rng, n, rng.uniform(20.0, 30.0)) for n in ns]
    df = 1.0 / (5.0 * max(x[-1] - x[0] for x in times))
    F = kmax - k0
    freq = df * (k0 + np.arange(F))
    fl = [flux(rng, x, freq[int(rng.integers(F // 8, F))]).astype(np.float32) for x in times]
    return times, fl, freq


@pytest.mark.parametrize("kmax", RAGGED_V2)
def test_ragged_nufft_every_transform_size(engine, kmax):
    import torch
    times, fl, freq = ragged_batch(kmax, kmax)
    out = engine.ls_power_ragged(times, fl, freq, "amplitude", algo="nufft")
    assert engine.ls_last_algo() == "nufft" and engine.ls_last_nufft_plan() == ragged_plan(kmax)
    compare(engine, "ragged v2 k0+F=%d plan %s" % (kmax, ragged_plan(kmax)[1:]), rows_of(out),
            reference(engine, times, fl, freq), times, fl, freq)
    perm = [2, 0, 1]
    out_p = engine.ls_power_ragged([times[i] for i in perm], [fl[i] for i in perm], freq, "amplitude", algo="nufft")
    assert np.array_equal(out_p, out[perm])
    offs = np.concatenate([[0], np.cumsum([len(x) for x in times])]).astype(np.int64)
    dev = engine.ls_power_ragged_device(torch.from_numpy(np.concatenate(times)).cuda(),
                                        torch.from_numpy(np.concatenate(fl)).cuda(), offs, torch.from_numpy(freq).cuda(),
                                        "amplitude", algo="nufft")
    torch.cuda.synchronize()
    assert np.array_equal(dev.cpu().numpy(), out)


@pytest.mark.parametrize("kmax", [2 ** 20 + 1, 2 ** 21, 2 ** 21 + 1])
def test_ragged_nufft_beyond_the_v2_range(engine, kmax):
    """k0 + F > 2^20: the window grid would need 2^24 cells or more.  algo="nufft" is refused; `auto` runs the direct
    kernel."""
    times, fl, freq = ragged_batch(kmax, kmax, ns=(1000, 700, 1100))
    expect_unsupported(lambda: engine.ls_power_ragged(times, fl, freq, "amplitude", algo="nufft"))
    out = engine.ls_power_ragged(times, fl, freq, "amplitude")
    assert engine.ls_last_algo() == "simt"
    compare(engine, "ragged auto, k0+F=%d -> direct" % kmax, rows_of(out), reference(engine, times, fl, freq), times, fl,
            freq)


def test_ragged_nufft_groups_of_one(engine, monkeypatch):
    monkeypatch.setenv("LKB_NUFFT_RAGGED_MB", "0.5")
    times, fl, freq = ragged_batch(7, 2049, ns=(900, 8, 1500, 300, 1200))      # odd batch; one light curve of 8 cadences
    out = engine.ls_power_ragged(times, fl, freq, "amplitude", algo="nufft")
    assert engine.ls_last_nufft_plan() == ragged_plan(2049)
    compare(engine, "ragged v2, groups of one, 8 cadences", rows_of(out), reference(engine, times, fl, freq), times, fl,
            freq)


def test_ragged_nufft_ineligible_light_curves(engine):
    """7 cadences, or a zero baseline: algo="nufft" is refused, `auto` runs the direct kernel for the whole call."""
    times, fl, freq = ragged_batch(9, 8001, ns=(2000, 7, 2500))
    expect_unsupported(lambda: engine.ls_power_ragged(times, fl, freq, "amplitude", algo="nufft"))
    out = engine.ls_power_ragged(times, fl, freq, "amplitude")
    assert engine.ls_last_algo() == "simt"
    compare(engine, "ragged auto, 7 cadences -> direct", rows_of(out), reference(engine, times, fl, freq), times, fl, freq)
    times[1] = np.full(10, 140.0)
    fl[1] = np.linspace(0.99, 1.01, 10).astype(np.float32)
    expect_unsupported(lambda: engine.ls_power_ragged(times, fl, freq, "amplitude", algo="nufft"))
    out = engine.ls_power_ragged(times, fl, freq, "amplitude")
    assert engine.ls_last_algo() == "simt"
    compare(engine, "ragged auto, zero baseline -> direct", rows_of(out), reference(engine, times, fl, freq), times, fl,
            freq, skip=(1,))


# ================================================================================== direct ragged kernel
DIRECT_NS = (767, 768, 769, 1535, 1536, 1537, 1001, 1002, 1003)


def direct_batch(seed, ns=DIRECT_NS, span=25.0):
    rng = np.random.default_rng(seed)
    times = [random_times(rng, n, span) for n in ns]
    fl = [flux(rng, x, rng.uniform(0.5, 3.0)).astype(np.float32) for x in times]
    return rng, times, fl


@pytest.mark.parametrize("F", [31, 32, 33])
@pytest.mark.parametrize("grid", ["regular", "irregular"])
def test_direct_tiles_and_blocks(engine, F, grid):
    rng, times, fl = direct_batch(F)
    if grid == "regular":
        freq = 0.01 + 0.1 * np.arange(F)
    else:
        freq = np.sort(rng.uniform(0.01, 3.5, F))
    out = engine.ls_power_ragged(times, fl, freq, "amplitude", algo="direct")
    assert engine.ls_last_algo() == "simt"
    compare(engine, "direct, %s grid, F=%d, N in %s" % (grid, F, DIRECT_NS[::3]), rows_of(out),
            reference(engine, times, fl, freq), times, fl, freq)


@pytest.mark.parametrize("one_irregular", [False, True])
def test_direct_per_light_curve_grids(engine, one_irregular):
    """Grids of 1, 31, 200 and 64 bins with their own f0 and df; with one irregular grid the whole call takes fp64
    phases."""
    rng, times, fl = direct_batch(11, ns=(900, 1536, 769, 2000))
    grids = [np.array([1.3]), 0.05 + 0.07 * np.arange(31), 0.2 + 0.011 * np.arange(200), 0.01 + 0.04 * np.arange(64)]
    if one_irregular:
        grids[2] = np.sort(rng.uniform(0.1, 2.5, 200))
    out = engine.ls_power_ragged(times, fl, grids, "amplitude", algo="direct")
    assert engine.ls_last_algo() == "simt"
    compare(engine, "direct, per-light-curve grids%s" % (", one irregular" if one_irregular else ""), out,
            reference(engine, times, fl, grids), times, fl, grids)


def test_direct_warp_straddles_the_low_rows(engine):
    """Bins from f T = 1.5 to 9.4 in steps of 0.125: the warp of bins 2 .. 5 holds f T = 1.75 .. 2.125."""
    rng = np.random.default_rng(12)
    times = []
    for n in (1000, 1537, 700):
        x = np.sort(rng.uniform(0.0, 25.0, n))
        x[0], x[-1] = 0.0, 25.0
        times.append(131.5 + x)
    fl = [flux(rng, x, 0.2).astype(np.float32) for x in times]
    freq = (1.5 + 0.125 * np.arange(64)) / 25.0
    out = engine.ls_power_ragged(times, fl, freq, "amplitude", algo="direct")
    compare(engine, "direct, warp across f T = 2", rows_of(out), reference(engine, times, fl, freq), times, fl, freq)


def test_direct_kepler_baseline_high_frequencies(engine):
    """A 1470-day baseline at 359 .. 360 / d: phases of 5e5 cycles, the fixed-point phase a + k b at large k."""
    rng = np.random.default_rng(13)
    times = [random_times(rng, n, 1470.0) for n in (5000, 3001)]
    df = 1.0 / (5.0 * 1470.0)
    freq = 359.0 + df * np.arange(int(round(1.0 / df)))
    fl = [flux(rng, x, freq[len(freq) // 3] + 0.3 * df, amp=3e-3).astype(np.float32) for x in times]
    out = engine.ls_power_ragged(times, fl, freq, "amplitude", algo="direct")
    assert engine.ls_last_algo() == "simt"
    compare(engine, "direct, Kepler baseline, 359-360 / d", rows_of(out), reference(engine, times, fl, freq), times, fl,
            freq)


# =========================================================================== shared grid, contraction kernels
CONTRACTION = [(63, 512, 128), (64, 512, 128), (65, 512, 129), (127, 256, 127), (128, 2048, 128), (129, 2049, 129),
               (127, 2047, 256), (64, 255, 200), (64, 256, 200), (65, 1023, 130), (65, 1025, 130)]


@pytest.mark.parametrize("B,N,F", CONTRACTION)
@pytest.mark.parametrize("grid", ["regular", "irregular"])
def test_contraction_kernels(engine, B, N, F, grid):
    rng = np.random.default_rng(B * 7 + N + F)
    t = random_times(rng, N, 30.0)
    if grid == "regular":
        df = 1.0 / (5.0 * (t[-1] - t[0]))
        freq = df * (1 + np.arange(F))
    else:
        freq = np.sort(rng.uniform(0.01, 4.0, F))
    Y32 = np.stack([flux(rng, t, rng.uniform(0.05, 3.5)) for _ in range(B)]).astype(np.float32)
    ref = reference(engine, [t] * B, list(Y32), freq)
    for algo in ("simt", "tcgen05"):
        if algo == "tcgen05" and not (B >= 64 and N >= 256 and F >= 128):
            expect_unsupported(lambda: engine.ls_power_shared(t, Y32, freq, "amplitude", algo="tcgen05"))
            continue
        out = engine.ls_power_shared(t, Y32, freq, "amplitude", algo=algo)
        assert engine.ls_last_algo() == algo
        compare(engine, "%s, %s grid, B=%d N=%d F=%d" % (algo, grid, B, N, F), rows_of(out), ref, [t] * B, list(Y32), freq)
