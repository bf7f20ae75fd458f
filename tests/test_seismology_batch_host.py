"""The batched ACF2D estimators (seismology.estimate_numax_acf2d_batch / estimate_deltanu_acf2d_batch) on the host:
the GPU autocorrelation (engine.acf_windows) is replaced, in this file only, by a numpy stand-in that runs the
loop's np.correlate on the same windows.  What is checked is everything around the kernel - validation, window
placement (numpy's slicing, wrap-around included), the per-series batching and the smoothing / argmax /
diagnostics - against the per-periodogram host estimators."""
import numpy as np
import pytest

from lightkurve_b200 import engine
from lightkurve_b200 import units as u
from lightkurve_b200.periodogram import SNRPeriodogram
from lightkurve_b200.seismology import (estimate_deltanu_acf2d, estimate_deltanu_acf2d_batch, estimate_numax_acf2d,
                                        estimate_numax_acf2d_batch)
from test_seismology import generate_test_spectrum


def red_giant_snr(rng, numax, F=5664, fs=0.05, f0=None, unit=u.microhertz):
    """Seeded SNR spectrum of a red giant: chi^2 (2 dof) noise times (1 + a Gaussian envelope of radial / dipole /
    quadrupole Lorentzian modes at 0.294 numax^0.772 spacing) on the grid f_k = f0 + k fs (f0 defaults to fs)."""
    f = (fs if f0 is None else f0) + fs * np.arange(F)
    dnu = 0.294 * numax ** 0.772
    sig = 0.66 * numax ** 0.88 / 2.355
    modes = np.concatenate([numax + dnu * (np.arange(-8, 9) + eps) for eps in (0.0, 0.5, -0.12)])
    height = np.concatenate([np.full(17, h) for h in (1.0, 1.2, 0.6)])
    comb = np.zeros(F)
    for m, h in zip(modes, height):
        comb += h / (1 + ((f - m) / 0.08) ** 2)
    env = 30.0 * np.exp(-0.5 * ((f - numax) / sig) ** 2)
    p = rng.exponential(size=F) * (1 + env * comb)
    fq = u.Quantity(f, u.microhertz)
    if unit != u.microhertz:
        fq = fq.to(unit)
    return SNRPeriodogram(fq, u.Quantity(p, None))


def numpy_acf_windows(series, starts, lengths, return_acf=False):
    """Stand-in for engine.acf_windows: the loop's own arithmetic on every window."""
    metrics, acfs = [], []
    for x, st, n in zip(series, starts, lengths):
        a = np.zeros((len(st), n))
        for k, s in enumerate(st):
            sel = np.array(x[s:s + n], dtype=float)
            sel -= np.nanmean(sel)
            a[k] = np.correlate(sel, sel, mode="full")[n - 1:]
        metrics.append((np.sum(np.abs(a), axis=1) - 1) / n)
        acfs.append(a)
    return (metrics, acfs) if return_acf else metrics


@pytest.fixture
def host_acf(monkeypatch):
    calls = []

    def fake(series, starts, lengths, return_acf=False):
        calls.append(len(series))
        return numpy_acf_windows(series, starts, lengths, return_acf)

    monkeypatch.setattr(engine, "acf_windows", fake)
    return calls


def _ms(unit=u.microhertz, chop=None):
    f, p, _, _ = generate_test_spectrum()
    pg = SNRPeriodogram(u.Quantity(f, u.microhertz), u.Quantity(p, None))
    if chop is not None:
        pg = pg[(pg.frequency.value > chop[0]) & (pg.frequency.value < chop[1])]
    if unit != u.microhertz:
        pg = SNRPeriodogram(pg.frequency.to(unit), pg.power)
    return pg


def assert_numax_equal(got, ref, acf2d=False):
    assert got.value == ref.value and got.unit == ref.unit
    assert (got.name, got.method) == (ref.name, ref.method)
    d, r = got.diagnostics, ref.diagnostics
    assert set(d) == set(r)
    np.testing.assert_array_equal(d["numaxs"], r["numaxs"])
    assert d["window_width"] == r["window_width"]
    np.testing.assert_array_equal(d["metric"], r["metric"])
    np.testing.assert_array_equal(d["metric_smooth"], r["metric_smooth"])
    if acf2d:
        assert d["acf2d"].shape == r["acf2d"].shape
        np.testing.assert_array_equal(d["acf2d"], r["acf2d"])
    else:
        assert d["acf2d"] is None


def assert_deltanu_equal(got, ref):
    assert got.value == ref.value and got.unit == ref.unit
    assert (got.name, got.method) == (ref.name, ref.method)
    for k in ("lags", "acf", "peaks", "sel"):
        np.testing.assert_array_equal(got.diagnostics[k], ref.diagnostics[k])
    assert got.diagnostics["deltanu_emp"] == ref.diagnostics["deltanu_emp"]


def test_batch_equals_loop_defaults_and_units(host_acf):
    """Red giants and main-sequence spectra, in microhertz and 1/day, a chopped periodogram (f0 > 0): one call."""
    rng = np.random.default_rng(1)
    pgs = [red_giant_snr(rng, 60.0), red_giant_snr(rng, 140.0, unit=1 / u.day), _ms(), _ms(unit=1 / u.day),
           _ms(chop=(1600, 3200)), red_giant_snr(rng, 95.0, F=3000, f0=40.0)]
    got = estimate_numax_acf2d_batch(pgs, return_acf2d=True)
    assert host_acf == [len(pgs)]
    for g, pg in zip(got, pgs):
        assert_numax_equal(g, estimate_numax_acf2d(pg), acf2d=True)
    plain = estimate_numax_acf2d_batch(pgs)
    for g, pg in zip(plain, pgs):
        assert_numax_equal(g, estimate_numax_acf2d(pg))
    dn = estimate_deltanu_acf2d_batch(pgs, got)
    for d, pg, nm in zip(dn, pgs, got):
        assert_deltanu_equal(d, estimate_deltanu_acf2d(pg, nm))
    assert abs(got[0].value - 60.0) < 6 and abs(got[1].to(u.microhertz).value - 140.0) < 14


def test_batch_equals_loop_custom_arguments(host_acf):
    rng = np.random.default_rng(2)
    pgs = [red_giant_snr(rng, 80.0), red_giant_snr(rng, 120.0)]
    numaxs = np.linspace(40.0, 200.0, 77)
    for kw in (dict(numaxs=numaxs), dict(window_width=18.0), dict(spacing=2.5), dict(numaxs=numaxs[:7]),
               dict(numaxs=u.Quantity(numaxs, u.microhertz).to(1 / u.day), window_width=30.0, spacing=1.5)):
        got = estimate_numax_acf2d_batch(pgs, return_acf2d=True, **kw)
        for g, pg in zip(got, pgs):
            assert_numax_equal(g, estimate_numax_acf2d(pg, **kw), acf2d=True)


def test_wrapped_window_is_reproduced(host_acf):
    """A trial numax far below the first bin of a chopped spectrum: both slice ends are negative, numpy wraps the
    window to the end of the array with its full length, and the loop accepts it."""
    pg = _ms(chop=(1000, 4000))
    numaxs = [200.0, 2500.0]
    ref = estimate_numax_acf2d(pg, numaxs=numaxs)
    got = estimate_numax_acf2d_batch([pg, pg], numaxs=numaxs, return_acf2d=True)
    for g in got:
        assert_numax_equal(g, estimate_numax_acf2d(pg, numaxs=numaxs), acf2d=True)
    F, fs = len(pg.frequency), np.median(np.diff(pg.frequency.value))
    spread = int(250.0 / 2 / fs)
    centre = int(200.0 / fs) - int(pg.frequency.value[0] / fs)
    assert centre + spread < 0
    np.testing.assert_array_equal(ref.diagnostics["acf2d"][:, 0] != 0, True)
    tail = np.array(pg.power.value[F + centre - spread:F + centre + spread])
    tail -= tail.mean()
    np.testing.assert_allclose(got[0].diagnostics["acf2d"][:, 0], np.correlate(tail, tail, "full")[len(tail) - 1:])


def test_truncated_numax_window_raises_like_the_loop(host_acf):
    rng = np.random.default_rng(3)
    good, pg = red_giant_snr(rng, 80.0, F=6000), red_giant_snr(rng, 80.0, F=3000, f0=40.0)
    top = pg.frequency.value[-1]
    for numaxs in ([60.0, top - 3.0], [pg.frequency.value[0] + 5.0, 100.0]):
        with pytest.raises(ValueError):
            estimate_numax_acf2d(pg, numaxs=numaxs)
        with pytest.raises(ValueError, match=r"periodogram 1\b"):
            estimate_numax_acf2d_batch([good, pg], numaxs=numaxs)
    assert host_acf == []                       # refused before any autocorrelation
    with pytest.raises(ValueError, match="uniformly spaced"):
        f = np.sort(np.random.default_rng(0).uniform(1, 200, 2000))
        estimate_numax_acf2d_batch([good, SNRPeriodogram(u.Quantity(f, u.microhertz), u.Quantity(np.ones(2000), None))])
    for kw in (dict(window_width=-5.0), dict(window_width=1e6), dict(spacing=0.001), dict(numaxs=[-1.0, 50.0]),
               dict(numaxs=[50.0, 1e5])):
        with pytest.raises(ValueError):
            estimate_numax_acf2d(good, **kw)
        with pytest.raises(ValueError):
            estimate_numax_acf2d_batch([good, pg], **kw)


def test_truncated_deltanu_window_gives_the_loops_shorter_acf(host_acf):
    """A numax near the top of the spectrum: the deltanu window runs past the last bin and numpy's slice is shorter."""
    rng = np.random.default_rng(4)
    pgs = [red_giant_snr(rng, 250.0, F=5300), red_giant_snr(rng, 100.0)]
    numaxs = [u.Quantity(pgs[0].frequency.value[-1] - 4.0, u.microhertz), 100.0]
    got = estimate_deltanu_acf2d_batch(pgs, numaxs)
    refs = [estimate_deltanu_acf2d(pg, nm) for pg, nm in zip(pgs, numaxs)]
    for g, r in zip(got, refs):
        assert_deltanu_equal(g, r)
    full = 2 * int(2 * int(np.floor(0.66 * numaxs[0].value ** 0.88)) / 2 / 0.05)
    assert len(refs[0].diagnostics["acf"]) < full
    with pytest.raises(ValueError, match="one numax per periodogram"):
        estimate_deltanu_acf2d_batch(pgs, numaxs[:1])
    with pytest.raises(ValueError):
        estimate_deltanu_acf2d_batch(pgs, [100.0, 1e5])


def test_engine_groups_by_byte_budget(monkeypatch):
    """engine.acf_windows splits the batch into groups of series under its staging budget, in order."""
    from lightkurve_b200 import _lib
    calls = []

    class FakeLib:
        def lkb_acf_windows(self, x, xo, B, wo, ws, wl, metric, acf, mem, stream):
            calls.append(B)
            return 0

    monkeypatch.setattr(_lib, "load", lambda: FakeLib())
    monkeypatch.setattr(engine, "ACF_STAGE_BYTES", 8 * 3000)
    series = [np.ones(1000)] * 5
    m, a = engine.acf_windows(series, [np.arange(3)] * 5, [100] * 5, return_acf=True)
    assert calls == [2, 2, 1]
    assert [x.shape for x in a] == [(3, 100)] * 5 and [len(x) for x in m] == [3] * 5
