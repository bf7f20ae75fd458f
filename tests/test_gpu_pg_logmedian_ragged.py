"""The log-median background kernels of csrc/pgops.cu on per-periodogram grids (lkb_pg_logmedian_ragged,
engine.pg_logmedian_ragged) and on one shared grid (lkb_pg_logmedian):
  - ragged grids (host and device mode, fp64 and fp32 power) against oracle.pg.smooth_logmedian;
  - the kernels' own arithmetic restated in numpy (exact window medians, then median * (1 / corr) accumulated by
    fused multiply-adds over the covering windows in ascending order, divided by their count), which both entries must equal bit for bit: this
    pins the shared-grid entry to the arithmetic it had before it became a case of the ragged kernels;
  - B copies of one grid through the ragged entry equal the shared entry bit for bit;
  - the SNR output is power / background bit for bit; a periodogram with no window gets NaN."""
import warnings
from fractions import Fraction

import numpy as np
import pytest
import torch

from lightkurve_b200 import engine as eng
from oracle import pg as opg

pytestmark = pytest.mark.gpu


def _fma(a, b, c):
    """a * b + c rounded once (the kernels are compiled with contraction, so the sum is a fused multiply-add)."""
    if not (np.isfinite(a) and np.isfinite(b) and np.isfinite(c)):
        return a * b + c
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def kernel_arith(freq, power, fw):
    lo, hi = eng.logmedian_windows(freq, fw)
    inv = 1.0 / (8.0 / 9.0) ** 3
    acc = [0.0] * len(freq)
    cnt = np.zeros(len(freq))
    p = np.asarray(power, dtype=np.float64)
    for a, b in zip(lo, hi):
        if b <= a:
            continue
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)
            m = float(np.nanmedian(p[a:b]))
        for i in range(a, b):
            acc[i] = _fma(m, inv, acc[i])
        cnt[a:b] += 1
    with np.errstate(all="ignore"):
        return np.asarray(acc) / cnt


def grids(rng):
    g = [(np.arange(2000) + 1) * 0.0137, np.sort(rng.uniform(0.01, 300, 777)), 2.5 + np.arange(40) * 0.5,
         (np.arange(9000) + 1) * 0.31, np.array([1.0, 2.0])]
    pw = [rng.chisquare(2, size=len(f)) * (1 + 5.0 / (1 + f)) for f in g]
    pw[0][5] = np.nan
    return g, pw


def test_ragged_against_the_oracle_and_the_kernel_arithmetic(engine):
    rng = np.random.default_rng(3)
    g, pw = grids(rng)
    for fw in (0.01, 0.1):
        bkg, snr = eng.pg_logmedian_ragged(g, pw, fw, snr=True)
        for f, p, b_, s_ in zip(g, pw, bkg, snr):
            np.testing.assert_allclose(b_, opg.smooth_logmedian(f, p, fw), rtol=1e-13, equal_nan=True)
            np.testing.assert_array_equal(b_, kernel_arith(f, p, fw))
            with np.errstate(all="ignore"):
                np.testing.assert_array_equal(s_, p / b_)


def test_device_mode_and_fp32_power(engine):
    rng = np.random.default_rng(4)
    g, pw = grids(rng)
    pw32 = [p.astype(np.float32) for p in pw]
    cat, off = eng._csr(pw32, np.float32)
    d = torch.from_numpy(cat).cuda()
    bkg, snr = eng.pg_logmedian_ragged(g, d, 0.01, bin_offsets=off, snr=True)
    bkg, snr = bkg.cpu().numpy(), snr.cpu().numpy()
    host = eng.pg_logmedian_ragged(g, [p.astype(np.float64) for p in pw32], 0.01)
    for k, (f, p) in enumerate(zip(g, pw32)):
        sl = slice(off[k], off[k + 1])
        np.testing.assert_array_equal(bkg[sl], host[k])
        np.testing.assert_array_equal(bkg[sl], kernel_arith(f, p.astype(np.float64), 0.01))
        with np.errstate(all="ignore"):
            np.testing.assert_array_equal(snr[sl], p.astype(np.float64) / bkg[sl])


def test_copies_of_one_grid_equal_the_shared_entry(engine):
    rng = np.random.default_rng(5)
    F, B = 20000, 5
    f = (np.arange(F) + 1) * 0.0137
    power = rng.chisquare(2, size=(B, F)) * (1 + 5.0 / (1 + f))
    power[0, 5] = np.nan
    shared = eng.pg_logmedian(f, power, 0.01)
    ragged = eng.pg_logmedian_ragged([f] * B, list(power), 0.01)
    for b in range(B):
        np.testing.assert_array_equal(ragged[b], shared[b])
        np.testing.assert_array_equal(shared[b], kernel_arith(f, power[b], 0.01))


def test_no_window_anywhere(engine):
    # a grid of one frequency has no window (x0 < log10 f[-1] never holds): the background is NaN
    bkg = eng.pg_logmedian_ragged([np.array([3.0]), np.array([5.0])], [np.array([1.0]), np.array([2.0])], 0.01)
    assert np.isnan(bkg[0]).all() and np.isnan(bkg[1]).all()
