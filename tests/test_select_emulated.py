"""The K6 order statistics (lightkurve_b200/csrc/select.cuh) executed on the CPU through tests/native/cuda_emu.h, with
the block sizes their callers use (256: flatten, nanmedian_std; 512: the regression sigma clip), on the inputs the
sampling select is built around: ties at the ends of its bracket, a bracket of one value, more candidates than its
buffer holds, brackets that miss, NaN on the sample positions, infinities, signed zeros, subnormals and values near
DBL_MAX.

Medians must equal np.nanmedian exactly (`==`, or both NaN).  `==` treats -0.0 and 0.0 as equal: the selects order
-0.0 before 0.0 (they compare raw bit patterns) where numpy's partition treats them as one value, so the sign of a zero
median may differ.  Standard deviations must agree with np.nanstd to rtol 1e-12.

Each case also checks which branch it took (tests/native/select_emu_driver.cpp reports it):
  observed   the one partition pass ran, and its observer saw every index exactly once (after the last reset), with the
             element's own value and a lower value lo <= median;
  resets     a stale caller bracket was detected and the pass repeated after reset();
  gets       reads of the data: about n for the sampling path, about 10 n when it fell back to the 8-pass radix select
             (candidate-buffer overflow or a bracket miss);
  bracket    a bracket left valid holds the returned median."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
CUDA_INC = "/usr/local/cuda/include"
c_vp, c_int = ctypes.c_void_p, ctypes.c_int
FS_SAMPLE, FS_GAP, FS_CAP = 2048, 64, 5632            # select.cuh
DBL_MAX = np.finfo(np.float64).max
MODE_RADIX, MODE_FAST, MODE_BRACKET = 0, 1, 2


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    out = str(tmp_path_factory.mktemp("emu") / "libselect_emu.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-pthread", "-I" + CUDA_INC, "-Wno-attributes", "-shared", "-fPIC",
                           "-Wl,-Bsymbolic", "-o", out, os.path.join(HERE, "native", "select_emu_driver.cpp")])
    lib = ctypes.CDLL(out)
    lib.emu_select.argtypes = [c_vp, c_vp, c_int, c_int, c_int, c_int] + [c_vp] * 15
    lib.emu_select.restype = c_int
    return lib


def run(emu, arrays, mode, threads, pass_m=False, brackets=None):
    """One launch, one CTA per array.  brackets: per array (lo, hi) or None (no valid bracket)."""
    B = len(arrays)
    off = np.zeros(B + 1, np.int64)
    np.cumsum([len(a) for a in arrays], out=off[1:])
    x = np.ascontiguousarray(np.concatenate(arrays).astype(np.float64)) if off[-1] else np.zeros(1)
    brackets = [None] * B if brackets is None else brackets
    blo = np.array([np.nan if br is None else br[0] for br in brackets])
    bhi = np.array([np.nan if br is None else br[1] for br in brackets])
    bval = np.array([br is not None for br in brackets], np.int32)
    r = {k: np.full(B, np.nan) for k in ("med", "sd", "obs_lo", "br_lo", "br_hi")}
    r.update({k: np.full(B, -1, np.int32) for k in ("observed", "resets", "br_valid")})
    r.update({k: np.full(B, -1, np.int64) for k in ("gets", "obs_calls", "obs_bad")})
    seen = np.zeros(max(int(off[-1]), 1), np.int32)
    emu.emu_select(x.ctypes.data, off.ctypes.data, B, threads, mode, int(pass_m), blo.ctypes.data, bhi.ctypes.data,
                   bval.ctypes.data, *[r[k].ctypes.data for k in ("med", "sd", "observed", "resets", "gets",
                                                                  "obs_calls", "obs_bad", "obs_lo", "br_lo", "br_hi",
                                                                  "br_valid")], seen.ctypes.data)
    r["seen"] = [seen[off[b]:off[b + 1]] for b in range(B)]
    return r


def check_values(arrays, r, check_std=None):
    for b, a in enumerate(arrays):
        ref = np.nanmedian(a) if np.any(~np.isnan(a)) else np.nan
        got = r["med"][b]
        assert got == ref or (np.isnan(got) and np.isnan(ref)), "array %d (n=%d): median %r, numpy %r" % (
            b, len(a), got, ref)
        if check_std is None or check_std[b]:
            sref = np.nanstd(a) if np.any(~np.isnan(a)) else np.nan
            np.testing.assert_allclose(r["sd"][b], sref, rtol=1e-12, atol=0, equal_nan=True,
                                       err_msg="array %d (n=%d): std" % (b, len(a)))


def check_observer(arrays, r):
    for b, a in enumerate(arrays):
        assert r["obs_bad"][b] == 0, "array %d: the observer saw a value other than the element's" % b
        if r["observed"][b]:
            assert np.all(r["seen"][b] == 1), "array %d: observer counts %s" % (b, np.unique(r["seen"][b]))
            assert r["obs_calls"][b] == len(a)
            assert r["obs_lo"][b] <= r["med"][b] or np.isnan(r["med"][b])
        if r["br_valid"][b]:
            assert r["br_lo"][b] <= r["med"][b] <= r["br_hi"][b], (b, r["br_lo"][b], r["med"][b], r["br_hi"][b])


def took_fast_path(r, b, n):
    """The partition pass ran and its buffer answered: no radix-select fallback (which reads the data ~10 more times)."""
    return bool(r["observed"][b]) and r["gets"][b] <= 2 * n + 2 * FS_SAMPLE


def fell_back(r, b, n):
    return r["gets"][b] >= 5 * n


def sample_positions(n):
    return np.arange(FS_SAMPLE) * (n // FS_SAMPLE)


# ---------------------------------------------------------------- data
def make(kind, n, seed):
    rng = np.random.default_rng(seed)
    x = rng.normal(size=n)
    if kind == "normal":
        return x
    if kind == "sorted":
        return np.sort(x)
    if kind == "quant3":
        return rng.integers(0, 3, n).astype(np.float64)
    if kind == "quant50":
        return rng.integers(0, 50, n) / 7.0
    if kind == "two_values":
        # an even count split 50/50: the two middle order statistics are distinct (median 2.5, not a data value)
        x = np.where(np.arange(n) < n // 2, 2.0, 3.0)
        return rng.permutation(x)
    sp = np.unique(sample_positions(n))                # (n < FS_SAMPLE: index 0 only)
    if kind == "sample_extreme":                        # the sample brackets everything: candidate overflow
        x[sp] = np.where(np.arange(len(sp)) % 2, 1e300, -1e300)
        return x
    if kind == "sample_high":                           # the sample's bracket is one value far above the median
        x[sp] = 1e300
        return x
    if kind == "sample_const":                          # one value (lo == hi) above the median
        x[sp] = 2.0
        return x
    if kind == "sample_nan":                            # no usable sample
        x[sp] = np.nan
        return x
    if kind == "nan90":
        x[rng.random(n) < 0.9] = np.nan
        return x
    if kind == "all_nan":
        return np.full(n, np.nan)
    if kind == "inf30":
        u = rng.random(n)
        x[u < 0.15] = -np.inf
        x[u > 0.85] = np.inf
        return x
    if kind == "inf_median":
        x[rng.random(n) < 0.6] = np.inf
        return x
    if kind == "zeros_subnormal":
        vals = np.array([-0.0, 0.0, 5e-324, -5e-324, 2.2e-308, -1e-310, 1e-310, 3e-320])
        return rng.choice(vals, n)
    if kind == "dbl_max":
        vals = np.array([-DBL_MAX, -0.9 * DBL_MAX, -1.0, 0.0, 1.0, 0.9 * DBL_MAX, DBL_MAX, np.nextafter(DBL_MAX, 0)])
        return rng.choice(vals, n)
    if kind == "spike":
        # more than FS_CAP distinct values strictly inside the sample's bracket: 97 % of the other positions within
        # 1e-12 of the sample's median (the sample itself stays normal, so its bracket is ~0.16 sigma wide)
        m = np.median(x[sp])
        k = rng.random(n) < 0.97
        k[sp] = False
        x[k] = m + 1e-12 * (rng.random(int(k.sum())) - 0.5)
        return x
    raise ValueError(kind)


KINDS = ["normal", "sorted", "quant3", "quant50", "two_values", "sample_extreme", "sample_high", "sample_const",
         "sample_nan", "nan90", "all_nan", "inf30", "inf_median", "zeros_subnormal", "dbl_max", "spike"]
# std over values near DBL_MAX overflows in the sum of squares (or the sum) in an order-dependent way: not compared
NO_STD = {"dbl_max"}
# the kinds whose sample brackets the median with few enough values inside
FAST_KINDS = ["normal", "sorted", "quant3", "quant50", "two_values", "inf30", "inf_median", "zeros_subnormal", "dbl_max"]


# ---------------------------------------------------------------- tests
@pytest.mark.parametrize("threads", [256, 512])
def test_small_arrays(emu, threads):
    """n = 1, 2, 3 on the radix select and on the fast variant (which must hand these sizes to the radix select
    without calling its observer)."""
    kinds = ["normal", "quant3", "two_values", "all_nan", "inf30", "inf_median", "zeros_subnormal", "dbl_max"]
    arrays = [make(k, n, 10 * i + n) for i, k in enumerate(kinds) for n in ((1, 2, 3) if threads == 256 else (3,))]
    arrays += [np.array([-0.0, 0.0]), np.array([0.0, -0.0, -0.0]), np.array([np.nan, 1.0]), np.array([np.inf, -np.inf]),
               np.array([np.inf, np.inf, 1.0]), np.zeros(0)]
    r = run(emu, arrays, MODE_RADIX if threads == 256 else MODE_FAST, threads)
    check_values(arrays, r)
    check_observer(arrays, r)
    assert not r["observed"].any() and not r["obs_calls"].any()


@pytest.mark.parametrize("kind", KINDS)
def test_kinds_at_sampling_sizes(emu, kind):
    """Every kind at n = 8192 = 4 FS_SAMPLE (the first size that samples), 65 000 (a Kepler light curve) and one of
    8191 (radix select only), 8193 and 12 288, through the fast variant at 512 threads; and, where that variant answers
    from its buffer, at 65 000 through the radix select at 256 threads (the other kinds reach it as the fallback)."""
    ns = [(8191, 8193, 12288)[KINDS.index(kind) % 3], 8192, 65000]
    arrays = [make(kind, n, 1000 + n) for n in ns]
    std_ok = [kind not in NO_STD] * len(arrays)
    rf = run(emu, arrays, MODE_FAST, 512)
    check_values(arrays, rf, std_ok)
    check_observer(arrays, rf)
    if kind in FAST_KINDS:
        rr = run(emu, arrays[2:], MODE_RADIX, 256)
        check_values(arrays[2:], rr, std_ok[2:])
        assert not rr["observed"].any()
    if ns[0] < 4 * FS_SAMPLE:                                      # n = 8191: below the sampling threshold
        assert not rf["observed"][0]
    big = [b for b in range(3) if ns[b] >= 4 * FS_SAMPLE]
    if kind in FAST_KINDS:
        for b in big:
            assert took_fast_path(rf, b, ns[b]), (kind, ns[b], rf["gets"][b])
    if kind in ("sample_nan", "all_nan", "nan90"):                 # fewer than 4 FS_GAP usable samples: radix select
        assert not rf["observed"][big].any()
    if kind in ("sample_extreme", "spike"):                         # lo <= median, candidate overflow: observed, fallback
        for b in big:
            assert rf["observed"][b] and not rf["br_valid"][b] and fell_back(rf, b, ns[b]), (kind, ns[b], rf["gets"][b])
    if kind in ("sample_high", "sample_const"):                     # the bracket misses above the median: the pass ran,
        for b in big:                                               # but obs had no lower bound - not `observed`
            assert not rf["observed"][b] and fell_back(rf, b, ns[b]), (kind, ns[b], rf["gets"][b])


def test_bracket_one_value_at_the_median(emu):
    """The sample's bracket is one value (lo == hi) holding the median, with many values equal to it on both sides of
    the median rank: odd and even counts (the two middle values both in the eq-lo block)."""
    rng = np.random.default_rng(5)
    arrays = []
    for n in (8192, 65001):
        x = rng.normal(size=n)
        x[rng.random(n) < 0.3] = np.median(x)
        arrays.append(x)
    arrays.append(rng.permutation(np.repeat([1.0, 2.0, 3.0], [30000, 5000, 30000])))     # median on a 5000-value tie
    r = run(emu, arrays, MODE_FAST, 512)
    check_values(arrays, r)
    check_observer(arrays, r)
    for b, a in enumerate(arrays):
        assert took_fast_path(r, b, len(a))


@pytest.mark.parametrize("threads,pass_m", [(256, True), (512, False)])
def test_caller_brackets(emu, threads, pass_m):
    """The caller's bracket: valid (no sample, no restart), stale (median outside: reset, then a fresh sample),
    degenerate lo == hi on the median value itself (odd count: valid) and elsewhere (stale); with the count of
    non-NaN values given (m_known, as flatten does) or counted in the pass (as the clip does)."""
    rng = np.random.default_rng(9)
    cases = []
    for n in (8193, 65000):
        x = rng.normal(size=n)
        x[rng.random(n) < 0.05] = np.nan
        if np.count_nonzero(~np.isnan(x)) % 2 == 0:               # an odd count: the median is a data value
            x[np.flatnonzero(~np.isnan(x))[0]] = np.nan
        s = np.sort(x[~np.isnan(x)])
        m = len(s)
        cases.append((x, (s[m // 2 - 300], s[m // 2 + 300]), "valid"))
        cases.append((x, (s[m // 2 + 50], s[m // 2 + 900]), "stale"))
        cases.append((x, (s[0] - 2.0, s[0] - 1.0), "stale"))
        cases.append((x, (s[m // 2], s[m // 2]), "valid"))
        cases.append((x, (s[m // 4], s[m // 4]), "stale"))
    arrays = [c[0] for c in cases]
    r = run(emu, arrays, MODE_BRACKET, threads, pass_m=pass_m, brackets=[c[1] for c in cases])
    check_values(arrays, r)
    check_observer(arrays, r)
    for b, (x, br, what) in enumerate(cases):
        assert r["observed"][b], (b, what)
        if what == "valid":
            assert r["resets"][b] == 0 and r["gets"][b] == len(x), (b, r["resets"][b], r["gets"][b])
            assert r["br_valid"][b] and (r["br_lo"][b], r["br_hi"][b]) == br
        else:
            assert r["resets"][b] == 1, (b, what, r["resets"][b])
            assert r["gets"][b] >= 2 * len(x)


def test_bracket_left_behind_is_reused(emu):
    """The bracket a call leaves behind (valid: it holds the median) answers a second call on slightly changed data
    without a sample or a restart - the regression clip's round-to-round reuse."""
    rng = np.random.default_rng(13)
    arrays = [rng.normal(size=n) for n in (8192, 65000)]
    r1 = run(emu, arrays, MODE_BRACKET, 512)
    check_values(arrays, r1)
    assert r1["br_valid"].all() and (r1["resets"] == 0).all()
    changed = []
    for a in arrays:
        a = a.copy()
        a[rng.choice(len(a), len(a) // 200, replace=False)] = np.nan                  # a clip round strikes 0.5 %
        changed.append(a)
    r2 = run(emu, changed, MODE_BRACKET, 512, brackets=list(zip(r1["br_lo"], r1["br_hi"])))
    check_values(changed, r2)
    check_observer(changed, r2)
    assert (r2["resets"] == 0).all() and (r2["gets"] == [len(a) for a in changed]).all()


def test_candidate_overflow_falls_back(emu):
    """More than FS_CAP values strictly inside the bracket: the partition pass is observed, the bracket is left
    invalid, and the radix select answers."""
    arrays = [make("spike", n, 77 + n) for n in (8192, 65000)]
    r = run(emu, arrays, MODE_BRACKET, 256)
    check_values(arrays, r)
    check_observer(arrays, r)
    for b, a in enumerate(arrays):
        assert r["observed"][b] and not r["br_valid"][b] and fell_back(r, b, len(a))
