"""Inputs shared by the K11/K12 tests on the CPU emulator (tests/test_clip_cdpp_emulated.py) and on the GPU
(tests/test_gpu_cdpp.py): sigma-clip cases with their clip parameters, and light curves for the CDPP."""
import numpy as np

# resident in shared memory up to this many cadences (clip.cuh: CL_RES_CAP)
RES_CAP = 20480


def _dips(rng, n, k, lo=2.0, hi=80.0, width=30):
    x = rng.normal(size=n)
    for s in rng.choice(n - width, k, replace=False):
        x[s:s + width] -= np.exp(rng.uniform(np.log(lo), np.log(hi)))
    return x


def clip_cases():
    """[(name, x, sigma_lower, sigma_upper, maxiters)]; maxiters None = until a round clips nothing."""
    rng = np.random.default_rng(2026)
    out = []
    x = rng.normal(size=20000)
    x[rng.choice(20000, 200, replace=False)] += rng.exponential(6.0, 200)
    x[::997] = np.nan
    out.append(("flares", x, 3.0, 3.0, 5))
    x = _dips(rng, 20000, 60)                          # one-sided deep dips: the median moves between rounds
    x[::997] = np.nan
    out.append(("deep_dips", x, 3.0, 3.0, 5))
    out.append(("deep_dips_sigma5", x, 5.0, 5.0, 5))
    out.append(("deep_dips_maxiters1", x, 3.0, 3.0, 1))
    out.append(("deep_dips_converged", x, 3.0, 3.0, None))
    out.append(("deep_dips_maxiters0", x, 3.0, 3.0, 0))
    x = rng.normal(size=5000) * 1e-3 + 1.0
    x[100:180] = np.nan
    x[rng.choice(5000, 20, replace=False)] = np.inf
    x[rng.choice(5000, 20, replace=False)] = -np.inf
    x[rng.choice(5000, 30, replace=False)] += 0.02
    out.append(("nan_inf", x, 5.0, 5.0, 5))
    x = _dips(rng, 12000, 30)
    x[rng.choice(12000, 100, replace=False)] += rng.exponential(6.0, 100)
    out.append(("asymmetric", x, 2.0, 4.0, 5))
    out.append(("lower_inf", x, np.inf, 3.0, None))
    out.append(("upper_inf", x, 3.0, np.inf, 5))
    x = np.round(2.0 * rng.normal(size=9000))          # integers: ties at the median
    x[rng.choice(9000, 90, replace=False)] += 15.0
    out.append(("quantised", x, 3.0, 3.0, 5))
    out.append(("constant", np.full(3000, 1.5), 3.0, 3.0, 5))
    out.append(("empty", np.zeros(0), 3.0, 3.0, 5))
    out.append(("no_finite", np.full(40, np.nan), 3.0, 3.0, 5))
    x = np.full(40, np.nan)
    x[7] = 2.5
    out.append(("one_finite", x, 3.0, 3.0, 5))
    x[30] = -1.0
    out.append(("two_finite", x, 1.0, 1.0, None))
    x = rng.normal(size=300)
    x[:3] += 40.0
    out.append(("short", x, 3.0, 3.0, 5))
    # streamed from global memory: one cadence past the shared-memory capacity, and a Kepler long-cadence length
    x = _dips(rng, RES_CAP + 1, 60)
    x[rng.choice(RES_CAP + 1, 200, replace=False)] += rng.exponential(6.0, 200)
    out.append(("stream_dips", x, 3.0, 3.0, 5))
    x = rng.normal(size=65000)
    x[rng.choice(65000, 650, replace=False)] += rng.exponential(6.0, 650)
    x[1000:1400] = np.nan
    out.append(("stream_kepler", x, 3.0, 3.0, None))
    return out


def light_curve(rng, n, noise_ppm, kind="plain", cadence=2.0 / 1440):
    """(time, flux) of n cadences: a slow trend, white noise, and per `kind` a box transit, flares, NaN runs and
    gaps in time."""
    t = 1325.0 + np.arange(n) * cadence
    if kind in ("gaps", "everything"):
        t = t + np.where(np.arange(n) > n // 2, 1.5, 0.0) + np.where(np.arange(n) > n // 4, 0.3, 0.0)
    f = 1.0 + 2e-3 * np.sin(2 * np.pi * (t - t[0]) / 7.3) + noise_ppm * 1e-6 * rng.normal(size=n)
    if kind in ("transit", "everything"):
        per = rng.uniform(1.0, 4.0)
        f[np.abs((t - t[0] - 0.4 + 0.5 * per) % per - 0.5 * per) < 0.06] -= 10 ** rng.uniform(-3.5, -2.5)
    if kind in ("flares", "everything"):
        k = rng.choice(n, max(1, n // 300), replace=False)
        f[k] += rng.exponential(20 * noise_ppm * 1e-6, len(k))
    if kind in ("nans", "everything"):
        s = rng.integers(0, max(1, n - 60))
        f[s:s + 50] = np.nan
        f[rng.choice(n, max(1, n // 500), replace=False)] = np.nan
    return t, f
