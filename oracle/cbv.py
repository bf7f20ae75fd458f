"""numpy restatement of the goodness metrics of CBVCorrector.correct and of its objective (TEST INFRASTRUCTURE).

Follows lightkurve's correctors/metrics.py (overfit_metric_lombscargle :23-123, underfit_metric_neighbors :178-255,
_compute_correlation) and cbvcorrector.py (_goodness_metric_obj_fun :781-854) formula for formula, on arrays: the
tests pin the K9 kernels (lightkurve_b200/csrc/goodness.cuh) and the host code of correct_batch to it.
"""
import numpy as np

BETA = (0.0007, 0.8083, -0.5023)
BAD_LIMIT = 0.95
LEAK = 0.01


def compute_correlation(flux_matrix):
    """_compute_correlation: [nCadences, nTargets] without NaNs -> target-target correlation matrix."""
    n = len(flux_matrix[:, 0])
    rms = np.sqrt(np.sum(flux_matrix ** 2.0, axis=0) / n)
    rms[np.nonzero(rms == 0.0)[0]] = np.inf
    unit = flux_matrix / np.tile(rms, (n, 1))
    return unit.T.dot(unit) / n


def underfit_metric(target, neighbors):
    """The under-fitting metric of one target: `target` [G] and `neighbors` [M, G] on one cadence grid, NaN where a
    value is absent.  Returns (metric, cadences used, nanmean of |c|^3 with the zeroed diagonal)."""
    target = np.asarray(target, dtype=np.float64)
    neighbors = np.atleast_2d(np.asarray(neighbors, dtype=np.float64))
    fm = np.zeros((len(target), len(neighbors) + 1))
    for i, row in enumerate(neighbors):
        fm[:, i] = row
    fm[:, -1] = target
    mask = np.zeros(fm.shape[0], dtype=bool)
    for i in range(fm.shape[1]):
        mask |= np.isnan(fm[:, i])
    fm = fm[~mask, :]
    with np.errstate(divide="ignore", invalid="ignore"):
        cm = compute_correlation(fm)
        n = len(fm[:, 0])
        wgn = BETA[0] + BETA[1] * (float(n) ** BETA[2]) if n > 0 else np.inf
        scale = 1 / wgn * np.log((2.0 / BAD_LIMIT) - 1.0)
        cm = np.tril(cm, k=-1) + np.triu(cm, k=+1)
        c3 = np.nanmean(np.abs(cm) ** 3, axis=0)[-1]
        metric = 2.0 / (1 + np.exp(scale * c3))
    return float(metric), n, float(c3)


def overfit_terms(corrected_power, original_power, noise_powers):
    """(n_positive, sum of the positive changes, [nanmean of each noise power row]) from power rows as the
    periodograms hold them (fp32 values, differences in fp64)."""
    change = np.asarray(corrected_power, dtype=np.float64) - np.asarray(original_power, dtype=np.float64)
    change = change[~np.isnan(change)]
    pos = change[change > 0.0]
    return len(pos), float(np.sum(pos)), [float(np.nanmean(np.asarray(p, dtype=np.float64))) for p in noise_powers]


def overfit_metric(n_positive, sum_positive, noise_means):
    """overfit_metric_lombscargle's mapping of the terms to [0, 1]."""
    per = []
    for m in noise_means:
        if n_positive == 0:
            per.append(0.0)
        else:
            den = n_positive * m
            per.append(np.inf if den == 0 else sum_positive / den)
    with np.errstate(over="ignore"):
        return float(2.0 / (1 + np.exp(np.max([np.mean(per), 0.0]))))


def objective(over, under, target_over, target_under):
    """_goodness_metric_obj_fun's penalty from the two metrics (a metric whose target is <= 0 counts as 1)."""
    if not target_over > 0:
        over = 1.0
    if not target_under > 0:
        under = 1.0
    if target_over > 0 and over >= target_over:
        over = target_over + LEAK * (over - target_over)
    if target_under > 0 and under >= target_under:
        under = target_under + LEAK * (under - target_under)
    return -(over + under)


def tess_like_batch(n=64, N=3000, seed=0):
    """TESS-like targets sharing eight systematic trends (the CBVs) with similar weights, a stellar sinusoid each,
    white noise, on one CCD."""
    import lightkurve_b200 as lk
    from lightkurve_b200 import units as u
    from lightkurve_b200.correctors import CotrendingBasisVectors
    rng = np.random.default_rng(seed)
    t = 2000.0 + np.arange(N) * (2.0 / 1440)
    cad = np.arange(10000, 10000 + N)
    x = np.linspace(-1, 1, N)
    sys = np.stack([x, x ** 2 - 1 / 3, np.sin(2.5 * x), np.cos(4 * x), np.sin(7 * x + 1), np.exp(-((x - 0.3) / 0.1) ** 2),
                    np.tanh(5 * x), np.cos(11 * x)])
    sys = (sys - sys.mean(axis=1, keepdims=True)) / sys.std(axis=1, keepdims=True)     # zero-mean, like real CBVs
    data = {"VECTOR_{}".format(i + 1): sys[i] for i in range(8)}
    data["CADENCENO"] = cad
    cbvs = CotrendingBasisVectors(data, t, cbv_type="SingleScale")
    lcs, injected = [], []
    w0 = rng.normal(scale=400.0, size=8)                 # systematics are common-mode across the CCD
    for b in range(n):
        w = w0 * (1.0 + 0.3 * rng.normal(size=8))
        period = rng.uniform(0.3, 1.0)
        star = 60.0 * np.sin(2 * np.pi * t / period)
        flux = 1e5 + w @ sys + star + rng.normal(scale=25.0, size=N)
        lc = lk.LightCurve(time=t, flux=flux, flux_err=np.full(N, 25.0), cadenceno=cad,
                           flux_unit=u.electron / u.second)
        lc.meta.update(MISSION="TESS", TARGETID=5000 + b, RA=80.0 + rng.uniform(-3, 3), DEC=10.0 + rng.uniform(-3, 3))
        lcs.append(lc)
        injected.append((w @ sys, star))
    return lcs, cbvs, injected
