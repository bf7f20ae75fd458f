"""Inputs, the fp64 oracle and the tolerance checks of the multi-term (nterms 1..4) Lomb-Scargle tests, shared by
tests/test_gpu_chi2_paths.py (GPU) and tests/test_nufft_chi2_emulated.py (the NUFFT path on the CPU emulator).

Oracle: astropy's lombscargle_chi2 (oracle/ls.py:ls_chi2_psd - fit_mean = center_data = True, dy = 1, psd) restated
for many bins at once: the design matrix [1, sin(2 pi j f t), cos(2 pi j f t)] (j <= nterms) in fp64 from t - t[0] with
the phase f t reduced to [0, 1) cycles first, its normal matrix X^T X, X^T y of the centred flux, one fp64 solve per
bin, and the condition number of X^T X.  A bin whose normal matrix is exactly singular (f = 0, or fewer cadences than
parameters) gives NaN, as ls_chi2_psd does through LinAlgError.

Tolerances are stated on the returned quantity X (power or amplitude) of every bin whose condition number is at most
COND_MAX, as |X - X_ref| <= a max(X_ref) + r X_ref; the worst ratio of the two sides ("excess") is printed and must be
<= 1.  Worse-conditioned bins are only required to be finite or NaN (never +-inf)."""
import numpy as np

from oracle import ls as ols

COND_MAX = 1e6
V2_P_MIN = 14             # smallest v2 fine grid (nufft_v2.cuh V2R_P_MIN)
V2_P_MAX = 23
LS_WARPS = 8              # ls.cu: frequency bins per block of the direct kernel (one per warp)
TOL_DIRECT = (1e-9, 1e-7)     # fp64 direct sums, fp32 output
TOL_NUFFT = (1e-5, 1e-4)      # the parity tolerance of the NUFFT family (amplitude spectrum)
N_WORST, N_RANDOM = 500, 200


# ------------------------------------------------------------------------------------------------------ plans
def fine_log2(kmax):
    """nufft_core.h fine_grid_log2 at upsampling 2: the smallest p >= 4 with 2^p >= 4 kmax."""
    p = 4
    while (1 << p) < 4 * kmax:
        p += 1
    return p


def chi2_plan(nterms, kmax):
    """("v2", p, p2) of ls_nufft_chi2_ragged_launch for the grid f_k = (k0 + k) df with k0 + F = kmax."""
    return ("v2", max(fine_log2(nterms * kmax), V2_P_MIN), max(fine_log2(2 * nterms * kmax), V2_P_MIN))


# ------------------------------------------------------------------------------------------------------ inputs
def irregular_times(rng, n, span, t0=1300.0):
    return t0 + np.sort(rng.uniform(0.0, span, n))


def cadence_times(rng, n, dt=2.0 / 1440.0, gap=0.2, t0=2000.0):
    """A strictly regular cadence (TESS 2-min by default) from a random start with one data gap of `gap` of the span."""
    t = t0 + rng.uniform(0, 1) + np.arange(int(n * (1 + gap))) * dt
    if len(t) == n:
        return t
    g0 = int(rng.integers(n // 8, n // 2))
    return np.delete(t, np.arange(g0, g0 + len(t) - n))


def signal(rng, t, f1, amp, noise=None, mean=1.0):
    """A non-sinusoidal signal (three harmonics) of fundamental f1 plus white noise (of a random level in [1e-4, 1e-3]
    by default)."""
    ph = 2 * np.pi * f1 * (t - t[0]) + rng.uniform(0, 2 * np.pi)
    noise = 10 ** rng.uniform(-4, -3) if noise is None else noise
    return mean + amp * (np.sin(ph) + 0.5 * np.cos(2 * ph + 0.3) + 0.25 * np.sin(3 * ph + 1.1)) \
        + noise * rng.normal(size=len(t))


def batch(kind, ns, seed):
    """Light curves of lengths `ns`: "irregular" (random times over 10-25 d, fundamentals 0.3-3 / d) or "tess" (2-min
    cadence with a gap, fundamentals 3-30 / d); signals of very different strengths."""
    rng = np.random.default_rng(seed)
    times, fluxes = [], []
    for b, n in enumerate(ns):
        if kind == "irregular":
            t = np.sort(rng.uniform(0, 25.0 * rng.uniform(0.4, 1.0), n))
        else:
            t = cadence_times(rng, n, gap=0.25)
        f1 = rng.uniform(0.3, 3.0) if kind == "irregular" else rng.uniform(3.0, 30.0)
        times.append(t)
        fluxes.append(signal(rng, t, f1, [1e-2, 1e-3, 3e-3, 1e-4, 5e-3][b % 5]))
    return times, fluxes


def hostile(rng, t, f_above):
    """A loud line above the frequency grid and only noise in band."""
    return 1 + 8e-3 * np.sin(2 * np.pi * f_above * t + 0.4) + 2e-4 * rng.normal(size=len(t))


def layout(times, fluxes):
    """The K1 prologue's layout of a ragged batch, as the NUFFT launcher takes it: times relative to each light curve's
    first cadence, the centred flux in fp32, padded CSR offsets (multiples of 4), span and sum of the fp32 flux."""
    B = len(times)
    off = np.zeros(B + 1, np.int64)
    poff = np.zeros(B + 1, np.int64)
    for b, t in enumerate(times):
        off[b + 1] = off[b] + len(t)
        poff[b + 1] = poff[b] + ((len(t) + 3) // 4) * 4
    ptotal = int(poff[-1])
    tt, yy = np.zeros(ptotal + 4), np.zeros(ptotal + 4, np.float32)
    span, ysum = np.zeros(B), np.zeros(B)
    for b, (t, y) in enumerate(zip(times, fluxes)):
        n = len(t)
        tr = t - t[0]
        yc = (np.asarray(y, np.float64) - np.mean(y)).astype(np.float32)
        tt[poff[b]:poff[b] + n] = tr
        yy[poff[b]:poff[b] + n] = yc
        span[b] = tr.max()
        ysum[b] = yc.astype(np.float64).sum()
    return dict(B=B, off=off, poff=poff, ptotal=ptotal, tt=tt, yy=yy, times=list(times), fluxes=list(fluxes),
                span=span, ysum=ysum, nmax=max(len(t) for t in times))


# ------------------------------------------------------------------------------------------------------ oracle
def _design(tr, f, nterms):
    """[len(f), n, 2 nterms + 1] design matrices, phases reduced to cycles in [0, 1) before the harmonics."""
    ph = np.multiply.outer(f, tr) % 1.0
    X = np.empty(ph.shape + (2 * nterms + 1,))
    X[..., 0] = 1.0
    for j in range(1, nterms + 1):
        a = (2 * np.pi * j) * ph
        X[..., 2 * j - 1] = np.sin(a)
        X[..., 2 * j] = np.cos(a)
    return X


def oracle(t, y, freq, nterms, theta=False):
    """psd_raw power (astropy lombscargle_chi2), the condition number of every bin's normal matrix and, with `theta`,
    the fitted parameters [offset, sin 1, cos 1, ...] of the centred flux (NaN where the normal matrix is singular)."""
    t = np.asarray(t, np.float64)
    freq = np.atleast_1d(np.asarray(freq, np.float64))
    M, n, F = 2 * nterms + 1, len(t), len(freq)
    P, cond, th = np.full(F, np.nan), np.full(F, np.inf), np.full((F, M), np.nan)
    if n == 0:
        return (P, cond, th) if theta else (P, cond)
    tr = t - t[0]
    y64 = np.asarray(y, np.float64)
    yc = y64 - y64.mean()
    chunk = max(1, int(4e6 // (n * M)))
    for i0 in range(0, F, chunk):
        X = _design(tr, freq[i0:i0 + chunk], nterms)
        A = np.matmul(X.transpose(0, 2, 1), X)
        rhs = np.matmul(yc, X)
        with np.errstate(all="ignore"):
            cond[i0:i0 + chunk] = np.linalg.cond(A)
        for i in range(len(A)):
            try:
                s = np.linalg.solve(A[i], rhs[i])
            except np.linalg.LinAlgError:
                continue
            th[i0 + i] = s
            P[i0 + i] = 0.5 * rhs[i] @ s
    return (P, cond, th) if theta else (P, cond)


def oracle_longdouble(t, y, f, nterms):
    """One bin in extended precision (np.longdouble design matrix, sums and Gaussian elimination): the arbiter where
    the kernel and the fp64 oracle disagree."""
    ld = np.longdouble
    tr = np.asarray(t, ld) - ld(t[0])
    y = np.asarray(y, ld)
    yc = y - y.sum() / ld(len(y))
    ph = (ld(f) * tr) % ld(1)
    cols = [np.ones(len(tr), ld)]
    two_pi = 2 * np.arccos(ld(-1))
    for j in range(1, nterms + 1):
        cols += [np.sin(two_pi * j * ph), np.cos(two_pi * j * ph)]
    X = np.stack(cols, axis=1)
    A = X.T @ X
    rhs = X.T @ yc
    M = len(rhs)
    Ab = np.concatenate([A, rhs[:, None]], axis=1)
    for c in range(M):
        piv = c + int(np.argmax(np.abs(Ab[c:, c])))
        Ab[[c, piv]] = Ab[[piv, c]]
        for r in range(c + 1, M):
            Ab[r] -= Ab[r, c] / Ab[c, c] * Ab[c]
    s = np.zeros(M, ld)
    for c in range(M - 1, -1, -1):
        s[c] = (Ab[c, M] - Ab[c, c + 1:M] @ s[c + 1:]) / Ab[c, c]
    return float(ld(0.5) * (rhs @ s)), s.astype(np.float64)


def normalise(P, norm, n, scale=1.0):
    """lightkurve's rescale of the psd_raw power (ls_common.cuh ls_normalize)."""
    if norm == "amplitude":
        with np.errstate(invalid="ignore"):
            return np.sqrt(P) * np.sqrt(4.0 / n)
    return P * scale if norm == "psd" else P


# ------------------------------------------------------------------------------------------------------ checks
def excess(got, ref, cond, tol):
    """Worst |got - ref| / (a max(ref) + r ref) over the bins with cond <= COND_MAX (0 if none), the index of that
    bin, and the number of bins left out.  The bins left out must not be +-inf."""
    got = np.asarray(got, np.float64)
    ref = np.asarray(ref, np.float64)
    good = (np.asarray(cond) <= COND_MAX) & np.isfinite(ref)
    assert not np.isinf(got).any(), "a bin is +-inf"
    if not good.any():
        return 0.0, -1, int((~good).sum())
    a, r = tol
    amax = float(np.max(ref[good]))
    with np.errstate(invalid="ignore", divide="ignore"):
        ex = np.abs(got[good] - ref[good]) / (a * amax + r * ref[good])
    ex[got[good] == ref[good]] = 0.0              # (a zero power, e.g. constant flux, with a zero tolerance)
    ex[np.isnan(ex)] = np.inf                     # a NaN where the oracle is finite and well conditioned
    i = int(np.argmax(ex))
    return float(ex[i]), int(np.flatnonzero(good)[i]), int((~good).sum())


def compare_to_reference(name, out, ref, times, fluxes, freq, nterms, norm="amplitude", scale=None, tol=TOL_NUFFT,
                         seed=17):
    """The NUFFT family against the fp64 direct kernel `ref` on EVERY (light curve, bin), and against the oracle on the
    N_WORST pairs where the two disagree most plus N_RANDOM random pairs.  Every pair over the tolerance against the
    direct kernel must be among the picks; the oracle decides them with the condition-number rule.  The direct kernel
    itself must agree with the oracle on the picked pairs to 1 % of the tolerance.  Returns the worst excesses."""
    out = np.asarray(out, np.float64)
    ref = np.asarray(ref, np.float64)
    a, r = tol
    assert not np.isinf(out).any() and not np.isinf(ref).any(), name
    amax = np.nanmax(np.where(np.isfinite(ref), ref, np.nan), axis=1, keepdims=True)
    with np.errstate(invalid="ignore"):
        d = np.abs(out - ref) / (a * amax + r * ref)
    d[np.isnan(out) != np.isnan(ref)] = np.inf     # NaN in one only: to the oracle
    d[np.isnan(d)] = 0.0                           # NaN in both
    over = int((d > 1.0).sum())
    assert over <= N_WORST, (name, over, "pairs over the tolerance against the direct kernel")
    rng = np.random.default_rng(seed)
    flat = np.argsort(d.ravel())[-N_WORST:]
    flat = np.unique(np.concatenate([flat, rng.choice(d.size, min(N_RANDOM, d.size), replace=False)]))
    bb, kk = np.unravel_index(flat, d.shape)
    worst_oracle, worst_ref, n_bad = 0.0, 0.0, 0
    for b in np.unique(bb):
        ks = kk[bb == b]
        sc = 1.0 if scale is None else scale[b]
        P, cond = oracle(times[b], fluxes[b], freq[ks], nterms)
        o = normalise(P, norm, len(times[b]), sc)
        good = (cond <= COND_MAX) & np.isfinite(o)
        n_bad += int((~good).sum())
        if not good.any():
            continue
        tolb = a * max(float(amax[b, 0]), float(np.max(o[good]))) + r * o[good]
        with np.errstate(invalid="ignore"):
            eo = np.abs(out[b, ks][good] - o[good]) / tolb
            er = np.abs(ref[b, ks][good] - o[good]) / tolb
        eo[np.isnan(eo)] = np.inf
        er[np.isnan(er)] = np.inf
        worst_oracle = max(worst_oracle, float(eo.max()))
        worst_ref = max(worst_ref, float(er.max()))
    worst_full = float(d.max())
    print("%-66s worst excess: vs fp64 direct %.3g (%d over), picked vs oracle %.3g (direct itself %.2g; %d picks "
          "ill-conditioned)" % (name, worst_full, over, worst_oracle, worst_ref, n_bad))
    assert worst_ref < 0.01, (name, "the direct kernel disagrees with the oracle", worst_ref)
    assert worst_oracle <= 1.0, (name, worst_oracle)
    return worst_full, worst_oracle
