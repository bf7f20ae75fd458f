"""The fp64 Gram pass that lkb_elasticnet (K8) and lkb_regress_ex (K5) share (`rg_gram_pass` in regress.cu), read back
from workspace slot D and compared with an extended-precision reference; the elastic net's and the exact-invariant
regression's independence of the batch; and the elastic net against oracle/enet.py at N >= 4096.

Which kernel a Gram pass takes (`rg_gram_pass`, restated by `gram_choice` below): with Ka = K + 1 columns ([X | y]) and
ntile = ceil(Ka / 8) DMMA tiles, tb = 4 (ntile <= 20) or 5 and nb5 = ceil(ntile / tb) select
`rg_gram_mma_kernel<nb5, tb>`, one of <1,4> <2,4> <3,4> <4,4> <5,4> <5,5>.  The first pass of a call splits a light
curve's 32-cadence stages over two CTAs when N >= 4096 and either the call is exact (lkb_elasticnet, and lkb_regress_ex
with LKB_REGRESS_EXACT_INVARIANT) or B < 4 SMs; the two CTAs add into a zeroed Gram matrix, which commutes exactly.
LKB_REGRESS_SIMT=1 takes the SIMT kernel `rg_accum_kernel` instead.  lkb_regress's tensor-core first pass (shared X,
B >= 64, N >= 4096, 16 <= K <= 160, not exact) sums with fp64 atomics and has its own accuracy test
(test_regress_paths' "tc" cases); no case here takes it.

The Gram matrices stay in slot D after a call: [B][K+1][K+1], upper triangle, column K = X^T W y, [K][K] = y^T W y.
lkb_elasticnet leaves the unit-weight Gram of the used cadences (the coordinate descent only reads it), lkb_regress_ex
the 1/flux_err^2-weighted Gram of the cadences its last fit used (after niters > 1 the first pass minus the downdate
passes of the clipped rows)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import detrend as odet
from oracle import enet as oen
from test_gpu_enet import batch as enet_batch, check as enet_check

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H100_SMS = 132
EPS = np.finfo(np.float64).eps
U = EPS / 2                                    # unit roundoff of fp64
U_LD = np.finfo(np.longdouble).eps / 2         # of the reference (80-bit on x86-64: 2^-64)
RG_RC = 32                                     # cadences per stage
KERNELS = [(1, 4), (2, 4), (3, 4), (4, 4), (5, 4), (5, 5)]


@pytest.fixture(scope="module")
def engine():
    from lightkurve_b200 import engine as eng
    if eng.device_count() == 0:
        pytest.skip("needs a CUDA device")
    eng.init(0)
    return eng


# ------------------------------------------------------------------ the kernel choice, restated
def gram_choice(B, N, K, first, exact, sms):
    """(kernel, CTAs per light curve) of `rg_gram_pass` without LKB_REGRESS_SIMT: kernel is (nb5, tb) of
    rg_gram_mma_kernel (every K <= 165 fits its tiling)."""
    Ka = K + 1
    ntile = (Ka + 7) // 8
    tb = 4 if ntile <= 20 else 5
    nb5 = (ntile + tb - 1) // tb
    return (nb5, tb), 2 if (first and (exact or B < 4 * sms) and N >= 4096) else 1


def regress_tc_taken(B, N, K, batched, exact):
    """lkb_regress's tensor-core first pass (`regress_tc_supported` and the conditions around it)."""
    return not exact and not batched and B >= 64 and N >= 4096 and 16 <= K <= 160


def resolve_B(B, sms):
    """Batch sizes relative to the SM count are written "4S", "4S-1", "4S+17"."""
    if isinstance(B, int):
        return B
    return 4 * sms + (int(B[2:]) if len(B) > 2 else 0)


# Used-cadence patterns of one light curve per batch entry: (count, where) with where "start", "end", "middle"
# (straddling N / 2); "ragged": a random mask keeping 60-100 %; "all".
FEW = [(n, w) for n in (1, 31, 32, 33) for w in ("start", "end", "middle")]

# (id, entry, B, N, K, options, expected kernel, expected CTAs of the first pass)
#   entry "enet": engine.elasticnet (unit weights); "regress": engine.regress (1/fe^2 weights over a factor of 100)
#   options: batched (per-light-curve X), used (pattern list, cycled over the batch), mix (e-/s and normalised flux
#   alternating in the batch), exact (exact_invariant), niters (regress; default 1)
CASES = [
    # every instantiation at the edges of its K range
    ("enet-k1-n777-mix", "enet", 3, 777, 1, dict(used=["ragged"], mix=True), (1, 4), 1),
    ("regress-k7-n4096-mix", "regress", 5, 4096, 7, dict(used=["ragged"], mix=True), (1, 4), 2),
    ("enet-k8-n4095-batched", "enet", 4, 4095, 8, dict(batched=True, used=["ragged", "all"]), (1, 4), 1),
    ("regress-k31-n4097-batched-exact-niters3", "regress", 3, 4097, 31,
     dict(batched=True, exact=True, niters=3, mix=True), (1, 4), 2),
    ("enet-k32-n4096-mix", "enet", 3, 4096, 32, dict(used=["ragged"], mix=True), (2, 4), 2),
    ("regress-k63-n2000", "regress", 3, 2000, 63, dict(used=["ragged"]), (2, 4), 1),
    ("enet-k64-n4096-batched", "enet", 2, 4096, 64, dict(batched=True, used=["ragged"]), (3, 4), 2),
    ("regress-k95-n4095-mix-niters2", "regress", 2, 4095, 95, dict(mix=True, niters=2), (3, 4), 1),
    ("enet-k96-n3000-mix", "enet", 2, 3000, 96, dict(mix=True), (4, 4), 1),
    ("regress-k127-n4096-batched", "regress", 2, 4096, 127, dict(batched=True, used=["ragged"]), (4, 4), 2),
    ("enet-k128-n4096-mix", "enet", 2, 4096, 128, dict(used=["ragged"], mix=True), (5, 4), 2),
    ("regress-k159-n1000", "regress", 2, 1000, 159, dict(mix=True), (5, 4), 1),
    ("enet-k160-n4096", "enet", 2, 4096, 160, dict(used=["ragged"]), (5, 5), 2),
    ("regress-k165-n4096-batched-niters2", "regress", 2, 4096, 165, dict(batched=True, niters=2, mix=True), (5, 5), 2),
    ("enet-k165-n500-batched", "enet", 3, 500, 165, dict(batched=True, mix=True), (5, 5), 1),
    # the split: N = 4095 / 4096, B on both sides of 4 SMs
    ("enet-k9-n4095-b1", "enet", 1, 4095, 9, {}, (1, 4), 1),
    ("enet-k9-n4096-b1", "enet", 1, 4096, 9, {}, (1, 4), 2),
    ("enet-k9-n4096-b4S-1-mix", "enet", "4S-1", 4096, 9, dict(used=["ragged", "all"], mix=True), (1, 4), 2),
    ("enet-k9-n4096-b4S-mix", "enet", "4S", 4096, 9, dict(used=["ragged", "all"], mix=True), (1, 4), 2),
    ("enet-k9-n4095-b4S-batched", "enet", "4S", 4095, 9, dict(batched=True, used=["ragged"]), (1, 4), 1),
    ("regress-k9-n4096-b4S-1", "regress", "4S-1", 4096, 9, dict(used=["ragged"], mix=True), (1, 4), 2),
    ("regress-k9-n4096-b4S", "regress", "4S", 4096, 9, dict(used=["ragged"], mix=True), (1, 4), 1),
    ("regress-k9-n4096-b4S-exact", "regress", "4S", 4096, 9, dict(used=["ragged"], mix=True, exact=True), (1, 4), 2),
    # one split half empty or tiny: 1, 31, 32, 33 used cadences at the start, the end or straddling the middle
    ("enet-k9-n4096-few", "enet", 12, 4096, 9, dict(used=FEW, mix=True), (1, 4), 2),
    ("regress-k20-n5000-few-exact", "regress", 12, 5000, 20, dict(used=FEW, mix=True, exact=True), (1, 4), 2),
    ("enet-k40-n65000-few-batched", "enet", 4, 65000, 40,
     dict(batched=True, used=[(65, "middle"), (95, "start"), (2049, "end"), (4063, "middle")]), (2, 4), 2),
    # fewer cadences than one stage
    ("enet-k3-n20", "enet", 4, 20, 3, dict(used=["ragged", "all"], mix=True), (1, 4), 1),
    ("regress-k5-n31-batched", "regress", 3, 31, 5, dict(batched=True, mix=True), (1, 4), 1),
]

# a few of the same cases on the SIMT kernel (LKB_REGRESS_SIMT=1, read once per process: run in a child process)
SIMT_CASES = ["enet-k9-n4096-few", "regress-k31-n4097-batched-exact-niters3", "enet-k165-n500-batched"]


def case_by_id(cid):
    return next(c for c in CASES if c[0] == cid)


def test_case_table_matches_the_selection_rules():
    """CPU: every case's expected kernel and split follow from rg_gram_pass's rule at the H100's 132 SMs (and at any
    other SM count, since the large batches are written relative to it); every instantiation is reached with one and
    with two CTAs; no regression case takes the tensor-core first pass."""
    seen = set()
    for sms in (H100_SMS, 114, 8):
        for cid, entry, B, N, K, opt, kernel, ctas in CASES:
            Bv = resolve_B(B, sms)
            exact = entry == "enet" or opt.get("exact", False)
            assert gram_choice(Bv, N, K, True, exact, sms) == (kernel, ctas), (cid, sms)
            if entry == "regress":
                assert not regress_tc_taken(Bv, N, K, opt.get("batched", False), exact), cid
            seen.add((kernel, ctas))
    assert seen == {(k, c) for k in KERNELS for c in (1, 2)}
    # the edges of each instantiation's K range
    for (nb5, tb), ks in zip(KERNELS, ([1, 31], [32, 63], [64, 95], [96, 127], [128, 159], [160, 165])):
        for k in ks:
            assert gram_choice(1, 100, k, True, False, H100_SMS)[0] == (nb5, tb), k
        assert {c[4] for c in CASES if c[6] == (nb5, tb)} >= set(ks)
    # the elastic net's split is decided by N alone; lkb_regress's (not exact) by B too
    for N in (4095, 4096):
        assert len({gram_choice(B, N, 9, True, True, H100_SMS) for B in (1, 527, 528, 545)}) == 1
    assert gram_choice(527, 4096, 9, True, False, H100_SMS)[1] == 2
    assert gram_choice(528, 4096, 9, True, False, H100_SMS)[1] == 1
    assert gram_choice(8, 4096, 9, False, True, H100_SMS)[1] == 1            # downdate passes: one CTA
    assert all(c in CASES for c in map(case_by_id, SIMT_CASES))


# ------------------------------------------------------------------ inputs
def design(rng, N, K):
    """K - 1 random-walk CBV-like columns of scales 0.1 to 10 and the constant column last."""
    V = np.cumsum(rng.normal(size=(N, K - 1)), axis=0) / np.sqrt(N) * 10 ** rng.uniform(-1, 1, K - 1)
    return np.hstack([V, np.ones((N, 1))])


def used_mask(rng, N, pattern):
    if pattern == "all":
        return np.ones(N, bool)
    if pattern == "ragged":
        return rng.random(N) > rng.uniform(0.0, 0.4)
    n, where = pattern
    m = np.zeros(N, bool)
    s = {"start": 0, "end": N - n, "middle": N // 2 - n // 2}[where]
    m[s:s + n] = True
    return m


def make_inputs(case, sms, seed=None):
    cid, entry, B, N, K, opt = case[:6]
    B = resolve_B(B, sms)
    rng = np.random.default_rng(sum(map(ord, cid)) if seed is None else seed)
    batched = opt.get("batched", False)
    X = np.stack([design(rng, N, K) for _ in range(B)]) if batched else design(rng, N, K)
    scale = np.where(np.arange(B) % 2 == 0, 10 ** rng.uniform(4, 5, B), 1.0) if opt.get("mix") else np.ones(B)
    W = rng.normal(size=(B, K)) * 0.01 / np.abs(X).max(axis=-2)
    W[:, -1] = 1.0
    XW = np.einsum("bnk,bk->bn", X, W) if batched else W @ X.T
    Y = scale[:, None] * (XW + 1e-3 * rng.normal(size=(B, N)))
    Y[:, ::97] += 8e-3 * scale[:, None]                               # outliers for the sigma clip
    fe = 1e-3 * scale[:, None] * 10 ** rng.uniform(0, 1, (B, N))      # weights 1/fe^2 over a factor of 100
    pats = opt.get("used", ["all"])
    M = np.stack([used_mask(rng, N, pats[b % len(pats)]) for b in range(B)])
    return dict(X=X, Y=Y, fe=fe, M=M, B=B, N=N, K=K, batched=batched)


def run(engine, case, inp):
    """The entry's call; returns (results, Gram [B][K+1][K+1] read back from slot D)."""
    cid, entry, _, N, K, opt = case[:6]
    B = inp["B"]
    if entry == "enet":
        r = engine.elasticnet(inp["X"], inp["Y"], inp["M"], alpha=1.0, l1_ratio=0.9)
    else:                       # a finite prior keeps the few-cadence systems solvable (it never enters slot D)
        r = engine.regress(inp["X"], inp["Y"], inp["fe"], inp["M"], np.zeros(K), np.full(K, 1e6), sigma=3,
                           niters=opt.get("niters", 1), exact_invariant=opt.get("exact", False))
    return r, engine.ws_read("D", B * (K + 1) ** 2, np.float64).reshape(B, K + 1, K + 1)


def last_fit_rows(case, inp, b):
    """(cadences of the first pass, cadences of the last fit) of light curve b: for niters > 1 the oracle's
    clip after niters - 1 fits removes its outliers, as in test_return_cov_is_the_inverse_of_the_last_fit."""
    entry, K, opt = case[1], case[4], case[5]
    m = inp["M"][b]
    niters = opt.get("niters", 1) if entry == "regress" else 1
    if niters == 1:
        return m, m
    X = inp["X"][b] if inp["batched"] else inp["X"]
    prev = odet.regress(X, inp["Y"][b], inp["fe"][b], m, np.zeros(K), np.full(K, 1e6), sigma=3,
                        niters=niters - 1)["outlier_mask"]
    return m, m & ~prev


def reference(case, inp, b, rows):
    """(G, A): [X | y]^T W [X | y] and sum |x_i x_j w| over `rows`, in long double."""
    X = inp["X"][b] if inp["batched"] else inp["X"]
    Z = np.hstack([X[rows], inp["Y"][b][rows, None]]).astype(np.longdouble)
    w = np.ones(len(Z), np.longdouble) if case[1] == "enet" else 1 / inp["fe"][b][rows].astype(np.longdouble) ** 2
    return (Z * w[:, None]).T @ Z, (np.abs(Z) * w[:, None]).T @ np.abs(Z)


def bound_units(cnt, ctas, removed_per_pass):
    """Worst-case |G - G_exact| / (u sum|x_i x_j w|), u = eps / 2, for the kernels' summation structure.

    A Gram entry is one lane's accumulator, carried through a CTA's whole stages in cadence order: each DMMA step
    (or SIMT FMA) adds exact products with at most one rounding per cadence of the chain, so a chain of r cadences
    contributes r (the chain of a CTA is at most ceil(stages / CTAs) whole 32-cadence stages; padding rows carry weight
    0 and add exact zeros).  Per product: the weight 1/(fe fe) is rounded twice, the weighted operand w x once, and
    the product once if the DMMA does not fuse it (4).  The second CTA's atomic add is one more rounding (1).  Each
    downdate pass adds its own chain of the removed rows, its 4 product roundings and the rounding of G -= acc (5 + r).
    The reference's own error (cnt roundings of 2^-64) is counted too."""
    stages = -(-cnt // RG_RC)
    chain = RG_RC * -(-stages // ctas)
    units = chain + 4 + (1 if ctas == 2 else 0)
    for r in removed_per_pass:
        units += r + 5
    return units + 2 * cnt * U_LD / U


def check_gram(case, inp, G, lcs, stats):
    """Every used upper-triangle entry of the light curves `lcs` within its bound; records the worst error as a
    multiple of eps sum|x_i x_j w_i| per (kernel, CTAs)."""
    kernel, ctas = case[6], case[7]
    K = case[4]
    iu = np.triu_indices(K + 1)
    for b in lcs:
        first, last = last_fit_rows(case, inp, b)
        Gr, _ = reference(case, inp, b, last)
        _, A = reference(case, inp, b, first)                       # downdates: errors scale with every row added
        npass = case[5].get("niters", 1) if case[1] == "regress" else 1
        removed = [int(np.count_nonzero(first & ~last))] * (npass - 1)
        units = bound_units(int(np.count_nonzero(first)), ctas, removed)
        err = np.abs(G[b].astype(np.longdouble) - Gr)[iu]
        scale = (U * A)[iu]
        ratio = np.where(scale > 0, err / np.where(scale > 0, scale, 1), np.where(err > 0, np.inf, 0))
        worst = float(ratio.max())
        key = "%s-%dcta" % (kernel, ctas)
        stats[key] = max(stats.get(key, 0.0), worst / 2)              # in units of eps
        assert worst <= units, "%s lc %d: Gram error %.3g u sum|...| > bound %.0f u (at %s)" % (
            case[0], b, worst, units, np.unravel_index(int(np.argmax(ratio)), ratio.shape))


def sample(B):
    """All light curves of a small batch; of a large one the ends, the middle and a few more."""
    if B <= 16:
        return list(range(B))
    return sorted({0, 1, B // 2 - 1, B // 2, B - 2, B - 1} | set(np.random.default_rng(B).choice(B, 6, replace=False)))


STATS = {}


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_gram_read_back_vs_long_double(engine, case):
    sms = engine.sm_count()
    B = resolve_B(case[2], sms)
    exact = case[1] == "enet" or case[5].get("exact", False)
    assert gram_choice(B, case[3], case[4], True, exact, sms) == (case[6], case[7])
    inp = make_inputs(case, sms)
    _, G = run(engine, case, inp)
    check_gram(case, inp, G, sample(B), STATS)
    print("worst Gram error / (eps sum|x_i x_j w_i|) so far:", {k: round(v, 3) for k, v in sorted(STATS.items())})


@pytest.mark.gpu
def test_gram_bound_catches_a_dropped_cadence_or_stage(engine):
    """The bound is tight enough to see the faults it is meant to catch: against a reference without any ONE of the
    used cadences, or without the stage on either side of the two-CTA split, some entry falls outside it."""
    case = ("enet-k9-n4096-b1-ragged", "enet", 1, 4096, 9, dict(used=["ragged"], mix=True), (1, 4), 2)
    inp = make_inputs(case, engine.sm_count(), seed=77)
    _, G = run(engine, case, inp)
    check_gram(case, inp, G, [0], {})
    rows = inp["M"][0]
    cnt = int(np.count_nonzero(rows))
    units = bound_units(cnt, 2, [])
    Gr, A = reference(case, inp, 0, rows)
    iu = np.triu_indices(10)
    tol = (units * U * A)[iu].astype(np.float64)
    D = (G[0].astype(np.longdouble) - Gr)[iu].astype(np.float64)
    Z = np.hstack([inp["X"][rows], inp["Y"][0][rows, None]])
    # dropping cadence c from the reference shifts entry (i, j) by z_ci z_cj
    shift = np.einsum("ci,cj->cij", Z, Z)[:, iu[0], iu[1]]
    excess = np.max(np.abs(D[None, :] + shift) / tol[None, :], axis=1)
    assert excess.min() > 1, "dropping cadence %d stays within the bound" % int(np.argmin(excess))
    stages = -(-cnt // RG_RC)
    for s in (stages // 2 - 1, stages // 2):                          # the last stage of CTA 0, the first of CTA 1
        sh = shift[s * RG_RC:(s + 1) * RG_RC].sum(axis=0)
        assert np.max(np.abs(D + sh) / tol) > 1, s
    print("Gram error %.3g of the bound; the least-visible dropped cadence exceeds it %.3g-fold"
          % (np.max(np.abs(D) / tol), excess.min()))


_SIMT_SCRIPT = r"""
import sys
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[1] + "/tests")
import numpy as np
from lightkurve_b200 import engine
import test_gpu_gram_pass as t
engine.init(0)
case = t.case_by_id(sys.argv[2])
inp = t.make_inputs(case, engine.sm_count())
_, G = t.run(engine, case, inp)
np.save(sys.argv[3], G)
"""


@pytest.mark.gpu
@pytest.mark.parametrize("cid", SIMT_CASES)
def test_simt_gram_read_back_vs_long_double(engine, tmp_path, cid):
    """The SIMT kernel rg_accum_kernel (one 64 x 64 block per CTA, each thread an 8 x 4 tile summed over every used
    cadence in one chain: one CTA, the same bound)."""
    case = case_by_id(cid)
    out = tmp_path / "gram.npy"
    env = dict(os.environ, LKB_REGRESS_SIMT="1")
    flags = ["-s"] if sys.flags.no_user_site else []
    subprocess.check_call([sys.executable] + flags + ["-c", _SIMT_SCRIPT, ROOT, cid, str(out)], env=env)
    G = np.load(out)
    inp = make_inputs(case, engine.sm_count())
    simt = ("simt",) + case[1:6] + ("simt", 1)
    stats = {}
    check_gram(simt, inp, G, sample(inp["B"]), stats)
    print(cid, stats)


# ------------------------------------------------------------------ batch independence (bitwise)
ENET_FIELDS = ("coefficients", "n_iter", "dual_gap", "converged", "model")


def neighbours(rng, X, B, N, K, batched, fixture):
    """B light curves, `fixture` (X_f, y_f, m_f) at position pos, random neighbours elsewhere."""
    Xf, yf, mf, pos = fixture
    W = rng.normal(size=(B, K)) * 0.01
    W[:, -1] = 1.0
    if batched:
        Xs = np.stack([Xf if b == pos else design(rng, N, K) for b in range(B)])
        XW = np.einsum("bnk,bk->bn", Xs, W)
    else:
        Xs, XW = X, W @ X.T
    Y = 1e4 * (XW + 1e-3 * rng.normal(size=(B, N)))
    M = rng.random((B, N)) > 0.1
    Y[pos], M[pos] = yf, mf
    return Xs, Y, M


@pytest.mark.gpu
@pytest.mark.parametrize("N,K,batched", [(4096, 9, False), (4096, 9, True), (4096, 165, False), (18000, 9, False),
                                         (18000, 165, False)])
def test_elasticnet_bitwise_independent_of_the_batch(engine, N, K, batched):
    """One light curve among B = 1, 4 SMs - 1, 4 SMs and 4 SMs + 17 random neighbours, at a different position each
    time: its Gram matrix, coefficients, n_iter, dual gap, convergence flag and model are bitwise the same.  (A
    per-light-curve X at K = 165 and 4 SMs light curves would take 2.9 GB of host memory: that combination is left to
    the small batches of test_gram_read_back_vs_long_double.)"""
    sms = engine.sm_count()
    rng = np.random.default_rng(N + K + batched)
    X = design(rng, N, K)
    w = rng.normal(size=K) * 0.01 * np.geomspace(1, 1e-2, K)
    w[-1] = 1.0
    yf = 1e4 * (X @ w + 1e-3 * rng.normal(size=N))
    mf = rng.random(N) > 0.2
    kw = dict(alpha=1e-20, l1_ratio=0.01) if K <= 9 else dict(alpha=1.0, l1_ratio=0.9)
    ref, fails = None, []
    for B in (1, 4 * sms - 1, 4 * sms, 4 * sms + 17):
        pos = {1: 0, 4 * sms - 1: 4 * sms - 2, 4 * sms: 2 * sms + 1, 4 * sms + 17: 7}[B]
        Xs, Y, M = neighbours(rng, X, B, N, K, batched, (X, yf, mf, pos))
        r = engine.elasticnet(Xs, Y, M, **kw)
        G = engine.ws_read("D", B * (K + 1) ** 2, np.float64).reshape(B, K + 1, K + 1)
        got = {k: r[k][pos].copy() for k in ENET_FIELDS}
        got["gram"] = np.triu(G[pos])
        del Xs, Y, M, r, G
        if ref is None:
            ref = got
            continue
        diffs = []
        for k in ("gram",) + ENET_FIELDS:
            a, b = np.asarray(got[k]), np.asarray(ref[k])
            if not np.array_equal(a, b):
                d = np.abs(a.astype(np.float64) - b.astype(np.float64))
                diffs.append("%s in %d entries, by up to %.3g (relative %.3g)" % (
                    k, np.count_nonzero(a != b), d.max(), np.max(d / np.maximum(np.abs(b.astype(np.float64)),
                                                                                  1e-300))))
        if diffs:
            fails.append("B = %d (position %d) against B = 1: %s" % (B, pos, "; ".join(diffs)))
    assert not fails, "\n".join(fails)


def _corrector(X, y, cbvs=None):
    import lightkurve_b200 as lk
    from lightkurve_b200 import units as u
    from lightkurve_b200.correctors import CBVCorrector, CotrendingBasisVectors
    N = len(y)
    cad = np.arange(100, 100 + N)
    lc = lk.LightCurve(time=np.arange(N) * 0.02, flux=y, flux_err=np.full(N, 3.0), cadenceno=cad,
                       flux_unit=u.electron / u.second)
    if cbvs is None:
        data = {"VECTOR_{}".format(i + 1): X[:, i] for i in range(X.shape[1] - 1)}
        data["CADENCENO"] = cad
        cbvs = CotrendingBasisVectors(data, np.arange(N) * 0.02, cbv_type="SingleScale")
    return CBVCorrector(lc, cbvs=[cbvs]), cbvs


@pytest.mark.gpu
def test_correct_elasticnet_batch_bitwise_equals_its_own_call(engine):
    """CBVCorrector at N = 4096 with synthetic CBVs shared by 4 SMs correctors: correct_elasticnet_batch leaves each
    corrector bitwise in the state of its own correct_elasticnet call (coefficients, n_iter, dual gap, model)."""
    from lightkurve_b200.correctors import CBVCorrector
    sms = engine.sm_count()
    N, B = 4096, 4 * engine.sm_count()
    X, _ = oen.cbv_fixture(5, N=N, K=9, scale=1e4)
    rng = np.random.default_rng(6)
    W = rng.normal(size=(B, 8)) * np.geomspace(1, 1e-2, 8)
    Y = 1e4 * (1 + 0.01 * W @ X[:, :-1].T + 1e-3 * rng.normal(size=(B, N)))
    masks = list(rng.random((B, N)) > 0.1)
    cbvs = None
    cs = []
    for b in range(B):
        c, cbvs = _corrector(X, Y[b], cbvs)
        cs.append(c)
    kw = dict(cbv_type=["SingleScale"], cbv_indices=[np.arange(1, 9)])
    CBVCorrector.correct_elasticnet_batch(cs, cadence_mask=masks, **kw)
    for b in (0, sms + 3, B - 1):
        one, _ = _corrector(X, Y[b], cbvs)
        one.correct_elasticnet(cadence_mask=masks[b], **kw)
        assert one.elasticnet_n_iter == cs[b].elasticnet_n_iter, b
        assert one.elasticnet_dual_gap == cs[b].elasticnet_dual_gap, b
        assert np.array_equal(one.coefficients, cs[b].coefficients), b
        assert np.array_equal(one.model_lc.flux.value, cs[b].model_lc.flux.value), b


@pytest.mark.gpu
@pytest.mark.parametrize("N", [4095, 4096])
@pytest.mark.parametrize("K", [9, 40, 70, 100, 140, 165])
def test_regress_ex_exact_invariant_at_the_gram_edges(engine, N, K):
    """LKB_REGRESS_EXACT_INVARIANT at one K of each Gram instantiation, on both sides of the two-CTA threshold: a light
    curve's outputs at B = 1 equal those at B = 4 SMs bitwise (shared X), and those with the same X passed per light
    curve (at B = 1; at B = 4 SMs too for K = 9)."""
    sms = engine.sm_count()
    B = 4 * sms
    case = ("k%d" % K, "regress", B, N, K, dict(used=["ragged"], mix=True, exact=True, niters=3))
    inp = make_inputs(case, sms)
    X, Y, fe, M = inp["X"], inp["Y"], inp["fe"], inp["M"]
    pm, ps = np.zeros(K), np.full(K, 1e6)

    def call(Xc, rows):
        return engine.regress(Xc, Y[rows], fe[rows], M[rows], pm, ps, sigma=3, niters=3, exact_invariant=True)

    full = call(X, slice(None))
    if K == 9:
        fullb = call(np.ascontiguousarray(np.broadcast_to(X, (B, N, K))), slice(None))
    for b in (0, B // 2 + 1, B - 1):
        one = call(X, slice(b, b + 1))
        oneb = call(X[None], slice(b, b + 1))
        for k in ("coefficients", "model", "outlier_mask", "status"):
            assert np.array_equal(full[k][b], one[k][0]), (b, k)
            assert np.array_equal(oneb[k][0], one[k][0]), (b, k)
            if K == 9:
                assert np.array_equal(fullb[k][b], one[k][0]), (b, k)


# ------------------------------------------------------------------ the elastic net against the oracle at N >= 4096
@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(alpha=1e-20, l1_ratio=0.01), dict(alpha=1.0, l1_ratio=0.9)],
                         ids=["defaults", "alpha1-l1r0.9"])
@pytest.mark.parametrize("K", [20, 70, 100, 140, 165])
def test_elasticnet_matches_oracle_at_n4096(engine, K, kw):
    """Two CTAs per light curve in every Gram instantiation: n_iter and convergence equal, coefficients to 1e-9 and
    the model to 1e-9 of its maximum, as tests/test_gpu_enet.py holds the smaller cases."""
    X, Y, M, refs = enet_batch(2, 4096, K, K, K % 20 == 0, kw)
    enet_check(engine.elasticnet(X, Y, M, **kw), refs)
