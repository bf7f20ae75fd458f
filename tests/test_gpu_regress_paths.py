"""K5 (RegressionCorrector: lkb_regress) across the kernel paths regress.cu chooses by shape, against
oracle.detrend.regress on EVERY light curve of every batch; and K6 (engine.nanmedian_std) at up to 1e6 values on the
hostile inputs of tests/test_select_emulated.py.

Which path a case takes follows from its shape and the switches it sets (regress.cu, regress_tc.cu):
  gram   "tc"      first Gram pass as one tensor-core GEMM + one refinement step: shared X, B >= 64, N >= 4096,
                   16 <= K <= 160 (RT_KX); later passes downdate with the fp64 DMMA kernel
         "dmma2"   fp64 DMMA, first pass split over two CTAs per light curve: not "tc", N >= 4096, B < 4 * SMs
         "dmma"    fp64 DMMA, one CTA per light curve: N < 4096
         "simt"    LKB_REGRESS_SIMT=1 (read once per process, so those cases run in a subprocess): rg_accum_kernel
  model  "mma"     rg_model_mma_kernel: shared X, B >= 8, not SIMT;  "rows": rg_model_rows otherwise
The table below states each case's expected path and test_case_table_matches_the_selection_rules restates the rules.

Tolerances: coefficients and model rtol 1e-7 on the fp64 paths and 1e-4 on "tc" (SURVEY 8c).  The absolute floors
scale with the light curve: `level` = max_k |w_k| max|X[:, k]|, the largest column contribution to the model (~1 for
normalised flux, ~1e5 for flux in e-/s); coefficient k's floor is 1e-10 level / max|X[:, k]| (tc: 1e-5), the model's
1e-10 level (tc: 1e-6).  Outlier masks must be identical."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import detrend as odet

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H100_SMS = 132
SIGMA, NITERS = 5.0, 5


def expected_paths(B, N, K, batched, simt):
    if simt:
        return "simt", "rows"
    if not batched and B >= 64 and N >= 4096 and 16 <= K <= 160:
        gram = "tc"
    else:
        gram = "dmma2" if (N >= 4096 and B < 4 * H100_SMS) else "dmma"
    return gram, ("mma" if (not batched and B >= 8) else "rows")


def design(rng, N, K):
    """A constant column and K - 1 smooth, mutually orthogonal, mean-free columns of scales 0.1 to 10 (CBV-like)."""
    if K == 1:
        return np.ones((N, 1))
    X = np.cumsum(rng.normal(size=(N, K - 1)), axis=0)
    X, _ = np.linalg.qr(X - X.mean(0))
    return np.hstack([X * np.sqrt(N) * 10 ** rng.uniform(-1, 1, K - 1), np.ones((N, 1))])


def make_case(seed, B, N, K, batched=False, eps=False, mask=False, prior=False, singular=()):
    """Seeded inputs.  eps: flux in e-/s (offset 1e5, noise 30, CBV amplitudes ~300 e-/s); else normalised (offset 1,
    noise 3e-4).  singular: light curves whose cadence mask removes every cadence (a zero matrix: status -4)."""
    rng = np.random.default_rng(seed)
    X = np.stack([design(rng, N, K) for _ in range(B)]) if batched else design(rng, N, K)
    off, noise, amp = (1e5, 30.0, 300.0) if eps else (1.0, 3e-4, 3e-3)
    cs = np.abs(X).max(axis=-2)                                     # [K] or [B, K]
    W = rng.normal(size=(B, K)) * amp / cs
    W[:, -1] = off
    Y = (np.einsum("bnk,bk->bn", X, W) if batched else W @ X.T) + noise * rng.normal(size=(B, N))
    for b in range(B):                                              # flares and transit-like dips
        Y[b, rng.choice(N, max(2, N // 500), replace=False)] += 8 * noise * rng.uniform(1, 3)
        s = rng.integers(0, N - 20)
        Y[b, s:s + 15] -= 6 * noise
    fe = noise * rng.uniform(0.8, 1.2, (B, N))
    cm = (rng.random((B, N)) > 0.03) if mask or singular else None
    for b in singular:
        cm[b] = False
    pm = ps = None
    if prior:
        c0 = cs if cs.ndim == 1 else cs[0]
        pm = rng.normal(size=K) * amp / c0
        pm[-1] = off
        ps = np.full(K, np.inf)
        ps[: max(1, K // 3)] = amp / c0[: max(1, K // 3)]        # a finite/inf mix
    return dict(X=X, Y=Y, fe=fe, cm=cm, pm=pm, ps=ps)


def oracle_one(c, b):
    X = c["X"][b] if c["X"].ndim == 3 else c["X"]
    cm = None if c["cm"] is None else c["cm"][b]
    return odet.regress(X, c["Y"][b], c["fe"][b], cm, c["pm"], c["ps"], sigma=SIGMA, niters=NITERS)


def check_against_oracle(c, r, fp64, singular=()):
    B = c["Y"].shape[0]
    for b in range(B):
        if b in singular:
            assert r["status"][b] == -4 and np.isnan(r["coefficients"][b]).all() and np.isnan(r["model"][b]).all()
            continue
        assert r["status"][b] == 0, b
        ref = oracle_one(c, b)
        X = c["X"][b] if c["X"].ndim == 3 else c["X"]
        cs = np.abs(X).max(axis=0)
        level = np.max(np.abs(ref["coefficients"]) * cs)
        rtol, fc, fm = (1e-7, 1e-10, 1e-10) if fp64 else (1e-4, 1e-5, 1e-6)
        assert np.array_equal(r["outlier_mask"][b], ref["outlier_mask"]), "light curve %d: %d outlier flags differ" % (
            b, np.count_nonzero(r["outlier_mask"][b] != ref["outlier_mask"]))
        err = np.abs(r["coefficients"][b] - ref["coefficients"])
        bound = rtol * np.abs(ref["coefficients"]) + fc * level / cs
        assert np.all(err <= bound), "light curve %d: coefficient error / bound %.3g" % (b, np.max(err / bound))
        np.testing.assert_allclose(r["model"][b], ref["model"], rtol=rtol, atol=fm * level,
                                   err_msg="light curve %d" % b)


def run_gpu(engine, c, **kw):
    return engine.regress(c["X"], c["Y"], c["fe"], c["cm"], c["pm"], c["ps"], sigma=SIGMA, niters=NITERS, **kw)


# (id, B, N, K, options, expected gram path, expected model path)
CASES = [
    ("k1-b1-n777", 1, 777, 1, {}, "dmma", "rows"),
    ("k2-b7-n777", 7, 777, 2, dict(mask=True), "dmma", "rows"),
    ("k16-b8-n777", 8, 777, 16, dict(prior=True), "dmma", "mma"),
    ("k165-b8-n777", 8, 777, 165, {}, "dmma", "mma"),
    ("k164-b65-n777-eps", 65, 777, 164, dict(eps=True), "dmma", "mma"),
    ("k17-b7-n8191", 7, 8191, 17, dict(mask=True), "dmma2", "rows"),
    ("k151-b8-n8193-eps-prior", 8, 8193, 151, dict(eps=True, prior=True), "dmma2", "mma"),
    ("k161-b3-n65000-eps", 3, 65000, 161, dict(eps=True), "dmma2", "rows"),
    ("k161-b65-n8192", 65, 8192, 161, {}, "dmma2", "mma"),
    ("k15-b65-n8192-eps", 65, 8192, 15, dict(eps=True), "dmma2", "mma"),
    ("k2-b8-n65000-batched", 8, 65000, 2, dict(batched=True), "dmma2", "rows"),
    ("k17-b7-n8193-batched-eps", 7, 8193, 17, dict(batched=True, eps=True, mask=True), "dmma2", "rows"),
    ("k151-b9-n777-batched-prior", 9, 777, 151, dict(batched=True, prior=True), "dmma", "rows"),
    ("k16-b65-n8192-tc", 65, 8192, 16, {}, "tc", "mma"),
    ("k17-b129-n8193-tc-eps", 129, 8193, 17, dict(eps=True, mask=True), "tc", "mma"),
    ("k160-b65-n8191-tc", 65, 8191, 160, {}, "tc", "mma"),
    ("k151-b64-n8192-tc-eps-prior", 64, 8192, 151, dict(eps=True, prior=True), "tc", "mma"),
    ("k17-b64-n65000-tc-eps", 64, 65000, 17, dict(eps=True), "tc", "mma"),
]


def test_case_table_matches_the_selection_rules():
    for cid, B, N, K, opt, gram, model in CASES:
        assert expected_paths(B, N, K, opt.get("batched", False), False) == (gram, model), cid
    seen = {(g, m) for *_, g, m in CASES}
    assert {"dmma", "dmma2", "tc"} <= {g for g, _ in seen} and {"mma", "rows"} <= {m for _, m in seen}


@pytest.mark.parametrize("cid,B,N,K,opt,gram,model", CASES, ids=[c[0] for c in CASES])
def test_regress_path_vs_oracle(engine, cid, B, N, K, opt, gram, model):
    c = make_case(sum(map(ord, cid)), B, N, K, **opt)
    r = run_gpu(engine, c)
    check_against_oracle(c, r, fp64=(gram != "tc"))


@pytest.mark.parametrize("gram", ["dmma2", "tc"])
def test_singular_light_curve_next_to_healthy_ones(engine, gram):
    B, N, K = (7, 8192, 17) if gram == "dmma2" else (65, 8192, 17)
    assert expected_paths(B, N, K, False, False)[0] == gram
    sing = (0, 4) if gram == "dmma2" else (3, 64)
    c = make_case(91, B, N, K, mask=True, singular=sing)
    r = run_gpu(engine, c)
    check_against_oracle(c, r, fp64=(gram != "tc"), singular=sing)


def test_return_cov_is_the_inverse_of_the_last_fit(engine):
    """The covariance of the last fit: np.linalg.inv of the oracle's matrix X^T W X + diag(1 / prior_sigma^2) over the
    cadences that fit used (cadence mask minus the outliers found by the first NITERS - 1 clips)."""
    B, N, K = 8, 8193, 17
    assert expected_paths(B, N, K, False, False) == ("dmma2", "mma")
    c = make_case(17, B, N, K, eps=True, mask=True, prior=True)
    r = run_gpu(engine, c, return_cov=True)
    for b in range(B):
        prev = odet.regress(c["X"], c["Y"][b], c["fe"][b], c["cm"][b], c["pm"], c["ps"], sigma=SIGMA,
                            niters=NITERS - 1)["outlier_mask"]
        tmp = c["cm"][b] & ~prev
        Xm = c["X"][tmp]
        A = Xm.T @ (Xm / c["fe"][b][tmp, None] ** 2) + np.diag(1.0 / c["ps"] ** 2)
        ref = np.linalg.inv(A)
        scale = np.sqrt(np.outer(np.diag(ref), np.diag(ref)))
        np.testing.assert_allclose(r["covariance"][b] / scale, ref / scale, rtol=0, atol=1e-9, err_msg="lc %d" % b)


@pytest.mark.parametrize("gram", ["dmma2", "tc"])
def test_batch_permutation(engine, gram):
    """A light curve's results do not depend on its place in the batch.  On the fp64 path a permuted batch of the same
    size returns the permuted results bitwise.  The tensor-core path sums its right-hand sides and refinement gradients
    over cadence slices with fp64 atomics (regress_tc.cu), so its last bits follow the scheduling: there the outlier
    masks must be identical and the values agree to the path's tolerance."""
    B, N, K = (40, 8192, 17) if gram == "dmma2" else (129, 8192, 17)
    assert expected_paths(B, N, K, False, False)[0] == gram
    c = make_case(23, B, N, K, eps=True, mask=True, prior=True)
    r1 = run_gpu(engine, c)
    perm = np.random.default_rng(5).permutation(B)
    cp = dict(c, Y=c["Y"][perm], fe=c["fe"][perm], cm=c["cm"][perm])
    r2 = run_gpu(engine, cp)
    for k in ("outlier_mask", "status"):
        assert np.array_equal(r2[k], r1[k][perm]), k
    if gram == "dmma2":
        for k in ("coefficients", "model"):
            assert np.array_equal(r2[k], r1[k][perm]), k
    else:
        cs = np.abs(c["X"]).max(axis=0)
        level = np.max(np.abs(r1["coefficients"]) * cs, axis=1, keepdims=True)
        assert np.all(np.abs(r2["coefficients"] - r1["coefficients"][perm])
                      <= 1e-4 * np.abs(r1["coefficients"][perm]) + 1e-5 * level[perm] / cs)
        assert np.all(np.abs(r2["model"] - r1["model"][perm]) <= 1e-6 * level[perm])


_SIMT_SCRIPT = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from lightkurve_b200 import engine
engine.init(0)
d = dict(np.load(sys.argv[2], allow_pickle=True))
get = lambda k: None if d[k].shape == () else d[k]
r = engine.regress(d["X"], d["Y"], d["fe"], get("cm"), get("pm"), get("ps"), sigma=float(d["sigma"]),
                   niters=int(d["niters"]))
np.savez(sys.argv[3], **r)
"""


@pytest.mark.parametrize("B,N,K,opt", [(9, 8193, 165, dict(eps=True, prior=True)),
                                       (8, 777, 64, dict(mask=True)),
                                       (3, 8192, 5, dict(batched=True))],
                         ids=["k165-b9-n8193-eps-prior", "k64-b8-n777", "k5-b3-n8192-batched"])
def test_simt_kernels_vs_oracle(engine, tmp_path, B, N, K, opt):
    """LKB_REGRESS_SIMT=1 (the SIMT Gram kernel rg_accum_kernel and rg_model_rows throughout).  The switch is read once
    per process, so the call runs in a child process."""
    c = make_case(7 * K + B, B, N, K, **opt)
    inp, out = tmp_path / "in.npz", tmp_path / "out.npz"
    none = np.array(None, dtype=object)
    np.savez(inp, X=c["X"], Y=c["Y"], fe=c["fe"], cm=none if c["cm"] is None else c["cm"],
             pm=none if c["pm"] is None else c["pm"], ps=none if c["ps"] is None else c["ps"], sigma=SIGMA,
             niters=NITERS)
    env = dict(os.environ, LKB_REGRESS_SIMT="1")
    flags = ["-s"] if sys.flags.no_user_site else []
    subprocess.check_call([sys.executable] + flags + ["-c", _SIMT_SCRIPT, ROOT, str(inp), str(out)], env=env)
    r = dict(np.load(out))
    check_against_oracle(c, r, fp64=True)


# ---------------------------------------------------------------- K6 at scale
def test_nanmedian_std_hostile_at_scale(engine):
    """engine.nanmedian_std (radix select, 256 threads) on the hostile kinds at 1e6 values and a few other lengths:
    medians equal to np.nanmedian (== : -0.0 equals 0.0), std to rtol 1e-12 (not over values near DBL_MAX)."""
    from test_select_emulated import KINDS, NO_STD, make
    arrays, kinds = [], []
    for i, kind in enumerate(KINDS):
        for n in (65000, 1_000_000) if i % 2 else (8193, 1_000_000):
            arrays.append(make(kind, n, 5000 + i))
            kinds.append(kind)
    med, sd = engine.nanmedian_std(arrays)
    for a, kind, m, s in zip(arrays, kinds, med, sd):
        ok = np.any(~np.isnan(a))
        ref = np.nanmedian(a) if ok else np.nan
        assert m == ref or (np.isnan(m) and np.isnan(ref)), (kind, len(a), m, ref)
        if kind not in NO_STD:
            sref = np.nanstd(a) if ok else np.nan
            np.testing.assert_allclose(s, sref, rtol=1e-12, equal_nan=True, err_msg="%s n=%d" % (kind, len(a)))
