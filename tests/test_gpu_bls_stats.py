"""K10 on the GPU: compute_stats_batch / get_transit_mask_batch against the host compute_stats / get_transit_mask on a
config-5-like batch plus the edge cases, and the invariances lkb_bls_stats promises (a light curve alone, in a batch
and in a permuted batch; two runs; device mode against host mode; too few transit slots)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _bls_stats_cases as C  # noqa: E402

from lightkurve_b200 import _lib as L  # noqa: E402
from lightkurve_b200.periodogram import BoxLeastSquaresPeriodogram as BLS  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def c5_like(n=300, seed=1005):
    """A few hundred light curves of bench.py's config 5 (tools/bench_bls_ragged.make_c5_bls), each with a
    candidate near its injected transit (or an arbitrary one where there is none)."""
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from tools.bench_bls_ragged import make_c5_bls
    times, fluxes, errs = make_c5_bls(seed=seed, B=n)
    rng = np.random.default_rng(seed)
    cs = []
    for b, (t, y, e) in enumerate(zip(times, fluxes, errs)):
        p, d = rng.uniform(0.5, 8), rng.uniform(0.05, 0.3)
        cs.append(("c5_%d" % b, t, y, e if b % 5 else None, p, d, t[0] + rng.uniform(-3, 30)))
    return cs


def all_cases():
    return c5_like() + C.cases() + [C.kepler_case()]


def call(engine, cs, return_mask=True, **kw):
    dys = [np.ones(len(c[1])) if c[3] is None else c[3] for c in cs]
    return engine.bls_stats([c[1] for c in cs], [c[2] for c in cs], dys, np.array([c[4] for c in cs]),
                            np.array([c[5] for c in cs]), np.array([c[6] for c in cs]), return_mask=return_mask, **kw)


def assert_same_lc(a, i, b, j):
    """Light curve i of result a is bitwise light curve j of result b."""
    np.testing.assert_array_equal(a["stats"][i], b["stats"][j])
    assert a["transit_first"][i] == b["transit_first"][j] and a["transit_n"][i] == b["transit_n"][j]
    assert a["status"][i] == b["status"][j]
    n = int(a["transit_n"][i])
    ta, tb = a["transit_offsets"][i], b["transit_offsets"][j]
    for k in ("per_transit_count", "per_transit_log_likelihood"):
        np.testing.assert_array_equal(a[k][ta:ta + n], b[k][tb:tb + n])
    oa, ob = a["offsets"], b["offsets"]
    np.testing.assert_array_equal(a["in_transit"][oa[i]:oa[i + 1]], b["in_transit"][ob[j]:ob[j + 1]])


def test_batch_against_host(engine):
    cs = all_cases()
    C.check_batch(cs, lambda pgs: BLS.compute_stats_batch(pgs, [c[4] for c in cs], [c[5] for c in cs],
                                                          [c[6] for c in cs]),
                  lambda pgs: BLS.get_transit_mask_batch(pgs, [c[4] for c in cs], [c[5] for c in cs],
                                                         [c[6] for c in cs]))


def test_max_power_defaults_against_host(engine):
    cs = C.cases()
    C.check_batch(cs, BLS.compute_stats_batch, BLS.get_transit_mask_batch)


def test_singular(engine):
    for name, t, y, dy, p, d, tt in C.singular_cases():
        pg = C.make_pg(t, y, dy, p, d, tt)
        res = call(engine, [(name, t, y, dy, p, d, tt)])
        assert res["status"][0] == L.E_SINGULAR, name
        with pytest.raises(np.linalg.LinAlgError):
            BLS.compute_stats_batch([pg])
        np.testing.assert_array_equal(BLS.get_transit_mask_batch([pg])[0], pg.get_transit_mask())


def test_alone_batched_permuted_and_repeated(engine):
    cs = all_cases() + C.singular_cases()
    full = call(engine, cs)
    again = call(engine, cs)
    perm = np.random.default_rng(7).permutation(len(cs))
    permuted = call(engine, [cs[i] for i in perm])
    inv = np.argsort(perm)
    for b in range(len(cs)):
        assert_same_lc(full, b, again, b)
        assert_same_lc(full, b, permuted, int(inv[b]))
    for b in list(range(0, len(cs), 37)) + list(range(len(cs) - 12, len(cs))):
        assert_same_lc(full, b, call(engine, [cs[b]]), 0)


def test_device_mode_equals_host_mode(engine):
    import torch
    cs = all_cases()
    host = call(engine, cs)
    dev = torch.device("cuda:0")
    cat = lambda xs: torch.from_numpy(np.concatenate(xs)).to(dev)
    dys = [np.ones(len(c[1])) if c[3] is None else c[3] for c in cs]
    res = engine.bls_stats(cat([c[1] for c in cs]), cat([c[2] for c in cs]), cat(dys),
                           torch.tensor([c[4] for c in cs], dtype=torch.float64, device=dev),
                           torch.tensor([c[5] for c in cs], dtype=torch.float64, device=dev),
                           torch.tensor([c[6] for c in cs], dtype=torch.float64, device=dev), return_mask=True,
                           offsets=host["offsets"], transit_offsets=host["transit_offsets"])
    torch.cuda.synchronize()
    for k in ("stats", "transit_first", "transit_n", "per_transit_count", "per_transit_log_likelihood", "status"):
        np.testing.assert_array_equal(res[k].cpu().numpy(), host[k], err_msg=k)
    np.testing.assert_array_equal(res["in_transit"].cpu().numpy().view(bool), host["in_transit"])


def test_too_few_transit_slots(engine):
    cs = C.cases()
    res = call(engine, cs)
    toff = res["transit_offsets"].copy()
    b = 0
    need = int(res["transit_n"][b])
    toff[b + 1:] -= int(toff[b + 1] - toff[b]) - (need - 1)        # one slot short for light curve 0
    with pytest.raises(ValueError, match="transit slots"):
        call(engine, cs, transit_offsets=toff)
    st = L.load().lkb_bls_stats
    assert st is not None
    # the raw entry returns LKB_E_ARG
    t, y = np.concatenate([c[1] for c in cs]), np.concatenate([c[2] for c in cs])
    B = len(cs)
    cand = [np.ascontiguousarray([c[i] for c in cs], dtype=np.float64) for i in (4, 5, 6)]
    outs = (np.empty((B, 15)), np.empty(B, np.int64), np.empty(B, np.int32), np.empty(max(1, toff[-1]), np.int32),
            np.empty(max(1, toff[-1])), np.empty(B, np.int32))
    rc = st(L.ptr(t), L.ptr(y), None, L.ptr(res["offsets"]), B, *[L.ptr(c) for c in cand], L.ptr(toff),
            L.ptr(outs[0]), L.ptr(outs[1]), L.ptr(outs[2]), L.ptr(outs[3]), L.ptr(outs[4]), None, L.ptr(outs[5]),
            L.MEM_HOST, None)
    assert rc == L.E_ARG
    assert outs[5][0] == L.E_ARG and outs[2][0] == need


def test_bad_candidates(engine):
    name, t, y, dy, p, d, tt = C.cases()[0]
    for bad in ((0.0, d, tt), (-1.0, d, tt), (p, 0.0, tt), (np.nan, d, tt), (p, d, np.inf)):
        with pytest.raises(ValueError):
            engine.bls_stats([t], [y], [dy], *bad)
