"""The K10 BLS vetting kernel (lightkurve_b200/csrc/bls_stats.cuh) executed on the CPU through tests/native/cuda_emu.h.
The emulated kernel stands in for lkb_bls_stats, so compute_stats_batch and get_transit_mask_batch run end to end
(engine packing, kernel, result objects) and are compared with the host compute_stats / get_transit_mask."""
import ctypes
import os
import shutil
import subprocess
import sys
import types

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _bls_stats_cases as C  # noqa: E402

from lightkurve_b200 import _lib as L  # noqa: E402
from lightkurve_b200 import engine  # noqa: E402
from lightkurve_b200.periodogram import BoxLeastSquaresPeriodogram as BLS  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
CUDA_INC = "/usr/local/cuda/include"
c_vp, c_int = ctypes.c_void_p, ctypes.c_int


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    out = str(tmp_path_factory.mktemp("emu") / "libbls_stats_emu.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-pthread", "-I" + CUDA_INC, "-Wno-attributes", "-shared", "-fPIC",
                           "-Wl,-Bsymbolic", "-o", out, os.path.join(HERE, "native", "bls_stats_emu_driver.cpp")])
    lib = ctypes.CDLL(out)
    lib.emu_bls_stats.argtypes = [c_vp, c_vp, c_vp, c_vp, c_int] + [c_vp] * 11
    lib.emu_bls_stats.restype = c_int
    lib.emu_last_error.restype = ctypes.c_char_p
    return lib


@pytest.fixture
def emu_engine(emu, monkeypatch):
    """lightkurve_b200's library with lkb_bls_stats served by the emulated kernel (host mode; the slot-capacity
    check of bls.cu restated: any light curve with status LKB_E_ARG fails the call)."""
    def lkb_bls_stats(t, y, dy, off, B, per, dur, tt, toff, stats, first, n, cnt, ll, mask, status, mem, stream):
        assert mem == L.MEM_HOST
        rc = emu.emu_bls_stats(t, y, dy, off, B, per, dur, tt, toff, stats, first, n, cnt, ll, mask, status)
        st = np.ctypeslib.as_array(ctypes.cast(status, ctypes.POINTER(ctypes.c_int32)), (B,))
        return L.E_ARG if rc == 0 and np.any(st == L.E_ARG) else rc

    fake = types.SimpleNamespace(lkb_bls_stats=lkb_bls_stats, lkb_last_error=lambda: b"emulated: too few transit slots")
    monkeypatch.setattr(L, "_lib", fake)
    return engine


def test_cases_against_host(emu_engine):
    C.check_batch(C.cases(), BLS.compute_stats_batch, BLS.get_transit_mask_batch)


def test_kepler_length_with_3000_transits(emu_engine):
    cs = [C.kepler_case()]
    _, got, _ = C.check_batch(cs, BLS.compute_stats_batch, BLS.get_transit_mask_batch)
    assert len(got[0]["per_transit_count"]) > 3000


def test_singular_sine_fit(emu_engine):
    """One cadence, or every time stamp equal to t[0]: numpy's LinAlgError, status LKB_E_SINGULAR; the mask is fine."""
    cs = C.singular_cases()
    for name, t, y, dy, p, d, tt in cs:
        pg = C.make_pg(t, y, dy, p, d, tt)
        with pytest.raises(np.linalg.LinAlgError):
            pg.compute_stats(p, d, tt)
        res = engine.bls_stats([t], [y], None if dy is None else [dy], p, d, tt)
        assert res["status"][0] == L.E_SINGULAR, name
        assert np.isnan(res["stats"][0, 10]) and np.isnan(res["stats"][0, 11])
        np.testing.assert_array_equal(BLS.get_transit_mask_batch([pg], p, d, tt)[0], pg.get_transit_mask(p, d, tt))
    # in a batch, the error names the first singular periodogram, as the loop would stop there
    pgs = C.pgs_of(C.cases()[:2] + cs)
    with pytest.raises(np.linalg.LinAlgError, match="periodogram 2"):
        BLS.compute_stats_batch(pgs, [c[4] for c in C.cases()[:2] + cs], [c[5] for c in C.cases()[:2] + cs],
                                [c[6] for c in C.cases()[:2] + cs])


def test_results_do_not_depend_on_the_batch(emu_engine):
    """A light curve alone, in a batch and in a permuted batch: bitwise the same outputs."""
    cs = C.cases()
    args = [([c[i] for c in cs]) for i in range(1, 7)]
    dys = [np.ones(len(c[1])) if c[3] is None else c[3] for c in cs]
    full = engine.bls_stats(args[0], args[1], dys, args[3], args[4], args[5], return_mask=True)
    perm = np.random.default_rng(3).permutation(len(cs))
    permuted = engine.bls_stats([args[0][i] for i in perm], [args[1][i] for i in perm], [dys[i] for i in perm],
                                np.array(args[3])[perm], np.array(args[4])[perm], np.array(args[5])[perm],
                                return_mask=True)
    for b in range(len(cs)):
        one = engine.bls_stats([args[0][b]], [args[1][b]], [dys[b]], args[3][b], args[4][b], args[5][b],
                               return_mask=True)
        for other, j in ((full, b), (permuted, int(np.flatnonzero(perm == b)[0]))):
            np.testing.assert_array_equal(other["stats"][j], one["stats"][0])
            assert other["transit_first"][j] == one["transit_first"][0]
            n = one["transit_n"][0]
            assert other["transit_n"][j] == n
            to, t1 = other["transit_offsets"][j], one["transit_offsets"][0]
            for k in ("per_transit_count", "per_transit_log_likelihood"):
                np.testing.assert_array_equal(other[k][to:to + n], one[k][t1:t1 + n])
            o = other["offsets"]
            np.testing.assert_array_equal(other["in_transit"][o[j]:o[j + 1]], one["in_transit"])


def test_too_few_transit_slots(emu_engine):
    name, t, y, dy, p, d, tt = C.cases()[0]
    need = engine.bls_transit_slots([t], [p], [tt])
    res = engine.bls_stats([t], [y], [dy], p, d, tt)
    assert res["transit_n"][0] <= need[1]
    with pytest.raises(ValueError):
        engine.bls_stats([t], [y], [dy], p, d, tt, transit_offsets=np.array([0, res["transit_n"][0] - 1]))
