"""Batched host-side entry points over the C ABI (``include/lkb200.h``).

Every function takes either host ``numpy`` arrays (the library stages them through
its device workspace; the call is synchronous) or CUDA ``torch`` tensors (raw device
pointers are handed over; the call is asynchronous on the current torch stream).
PyTorch is only the allocator / stream provider here - no torch op is on the
compute path.  No CPU fallback exists: without the built library or without a GPU
these functions raise.
"""
import numpy as np

from . import _lib as L

_NORMS = {"psd_raw": L.LS_NORM_PSD_RAW, "psd": L.LS_NORM_PSD_SCALE, "amplitude": L.LS_NORM_AMPLITUDE}
_ALGOS = {"auto": L.LS_ALGO_AUTO, "simt": L.LS_ALGO_SIMT, "tcgen05": L.LS_ALGO_TCGEN05, "nufft": L.LS_ALGO_NUFFT}


def _is_torch(x):
    return hasattr(x, "data_ptr") and hasattr(x, "is_cuda")


def _stream_ptr():
    import torch
    return torch.cuda.current_stream().cuda_stream


def device_count():
    return L.load().lkb_device_count()


def init(device=0):
    """Bind this process to one GPU (one process per GPU, like torch.distributed ranks)."""
    L.check(L.load().lkb_init(int(device)))


def shutdown():
    L.check(L.load().lkb_shutdown())


def launch_count():
    return int(L.load().lkb_launch_count())


def ls_last_algo():
    """Kernel family the most recent Lomb-Scargle call ran: "simt" (direct sums), "tcgen05" or "nufft"."""
    return {L.LS_ALGO_SIMT: "simt", L.LS_ALGO_TCGEN05: "tcgen05", L.LS_ALGO_NUFFT: "nufft"}.get(
        int(L.load().lkb_ls_last_algo()), "none")


def flatten_last_path():
    """Kernel path the most recent flatten call ran: "v2-moments" or "v2-direct" (streaming kernel, interior from
    sliding moments or direct taps), "v1" (FIR kernel) or "v1-rerun" (FIR kernel after more than 1022 gap cuts)."""
    return {L.FLATTEN_PATH_V2_MOMENTS: "v2-moments", L.FLATTEN_PATH_V2_DIRECT: "v2-direct", L.FLATTEN_PATH_V1: "v1",
            L.FLATTEN_PATH_V1_RERUN: "v1-rerun"}.get(int(L.load().lkb_flatten_last_path()), "none")


def ls_last_escalated():
    """Light curves of the most recent shared-grid NUFFT call that took the double-precision pass (lkb200.h)."""
    return int(L.load().lkb_ls_last_escalated())


def ls_last_nufft_plan():
    """Transform of the most recent NUFFT Lomb-Scargle call: ("v2" or "round-1", p, p2) - the flux and window-term fine
    grids have 2^p and 2^p2 cells - or None before the first one."""
    out = np.zeros(3, dtype=np.int32)
    L.check(L.load().lkb_ls_last_nufft_plan(L.ptr(out)))
    if out[0] < 0:
        return None
    return ("v2" if out[0] == 1 else "round-1", int(out[1]), int(out[2]))


def profile_enable(on=True):
    """Record CUDA events around the dominant kernel of each subsequent call (see lkb200.h)."""
    L.check(L.load().lkb_profile_enable(1 if on else 0))


def profile_read(max_n=512):
    """Durations [ms] of the dominant kernels launched since profile_enable / the last read."""
    buf = np.zeros(max_n, dtype=np.float64)
    n = L.load().lkb_profile_read(L.ptr(buf), max_n)
    if n < 0:
        L.check(n)
    return buf[:n].copy()


# workspace slot numbers (enum Slot in csrc/common.cuh) for the diagnostic read-back
WS_SLOTS = {name: i for i, name in enumerate(
    ["A", "B", "C", "D", "E", "F", "G", "H", "I", "J", "K", "L", "M", "N", "O", "P"]
    + ["IN%d" % i for i in range(8)] + ["OUT%d" % i for i in range(8)] + ["X%d" % i for i in range(8)] + ["Y%d" % i for i in range(8)])}


def ws_read(slot, count, dtype, offset_bytes=0):
    """Diagnostic: `count` items of `dtype` from workspace slot `slot` ("A".."P", "IN0".., "OUT0"..) as left by
    the last call (device synchronised first)."""
    out = np.empty(count, dtype=dtype)
    L.check(L.load().lkb_ws_read(WS_SLOTS[slot], int(offset_bytes), int(out.nbytes), L.ptr(out)))
    return out


def sm_count():
    return int(L.load().lkb_sm_count())


def _csr(arrays, dtype=np.float64):
    lens = [len(a) for a in arrays]
    offsets = np.zeros(len(arrays) + 1, dtype=np.int64)
    np.cumsum(lens, out=offsets[1:])
    cat = np.ascontiguousarray(np.concatenate([np.asarray(a, dtype=dtype) for a in arrays])) if arrays else \
        np.zeros(0, dtype)
    return cat, offsets


def _y_dtype_code(dt):
    if dt == np.float32:
        return L.DTYPE_F32
    if dt == np.float64:
        return L.DTYPE_F64
    raise TypeError("flux must be float32 or float64")


# --------------------------------------------------------------------------------------
# Lomb-Scargle
# --------------------------------------------------------------------------------------
_RAGGED_ALGOS = {"auto": L.LS_ALGO_AUTO, "direct": L.LS_ALGO_SIMT, "simt": L.LS_ALGO_SIMT, "nufft": L.LS_ALGO_NUFFT}


def ls_power_ragged(times, fluxes, frequency, normalization="amplitude", norm_scale=None, algo="auto"):
    """K1.  `times`/`fluxes`: lists of 1-D arrays (one per light curve, no NaNs).
    `frequency`: one 1-D grid shared by all light curves, or a list of per-LC grids.
    `algo`: "auto" (the NUFFT kernels for a large job on one shared regular grid with sorted times, else the direct
    sums), "direct" (always the exact direct sums - astropy method="slow") or "nufft" (raises when the grid or the
    times do not qualify - the reference's ls_method="fastnifty").
    Returns a [B, F] float32 array (shared grid) or a list of float32 arrays."""
    lib = L.load()
    B = len(times)
    if B == 0:
        return []
    if algo not in _RAGGED_ALGOS:
        raise ValueError("algo must be one of %s" % sorted(_RAGGED_ALGOS))
    t, offsets = _csr(times)
    ydt = np.float32 if all(np.asarray(f).dtype == np.float32 for f in fluxes) else np.float64
    y, yoff = _csr(fluxes, ydt)
    if not np.array_equal(offsets, yoff):
        raise ValueError("time and flux lengths differ")
    per_lc = isinstance(frequency, (list, tuple))
    if per_lc:
        freq, foff = _csr(frequency)
        F = 0
        out = np.empty(int(foff[-1]), dtype=np.float32)
    else:
        freq = np.ascontiguousarray(frequency, dtype=np.float64)
        foff = None
        F = len(freq)
        out = np.empty((B, F), dtype=np.float32)
    ns = None if norm_scale is None else np.ascontiguousarray(np.broadcast_to(norm_scale, (B,)), dtype=np.float64)
    L.check(lib.lkb_ls_power_ex(L.ptr(t), L.ptr(y), _y_dtype_code(ydt), L.ptr(offsets), B, L.ptr(freq), L.ptr(foff), F,
                                _NORMS[normalization], L.ptr(ns), L.ptr(out), L.MEM_HOST, None, _RAGGED_ALGOS[algo]))
    if per_lc:
        return [out[foff[b]:foff[b + 1]] for b in range(B)]
    return out


def ls_power_ragged_device(t_cat, y_cat, offsets, frequency, normalization="amplitude", norm_scale=None, algo="auto",
                           out=None):
    """K1 with DEVICE-resident inputs: `t_cat` (float64) and `y_cat` (float32 / float64) are CUDA torch tensors
    holding the light curves back to back, `offsets` the int64 [B + 1] CSR boundaries (host metadata, numpy),
    `frequency` a CUDA float64 tensor [F] shared by all light curves, `norm_scale` None or a CUDA float64 [B].
    Returns a CUDA float32 [B, F] tensor (`out` if given).  The kernels run on the current torch stream; the call
    synchronises that stream for its metadata read-backs."""
    import torch
    lib = L.load()
    if algo not in _RAGGED_ALGOS:
        raise ValueError("algo must be one of %s" % sorted(_RAGGED_ALGOS))
    offsets = np.ascontiguousarray(offsets, dtype=np.int64)
    B = len(offsets) - 1
    if B <= 0:
        raise ValueError("empty batch")
    for name, x in (("t_cat", t_cat), ("y_cat", y_cat), ("frequency", frequency)):
        if not (_is_torch(x) and x.is_cuda and x.is_contiguous() and x.dim() == 1):
            raise ValueError("%s must be a contiguous one-dimensional CUDA tensor" % name)
    if t_cat.dtype != torch.float64 or frequency.dtype != torch.float64:
        raise TypeError("t_cat and frequency must be float64")
    if y_cat.dtype not in (torch.float32, torch.float64):
        raise TypeError("flux must be float32 or float64, not %s" % (y_cat.dtype,))
    if offsets[0] != 0 or np.any(np.diff(offsets) < 0) or t_cat.numel() != offsets[-1] or y_cat.numel() != offsets[-1]:
        raise ValueError("offsets do not describe t_cat / y_cat")
    F = frequency.numel()
    if out is None:
        out = torch.empty((B, F), dtype=torch.float32, device=y_cat.device)
    elif not (_is_torch(out) and out.is_cuda and out.dtype == torch.float32 and tuple(out.shape) == (B, F)
              and out.is_contiguous()):
        raise ValueError("`out` must be a contiguous CUDA float32 tensor of shape (%d, %d)" % (B, F))
    if norm_scale is not None and not (_is_torch(norm_scale) and norm_scale.is_cuda and
                                       norm_scale.dtype == torch.float64 and norm_scale.numel() == B):
        raise ValueError("norm_scale must be a CUDA float64 tensor with one entry per light curve")
    ycode = L.DTYPE_F32 if y_cat.dtype == torch.float32 else L.DTYPE_F64
    L.check(lib.lkb_ls_power_ex(L.ptr(t_cat), L.ptr(y_cat), ycode, L.ptr(offsets), B, L.ptr(frequency), None, F,
                                _NORMS[normalization], L.ptr(norm_scale), L.ptr(out), L.MEM_DEVICE, _stream_ptr(),
                                _RAGGED_ALGOS[algo]))
    return out


def ls_power_chi2(times, fluxes, frequency, nterms=1, normalization="amplitude", norm_scale=None,
                  return_theta=False, algo="auto"):
    """K1n.  Multi-term periodogram (astropy method="chi2"/"fastchi2", nterms in [1, 4]); same
    arguments as ls_power_ragged.  With return_theta also returns the 2*nterms+1 fitted parameters
    per (light curve, frequency): [offset, sin 1, cos 1, sin 2, cos 2, ...].
    `algo`: "auto" (the NUFFT kernels for a large job on one shared regular grid with sorted times and no theta, to
    the parity tolerance of DESIGN.md section 2; else the direct sums), "direct" (always the exact fp64 direct sums)
    or "nufft" (raises with status -5 when the grid, the times or return_theta do not qualify)."""
    lib = L.load()
    B = len(times)
    if B == 0:
        return []
    if algo not in _RAGGED_ALGOS:
        raise ValueError("algo must be one of %s" % sorted(_RAGGED_ALGOS))
    t, offsets = _csr(times)
    ydt = np.float32 if all(np.asarray(f).dtype == np.float32 for f in fluxes) else np.float64
    y, yoff = _csr(fluxes, ydt)
    if not np.array_equal(offsets, yoff):
        raise ValueError("time and flux lengths differ")
    M = 2 * int(nterms) + 1
    per_lc = isinstance(frequency, (list, tuple))
    if per_lc:
        freq, foff = _csr(frequency)
        F = 0
        out = np.empty(int(foff[-1]), dtype=np.float32)
        theta = np.empty((int(foff[-1]), M), dtype=np.float64) if return_theta else None
    else:
        freq = np.ascontiguousarray(frequency, dtype=np.float64)
        foff = None
        F = len(freq)
        out = np.empty((B, F), dtype=np.float32)
        theta = np.empty((B, F, M), dtype=np.float64) if return_theta else None
    ns = None if norm_scale is None else np.ascontiguousarray(np.broadcast_to(norm_scale, (B,)), dtype=np.float64)
    L.check(lib.lkb_ls_power_chi2_ex(L.ptr(t), L.ptr(y), _y_dtype_code(ydt), L.ptr(offsets), B, L.ptr(freq),
                                     L.ptr(foff), F, int(nterms), _NORMS[normalization], L.ptr(ns), L.ptr(out),
                                     L.ptr(theta), L.MEM_HOST, None, _RAGGED_ALGOS[algo]))
    if per_lc:
        out = [out[foff[b]:foff[b + 1]] for b in range(B)]
        if return_theta:
            theta = [theta[foff[b]:foff[b + 1]] for b in range(B)]
    return (out, theta) if return_theta else out


def ls_power_shared(t, Y, frequency, normalization="amplitude", norm_scale=None, algo="auto", out=None):
    """K2.  One cadence grid `t` [N] shared by the batch `Y` [B, N]; `frequency` [F].
    numpy in -> numpy out (host mode); CUDA torch tensors in -> torch tensor out (device mode: the kernels are
    enqueued on the current torch stream, but the call itself synchronises that stream once for a small metadata
    read-back, and the library's grow-only workspaces are shared by all calls - use ONE stream per process).
    `algo`: "auto" (the spread + FFT path of DESIGN.md K2n when the grid is regular with integer f0/df,
    df * baseline <= 1 and the times ascend; else the tensor-core (wgmma) path, named "tcgen05", when the shape allows; else the CUDA-core
    contraction), "simt", "tcgen05", or "nufft" (raises for grids / times it does not support)."""
    lib = L.load()
    if algo not in _ALGOS:
        raise ValueError("algo must be one of %s" % sorted(_ALGOS))
    if _is_torch(Y):
        import torch
        if not (_is_torch(t) and _is_torch(frequency) and Y.is_cuda and t.is_cuda and frequency.is_cuda):
            raise ValueError("device mode needs CUDA tensors for t, Y and frequency")
        if Y.dim() != 2 or t.dim() != 1 or frequency.dim() != 1:
            raise ValueError("Y must be [B, N], t [N] and frequency [F]")
        B, N = Y.shape
        F = frequency.numel()
        if t.numel() != N:
            raise ValueError("t has %d cadences but Y has %d columns" % (t.numel(), N))
        if t.dtype != torch.float64 or frequency.dtype != torch.float64:
            raise TypeError("t and frequency must be float64")
        if Y.dtype not in (torch.float32, torch.float64):
            raise TypeError("flux must be float32 or float64, not %s" % (Y.dtype,))
        if not (Y.is_contiguous() and t.is_contiguous() and frequency.is_contiguous()):
            raise ValueError("t, Y and frequency must be contiguous")
        ycode = L.DTYPE_F32 if Y.dtype == torch.float32 else L.DTYPE_F64
        if out is None:
            out = torch.empty((B, F), dtype=torch.float32, device=Y.device)
        elif not (_is_torch(out) and out.is_cuda and out.device == Y.device and out.dtype == torch.float32
                  and tuple(out.shape) == (B, F) and out.is_contiguous()):
            raise ValueError("`out` must be a contiguous CUDA float32 tensor of shape (%d, %d) on %s" % (B, F, Y.device))
        ns = None
        if norm_scale is not None:
            ns = torch.tensor([float(norm_scale)], dtype=torch.float64, device=Y.device)
        L.check(lib.lkb_ls_power_shared(L.ptr(t), L.ptr(Y), ycode, int(B), int(N), L.ptr(frequency), int(F),
                                        _NORMS[normalization], L.ptr(ns), L.ptr(out), L.MEM_DEVICE, _stream_ptr(),
                                        _ALGOS[algo]))
        return out
    t = np.ascontiguousarray(t, dtype=np.float64)
    Y = np.ascontiguousarray(Y)
    if Y.dtype not in (np.float32, np.float64):
        Y = Y.astype(np.float64)
    if Y.ndim != 2 or t.ndim != 1:
        raise ValueError("Y must be [B, N] and t [N]")
    B, N = Y.shape
    if t.shape != (N,):
        raise ValueError("t has %d cadences but Y has %d columns" % (len(t), N))
    freq = np.ascontiguousarray(frequency, dtype=np.float64)
    if freq.ndim != 1:
        raise ValueError("frequency must be one-dimensional")
    if out is None:
        out = np.empty((B, len(freq)), dtype=np.float32)
    elif not (isinstance(out, np.ndarray) and out.dtype == np.float32 and out.shape == (B, len(freq))
              and out.flags.c_contiguous and out.flags.writeable):
        raise ValueError("`out` must be a writeable C-contiguous float32 array of shape (%d, %d)" % (B, len(freq)))
    ns = None if norm_scale is None else np.array([float(norm_scale)], dtype=np.float64)
    L.check(lib.lkb_ls_power_shared(L.ptr(t), L.ptr(Y), _y_dtype_code(Y.dtype), B, N, L.ptr(freq), len(freq),
                                    _NORMS[normalization], L.ptr(ns), L.ptr(out), L.MEM_HOST, None, _ALGOS[algo]))
    return out


# --------------------------------------------------------------------------------------
# Box Least Squares
# --------------------------------------------------------------------------------------
BLS_FIELDS = ("power", "depth", "depth_err", "duration", "transit_time", "depth_snr", "log_likelihood")


def bls_power(times, fluxes, flux_errs, period, duration, oversample=10, objective="likelihood",
              return_bins=False):
    """K3.  Lists of per-LC arrays (flux_errs: list or None => unit weights) and one duration grid [D].
    `period`: one grid [P] shared by all light curves - returns a dict of [B, P] float64 arrays - or a list of
    B one-dimensional per-light-curve grids (one GPU call; each light curve's result is bitwise what a call on its own grid
    gives) - then every field, "bins" and "period" included, is a list of per-light-curve arrays."""
    lib = L.load()
    B = len(times)
    t, offsets = _csr(times)
    y, yoff = _csr(fluxes)
    if not np.array_equal(offsets, yoff):
        raise ValueError("time and flux lengths differ")
    dy = None
    if flux_errs is not None:
        dy, doff = _csr(flux_errs)
        if not np.array_equal(offsets, doff):
            raise ValueError("time and flux_err lengths differ")
    duration = np.ascontiguousarray(np.atleast_1d(duration), dtype=np.float64)
    D = len(duration)
    # a list of arrays is one grid per light curve; a list of numbers is one shared grid, as it always was
    per_lc = isinstance(period, (list, tuple)) and len(period) > 0 and all(np.ndim(p) == 1 for p in period)
    if per_lc:
        if len(period) != B:
            raise ValueError("%d period grids for %d light curves" % (len(period), B))
        period, pofs = _csr([np.atleast_1d(p) for p in period])
        P = int(pofs[-1])
        shape = (P,)
    else:
        period = np.ascontiguousarray(np.atleast_1d(period), dtype=np.float64)
        pofs = None
        P = len(period)
        shape = (B, P)
    outs = [np.empty(shape, dtype=np.float64) for _ in range(7)]
    bins = np.empty(shape + (2,), dtype=np.int32) if return_bins else None
    L.check(lib.lkb_bls_power_ex(L.ptr(t), L.ptr(y), L.ptr(dy), L.ptr(offsets), B, L.ptr(period), L.ptr(pofs), P,
                                 L.ptr(duration), D, int(oversample), L.BLS_SNR if objective == "snr" else L.BLS_LIKELIHOOD,
                                 *[L.ptr(o) for o in outs], L.ptr(bins), L.MEM_HOST, None))
    res = dict(zip(BLS_FIELDS, outs))
    res["period"] = period
    if return_bins:
        res["bins"] = bins
    if per_lc:
        res = {k: [v[pofs[b]:pofs[b + 1]] for b in range(B)] for k, v in res.items()}
    return res


BLS_STATS_COLUMNS = ("depth", "depth_err", "depth_odd", "depth_odd_err", "depth_even", "depth_even_err", "depth_half",
                     "depth_half_err", "depth_phased", "depth_phased_err", "harmonic_amplitude",
                     "harmonic_delta_log_likelihood", "y_in", "y_out", "n_in")     # LKB_BLS_STATS_* in lkb200.h


def bls_transit_slots(times, period, transit_time):
    """Per-transit slot capacity of each light curve as a HOST CSR int64 [B + 1] (the bound of lkb200.h): with times
    and tt = transit_time - t[0] measured from the first cadence, rint((max t - tt) / P) - rint((min t - tt) / P) + 1."""
    caps = np.zeros(len(times) + 1, dtype=np.int64)
    for b, (t, p, tt) in enumerate(zip(times, period, transit_time)):
        t = np.asarray(t, dtype=np.float64)
        t0 = t[0]
        ttr = float(tt) - t0
        lo = np.rint((t.min() - t0 - ttr) / float(p))
        hi = np.rint((t.max() - t0 - ttr) / float(p))
        caps[b + 1] = int(hi - lo) + 1
    return np.cumsum(caps)


def bls_stats(times, fluxes, flux_errs, period, duration, transit_time, return_mask=False, offsets=None,
              transit_offsets=None):
    """K10.  The vetting statistics of BoxLeastSquaresPeriodogram.compute_stats and the mask of get_transit_mask for one
    candidate per light curve.  `period`, `duration`, `transit_time` (absolute): [B] or scalars.
    Host mode: lists of per-light-curve arrays (flux_errs: list or None => unit weights); the slot capacity is
    computed here (bls_transit_slots).  Device mode: `times`, `fluxes` (and `flux_errs` or None) are the concatenated
    CUDA float64 tensors with `offsets` (host int64 [B + 1]), the candidates CUDA float64 tensors [B], and
    `transit_offsets` (host int64 [B + 1]) is required.
    Returns dict(stats [B, len(BLS_STATS_COLUMNS)], transit_first int64 [B], transit_n int32 [B],
    per_transit_count int32 and per_transit_log_likelihood [transit_offsets[-1]] (light curve b's transits at
    transit_offsets[b], transit_n[b] of them), status int32 [B] (0 or -4 = singular sine fit), offsets,
    transit_offsets and, with return_mask, in_transit (bool on the host, uint8 on the device) [offsets[-1]])."""
    lib = L.load()
    if _is_torch(times):
        return _bls_stats_device(lib, times, fluxes, flux_errs, period, duration, transit_time, return_mask, offsets,
                                 transit_offsets)
    B = len(times)
    t, offsets = _csr(times)
    y, yoff = _csr(fluxes)
    if not np.array_equal(offsets, yoff):
        raise ValueError("time and flux lengths differ")
    dy = None
    if flux_errs is not None:
        dy, doff = _csr(flux_errs)
        if not np.array_equal(offsets, doff):
            raise ValueError("time and flux_err lengths differ")
    cand = [np.ascontiguousarray(np.broadcast_to(np.asarray(x, dtype=np.float64), (B,))) for x in
            (period, duration, transit_time)]
    if np.any(np.diff(offsets) < 1):
        raise ValueError("light curve %d has no cadences" % int(np.flatnonzero(np.diff(offsets) < 1)[0]))
    bad = ~((cand[0] > 0) & np.isfinite(cand[0]) & (cand[1] > 0) & np.isfinite(cand[1]) & np.isfinite(cand[2]))
    if np.any(bad):
        b = int(np.flatnonzero(bad)[0])
        raise ValueError("light curve %d: period (%g) and duration (%g) must be positive and finite, transit_time (%g) "
                         "finite" % (b, cand[0][b], cand[1][b], cand[2][b]))
    if transit_offsets is None:
        transit_offsets = bls_transit_slots(times, cand[0], cand[2])
    toff = np.ascontiguousarray(transit_offsets, dtype=np.int64)
    slots = int(toff[-1])
    stats = np.empty((B, len(BLS_STATS_COLUMNS)))
    first, n_tr, status = np.empty(B, np.int64), np.empty(B, np.int32), np.empty(B, np.int32)
    cnt, ll = np.empty(slots, np.int32), np.empty(slots)
    mask = np.empty(len(t), np.uint8) if return_mask else None
    L.check(lib.lkb_bls_stats(L.ptr(t), L.ptr(y), L.ptr(dy), L.ptr(offsets), B, *[L.ptr(c) for c in cand], L.ptr(toff),
                              L.ptr(stats), L.ptr(first), L.ptr(n_tr), L.ptr(cnt) if slots else None,
                              L.ptr(ll) if slots else None, L.ptr(mask), L.ptr(status), L.MEM_HOST, None))
    res = dict(stats=stats, transit_first=first, transit_n=n_tr, per_transit_count=cnt, per_transit_log_likelihood=ll,
               status=status, offsets=offsets, transit_offsets=toff)
    if return_mask:
        res["in_transit"] = mask.view(bool)
    return res


def _bls_stats_device(lib, t, y, dy, period, duration, transit_time, return_mask, offsets, transit_offsets):
    import torch
    if offsets is None or transit_offsets is None:
        raise ValueError("device mode needs the host CSR `offsets` and `transit_offsets`")
    for name, x in (("times", t), ("fluxes", y), ("flux_errs", dy), ("period", period), ("duration", duration),
                    ("transit_time", transit_time)):
        if x is not None and not (_is_torch(x) and x.is_cuda and x.is_contiguous() and x.dtype == torch.float64):
            raise ValueError("device mode: %s must be a contiguous CUDA float64 tensor" % name)
    off = np.ascontiguousarray(offsets, dtype=np.int64)
    toff = np.ascontiguousarray(transit_offsets, dtype=np.int64)
    B = len(off) - 1
    if t.numel() != off[-1] or y.numel() != off[-1] or (dy is not None and dy.numel() != off[-1]):
        raise ValueError("offsets end at %d but the arrays hold %d values" % (off[-1], t.numel()))
    if period.numel() != B or duration.numel() != B or transit_time.numel() != B:
        raise ValueError("period, duration and transit_time need one value per light curve")
    dev, slots = t.device, int(toff[-1])
    stats = torch.empty((B, len(BLS_STATS_COLUMNS)), dtype=torch.float64, device=dev)
    first = torch.empty(B, dtype=torch.int64, device=dev)
    n_tr = torch.empty(B, dtype=torch.int32, device=dev)
    status = torch.empty(B, dtype=torch.int32, device=dev)
    cnt = torch.empty(max(slots, 1), dtype=torch.int32, device=dev)
    ll = torch.empty(max(slots, 1), dtype=torch.float64, device=dev)
    mask = torch.empty(int(off[-1]), dtype=torch.uint8, device=dev) if return_mask else None
    L.check(lib.lkb_bls_stats(L.ptr(t), L.ptr(y), L.ptr(dy), L.ptr(off), B, L.ptr(period), L.ptr(duration),
                              L.ptr(transit_time), L.ptr(toff), L.ptr(stats), L.ptr(first), L.ptr(n_tr), L.ptr(cnt),
                              L.ptr(ll), L.ptr(mask), L.ptr(status), L.MEM_DEVICE, _stream_ptr()))
    res = dict(stats=stats, transit_first=first, transit_n=n_tr, per_transit_count=cnt[:slots],
               per_transit_log_likelihood=ll[:slots], status=status, offsets=off, transit_offsets=toff)
    if return_mask:
        res["in_transit"] = mask
    return res


BLS_CANDIDATE_FIELDS = ("period", "duration", "transit_time", "depth", "depth_err", "depth_snr", "power")


def _named_error(e, b, r):
    """`e` again, of the same type, with the light curve and round in front of its message."""
    try:
        return type(e)("light curve %d, round %d: %s" % (b, r, e))
    except Exception:                                  # an exception type that needs other arguments
        return e


def bls_find_candidates(times, fluxes, flux_errs, grid, n_candidates, shared_grid=False, return_stats=False):
    """K3 + K14 + K10 + K6.  `n_candidates` rounds of search, take the best candidate, remove its transits, for every
    light curve at once, with the cadences on the device throughout:
      1. lkb_bls_power_ex on each light curve's survivors (round 0: all its cadences), weights flux_err where every
         surviving flux_err is finite, else unit weights;
      2. lkb_bls_best: the candidate at np.nanargmax of the power;
      3. lkb_bls_stats at the candidate: in-transit flags and box levels (and, with return_stats, its statistics);
      4. lkb_transit_compact: lc[~get_transit_mask] and what the next grid needs;
      5. lkb_nanmedian_std of the survivors' time steps.
    `times`, `fluxes`, `flux_errs`: lists of host arrays (finite times; any flux_err).  `grid(b, r, tmin, tmax,
    median_dt)` returns dict(period, duration, oversample, objective) for light curve b in round r from its survivors'
    time span (tmin / tmax None without survivors) and np.median(np.diff(t)) - or raises as the single-curve loop would;
    duration, oversample and objective must be the same for all.  With `shared_grid` every call returns the same
    period grid and K3 runs its shared-grid entry.
    Returns dict of [B, n_candidates] float64 arrays (BLS_CANDIDATE_FIELDS), "masked_in" (list of B int8 arrays: the
    round that removed each cadence, -1 if none) and, with return_stats, "stats": per round, a host-mode-style
    bls_stats result (plus "tstart", each light curve's first surviving time).  The first error in the order of the
    single-curve loop (light curve by light curve, round by round) is raised with its type, naming both."""
    import torch
    lib = L.load()
    B = len(times)
    if not 0 < B <= 65535:
        raise ValueError("bls_find_candidates needs 1 .. 65535 light curves, got %d" % B)
    if not 1 <= int(n_candidates) <= 127:
        raise ValueError("n_candidates must be in 1 .. 127, got %r" % (n_candidates,))
    n_candidates = int(n_candidates)
    t_h, off0 = _csr(times)
    y_h, _ = _csr(fluxes)
    dy_h, _ = _csr(flux_errs)
    if len(y_h) != len(t_h) or len(dy_h) != len(t_h):
        raise ValueError("time, flux and flux_err lengths differ")
    dev = torch.device("cuda", torch.cuda.current_device())
    f64 = dict(dtype=torch.float64, device=dev)
    n_h = np.diff(off0)
    # round 0's grid inputs straight from the host arrays (numpy's own reductions)
    tinfo = np.full((B, 3), np.nan)
    med = np.full(B, np.nan)
    w_h = dy_h.copy()
    for b in range(B):
        tb = t_h[off0[b]:off0[b + 1]]
        if len(tb):
            tinfo[b] = tb[0], np.min(tb), np.max(tb)
        if len(tb) > 1:
            med[b] = np.median(np.diff(tb))
        if not np.isfinite(dy_h[off0[b]:off0[b + 1]]).all():
            w_h[off0[b]:off0[b + 1]] = 1.0

    def up(a, dtype=torch.float64):
        x = torch.empty(max(len(a), 1), dtype=dtype, device=dev)
        x[:len(a)].copy_(torch.from_numpy(np.ascontiguousarray(a)))
        return x

    d_t, d_y, d_dy, d_w = up(t_h), up(y_h), up(dy_h), up(w_h)
    d_idx = up(np.concatenate([np.arange(n, dtype=np.int32) for n in n_h]) if len(t_h) else np.zeros(0, np.int32),
               torch.int32)
    masked = torch.full((max(int(off0[-1]), 1),), -1, dtype=torch.int8, device=dev)
    off = off0.copy()
    out = {k: np.full((B, n_candidates), np.nan) for k in BLS_CANDIDATE_FIELDS}
    rounds_stats = []
    err = None                                         # (b, r, exception): the loop's first error so far
    Bc = B                                             # light curves still searched: those before the first error
    dur_t = None
    for r in range(n_candidates):
        # 1. the grids, on the host; an error truncates the batch to the light curves before it
        grids = []
        for b in range(Bc):
            try:
                g = grid(b, r, None if n_h[b] == 0 else np.float64(tinfo[b, 1]),
                         None if n_h[b] == 0 else np.float64(tinfo[b, 2]), np.float64(med[b]))
            except Exception as e:                     # noqa: BLE001 - whatever the loop raises is raised
                err, Bc = (b, r, e), b
                break
            grids.append(g)
        if Bc == 0:
            break
        g0 = grids[0]
        if dur_t is None:
            duration = np.ascontiguousarray(g0["duration"], dtype=np.float64)
            dur_t = up(duration)
            oversample, objective = int(g0["oversample"]), (L.BLS_SNR if g0["objective"] == "snr" else L.BLS_LIKELIHOOD)
        if shared_grid:
            per_h, pofs = np.ascontiguousarray(g0["period"], dtype=np.float64), None
            P = len(per_h)
            total_p = Bc * P
        else:
            per_h, pofs = _csr([g["period"] for g in grids])
            P = int(pofs[-1])
            total_p = P
        d_per = up(per_h)
        k3 = [torch.empty(total_p, **f64) for _ in range(7)]
        o = np.ascontiguousarray(off[:Bc + 1])
        L.check(lib.lkb_bls_power_ex(L.ptr(d_t), L.ptr(d_y), L.ptr(d_w), L.ptr(o), Bc, L.ptr(d_per), L.ptr(pofs), P,
                                     L.ptr(dur_t), len(duration), oversample, objective,
                                     *[L.ptr(x) for x in k3], None, L.MEM_DEVICE, _stream_ptr()))
        # 2. the candidates
        cand = torch.empty((7, Bc), **f64)
        idx = torch.empty(Bc, dtype=torch.int64, device=dev)
        L.check(lib.lkb_bls_best(*[L.ptr(x) for x in k3[:6]], L.ptr(d_per), L.ptr(pofs), Bc, P,
                                 *[L.ptr(cand[k]) for k in range(7)], L.ptr(idx), L.MEM_DEVICE, _stream_ptr()))
        del k3
        cand_h, idx_h = cand.cpu().numpy(), idx.cpu().numpy()
        nan_lc = np.flatnonzero(idx_h < 0)
        if len(nan_lc):
            err, Bc = (int(nan_lc[0]), r, ValueError("All-NaN slice encountered")), int(nan_lc[0])
            if Bc == 0:
                break
        for k, name in enumerate(BLS_CANDIDATE_FIELDS):
            out[name][:Bc, r] = cand_h[k, :Bc]
        # 3. in-transit flags and levels (and the statistics) at the candidates
        per_c, dur_c, tt_c = cand_h[0, :Bc], cand_h[1, :Bc], cand_h[2, :Bc]
        t0 = tinfo[:Bc, 0]
        ttr = tt_c - t0
        caps = np.rint((tinfo[:Bc, 2] - t0 - ttr) / per_c) - np.rint((tinfo[:Bc, 1] - t0 - ttr) / per_c) + 1
        toff = np.zeros(Bc + 1, np.int64)
        np.cumsum(caps.astype(np.int64), out=toff[1:])
        o = np.ascontiguousarray(off[:Bc + 1])
        n_now = int(o[-1])
        st = _bls_stats_device(lib, d_t[:n_now], d_y[:n_now], d_w[:n_now], cand[0, :Bc].contiguous(),
                               cand[1, :Bc].contiguous(), cand[2, :Bc].contiguous(), True, o, toff)
        if return_stats:
            sh = {k: (v.cpu().numpy() if torch.is_tensor(v) else v) for k, v in st.items() if k != "in_transit"}
            sh["tstart"] = t0.copy()
            bad = np.flatnonzero(sh["status"] == L.E_SINGULAR)
            if len(bad):
                err, Bc = (int(bad[0]), r, np.linalg.LinAlgError("Singular matrix")), int(bad[0])
                if Bc == 0:
                    break
                o = np.ascontiguousarray(off[:Bc + 1])
                n_now = int(o[-1])
            rounds_stats.append(sh)
        # 4. lc[~mask], with what the next round's grid needs
        nt, ny, ndy, nw = (torch.empty(max(n_now, 1), **f64) for _ in range(4))
        nidx = torch.empty(max(n_now, 1), dtype=torch.int32, device=dev)
        steps = torch.empty(max(n_now, 1), **f64)
        ti = torch.empty((Bc, 3), **f64)
        fin = torch.empty(Bc, dtype=torch.uint8, device=dev)
        noff, soff = np.zeros(Bc + 1, np.int64), np.zeros(Bc + 1, np.int64)
        L.check(lib.lkb_transit_compact(L.ptr(d_t), L.ptr(d_y), L.ptr(d_dy), L.ptr(d_idx), L.ptr(o), Bc,
                                        L.ptr(st["in_transit"]), L.ptr(st["stats"][:Bc]), r,
                                        L.ptr(np.ascontiguousarray(off0[:Bc + 1])), L.ptr(masked), L.ptr(nt),
                                        L.ptr(ny), L.ptr(ndy), L.ptr(nw), L.ptr(nidx), L.ptr(noff), L.ptr(soff),
                                        L.ptr(ti), L.ptr(fin), L.ptr(steps), L.MEM_DEVICE, _stream_ptr()))
        d_t, d_y, d_dy, d_w, d_idx = nt, ny, ndy, nw, nidx
        off = noff
        n_h = np.diff(off)
        # 5. the median time step of the survivors
        if r + 1 < n_candidates:
            md = torch.empty(Bc, **f64)
            L.check(lib.lkb_nanmedian_std(L.ptr(steps), L.ptr(soff), Bc, L.ptr(md), None, L.MEM_DEVICE,
                                          _stream_ptr()))
            tinfo[:Bc] = ti.cpu().numpy()
            med[:Bc] = md.cpu().numpy()
    if err is not None:
        b, r, e = err
        raise _named_error(e, b, r) from e
    m = masked.cpu().numpy()
    out["masked_in"] = [m[off0[b]:off0[b + 1]].copy() for b in range(B)]
    if return_stats:
        out["stats"] = rounds_stats
    return out


def bls_bin_index(t_rel, min_t, period, bin_duration):
    lib = L.load()
    t_rel = np.ascontiguousarray(t_rel, dtype=np.float64)
    out = np.empty(len(t_rel), dtype=np.int32)
    L.check(lib.lkb_bls_bin_index(L.ptr(t_rel), len(t_rel), float(min_t), float(period), float(bin_duration),
                                  L.ptr(out), L.MEM_HOST, None))
    return out


# --------------------------------------------------------------------------------------
# flatten
# --------------------------------------------------------------------------------------
def flatten_csr(t, f, fe, exclude, offsets, window_length=101, polyorder=2, break_tolerance=5, niters=3, sigma=3,
                flat=None, flat_err=None, trend=None):
    """K4 on already concatenated host arrays (CSR `offsets` [B + 1]): `t`, `f`, `fe` (or None) float64 [total],
    `exclude` uint8 [total] or None (1 = leave the cadence out of the fit).  Output arrays may be passed in (e.g.
    page-locked buffers).  Returns (flat, flat_err, trend) float64 [total]."""
    lib = L.load()
    offsets = np.ascontiguousarray(offsets, dtype=np.int64)
    B = len(offsets) - 1
    total = int(offsets[-1])
    for name, a in (("t", t), ("f", f), ("fe", fe)):
        if a is not None and not (isinstance(a, np.ndarray) and a.dtype == np.float64 and a.shape == (total,)
                                  and a.flags.c_contiguous):
            raise ValueError("%s must be a C-contiguous float64 array of %d cadences" % (name, total))
    if exclude is not None and not (isinstance(exclude, np.ndarray) and exclude.dtype == np.uint8
                                    and exclude.shape == (total,) and exclude.flags.c_contiguous):
        raise ValueError("exclude must be a C-contiguous uint8 array of %d cadences" % total)
    outs = []
    for name, a in (("flat", flat), ("flat_err", flat_err), ("trend", trend)):
        if a is None:
            a = np.empty(total, dtype=np.float64)
        elif not (isinstance(a, np.ndarray) and a.dtype == np.float64 and a.shape == (total,) and a.flags.c_contiguous
                  and a.flags.writeable):
            raise ValueError("%s must be a writeable C-contiguous float64 array of %d cadences" % (name, total))
        outs.append(a)
    flat, flat_err, trend = outs
    bt = np.nan if break_tolerance is None else float(break_tolerance)
    L.check(lib.lkb_flatten(L.ptr(t), L.ptr(f), L.ptr(fe), L.ptr(exclude), L.ptr(offsets), B, int(window_length),
                            int(polyorder), bt, int(niters), float(sigma), L.ptr(flat), L.ptr(flat_err),
                            L.ptr(trend), L.MEM_HOST, None))
    return flat, flat_err, trend


def flatten(times, fluxes, flux_errs=None, masks=None, window_length=101, polyorder=2, break_tolerance=5,
            niters=3, sigma=3):
    """K4.  Lists of per-LC arrays.  `masks`: list of bool arrays, True = exclude (lightkurve
    semantics) or None.  Returns (flat, flat_err, trend) as lists of float64 arrays."""
    B = len(times)
    t, offsets = _csr(times)
    f, foff = _csr(fluxes)
    if not np.array_equal(offsets, foff):
        raise ValueError("time and flux lengths differ")
    fe = None
    if flux_errs is not None:
        fe, eoff = _csr(flux_errs)
        if not np.array_equal(offsets, eoff):
            raise ValueError("time and flux_err lengths differ")
    ex = None
    if masks is not None:
        if len(masks) != B or any(len(m) != len(tt) for m, tt in zip(masks, times)):
            raise ValueError("time and mask lengths differ")
        ex = np.ascontiguousarray(np.concatenate([np.asarray(m, dtype=bool) for m in masks]).astype(np.uint8))
    flat, flat_err, trend = flatten_csr(t, f, fe, ex, offsets, window_length, polyorder, break_tolerance, niters, sigma)
    sp = lambda a: [a[offsets[b]:offsets[b + 1]] for b in range(B)]
    return sp(flat), sp(flat_err), sp(trend)


# --------------------------------------------------------------------------------------
# regression
# --------------------------------------------------------------------------------------
def regress(X, Y, flux_err=None, cadence_mask=None, prior_mu=None, prior_sigma=None, sigma=5, niters=5,
            return_cov=False, exact_invariant=False):
    """K5.  X [N, K] (shared) or [B, N, K]; Y [B, N]; flux_err [B, N] or None (ones);
    cadence_mask bool [B, N] or None; prior_mu / prior_sigma [K] (shared) or [B, K] (one prior per light curve).
    `exact_invariant`: each light curve's results are bitwise independent of the batch and of a shared or batched X
    (LKB_REGRESS_EXACT_INVARIANT).  Returns dict(coefficients [B,K], model [B,N] (median-subtracted), outlier_mask
    bool [B,N], status int32 [B]).  With CUDA torch tensors (float64; cadence_mask uint8) the call runs in device
    mode on the current stream and returns tensors (outlier_mask uint8)."""
    if _is_torch(Y):
        return _regress_device(X, Y, flux_err, cadence_mask, prior_mu, prior_sigma, sigma, niters, exact_invariant)
    lib = L.load()
    X = np.ascontiguousarray(X, dtype=np.float64)
    Y = np.ascontiguousarray(np.atleast_2d(Y), dtype=np.float64)
    B, N = Y.shape
    batched = X.ndim == 3
    K = X.shape[-1]
    if X.shape[-2] != N or (batched and X.shape[0] != B):
        raise ValueError("X shape %s does not match Y shape %s" % (X.shape, Y.shape))
    fe = None if flux_err is None else np.ascontiguousarray(np.broadcast_to(flux_err, Y.shape), dtype=np.float64)
    cm = None if cadence_mask is None else \
        np.ascontiguousarray(np.broadcast_to(np.asarray(cadence_mask, dtype=bool), Y.shape).astype(np.uint8))
    pm = None if prior_mu is None else np.ascontiguousarray(prior_mu, dtype=np.float64)
    ps = None if prior_sigma is None else np.ascontiguousarray(prior_sigma, dtype=np.float64)
    prior_batched = ps is not None and ps.ndim == 2
    for name, v in (("prior_mu", pm), ("prior_sigma", ps)):
        if v is not None and v.shape != ((B, K) if prior_batched else (K,)):
            raise ValueError("%s must have shape (%d,) or (%d, %d), got %s" % (name, K, B, K, v.shape))
    coeff = np.empty((B, K), dtype=np.float64)
    model = np.empty((B, N), dtype=np.float64)
    om = np.empty((B, N), dtype=np.uint8)
    status = np.empty(B, dtype=np.int32)
    cov = np.empty((B, K, K), dtype=np.float64) if return_cov else None
    L.check(lib.lkb_regress_ex(L.ptr(X), 1 if batched else 0, L.ptr(Y), L.ptr(fe), L.ptr(cm), L.ptr(pm), L.ptr(ps),
                               B, N, K, float(sigma), int(niters), L.ptr(coeff), L.ptr(model), L.ptr(om),
                               L.ptr(status), L.ptr(cov), L.MEM_HOST, None, 1 if prior_batched else 0,
                               L.REGRESS_EXACT_INVARIANT if exact_invariant else 0))
    out = dict(coefficients=coeff, model=model, outlier_mask=om.astype(bool), status=status)
    if return_cov:
        out["covariance"] = cov
    return out


def _regress_device(X, Y, flux_err, cadence_mask, prior_mu, prior_sigma, sigma, niters, exact_invariant):
    import torch
    lib = L.load()
    for name, t, dt in (("X", X, torch.float64), ("Y", Y, torch.float64), ("flux_err", flux_err, torch.float64),
                        ("cadence_mask", cadence_mask, torch.uint8), ("prior_mu", prior_mu, torch.float64),
                        ("prior_sigma", prior_sigma, torch.float64)):
        if t is not None and not (_is_torch(t) and t.is_cuda and t.is_contiguous() and t.dtype == dt):
            raise ValueError("%s must be a contiguous CUDA %s tensor in device mode" % (name, dt))
    if Y.dim() != 2:
        raise ValueError("Y must be [B, N]")
    B, N = Y.shape
    batched = X.dim() == 3
    K = X.shape[-1]
    if X.shape[-2] != N or (batched and X.shape[0] != B):
        raise ValueError("X shape %s does not match Y shape %s" % (tuple(X.shape), tuple(Y.shape)))
    for name, t in (("flux_err", flux_err), ("cadence_mask", cadence_mask)):
        if t is not None and tuple(t.shape) != (B, N):
            raise ValueError("%s must be [B, N]" % name)
    if (prior_mu is None) != (prior_sigma is None):
        raise ValueError("Please specify both `prior_mu` and `prior_sigma`")
    prior_batched = prior_sigma is not None and prior_sigma.dim() == 2
    for name, v in (("prior_mu", prior_mu), ("prior_sigma", prior_sigma)):
        if v is not None and tuple(v.shape) != ((B, K) if prior_batched else (K,)):
            raise ValueError("%s must have shape (%d,) or (%d, %d)" % (name, K, B, K))
    dev = Y.device
    coeff = torch.empty((B, K), dtype=torch.float64, device=dev)
    model = torch.empty((B, N), dtype=torch.float64, device=dev)
    om = torch.empty((B, N), dtype=torch.uint8, device=dev)
    status = torch.empty(B, dtype=torch.int32, device=dev)
    L.check(lib.lkb_regress_ex(L.ptr(X), 1 if batched else 0, L.ptr(Y), L.ptr(flux_err), L.ptr(cadence_mask),
                               L.ptr(prior_mu), L.ptr(prior_sigma), B, N, K, float(sigma), int(niters), L.ptr(coeff),
                               L.ptr(model), L.ptr(om), L.ptr(status), None, L.MEM_DEVICE, _stream_ptr(),
                               1 if prior_batched else 0, L.REGRESS_EXACT_INVARIANT if exact_invariant else 0))
    return dict(coefficients=coeff, model=model, outlier_mask=om, status=status)


def elasticnet(X, Y, cadence_mask=None, alpha=1e-20, l1_ratio=0.01, max_iter=1000, tol=1e-4, positive=False):
    """K8.  scikit-learn's ElasticNet(alpha, l1_ratio, fit_intercept=False, max_iter, tol, positive).fit on the used
    cadences of each light curve, and the CBVCorrector model.  X [N, K] (shared) or [B, N, K]; Y [B, N]; cadence_mask
    bool [B, N] or None (all).  Returns dict(coefficients [B, K], model [B, N] (= X[:, :-1] coef[:-1] minus its
    median over all cadences), n_iter int32 [B], dual_gap [B], converged bool [B])."""
    lib = L.load()
    X = np.ascontiguousarray(X, dtype=np.float64)
    Y = np.ascontiguousarray(np.atleast_2d(Y), dtype=np.float64)
    B, N = Y.shape
    batched = X.ndim == 3
    K = X.shape[-1]
    if X.ndim not in (2, 3) or X.shape[-2] != N or (batched and X.shape[0] != B):
        raise ValueError("X shape %s does not match Y shape %s" % (X.shape, Y.shape))
    cm = None if cadence_mask is None else \
        np.ascontiguousarray(np.broadcast_to(np.asarray(cadence_mask, dtype=bool), Y.shape).astype(np.uint8))
    coeff = np.empty((B, K), dtype=np.float64)
    model = np.empty((B, N), dtype=np.float64)
    n_iter = np.empty(B, dtype=np.int32)
    gap = np.empty(B, dtype=np.float64)
    conv = np.empty(B, dtype=np.uint8)
    L.check(lib.lkb_elasticnet(L.ptr(X), 1 if batched else 0, L.ptr(Y), L.ptr(cm), B, N, K, float(alpha),
                               float(l1_ratio), int(max_iter), float(tol), 1 if positive else 0, L.ptr(coeff),
                               L.ptr(model), L.ptr(n_iter), L.ptr(gap), L.ptr(conv), L.MEM_HOST, None))
    return dict(coefficients=coeff, model=model, n_iter=n_iter, dual_gap=gap, converged=conv.astype(bool))


def _k9_array(x, dtype, torch_dtype_name):
    """(array or tensor, mem) for a K9 input: CUDA torch tensors are passed through (device mode)."""
    if _is_torch(x):
        if not (x.is_cuda and x.is_contiguous() and str(x.dtype) == "torch." + torch_dtype_name):
            raise ValueError("device inputs must be contiguous CUDA %s tensors" % torch_dtype_name)
        return x, L.MEM_DEVICE
    return np.ascontiguousarray(x, dtype=dtype), L.MEM_HOST


def underfit_metric(pool, target, nb_offsets, nb_index):
    """K9.  The under-fitting metric of metrics.py:178-255 for B targets whose neighbours are rows of one pool.
    pool [P, G] and target [B, G] fp64 on one cadence grid, NaN where a value is absent (numpy, or CUDA torch tensors
    for device mode); nb_offsets int64 [B + 1] and nb_index [nb_offsets[-1]] (host): the pool rows of each target.
    Returns dict(metric [B], n_used int32 [B] (cadences used), c3_mean [B] (the nanmean of |c|^3)), numpy or torch."""
    lib = L.load()
    pool, mem = _k9_array(pool, np.float64, "float64")
    target, mem_t = _k9_array(target, np.float64, "float64")
    if mem != mem_t:
        raise ValueError("pool and target must both be host arrays or both CUDA tensors")
    if pool.ndim != 2 or target.ndim != 2 or pool.shape[1] != target.shape[1]:
        raise ValueError("pool [P, G] and target [B, G] must share G")
    P, G = pool.shape
    B = target.shape[0]
    off = np.ascontiguousarray(nb_offsets, dtype=np.int64)
    idx = np.ascontiguousarray(nb_index, dtype=np.int32)
    if off.shape != (B + 1,) or len(idx) != off[-1]:
        raise ValueError("nb_offsets must have B + 1 entries and end at len(nb_index)")
    if mem == L.MEM_DEVICE:
        import torch
        metric = torch.empty(B, dtype=torch.float64, device=target.device)
        n_used = torch.empty(B, dtype=torch.int32, device=target.device)
        c3 = torch.empty(B, dtype=torch.float64, device=target.device)
        stream = _stream_ptr()
    else:
        metric, n_used, c3, stream = np.empty(B), np.empty(B, np.int32), np.empty(B), None
    L.check(lib.lkb_underfit_metric(L.ptr(pool), P, L.ptr(target), B, G, L.ptr(off), L.ptr(idx), L.ptr(metric),
                                    L.ptr(n_used), L.ptr(c3), mem, stream))
    return dict(metric=metric, n_used=n_used, c3_mean=c3)


def overfit_terms(corrected, original, noise, offsets=None, n_samples=1):
    """K9.  The per-light-curve terms of the over-fitting metric (metrics.py:23-123) from float32 power rows.
    corrected / original: [B, F] (one grid) or the rows back to back with `offsets` int64 [B + 1] (host); noise: the
    `n_samples` noise rows of each light curve back to back (light curve b's rows at n_samples * offsets[b]).  numpy,
    or CUDA torch tensors for device mode.  Returns dict(n_positive int32 [B], sum_positive [B],
    noise_mean [B, n_samples])."""
    lib = L.load()
    corrected, mem = _k9_array(corrected, np.float32, "float32")
    original, _ = _k9_array(original, np.float32, "float32")
    S = int(n_samples)
    if offsets is None:
        if corrected.ndim != 2:
            raise ValueError("without offsets the power rows must be [B, F]")
        B, F = corrected.shape
        off = None
    else:
        off = np.ascontiguousarray(offsets, dtype=np.int64)
        if off.ndim != 1 or len(off) < 2 or off[0] != 0 or np.any(np.diff(off) < 0):
            raise ValueError("offsets must be an ascending int64 CSR array starting at 0")
        B, F = len(off) - 1, 0
    if tuple(original.shape) != tuple(corrected.shape):
        raise ValueError("corrected and original power must have the same shape")
    n_tot = B * F if off is None else int(off[-1])
    n_rows = corrected.numel() if mem == L.MEM_DEVICE else corrected.size
    if n_rows != n_tot:
        raise ValueError("offsets end at %d but the power rows hold %d values" % (n_tot, n_rows))
    if S > 0:
        noise, _ = _k9_array(noise, np.float32, "float32")
        if (noise.numel() if mem == L.MEM_DEVICE else noise.size) != S * n_tot:
            raise ValueError("noise must hold n_samples rows per light curve")
    else:
        noise = None
    if mem == L.MEM_DEVICE:
        import torch
        dev = corrected.device
        npos = torch.empty(B, dtype=torch.int32, device=dev)
        spos = torch.empty(B, dtype=torch.float64, device=dev)
        nmean = torch.empty((B, S), dtype=torch.float64, device=dev)
        stream = _stream_ptr()
    else:
        npos, spos, nmean, stream = np.empty(B, np.int32), np.empty(B), np.empty((B, S)), None
    L.check(lib.lkb_overfit_terms(L.ptr(corrected), L.ptr(original), L.ptr(noise), L.ptr(off), B, F, S, L.ptr(npos),
                                  L.ptr(spos), L.ptr(nmean) if S else None, mem, stream))
    return dict(n_positive=npos, sum_positive=spos, noise_mean=nmean)


def nanmedian_std(arrays):
    """K6.  np.nanmedian and np.nanstd of each array."""
    lib = L.load()
    x, offsets = _csr(arrays)
    B = len(arrays)
    med = np.empty(B, dtype=np.float64)
    sd = np.empty(B, dtype=np.float64)
    L.check(lib.lkb_nanmedian_std(L.ptr(x), L.ptr(offsets), B, L.ptr(med), L.ptr(sd), L.MEM_HOST, None))
    return med, sd


def sigma_clip(arrays, sigma_lower=3.0, sigma_upper=3.0, maxiters=5, offsets=None):
    """K11.  astropy.stats.sigma_clip(x, sigma_lower=, sigma_upper=, maxiters=).mask (cenfunc="median", stdfunc="std")
    of each light curve; maxiters None (or < 0) clips until a round clips nothing.  `arrays`: a list of 1-D arrays
    (host mode), or the concatenated CUDA float64 tensor with the host int64 CSR `offsets` [B + 1] (device mode, on
    the current torch stream).  Returns dict(mask (host: a list of bool arrays; device: a uint8 tensor), center,
    std (median and standard deviation, ddof 0, of the kept values), n_kept, offsets)."""
    lib = L.load()
    mi = -1 if maxiters is None else int(maxiters)
    if _is_torch(arrays):
        import torch
        if offsets is None:
            raise ValueError("device mode needs the host CSR `offsets`")
        if not (arrays.is_cuda and arrays.is_contiguous() and arrays.dim() == 1 and arrays.dtype == torch.float64):
            raise ValueError("device mode: the values must be a contiguous one-dimensional CUDA float64 tensor")
        off = np.ascontiguousarray(offsets, dtype=np.int64)
        B = len(off) - 1
        if B <= 0 or off[0] != 0 or np.any(np.diff(off) < 0) or off[-1] != arrays.numel():
            raise ValueError("offsets do not describe the %d values" % arrays.numel())
        dev = arrays.device
        mask = torch.empty(max(int(off[-1]), 1), dtype=torch.uint8, device=dev)
        center, sd = torch.empty(B, dtype=torch.float64, device=dev), torch.empty(B, dtype=torch.float64, device=dev)
        nk = torch.empty(B, dtype=torch.int64, device=dev)
        L.check(lib.lkb_sigma_clip(L.ptr(arrays), L.ptr(off), B, float(sigma_lower), float(sigma_upper), mi,
                                   L.ptr(mask), L.ptr(center), L.ptr(sd), L.ptr(nk), L.MEM_DEVICE, _stream_ptr()))
        return dict(mask=mask[:int(off[-1])], center=center, std=sd, n_kept=nk, offsets=off)
    B = len(arrays)
    if B == 0:
        return dict(mask=[], center=np.zeros(0), std=np.zeros(0), n_kept=np.zeros(0, np.int64),
                    offsets=np.zeros(1, np.int64))
    x, off = _csr(arrays)
    mask = np.empty(max(len(x), 1), dtype=np.uint8)
    center, sd, nk = np.empty(B), np.empty(B), np.empty(B, dtype=np.int64)
    L.check(lib.lkb_sigma_clip(L.ptr(x), L.ptr(off), B, float(sigma_lower), float(sigma_upper), mi, L.ptr(mask),
                               L.ptr(center), L.ptr(sd), L.ptr(nk), L.MEM_HOST, None))
    m = mask.view(bool)
    return dict(mask=[m[off[b]:off[b + 1]] for b in range(B)], center=center, std=sd, n_kept=nk, offsets=off)


def cdpp(times, fluxes, durations=13, savgol_window=101, savgol_polyorder=2, sigma=5.0, offsets=None):
    """K4 + K11 + K12.  LightCurve.estimate_cdpp (lightcurve.py:1764-1833) of each light curve at each transit
    duration (in cadences, ints >= 1): flatten, remove_outliers(sigma), normalize("ppm") and the standard deviation of
    the running means, with the flattened flux kept on the device.  `times` / `fluxes`: lists of 1-D arrays (host
    mode), or the concatenated CUDA float64 tensors with the host int64 CSR `offsets` [B + 1] (device mode, on the
    current torch stream).  Returns the [B, D] ppm values (numpy, or a CUDA float64 tensor); NaN where a light
    curve keeps no cadence."""
    lib = L.load()
    dur = np.ascontiguousarray(np.atleast_1d(durations), dtype=np.int32)
    if dur.ndim != 1 or len(dur) == 0 or not np.array_equal(dur, np.atleast_1d(durations)):
        raise ValueError("durations must be a non-empty sequence of integers")
    D = len(dur)
    if _is_torch(fluxes):
        import torch
        if offsets is None:
            raise ValueError("device mode needs the host CSR `offsets`")
        for name, v in (("times", times), ("fluxes", fluxes)):
            if not (_is_torch(v) and v.is_cuda and v.is_contiguous() and v.dim() == 1 and v.dtype == torch.float64):
                raise ValueError("device mode: %s must be a contiguous one-dimensional CUDA float64 tensor" % name)
        off = np.ascontiguousarray(offsets, dtype=np.int64)
        B = len(off) - 1
        if B <= 0 or off[0] != 0 or np.any(np.diff(off) < 0) or off[-1] != fluxes.numel() or \
                times.numel() != fluxes.numel():
            raise ValueError("offsets do not describe the time and flux tensors")
        out = torch.empty((B, D), dtype=torch.float64, device=fluxes.device)
        L.check(lib.lkb_cdpp(L.ptr(times), L.ptr(fluxes), L.ptr(off), B, L.ptr(dur), D, int(savgol_window),
                             int(savgol_polyorder), float(sigma), L.ptr(out), L.MEM_DEVICE, _stream_ptr()))
        return out
    B = len(times)
    if B == 0:
        return np.zeros((0, D))
    t, off = _csr(times)
    f, foff = _csr(fluxes)
    if not np.array_equal(off, foff):
        raise ValueError("time and flux lengths differ")
    out = np.empty((B, D))
    L.check(lib.lkb_cdpp(L.ptr(t), L.ptr(f), L.ptr(off), B, L.ptr(dur), D, int(savgol_window), int(savgol_polyorder),
                         float(sigma), L.ptr(out), L.MEM_HOST, None))
    return out


def _device_csr(x, name, dtype, n=None):
    """Checks that `x` is a contiguous one-dimensional CUDA tensor of `dtype` (of n values when n is given)."""
    if not (_is_torch(x) and x.is_cuda and x.is_contiguous() and x.dim() == 1 and x.dtype == dtype):
        raise ValueError("device mode: %s must be a contiguous one-dimensional CUDA %s tensor" % (name, dtype))
    if n is not None and x.numel() != n:
        raise ValueError("device mode: %s has %d values, the offsets describe %d" % (name, x.numel(), n))


def _host_offsets(offsets, what):
    off = np.ascontiguousarray(offsets, dtype=np.int64)
    if off.ndim != 1 or len(off) < 2 or off[0] != 0 or np.any(np.diff(off) < 0):
        raise ValueError("%s must be a non-decreasing int64 CSR starting at 0" % what)
    return off


def fold(times, t0, shift, period, wrap, normalize=False, offsets=None):
    """K13.  LightCurve.fold's phase of each light curve, rel = ((t - t0) + shift + (period - wrap)) % period -
    (period - wrap) (numpy's remainder), stably sorted, divided by the period when `normalize`.  `t0`, `shift`,
    `period`, `wrap`: one value per light curve (days).  `times`: a list of 1-D arrays (host mode), or the
    concatenated CUDA float64 tensor with the host int64 CSR `offsets` [B + 1] (device mode, on the current torch
    stream).  Returns dict(phase, perm): the sorted phases and the int32 permutation (each light curve's own cadence
    index of each sorted position), as lists of arrays (host) or concatenated tensors (device)."""
    lib = L.load()
    if _is_torch(times):
        import torch
        if offsets is None:
            raise ValueError("device mode needs the host CSR `offsets`")
        off = _host_offsets(offsets, "offsets")
        _device_csr(times, "times", torch.float64, int(off[-1]))
        B = len(off) - 1
    else:
        B = len(times)
        if B == 0:
            return dict(phase=[], perm=[])
        t, off = _csr(times)
    pars = [np.ascontiguousarray(np.broadcast_to(np.asarray(v, dtype=np.float64), (B,))) for v in (t0, shift, period,
                                                                                                   wrap)]
    n = int(off[-1])
    if _is_torch(times):
        import torch
        phase = torch.empty(max(n, 1), dtype=torch.float64, device=times.device)
        perm = torch.empty(max(n, 1), dtype=torch.int32, device=times.device)
        L.check(lib.lkb_fold(L.ptr(times), L.ptr(off), B, *[L.ptr(p) for p in pars], int(bool(normalize)),
                             L.ptr(phase), L.ptr(perm), L.MEM_DEVICE, _stream_ptr()))
        return dict(phase=phase[:n], perm=perm[:n])
    phase = np.empty(max(n, 1))
    perm = np.empty(max(n, 1), dtype=np.int32)
    L.check(lib.lkb_fold(L.ptr(t), L.ptr(off), B, *[L.ptr(p) for p in pars], int(bool(normalize)), L.ptr(phase),
                         L.ptr(perm), L.MEM_HOST, None))
    return dict(phase=[phase[off[b]:off[b + 1]] for b in range(B)], perm=[perm[off[b]:off[b + 1]] for b in range(B)])


_BIN_AGGREGATES = {"nanmean": L.BIN_NANMEAN, "nanmedian": L.BIN_NANMEDIAN}


def bin(times, fluxes, flux_errs, starts, ends, index_edges=False, aggregate="nanmean", offsets=None,
        bin_offsets=None):
    """K13.  LightCurve.bin of each light curve with the given bin edges: the cadences are stably sorted by time and
    cadence t falls in bin j = searchsorted(starts, t, "right") - 1 when t < ends[j] (t <= ends[-1] in the last bin).
    `starts` / `ends`: per light curve, times (float64) or, with `index_edges`, indices into its time-sorted cadences.
    `aggregate`: "nanmean" or "nanmedian" of the flux; the error is the root mean square of the finite errors when the
    light curve has any, else the bin's nanstd of the flux; `flux_errs` may be None (no errors).  Host mode: lists of
    1-D arrays.  Device mode: concatenated CUDA tensors (float64; int32 index edges) with the host int64 CSRs
    `offsets` of the cadences and `bin_offsets` of the bins.  Returns dict(time (bin centres), flux, flux_err, count),
    lists of arrays (host) or concatenated tensors (device)."""
    lib = L.load()
    if aggregate not in _BIN_AGGREGATES:
        raise ValueError("aggregate must be one of %s" % sorted(_BIN_AGGREGATES))
    agg = _BIN_AGGREGATES[aggregate]
    if _is_torch(times):
        import torch
        if offsets is None or bin_offsets is None:
            raise ValueError("device mode needs the host CSRs `offsets` and `bin_offsets`")
        off = _host_offsets(offsets, "offsets")
        boff = _host_offsets(bin_offsets, "bin_offsets")
        if len(boff) != len(off):
            raise ValueError("offsets and bin_offsets describe different numbers of light curves")
        n, nb = int(off[-1]), int(boff[-1])
        _device_csr(times, "times", torch.float64, n)
        _device_csr(fluxes, "fluxes", torch.float64, n)
        if flux_errs is not None:
            _device_csr(flux_errs, "flux_errs", torch.float64, n)
        edt = torch.int32 if index_edges else torch.float64
        _device_csr(starts, "starts", edt, nb)
        _device_csr(ends, "ends", edt, nb)
        B, dev = len(off) - 1, times.device
        centre, flux, err = (torch.empty(max(nb, 1), dtype=torch.float64, device=dev) for _ in range(3))
        count = torch.empty(max(nb, 1), dtype=torch.int32, device=dev)
        e_t = [L.ptr(starts), L.ptr(ends), None, None] if not index_edges else [None, None, L.ptr(starts), L.ptr(ends)]
        L.check(lib.lkb_bin(L.ptr(times), L.ptr(fluxes), None if flux_errs is None else L.ptr(flux_errs), L.ptr(off),
                            B, L.ptr(boff), *e_t, agg, L.ptr(centre), L.ptr(flux), L.ptr(err), L.ptr(count),
                            L.MEM_DEVICE, _stream_ptr()))
        return dict(time=centre[:nb], flux=flux[:nb], flux_err=err[:nb], count=count[:nb])
    B = len(times)
    if B == 0:
        return dict(time=[], flux=[], flux_err=[], count=[])
    t, off = _csr(times)
    f, foff = _csr(fluxes)
    fe = None
    if flux_errs is not None:
        fe, eoff = _csr(flux_errs)
        if not np.array_equal(off, eoff):
            raise ValueError("time and flux_err lengths differ")
    if not np.array_equal(off, foff):
        raise ValueError("time and flux lengths differ")
    edt = np.int32 if index_edges else np.float64
    s, boff = _csr(starts, edt)
    e, eboff = _csr(ends, edt)
    if len(boff) != B + 1 or not np.array_equal(boff, eboff):
        raise ValueError("starts and ends must have one array per light curve, of the same lengths")
    nb = int(boff[-1])
    centre, flux, err = np.empty(max(nb, 1)), np.empty(max(nb, 1)), np.empty(max(nb, 1))
    count = np.empty(max(nb, 1), dtype=np.int32)
    e_t = [L.ptr(s), L.ptr(e), None, None] if not index_edges else [None, None, L.ptr(s), L.ptr(e)]
    L.check(lib.lkb_bin(L.ptr(t), L.ptr(f), None if fe is None else L.ptr(fe), L.ptr(off), B, L.ptr(boff), *e_t, agg,
                        L.ptr(centre), L.ptr(flux), L.ptr(err), L.ptr(count), L.MEM_HOST, None))
    sl = [slice(boff[b], boff[b + 1]) for b in range(B)]
    return dict(time=[centre[x] for x in sl], flux=[flux[x] for x in sl], flux_err=[err[x] for x in sl],
                count=[count[x] for x in sl])


def logmedian_windows(frequency, filter_width):
    """Half-open bin ranges of the reference's moving log10-frequency window (periodogram.py:267-277) for an
    ASCENDING frequency grid: window w = { i : |log10 f_i - x0_w| < filter_width }, x0 advancing by
    filter_width / 2 from log10 f_0 (the same fp64 accumulation).  Empty windows are kept (they add nothing)."""
    logf = np.log10(np.asarray(frequency, dtype=np.float64))
    F = len(logf)
    x0s = []
    x0 = logf[0]
    while x0 < logf[-1]:
        x0s.append(x0)
        x0 += 0.5 * filter_width
    x0s = np.asarray(x0s, dtype=np.float64)
    lo = np.searchsorted(logf, x0s - filter_width, side="right")
    hi = np.searchsorted(logf, x0s + filter_width, side="left")
    # the reference's expression is |logf - x0| < w in fp64: settle the edge bins with exactly that
    inside = lambda i, c: np.abs(logf[np.clip(i, 0, F - 1)] - c) < filter_width
    for _ in range(3):
        grow = (lo > 0) & inside(lo - 1, x0s)
        lo = np.where(grow, lo - 1, lo)
        shrink = (lo < hi) & ~inside(lo, x0s)
        lo = np.where(shrink, lo + 1, lo)
        grow = (hi < F) & inside(hi, x0s)
        hi = np.where(grow, hi + 1, hi)
        shrink = (hi > lo) & ~inside(hi - 1, x0s)
        hi = np.where(shrink, hi - 1, hi)
    return lo.astype(np.int32), np.maximum(hi, lo).astype(np.int32)


def pg_logmedian(frequency, power, filter_width):
    """Background of B periodograms on one frequency grid (Periodogram.smooth(method="logmedian")).
    power [B, F] (or [F]); returns the same shape, fp64."""
    lib = L.load()
    freq = np.asarray(frequency, dtype=np.float64)
    p = np.asarray(power, dtype=np.float64)
    one = p.ndim == 1
    p = np.ascontiguousarray(np.atleast_2d(p))
    B, F = p.shape
    if len(freq) != F:
        raise ValueError("frequency and power must have the same length")
    order = None
    if F > 1 and not np.all(np.diff(freq) >= 0):
        order = np.argsort(freq, kind="stable")
        freq, p = freq[order], np.ascontiguousarray(p[:, order])
    lo, hi = logmedian_windows(freq, filter_width)
    out = np.empty((B, F), dtype=np.float64)
    if len(lo) == 0:
        out[:] = np.nan
    else:
        lo, hi = np.ascontiguousarray(lo), np.ascontiguousarray(hi)
        L.check(lib.lkb_pg_logmedian(L.ptr(p), B, F, L.ptr(lo), L.ptr(hi), len(lo), (8.0 / 9.0) ** 3, L.ptr(out),
                                     L.MEM_HOST, None))
    if order is not None:
        inv = np.empty_like(order)
        inv[order] = np.arange(F)
        out = out[:, inv]
    return out[0] if one else out


def pg_logmedian_ragged(frequencies, power, filter_width, bin_offsets=None, snr=False):
    """Periodogram.smooth(method="logmedian") of B periodograms on their own ascending frequency grids
    (`frequencies`: list of host arrays).  `power`: list of host arrays (host mode), or the concatenated CUDA float32
    / float64 tensor with its host int64 CSR `bin_offsets` (device mode, on the current torch stream).  Returns the
    backgrounds and, with `snr`, also power / background (Periodogram.flatten), fp64: lists of arrays (host) or
    concatenated tensors (device)."""
    lib = L.load()
    B = len(frequencies)
    wins = [logmedian_windows(f, filter_width) for f in frequencies]
    lo, woff = _csr([w[0] for w in wins], np.int32)
    hi, _ = _csr([w[1] for w in wins], np.int32)
    if _is_torch(power):
        import torch
        boff = _host_offsets(bin_offsets, "bin_offsets")
        if len(boff) != B + 1 or any(boff[b + 1] - boff[b] != len(f) for b, f in enumerate(frequencies)):
            raise ValueError("bin_offsets do not describe the frequency grids")
        if power.dtype not in (torch.float32, torch.float64):
            raise TypeError("power must be float32 or float64")
        _device_csr(power, "power", power.dtype, int(boff[-1]))
        n = max(int(boff[-1]), 1)
        bkg = torch.empty(n, dtype=torch.float64, device=power.device)
        out_snr = torch.empty(n, dtype=torch.float64, device=power.device) if snr else None
        L.check(lib.lkb_pg_logmedian_ragged(L.ptr(power), L.DTYPE_F32 if power.dtype == torch.float32 else L.DTYPE_F64,
                                            L.ptr(boff), B, L.ptr(lo), L.ptr(hi), L.ptr(woff), (8.0 / 9.0) ** 3,
                                            L.ptr(bkg), L.ptr(out_snr), L.MEM_DEVICE, _stream_ptr()))
        nb = int(boff[-1])
        return (bkg[:nb], out_snr[:nb]) if snr else bkg[:nb]
    p, boff = _csr(power)
    if len(boff) != B + 1 or any(boff[b + 1] - boff[b] != len(f) for b, f in enumerate(frequencies)):
        raise ValueError("power and frequency lengths differ")
    bkg = np.empty(max(len(p), 1))
    out_snr = np.empty(max(len(p), 1)) if snr else None
    L.check(lib.lkb_pg_logmedian_ragged(L.ptr(p), L.DTYPE_F64, L.ptr(boff), B, L.ptr(lo), L.ptr(hi), L.ptr(woff),
                                        (8.0 / 9.0) ** 3, L.ptr(bkg), L.ptr(out_snr), L.MEM_HOST, None))
    sp = lambda x: [x[boff[b]:boff[b + 1]] for b in range(B)]
    return (sp(bkg), sp(out_snr)) if snr else sp(bkg)


# --------------------------------------------------------------------------------------
# gap filling and the seismology spectra (K15)
# --------------------------------------------------------------------------------------
GAP_DECREASING, GAP_POSITIVE, GAP_TOO_LONG = 1, 2, 4


def _gap_reject(b, flags, dt):
    """The ValueError for light curve b that fill_gaps refuses (the loop would mis-assign or never end), or None."""
    if flags & GAP_DECREASING:
        return ValueError("light curve %d: its times decrease; fill_gaps needs them in order" % b)
    if flags & GAP_POSITIVE and not dt > 0:
        return ValueError("light curve %d: the median time step is %r while some step is positive; the gap "
                          "filling loop would never end" % (b, float(dt)))
    if flags & GAP_TOO_LONG:
        return ValueError("light curve %d: a gap spans more than 2**24 median time steps, or the median step is too "
                          "small to advance the time" % b)
    return None


def fill_gaps_device(d_t, d_y, d_e, offsets, std):
    """K15 (+ K6 for the median step): LightCurve.fill_gaps(method="gaussian_noise") of the NaN-free light curves in
    the concatenated CUDA float64 tensors `d_t` (finite times), `d_y`, `d_e` with the host int64 CSR `offsets`.
    `std(plan)` returns the host [B] noise levels, given plan = dict(dt, mean, n_ins, flags) (host arrays; called
    after the plan's one synchronisation).  Refused light curves raise ValueError naming the first; then the normal
    deviates come from ONE np.random.standard_normal(sum of n_ins) draw, which equals the loop's consecutive
    np.random.normal(mean, std, n_ins[b]) draws.  Returns (t, flux, flux_err, out_offsets, plan), CUDA tensors and
    host arrays."""
    import torch
    lib = L.load()
    off = _host_offsets(offsets, "offsets")
    B, n = len(off) - 1, int(off[-1])
    for name, x in (("t", d_t), ("flux", d_y), ("flux_err", d_e)):
        _device_csr(x, name, torch.float64)
        if x.numel() < max(n, 1):
            raise ValueError("device mode: %s has fewer values than the offsets describe" % name)
    dev = d_t.device
    dt, mean = torch.empty(B, dtype=torch.float64, device=dev), torch.empty(B, dtype=torch.float64, device=dev)
    n_ins = torch.empty(B, dtype=torch.int64, device=dev)
    flags = torch.empty(B, dtype=torch.int32, device=dev)
    L.check(lib.lkb_fill_gaps_plan(L.ptr(d_t), L.ptr(d_y), L.ptr(off), B, L.ptr(dt), L.ptr(mean), L.ptr(n_ins),
                                   L.ptr(flags), L.MEM_DEVICE, _stream_ptr()))
    plan = dict(dt=dt.cpu().numpy(), mean=mean.cpu().numpy(), n_ins=n_ins.cpu().numpy(), flags=flags.cpu().numpy())
    for b in range(B):
        e = _gap_reject(b, int(plan["flags"][b]), plan["dt"][b])
        if e is not None:
            raise e
    s = np.ascontiguousarray(std(plan), dtype=np.float64)
    noff = off.copy()
    noff[1:] += np.cumsum(plan["n_ins"])
    nz = int(noff[-1] - off[-1])
    z = torch.from_numpy(np.ascontiguousarray(np.random.standard_normal(nz))).to(dev) if nz else None
    d_s = torch.from_numpy(s).to(dev)
    nn = max(int(noff[-1]), 1)
    t2, y2, e2 = (torch.empty(nn, dtype=torch.float64, device=dev) for _ in range(3))
    L.check(lib.lkb_fill_gaps(L.ptr(d_t), L.ptr(d_y), L.ptr(d_e), L.ptr(off), B, L.ptr(dt), L.ptr(mean), L.ptr(d_s),
                              L.ptr(z), L.ptr(noff), L.ptr(t2), L.ptr(y2), L.ptr(e2), L.MEM_DEVICE, _stream_ptr()))
    plan["std"] = s
    return t2, y2, e2, noff, plan


def fill_gaps(times, fluxes, flux_errs, std):
    """`fill_gaps_device` for lists of host float64 arrays (NaN-free flux, finite times), uploaded once.  `std(cdpp)`
    gets the [B] CDPP in ppm (lkb_cdpp with estimate_cdpp's defaults, on the device copies) and returns the [B]
    noise levels.  Returns the filled times, fluxes and flux errors as lists of host arrays."""
    import torch
    t_h, off = _csr(times)
    B, n = len(times), int(off[-1])
    dev = torch.device("cuda", torch.cuda.current_device())
    d_t, d_y, d_e = (torch.from_numpy(_csr(a)[0] if n else np.zeros(1)).to(dev) for a in (times, fluxes, flux_errs))

    def level(plan):
        return std(cdpp(d_t[:n], d_y[:n], 13, offsets=off).cpu().numpy()[:, 0] if n else np.zeros(B))

    t2, y2, e2, noff, _ = fill_gaps_device(d_t, d_y, d_e, off, level)
    tt, yy, ee = (x.cpu().numpy() for x in (t2, y2, e2))
    sl = [slice(noff[b], noff[b + 1]) for b in range(B)]
    return [tt[x].copy() for x in sl], [yy[x].copy() for x in sl], [ee[x].copy() for x in sl]


SEISMOLOGY_MAX_B = 65535


def seismology_spectra(times, fluxes, flux_errs, grid, on_median=None, filter_width=0.01):
    """K6 + normalize/compact + K15 + K4/K11/K12 + K1 (or K1n) + the ragged log-median: the SNR spectra of
    ``lc.normalize().remove_nans().fill_gaps().to_periodogram(**kwargs).flatten()`` for every light curve.
    `times`, `fluxes`, `flux_errs`: lists of host float64 arrays, the raw light curves, uploaded once.  On the device:
    the K6 nanmedian and nanstd of the flux (`on_median(median, std)` gets them on the host, for normalize's
    warnings), flux and flux_err divided by the median with the NaN fluxes dropped (lkb_normalize_compact), K15 with
    the CDPP (lkb_cdpp, estimate_cdpp's defaults, converted from ppm to the dimensionless flux) as the noise level,
    K15's plan again for the median step of the filled times, the periodograms and their log-median SNR.
    `grid(b, median_dt, t_first, t_last, n)` returns dict(frequency (1/day), freq (the grid in its own unit),
    scale (psd scale or None), normalization, nterms, multiterm) or raises as the loop would.  Kept times must be
    finite (ValueError naming the light curve); fill_gaps' refusals come next, then the first grid error.
    Returns the list of SNR arrays (in each grid's order)."""
    import torch
    lib = L.load()
    from . import units as u
    B = len(times)
    if not 0 < B <= SEISMOLOGY_MAX_B:
        raise ValueError("seismology_spectra needs 1 .. %d light curves, got %d" % (SEISMOLOGY_MAX_B, B))
    t_h, off = _csr(times)
    y_h, yoff = _csr(fluxes)
    e_h, eoff = _csr(flux_errs)
    if not (np.array_equal(off, yoff) and np.array_equal(off, eoff)):
        raise ValueError("time, flux and flux_err lengths differ")
    dev = torch.device("cuda", torch.cuda.current_device())
    f64 = dict(dtype=torch.float64, device=dev)

    def up(a):
        x = torch.empty(max(len(a), 1), **f64)
        x[:len(a)].copy_(torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)))
        return x

    n0 = int(off[-1])
    d_t, d_y, d_e = up(t_h), up(y_h), up(e_h)
    # 1. normalize().remove_nans(): the K6 median (only [B] values come back), the division and the compaction
    med, sd = torch.empty(B, **f64), torch.empty(B, **f64)
    L.check(lib.lkb_nanmedian_std(L.ptr(d_y), L.ptr(off), B, L.ptr(med), L.ptr(sd), L.MEM_DEVICE, _stream_ptr()))
    if on_median is not None:
        on_median(med.cpu().numpy(), sd.cpu().numpy())
    noff = np.zeros(B + 1, np.int64)
    bad = np.zeros(B, np.int32)
    t1, y1, e1 = (torch.empty(max(n0, 1), **f64) for _ in range(3))
    ends = torch.empty(2 * B, **f64)
    L.check(lib.lkb_normalize_compact(L.ptr(d_t), L.ptr(d_y), L.ptr(d_e), L.ptr(off), B, L.ptr(med), L.ptr(noff),
                                      L.ptr(bad), L.ptr(t1), L.ptr(y1), L.ptr(e1), L.ptr(ends), L.MEM_DEVICE,
                                      _stream_ptr()))
    del d_t, d_y, d_e
    for b in np.flatnonzero(bad):
        raise ValueError("light curve %d has non-finite times" % b)
    ends_h = ends.cpu().numpy().reshape(B, 2)
    n = int(noff[-1])
    ppm = float(u.Quantity(1.0, u.ppm).to(u.dimensionless_unscaled).value)

    def std(plan):
        if n == 0:
            return np.zeros(B)
        return cdpp(t1[:n], y1[:n], 13, offsets=noff).cpu().numpy()[:, 0] * ppm

    # 2. fill_gaps
    t2, y2, e2, foff, plan = fill_gaps_device(t1, y1, e1, noff, std)
    del t1, y1, e1
    if np.any((plan["n_ins"] > 0) & ~np.isfinite(plan["mean"] + plan["std"])):
        # NaN inserted flux: the periodogram's own remove_nans drops those cadences
        tt, yy, ee = (x.cpu().numpy()[:int(foff[-1])] for x in (t2, y2, e2))
        keep = ~np.isnan(yy)
        lens = np.array([int(keep[foff[b]:foff[b + 1]].sum()) for b in range(B)], dtype=np.int64)
        foff = np.zeros(B + 1, np.int64)
        np.cumsum(lens, out=foff[1:])
        t2, y2, e2 = up(tt[keep]), up(yy[keep]), up(ee[keep])
    # 3. the grids: median step of the filled times (K15's plan entry runs K6 on the steps), first and last time, N
    N = np.diff(foff)
    md = torch.empty(B, **f64)
    scratch = [torch.empty(B, **f64), torch.empty(B, dtype=torch.int64, device=dev),
               torch.empty(B, dtype=torch.int32, device=dev)]
    L.check(lib.lkb_fill_gaps_plan(L.ptr(t2), L.ptr(y2), L.ptr(foff), B, L.ptr(md), L.ptr(scratch[0]),
                                   L.ptr(scratch[1]), L.ptr(scratch[2]), L.MEM_DEVICE, _stream_ptr()))
    md_h = md.cpu().numpy()
    grids = [grid(b, md_h[b], ends_h[b, 0] if N[b] else None, ends_h[b, 1] if N[b] else None, int(N[b]))
             for b in range(B)]
    # 4. the periodograms, on grids in ascending frequency (Periodogram.smooth sorts a descending one)
    orders = [None if len(g["freq"]) < 2 or np.all(np.diff(g["freq"]) >= 0) else np.argsort(g["freq"], kind="stable")
              for g in grids]
    sorted_f = [g["frequency"] if o is None else g["frequency"][o] for g, o in zip(grids, orders)]
    freq_h, pofs = _csr(sorted_f)
    g0 = grids[0]
    scale = None
    if g0["scale"] is not None:
        scale = torch.from_numpy(np.ascontiguousarray([g["scale"] for g in grids], dtype=np.float64)).to(dev)
    d_f = up(freq_h)
    F = int(pofs[-1])
    power = torch.empty(max(F, 1), dtype=torch.float32, device=dev)
    if g0["multiterm"]:
        L.check(lib.lkb_ls_power_chi2_ex(L.ptr(t2), L.ptr(y2), L.DTYPE_F64, L.ptr(foff), B, L.ptr(d_f), L.ptr(pofs), F,
                                         int(g0["nterms"]), _NORMS[g0["normalization"]], L.ptr(scale), L.ptr(power),
                                         None, L.MEM_DEVICE, _stream_ptr(), L.LS_ALGO_SIMT))
    else:
        L.check(lib.lkb_ls_power_ex(L.ptr(t2), L.ptr(y2), L.DTYPE_F64, L.ptr(foff), B, L.ptr(d_f), L.ptr(pofs), F,
                                    _NORMS[g0["normalization"]], L.ptr(scale), L.ptr(power), L.MEM_DEVICE,
                                    _stream_ptr(), L.LS_ALGO_AUTO))
    # 5. the log-median background and the SNR
    _, snr = pg_logmedian_ragged([g["freq"] if o is None else g["freq"][o] for g, o in zip(grids, orders)],
                                 power[:F] if F else power, filter_width, bin_offsets=pofs, snr=True)
    snr_h = snr.cpu().numpy()
    out = []
    for b, o in enumerate(orders):
        x = snr_h[pofs[b]:pofs[b + 1]]
        if o is not None:
            inv = np.empty_like(o)
            inv[o] = np.arange(len(o))
            x = x[inv]
        out.append(x.copy())
    return out


# bytes of series + outputs staged on the device by one lkb_acf_windows call; larger batches are split by series
ACF_STAGE_BYTES = 2 << 30


def acf_windows(series, starts, lengths, return_acf=False):
    """K7.  Windowed autocorrelation (the seismology ACF2D step) of B series: `series` a list of 1-D arrays,
    `starts` a list of int arrays (first bin of each window of series b), `lengths` a list of ints (the window
    length = lag count of series b).  Window k of series b gives, with y = window - nanmean(window),
    acf = np.correlate(y, y, "full")[n-1:] and metric = (sum |acf| - 1) / n.
    Returns the list of metric arrays [n_windows_b] and, with return_acf, the list of [n_windows_b, n_b] acf arrays.
    The batch goes to the GPU in groups of series whose staged input and output stay under ACF_STAGE_BYTES."""
    lib = L.load()
    B = len(series)
    if len(starts) != B or len(lengths) != B:
        raise ValueError("series, starts and lengths must have one entry per series")
    xs = [np.asarray(s, dtype=np.float64).ravel() for s in series]
    st = [np.asarray(s, dtype=np.int64).ravel() for s in starts]
    ln = [int(n) for n in lengths]
    cost = [8 * (len(x) + len(s) + (len(s) * n if return_acf else 0)) for x, s, n in zip(xs, st, ln)]
    metrics, acfs = [None] * B, [None] * B
    b0 = 0
    while b0 < B:
        b1, used = b0 + 1, cost[b0]
        while b1 < B and used + cost[b1] <= ACF_STAGE_BYTES:
            used += cost[b1]
            b1 += 1
        x, xoff = _csr(xs[b0:b1])
        ws, woff = _csr(st[b0:b1], np.int64)
        wl = np.ascontiguousarray(ln[b0:b1], dtype=np.int64)
        W = int(woff[-1])
        metric = np.empty(W, dtype=np.float64)
        nlag = sum(len(s) * n for s, n in zip(st[b0:b1], ln[b0:b1]))
        acf = np.empty(nlag, dtype=np.float64) if return_acf else None
        L.check(lib.lkb_acf_windows(L.ptr(x), L.ptr(xoff), b1 - b0, L.ptr(woff), L.ptr(ws), L.ptr(wl),
                                    L.ptr(metric), L.ptr(acf), L.MEM_HOST, None))
        a0 = 0
        for j, b in enumerate(range(b0, b1)):
            metrics[b] = metric[woff[j]:woff[j + 1]]
            if return_acf:
                k = len(st[b])
                acfs[b] = acf[a0:a0 + k * ln[b]].reshape(k, ln[b])
                a0 += k * ln[b]
        b0 = b1
    return (metrics, acfs) if return_acf else metrics


# --------------------------------------------------------------------------------------
# multi-GPU exchange step (SURVEY.md 8e): NCCL all-gather through the C ABI
# --------------------------------------------------------------------------------------
def nccl_version():
    """NCCL_VERSION_CODE of the library the C ABI bound at run time (0: none could be loaded)."""
    return int(L.load().lkb_nccl_version())


def nccl_unique_id():
    """128-byte NCCL id (bytes).  Rank 0 creates it; the host program carries it to the other ranks."""
    buf = np.zeros(L.NCCL_ID_BYTES, dtype=np.uint8)
    L.check(L.load().lkb_nccl_unique_id(L.ptr(buf)))
    return buf.tobytes()


def nccl_init(rank, world_size, unique_id):
    """Collective: every rank calls this with the SAME id after ``init(device)``."""
    buf = np.frombuffer(bytes(unique_id), dtype=np.uint8).copy()
    if buf.size != L.NCCL_ID_BYTES:
        raise ValueError("an NCCL unique id has %d bytes, got %d" % (L.NCCL_ID_BYTES, buf.size))
    L.check(L.load().lkb_nccl_init(int(rank), int(world_size), L.ptr(buf)))


def nccl_shutdown():
    L.check(L.load().lkb_nccl_shutdown())


def nccl_rank_world():
    lib = L.load()
    return int(lib.lkb_nccl_rank()), int(lib.lkb_nccl_world_size())


def allgather_f32(local, out=None):
    """One ncclAllGather of a contiguous CUDA float32 torch tensor `local` ([n, ...], same shape on every
    rank) into `out` ([world * n, ...], rank-major), asynchronous on the current torch stream."""
    import torch
    lib = L.load()
    world = int(lib.lkb_nccl_world_size())
    if world <= 0:
        raise ValueError("allgather_f32: no communicator (call engine.nccl_init on every rank first)")
    if not (_is_torch(local) and local.is_cuda and local.dtype == torch.float32 and local.is_contiguous()):
        raise TypeError("allgather_f32 needs a contiguous CUDA float32 tensor")
    shape = (world * local.shape[0],) + tuple(local.shape[1:])
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=local.device)
    elif tuple(out.shape) != shape or out.dtype != torch.float32 or not out.is_cuda or not out.is_contiguous():
        raise ValueError("allgather_f32: `out` must be a contiguous CUDA float32 tensor of shape %r" % (shape,))
    L.check(lib.lkb_allgather_f32(L.ptr(local), int(local.numel()), L.ptr(out), _stream_ptr()))
    return out
