"""The precision-escalation pass of the shared-grid NUFFT (ls_nufft.cu + nufft_v2.cuh) when it lists no light curve, run
through the CPU emulator of the whole translation unit (tests/native/cuda_emu.h)."""
import numpy as np

from test_nufft_emulated import _shared_inputs, _window_rows, emu  # noqa: F401  (emu: the module's fixture)


def test_escalation_pass_with_no_listed_light_curve_leaves_the_power_alone(emu, monkeypatch):  # noqa: F811
    """A threshold no light curve reaches: the flag kernel lists none, and the double-precision rounds (sized before the
    host knows the count) find a count of 0 and write nothing.  The power is bitwise that of the fp32 kernels alone
    (escalation switched off), and no light curve is reported as escalated."""
    B, N, F = 5, 500, 3500
    t, trel, Y, ycp, Npad, ysum, absmax, freq, f0, df = _shared_inputs(31, N, F, B, 5.0, 1)
    F_low = int((freq * trel[-1] <= 2.0).sum()) + 1
    rot, rot2 = _window_rows(trel, freq, F_low)

    def run(ratio):
        monkeypatch.setenv("LKB_NUFFT_ESCALATE", ratio)
        power = np.zeros((B, F), np.float32)
        rc = emu.emu_nufft_shared(trel.ctypes.data, N, ycp.ctypes.data, Npad, ysum.ctypes.data, absmax.ctypes.data, B,
                                  freq.ctypes.data, F, f0, df, rot.ctypes.data, rot2.ctypes.data, F_low, 2,
                                  2.0 / (N * 5.0 * df), power.ctypes.data)
        assert rc == 0, emu.emu_last_error()
        return power, emu.emu_last_escalated()

    off, n_off = run("0")
    none, n_none = run("1e30")
    assert n_off == 0 and n_none == 0
    assert np.array_equal(none, off)
    # and with every light curve listed, the pass does replace rows (the same call path is live)
    everything, n_all = run("1e-6")
    assert n_all == B and not np.array_equal(everything, off)
