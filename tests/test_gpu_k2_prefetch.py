"""The row sweeps of the three-vector predictor-corrector kernel (n_y = 4096) issue L2 prefetches ahead of their row
loads.  A prefetch changes no arithmetic, so every prefetch setting walks the same iterates bit for bit: same nIters,
counts, active rows and y*.  ICNN_PC_PREFETCH="a,b" sets the distances at every K2 launch ("0,0" = off), so a switch in
the middle of a run is checked as well."""
import os

import numpy as np
import pytest

from oracle import picnn_np, synth

pytestmark = pytest.mark.gpu
np.seterr(all="ignore")


def r32(fg):
    def w(y):
        f, g = fg(y)
        return f.astype(np.float32).astype(np.float64), g.astype(np.float32).astype(np.float64)
    return w


def switching(fg, at, value, monkeypatch):
    """fg that sets ICNN_PC_PREFETCH=value from its call `at` on (K2 of iteration t runs after the t-th fg call)."""
    calls = [0]

    def w(y):
        if calls[0] == at:
            monkeypatch.setenv("ICNN_PC_PREFETCH", value)
        calls[0] += 1
        return fg(y)
    return w


def check_same(ref, alt):
    assert np.array_equal(np.array(ref[5]), np.array(alt[5]))                     # nIters
    assert [len(r) for r in ref[1]] == [len(r) for r in alt[1]]                  # counts
    for a, b in zip(ref[1], alt[1]):                                             # active rows, in order
        assert np.array_equal(np.asarray(a), np.asarray(b))
    assert np.array_equal(ref[0], alt[0])                                        # y*, bit for bit
    assert np.all((alt[0] > 0) & (alt[0] < 1))


@pytest.mark.parametrize("setting", ["1,0", "0,8", "2,16"])
def test_prefetch_settings_match_no_prefetch(setting, monkeypatch):
    from icnn_b200 import bundle_entropy as be
    p, x, y0 = synth.make_inputs("C5", B=3)
    fg = r32(picnn_np.make_fg(p, x))
    monkeypatch.setenv("ICNN_PC_PREFETCH", "0,0")
    off = be.solveBatch(fg, y0.copy(), nIter=45)
    monkeypatch.setenv("ICNN_PC_PREFETCH", setting)
    on = be.solveBatch(fg, y0.copy(), nIter=45)
    monkeypatch.delenv("ICNN_PC_PREFETCH")
    dflt = be.solveBatch(fg, y0.copy(), nIter=45)
    check_same(off, on)
    check_same(off, dflt)
    assert max(len(r) for r in on[1]) + 2 > 32    # the one-pass rb = 5 sweep ran (largest tile set)


def test_prefetch_switch_mid_run(monkeypatch):
    from icnn_b200 import bundle_entropy as be
    p, x, y0 = synth.make_inputs("C5", B=3)
    fg = r32(picnn_np.make_fg(p, x))
    monkeypatch.setenv("ICNN_PC_PREFETCH", "0,0")
    off = be.solveBatch(fg, y0.copy(), nIter=45)
    mixed = be.solveBatch(switching(fg, 20, "2,16", monkeypatch), y0.copy(), nIter=45)
    assert os.environ.get("ICNN_PC_PREFETCH") == "2,16"
    monkeypatch.delenv("ICNN_PC_PREFETCH")
    check_same(off, mixed)
