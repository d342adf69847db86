"""Sweep A of the three-vector predictor-corrector kernel (n_y = 4096) builds the Gram of k + 2 <= 40 sweep rows in one
pass over the bundle rows; ICNN_PC_LEGACY=1 keeps the four-sweep composition it replaced for 32 < k + 2 <= 40.  Both
accumulate every Gram tile over the same columns in the same order, so the solves walk the same iterates: same active
sets, counts and nIters, y* within 1e-9.  The build is read from the environment at every K2 launch, so a switch in the
middle of a run is checked as well."""
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


def switching(fg, at, monkeypatch):
    """fg that sets ICNN_PC_LEGACY=1 from its call `at` on (K2 of iteration t runs after the t-th fg call)."""
    calls = [0]

    def w(y):
        if calls[0] == at:
            monkeypatch.setenv("ICNN_PC_LEGACY", "1")
        calls[0] += 1
        return fg(y)
    return w


def check_same(ref, alt):
    assert np.array_equal(np.array(ref[5]), np.array(alt[5]))                     # nIters
    assert [len(r) for r in ref[1]] == [len(r) for r in alt[1]]                  # counts
    for a, b in zip(ref[1], alt[1]):                                             # active rows, in order
        assert np.allclose(np.asarray(a), np.asarray(b), rtol=1e-5, atol=1e-6)
    assert np.abs(ref[0] - alt[0]).max() <= 1e-9
    assert np.all((alt[0] > 0) & (alt[0] < 1))


@pytest.mark.parametrize("nIter", [12, 45])
def test_one_pass_sweep_a_matches_composition(nIter, monkeypatch):
    from icnn_b200 import bundle_entropy as be
    p, x, y0 = synth.make_inputs("C5", B=3)
    fg = r32(picnn_np.make_fg(p, x))
    monkeypatch.delenv("ICNN_PC_LEGACY", raising=False)
    new = be.solveBatch(fg, y0.copy(), nIter=nIter)
    monkeypatch.setenv("ICNN_PC_LEGACY", "1")
    old = be.solveBatch(fg, y0.copy(), nIter=nIter)
    monkeypatch.delenv("ICNN_PC_LEGACY")
    check_same(old, new)
    if nIter == 45:
        assert max(len(r) for r in new[1]) + 2 > 32    # the one-pass rb = 5 sweep ran


def test_build_switch_mid_run_matches_either_build(monkeypatch):
    from icnn_b200 import bundle_entropy as be
    p, x, y0 = synth.make_inputs("C5", B=3)
    fg = r32(picnn_np.make_fg(p, x))
    monkeypatch.delenv("ICNN_PC_LEGACY", raising=False)
    new = be.solveBatch(fg, y0.copy(), nIter=45)
    mixed = be.solveBatch(switching(fg, 38, monkeypatch), y0.copy(), nIter=45)
    assert os.environ.get("ICNN_PC_LEGACY") == "1"
    monkeypatch.delenv("ICNN_PC_LEGACY")
    check_same(new, mixed)
