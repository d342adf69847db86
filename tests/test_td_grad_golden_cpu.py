"""The float64 oracle of the RL TD training step (oracle/td_grad_np.py) against the reference's own Agent graph executed
on the TF shim (tests/golden/rl/td_grad.npz, written by oracle/gen_golden_td_grad.py)."""
import os

import numpy as np
import pytest

from oracle import td_grad_np as tg
from oracle.gen_golden_bundle_grad import tf_name_to_param


@pytest.mark.parametrize("tag", ["small", "c4"])
def test_oracle_reproduces_golden(tag, golden_dir):
    gold = np.load(os.path.join(golden_dir, "rl", "td_grad.npz"))
    c = tg.case(tag)
    loss, td, g = tg.td_grad(c["p"], c["pt"], c["obs"], c["act"], c["rew"], c["ob2"], c["act2"], c["term"])
    assert abs(loss - float(gold[tag + "_loss_q"])) <= 1e-9 * max(1.0, abs(loss))
    np.testing.assert_allclose(td, gold[tag + "_td"], rtol=0, atol=1e-9)
    names = [str(s) for s in gold[tag + "_theta"]]
    assert len(names) == 25 and all(s.startswith("q/") for s in names)
    stored = 0
    for name in names:
        key = "%s_gv_%s" % (tag, name.replace("/", "__"))
        if key not in gold.files:
            continue
        k, i = tf_name_to_param(name[2:])
        ref = gold[key]
        np.testing.assert_allclose(np.reshape(g[k][i], ref.shape), ref, rtol=0,
                                   atol=1e-9 * max(1.0, np.abs(ref).max()), err_msg=name)
        stored += 1
    assert stored == (25 if tag == "small" else stored) and stored >= 15


@pytest.mark.parametrize("tag", ["small", "c4"])
def test_golden_rows_cover_the_cases(tag):
    """Terminal and non-terminal rows, the clamp active from both sides and inactive, actions at the entropy clip's
    ends, and no row near a clamp boundary."""
    c = tg.case(tag)
    td, q, y0 = tg.td_parts(c["p"], c["pt"], c["obs"], c["act"], c["rew"], c["ob2"], c["act2"], c["term"])
    assert c["term"].any() and (~c["term"]).any()
    assert (y0 > q + 1).any() and (y0 < q - 1).any() and (np.abs(y0 - q) < 1).any()
    assert (c["act"] == 1).any() and (c["act"] == -1).any() and (c["act2"] == 1).any() and (c["act2"] == -1).any()
    assert tg.clamp_gap(q, y0).min() > tg.CLAMP_GAP
    assert np.abs(td).max() <= 1.0 + 1e-12
