"""The float64 conv GD training-gradient oracle (oracle/conv_gd_grad_torch.py) against the reference's own
back-optimisation graph (tests/golden/conv/conv_gd_grad.npz: completion/icnn.back.py's Model on the TF shim, nGdIter
unrolled momentum-GD steps, mse_ and gv_ = compute_gradients(mse_, theta_)), and the regeneration of that golden from
a reference checkout (skipped without one)."""
import os
import types

import numpy as np
import pytest

from oracle import conv_gd_grad_torch as O
from oracle.gen_golden_conv_gd_grad import CASES, case_inputs
from oracle.gen_golden_conv_grad import probe

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "conv", "conv_gd_grad.npz")


def _case(tag):
    from icnn_b200.conv_picnn import parse_variables
    v, x, y0, trueY, H, W = case_inputs(tag)
    return parse_variables(v, H, W), x, y0, trueY


@pytest.mark.parametrize("tag", list(CASES))
def test_gradient_set_is_the_reference_gv(tag):
    """The variables with a gradient are exactly gv_'s (49 for the reference architecture), for
    conv_gd_trainable and for the oracle's literal double backward."""
    from icnn_b200.gd_grad import conv_gd_trainable
    gold = np.load(GOLDEN)
    names = set(str(s) for s in gold[tag + "_gv_names"])
    spec, x, y0, trueY = _case(tag)
    Lc, Ld = len(spec.convs), len(spec.fcs)
    assert set(conv_gd_trainable(types.SimpleNamespace(vars=spec.vars, Lc=Lc, Ld=Ld))) == names
    _yN, _l, grads, _adj, _rel = O.gd_grad(spec, x[:1], y0[:1], trueY[:1], 2)
    assert set(grads) == names
    assert len(names) == 49


@pytest.mark.parametrize("tag", list(CASES))
def test_oracle_reproduces_the_reference_graph(tag):
    """Per sample (the golden's Model is built on one sample, so mse_ is the mean over its n pixels: loss_scale =
    2 255^2 / n), yn_, mse_ and every stored gradient, whole or probed, to 1e-9 * max(1, its largest entry)."""
    gold = np.load(GOLDEN)
    spec, x, y0, trueY = _case(tag)
    n = spec.H * spec.W
    nIter = int(gold[tag + "_nGdIter"])
    stored = [(k, kind) for k in gold.files for kind in ("_grad_", "_probe_") if k.startswith(tag + kind)]
    assert len(stored) == 49
    tol = lambda ref: 1e-9 * max(1.0, np.abs(ref).max())   # noqa: E731
    for u in range(len(x)):
        s = slice(u, u + 1)
        yN, loss, grads, _adj, _rel = O.gd_grad(spec, x[s], y0[s], trueY[s], nIter, loss_scale=2 * 255.0 ** 2 / n)
        # loss = loss_scale / 2 sum (yN - trueY)^2 = mean of square(255 (yN - trueY)) over the sample
        assert abs(loss - gold[tag + "_mse"][u]) <= tol(gold[tag + "_mse"][u])
        assert np.abs(yN[0] - gold[tag + "_yn"][u]).max() <= tol(gold[tag + "_yn"][u])
        for k, kind in stored:
            name = k[len(tag + kind):]
            ref = gold[k][u]
            got = grads[name] if kind == "_grad_" else probe(grads[name].reshape(-1))
            err = np.abs(got - ref).max()
            assert err <= tol(ref), (u, name, err)


def test_golden_regenerates_from_the_reference():
    ref = os.environ.get("ICNN_REFERENCE_DIR", "")
    if not ref or not os.path.isfile(os.path.join(ref, "completion", "icnn.back.py")):
        pytest.skip("no reference checkout at $ICNN_REFERENCE_DIR")
    from oracle.gen_golden_conv_gd_grad import generate
    gold = np.load(GOLDEN)
    out = generate()
    assert set(out) == set(gold.files)
    for k, a in out.items():
        np.testing.assert_array_equal(np.asarray(a, dtype=gold[k].dtype), gold[k], err_msg=k)
