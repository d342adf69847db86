"""The float64 conv training-gradient oracle (oracle/conv_train_grad_torch.py) against the reference's own training
step (tests/golden/conv/conv_train_grad.npz: solveBatch, mseGrad, Model.train_step_fd and Model.__init__'s gv_ on the
TF shim)."""
import os
import types

import numpy as np
import pytest

from oracle import conv_train_grad_torch as O
from oracle.gen_golden_conv_grad import CASES, case_rows_inputs, probe

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "conv", "conv_train_grad.npz")


def _spec(tag):
    from icnn_b200.conv_picnn import parse_variables
    v, x, _y0, _tY, H, W, _n = case_rows_inputs(tag)
    return parse_variables(v, H, W), x


@pytest.mark.parametrize("tag", list(CASES))
def test_gradient_set_is_the_reference_gv(tag):
    """The variables with a gradient are exactly gv_'s, for the oracle and for bundle_grad.conv_trainable."""
    from icnn_b200.bundle_grad import conv_trainable
    gold = np.load(GOLDEN)
    names = set(str(s) for s in gold[tag + "_gv_names"])
    spec, _x = _spec(tag)
    Lc, Ld = len(spec.convs), len(spec.fcs)
    assert set(O.trainable(list(spec.vars), Lc, Ld)) == names
    assert set(conv_trainable(types.SimpleNamespace(vars=spec.vars, Lc=Lc, Ld=Ld))) == names
    assert len(names) == 51


@pytest.mark.parametrize("tag", list(CASES))
def test_oracle_reproduces_the_reference_training_step(tag):
    """Per sample (the golden's Model is built on one sample's rows), every stored gradient, whole or probed, to
    1e-9 * max(1, its largest entry) (tests/test_oracle_bundle_grad.py's rule)."""
    gold = np.load(GOLDEN)
    spec, x = _spec(tag)
    f64 = lambda k: gold[tag + "_" + k].astype(np.float64)   # noqa: E731
    Y, V, c, counts = f64("Y"), f64("V"), f64("c"), gold[tag + "_counts"]
    off = np.concatenate([[0], np.cumsum(counts)])
    stored = [(k, kind) for k in gold.files for kind in ("_grad_", "_probe_") if k.startswith(tag + kind)]
    assert len(stored) == 51
    for u in range(len(counts)):
        s = slice(off[u], off[u + 1])
        grads, _adj, _rel, _bs = O.train_grad(spec, x[u:u + 1], Y[s], V[s], c[s], counts[u:u + 1])
        for k, kind in stored:
            name = k[len(tag + kind):]
            ref = gold[k][u]
            got = grads[name] if kind == "_grad_" else probe(grads[name].reshape(-1))
            err = np.abs(got - ref).max()
            assert err <= 1e-9 * max(1.0, np.abs(ref).max()), (u, name, err)

