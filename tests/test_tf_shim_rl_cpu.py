"""The RL primitives of oracle/tf_shim_rl.py against torch, the way test_tf_shim_cpu.py checks the shim's others."""
import numpy as np
import torch

from oracle.tf_shim_rl import RLShim


def _shim():
    rs = np.random.RandomState(0)
    v = {"q/u0/W": rs.randn(3, 4), "q/u0/b": rs.randn(4), "q/z0_yu/W": rs.randn(4, 2),
         "q_target/u0/W": rs.randn(3, 4), "q_target/u0/b": rs.randn(4)}
    return RLShim(v), v


def test_select():
    sh, _ = _shim()
    c = torch.tensor([True, False, True])
    a, b = torch.arange(3.0, dtype=torch.float64), -torch.arange(3.0, dtype=torch.float64)
    assert torch.equal(sh.tf.select(c, a, b), torch.where(c, a, b))


def test_l2_regularizer_and_collections():
    sh, v = _shim()
    tf, tl = sh.tf, sh.tflearn
    x = torch.tensor(np.random.RandomState(1).randn(5, 3))
    for scope in ("q", "q_target"):
        with tf.variable_scope(scope):
            with tf.variable_scope("u0") as s:
                out = tl.fully_connected(x, 4, scope=s, regularizer="L2", weight_decay=0.002)
            with tf.variable_scope("z0_yu") as s:
                if scope == "q":
                    tl.fully_connected(out, 2, scope=s, bias=False, regularizer="L2")
    ref = torch.as_tensor(x) @ torch.as_tensor(v["q_target/u0/W"]) + torch.as_tensor(v["q_target/u0/b"])
    assert torch.allclose(out, ref)
    reg = tf.get_collection(tf.GraphKeys.REGULARIZATION_LOSSES, scope="q/")
    exp = [0.002 * (torch.as_tensor(v["q/u0/W"]) ** 2).sum() / 2, 0.001 * (torch.as_tensor(v["q/z0_yu/W"]) ** 2).sum() / 2]
    assert len(reg) == 2 and all(torch.allclose(a, b) for a, b in zip(reg, exp))   # W only, never b
    assert torch.allclose(tf.reduce_sum(reg), exp[0] + exp[1])
    th = tf.get_collection(tf.GraphKeys.TRAINABLE_VARIABLES, scope="q/")
    assert [t.name for t in th] == ["q/u0/W:0", "q/u0/b:0", "q/z0_yu/W:0"]
    tt = tf.get_collection(tf.GraphKeys.TRAINABLE_VARIABLES, scope="q_target/")
    assert [t.name for t in tt] == ["q_target/u0/W:0", "q_target/u0/b:0"]


def test_variable_arithmetic_and_assign_sub():
    sh, v = _shim()
    with sh.tf.variable_scope("q"):
        with sh.tf.variable_scope("u0") as s:
            sh.tflearn.fully_connected(torch.zeros(1, 3, dtype=torch.float64), 4, scope=s)
    a, b = sh.vars["q_target/u0/W"], sh.vars["q/u0/W"]
    A, Bv = torch.as_tensor(v["q_target/u0/W"]), torch.as_tensor(v["q/u0/W"])
    assert torch.allclose(0.01 * (a - b), 0.01 * (A - Bv))
    assert torch.allclose(a + b, A + Bv) and torch.allclose(-a, -A) and torch.allclose(2.0 * a, 2 * A)
    assert torch.allclose(1.0 - a, 1 - A) and torch.allclose(a * 3.0, 3 * A)
    assert a.assign_sub(0.01 * (a - b)) == ("assign_sub", "q_target/u0/W:0")
    assert torch.equal(a.value.detach(), A)        # built, never run
