"""The TensorFlow / tflearn primitives RL/src/icnn.py:55-108 needs beyond oracle/tf_shim.py (test infrastructure).

``RLShim`` is a ``tf_shim.Shim`` whose ``tf`` / ``tflearn`` also answer the calls the RL agent's training graph makes
(Agent.__init__ from ``obs = tf.placeholder`` through ``optim_q.compute_gradients(loss_q)``).  Restated from the
libraries' published semantics, one line each:

  tf.select(cond, a, b)                               elementwise a where cond else b (TensorFlow 0.x; tf.where later)
  tf.GraphKeys.REGULARIZATION_LOSSES / TRAINABLE_VARIABLES     the two collection keys
  tf.get_collection(key, scope)                       the collection's items whose name starts with ``scope``
                                                      (re.match), in insertion order
  tflearn.fully_connected(.., regularizer='L2', weight_decay)  adds weight_decay * sum(W^2) / 2 (tflearn.losses.L2 =
                                                      wd * tf.nn.l2_loss) of its W -- never of its b -- to
                                                      REGULARIZATION_LOSSES under the layer's scope
  TRAINABLE_VARIABLES                                 the trainable variables in creation order
  tf.reduce_sum(list)                                 sum of the packed list
  Variable arithmetic (v - w, tau * v, -v, ...)       on the variable's value
  Variable.assign_sub(delta)                          an op that is built, never run here
"""
from __future__ import annotations

import re
import types

import torch

from oracle import tf_shim
from oracle.tf_shim import Shim, _t

REG_LOSSES, TRAINABLE = "regularization_losses", "trainable_variables"


class RLVariable(tf_shim.Variable):
    def assign_sub(self, _delta):        # update_target (:102-103) is built, never run, by the code executed here
        return ("assign_sub", self.name)

    def __add__(self, o): return self.value + _t(o)
    def __radd__(self, o): return _t(o) + self.value
    def __sub__(self, o): return self.value - _t(o)
    def __rsub__(self, o): return _t(o) - self.value
    def __mul__(self, o): return self.value * _t(o)
    def __rmul__(self, o): return _t(o) * self.value
    def __neg__(self): return -self.value


class RLShim(Shim):
    def __init__(self, variables, feeds=None):
        super().__init__(variables, feeds)
        self.vars = {k: RLVariable(k, v) for k, v in variables.items()}
        self.reg_losses = []                 # (name, scalar) in insertion order

    def _make_tf(self):
        tf = super()._make_tf()
        sh = self
        tf.select = lambda cond, a, b: torch.where(_t(cond).bool(), _t(a), _t(b))
        tf.GraphKeys = types.SimpleNamespace(REGULARIZATION_LOSSES=REG_LOSSES, TRAINABLE_VARIABLES=TRAINABLE)

        def get_collection(key, scope=None):
            if key == REG_LOSSES:
                items = sh.reg_losses
            elif key == TRAINABLE:
                items = [(v.name, v) for v in tf.trainable_variables()]
            else:
                raise KeyError(key)
            return [v for name, v in items if scope is None or re.match(scope, name)]
        tf.get_collection = get_collection

        red = tf.reduce_sum

        def reduce_sum(x, axis=None, reduction_indices=None):
            if isinstance(x, (list, tuple)):
                x = torch.stack([_t(v) for v in x])
            return red(x, axis=axis, reduction_indices=reduction_indices)
        tf.reduce_sum = reduce_sum
        return tf

    def _make_tflearn(self):
        tl = super()._make_tflearn()
        sh = self
        fc = tl.fully_connected

        def fully_connected(incoming, n_units, activation="linear", bias=True, weights_init=None, bias_init=None,
                            regularizer=None, weight_decay=0.001, trainable=True, restore=True, reuse=False,
                            scope=None, name="FullyConnected"):
            out = fc(incoming, n_units, activation=activation, bias=bias, weights_init=weights_init,
                     bias_init=bias_init, regularizer=regularizer, weight_decay=weight_decay, trainable=trainable,
                     restore=restore, reuse=reuse, scope=scope, name=name)
            if regularizer is not None:
                assert regularizer == "L2", regularizer
                W = sh.get(scope.name + "/W")
                sh.reg_losses.append((scope.name + "/W/Regularizer/L2Loss:0", weight_decay * (W ** 2).sum() / 2))
            return out
        tl.fully_connected = fully_connected
        return tl
