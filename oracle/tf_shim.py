"""A minimal eager stand-in for the TensorFlow-0.x / tflearn calls the reference's ICNN graph code makes,
backed by torch float64 autograd.  TEST INFRASTRUCTURE ONLY (see oracle/__init__.py); used by
oracle/gen_golden_tfshim.py in the build container to EXECUTE THE REFERENCE'S OWN, UNMODIFIED graph-construction
code (cut out of its files with ``ast``; TensorFlow and tflearn themselves are not installed and there is no
network):

  * multi-label-cls/icnn_ebundle.py:120-166,316-388  Model.__init__ / Model.f        (E_, dE_dy_ = tf.gradients)
  * multi-label-cls/icnn-back.py:104-147,233-305     Model.__init__ / Model.f        (unrolled momentum GD, mse_,
                                                                                      opt.compute_gradients)
  * RL/src/icnn.py:325-404, 148-158                  Agent.negQ / Agent.bundle_entropy
  * completion/icnn_ebundle.py:105-161,337-452       Model.__init__ / Model.f        (the conv PICNN used on Olivetti)

What this pins: WHICH tensor multiplies which, which layers carry a bias / an activation / a batch-norm, the
variable naming, the unrolled recurrence and what is differentiated with respect to what -- all decided by the
reference's code as it executes.  What it cannot pin: the primitives themselves.  They are restated here from
the libraries' published semantics, one line each:

  tflearn.fully_connected(x, n, activation, bias)   x @ W [+ b], W laid out [n_in, n_units]; 'relu' / 'linear'
  tflearn.conv_2d(x, nf, k, strides, 'same', bias)    NHWC cross-correlation, W laid out [k, k, c_in, nf]; TensorFlow 'SAME'
                                                    padding: out = ceil(in / s), total = max((out-1) s + k - in, 0),
                                                    floor(total / 2) before, the rest after
  tflearn.batch_normalization (is_training False)   (x - moving_mean) / sqrt(moving_variance + 1e-5) * gamma + beta
  tflearn.activations.leaky_relu(x, alpha)          relu(x) - alpha * relu(-x)
  tf.gradients(ys, xs)                              d sum(ys) / d xs  (TensorFlow sums over ys)
  tf.nn.relu, tf.mul, tf.add_n, tf.reshape, tf.reduce_*, tf.square, tf.log, tf.clip_by_value, ...   elementwise
  opt.compute_gradients(loss, var_list)             [(d sum(loss) / d v, v)], None for unreachable variables

Eager instead of graph mode: ``tf.placeholder(.., name=N)`` returns the tensor registered under N in ``feeds``
BEFORE the reference code runs, so building the "graph" evaluates it.  Everything is float64 (the reference
declares float32 placeholders; the goldens are the float64 value of the same expressions, which is what the
float64 oracle is compared with).  Variables come from a store filled by the caller: a name the reference asks for
that the store lacks raises KeyError, and ``unused_variables()`` lists what the reference never touched -- both are
asserted empty by the generator, i.e. the oracle's parameterisation and the reference's variable set coincide.
"""
from __future__ import annotations

import contextlib
import types

import numpy as np
import torch

DT = torch.float64
BN_EPS = 1e-5        # tflearn.layers.normalization.batch_normalization(epsilon=1e-5)


@contextlib.contextmanager
def tensor_get_shape():
    """While active, torch tensors answer ``t.get_shape()[i].value`` like TensorFlow tensors
    (completion/icnn_ebundle.py:416 asks ``prevU.get_shape()[1].value``); removed again on exit."""
    torch.Tensor.get_shape = lambda self: [types.SimpleNamespace(value=int(d)) for d in self.shape]
    try:
        yield
    finally:
        del torch.Tensor.get_shape


class Variable:
    """A trainable variable: ``.name`` as TensorFlow prints it ('u0/W:0'), ``.value`` the torch leaf."""

    def __init__(self, name, array):
        self.name = name + ":0"
        self.value = torch.tensor(np.asarray(array, dtype=np.float64), dtype=DT, requires_grad=True)
        self.used = False

    def assign(self, _value):            # makeCvx / proj ops are built, never run, by the code paths executed here
        return ("assign", self.name)

    def get_shape(self):
        return types.SimpleNamespace(num_elements=lambda: int(self.value.numel()))


def _t(v):
    if isinstance(v, Variable):
        return v.value
    if isinstance(v, torch.Tensor):
        return v
    return torch.as_tensor(v, dtype=DT)


class _Scope:
    def __init__(self, name):
        self.name = name
        self.reuse = False

    def reuse_variables(self):
        self.reuse = True


class Shim:
    """One instance = one "default graph": variable store, feeds, scope stack, and the two module objects
    ``tf`` / ``tflearn`` to put in the namespace the reference code is exec'd in."""

    def __init__(self, variables, feeds=None):
        self.vars = {k: Variable(k, v) for k, v in variables.items()}
        self.feeds = dict(feeds or {})
        self.stack = [_Scope("")]
        self.created = []               # variable names in the order the reference code first asked for them
        self.tf = self._make_tf()
        self.tflearn = self._make_tflearn()

    # ---- variable store -----------------------------------------------------------------------------
    def get(self, name):
        v = self.vars[name]             # KeyError = the reference wants a variable the oracle does not have
        if not v.used:
            v.used = True
            self.created.append(name)
        return v.value

    def unused_variables(self):
        return sorted(k for k, v in self.vars.items() if not v.used)

    def feed(self, name, array, requires_grad=False):
        self.feeds[name] = torch.tensor(np.asarray(array, dtype=np.float64), dtype=DT, requires_grad=requires_grad)
        return self.feeds[name]

    # ---- tf -------------------------------------------------------------------------------------------
    def _make_tf(self):
        sh = self
        tf = types.SimpleNamespace()
        tf.float32, tf.float64, tf.bool = "float32", "float64", "bool"

        def placeholder(dtype, shape=None, name=None):
            return sh.feeds[name]
        tf.placeholder = placeholder

        @contextlib.contextmanager
        def variable_scope(name_or_scope, reuse=None):
            if isinstance(name_or_scope, _Scope):
                s = name_or_scope
            else:
                parent = sh.stack[-1].name
                s = _Scope(parent + "/" + name_or_scope if parent else name_or_scope)
                s.reuse = sh.stack[-1].reuse
            sh.stack.append(s)
            try:
                yield s
            finally:
                sh.stack.pop()
        tf.variable_scope = variable_scope
        tf.get_variable_scope = lambda: sh.stack[-1]

        @contextlib.contextmanager
        def name_scope(_name):
            yield None
        tf.name_scope = name_scope

        tf.nn = types.SimpleNamespace(relu=lambda x: torch.relu(_t(x)))
        tf.mul = tf.multiply = lambda a, b: _t(a) * _t(b)

        def add_n(xs):
            acc = _t(xs[0])
            for x in xs[1:]:
                acc = acc + _t(x)
            return acc
        tf.add_n = add_n
        tf.reshape = lambda x, shape, name=None: _t(x).reshape(*shape)
        tf.square = lambda x: _t(x) ** 2
        tf.sqrt = lambda x: torch.sqrt(_t(x))
        tf.log = lambda x: torch.log(_t(x))
        tf.abs = lambda x: torch.abs(_t(x))
        tf.maximum = lambda a, b: torch.maximum(_t(a), _t(b))
        tf.minimum = lambda a, b: torch.minimum(_t(a), _t(b))
        tf.clip_by_value = lambda x, lo, hi: torch.clamp(_t(x), lo, hi)
        tf.stop_gradient = lambda x: _t(x).detach()
        tf.contrib = types.SimpleNamespace(layers=types.SimpleNamespace(flatten=lambda x: _t(x).reshape(_t(x).shape[0], -1)))

        def _red(fn):
            def red(x, axis=None, reduction_indices=None):
                ax = axis if axis is not None else reduction_indices
                return fn(_t(x)) if ax is None else fn(_t(x), ax)
            return red
        tf.reduce_sum = _red(torch.sum)
        tf.reduce_mean = _red(torch.mean)
        tf.reduce_max = lambda x, axis=None: _t(x).max() if axis is None else _t(x).max(axis).values
        tf.reduce_min = lambda x, axis=None: _t(x).min() if axis is None else _t(x).min(axis).values

        def gradients(ys, xs):
            single = not isinstance(xs, (list, tuple))
            xl = [_t(x) for x in ([xs] if single else xs)]
            g = torch.autograd.grad(_t(ys).sum(), xl, create_graph=True, allow_unused=True)
            return list(g)
        tf.gradients = gradients

        # TensorFlow lists trainable variables in creation order; batch-norm moving statistics are not trainable
        tf.trainable_variables = lambda: [sh.vars[k] for k in sh.created if "/moving_" not in k]
        noop = lambda *a, **k: None     # noqa: E731
        tf.summary = types.SimpleNamespace(scalar=noop, histogram=noop, merge_all=noop, FileWriter=noop)
        tf.scalar_summary = tf.histogram_summary = tf.merge_all_summaries = noop
        tf.constant_initializer = lambda v: ("constant", v)

        class AdamOptimizer:
            def __init__(self, learning_rate=0.001):
                self.lr = learning_rate

            def compute_gradients(self, loss, var_list=None):
                vl = list(var_list) if var_list is not None else tf.trainable_variables()
                gs = torch.autograd.grad(_t(loss).sum(), [v.value for v in vl], allow_unused=True, retain_graph=True)
                return list(zip(gs, vl))

            def apply_gradients(self, _gv):
                return ("train_step",)
        tf.train = types.SimpleNamespace(AdamOptimizer=AdamOptimizer, Saver=lambda **k: None)
        return tf

    # ---- tflearn --------------------------------------------------------------------------------------
    def _make_tflearn(self):
        sh = self
        tl = types.SimpleNamespace()

        def fully_connected(incoming, n_units, activation="linear", bias=True, weights_init=None, bias_init=None,
                            regularizer=None, weight_decay=0.001, trainable=True, restore=True, reuse=False,
                            scope=None, name="FullyConnected"):
            x = _t(incoming)
            if x.dim() > 2:                                     # tflearn flattens a conv feature map (NHWC order)
                x = x.reshape(x.shape[0], -1)
            W = sh.get(scope.name + "/W")
            assert W.shape == (x.shape[1], n_units), (scope.name, tuple(W.shape), (x.shape[1], n_units))
            out = x @ W
            if bias:
                b = sh.get(scope.name + "/b")
                assert b.shape == (n_units,)
                out = out + b
            else:
                assert scope.name + "/b" not in sh.vars, scope.name + " is bias-free in the reference"
            if activation == "relu":
                out = torch.relu(out)
            else:
                assert activation == "linear", activation
            return out
        tl.fully_connected = fully_connected

        def batch_normalization(incoming, reuse=False, scope=None, name="BatchNormalization", **kw):
            pre = scope.name + "/" + name + "/"
            g, b = sh.get(pre + "gamma"), sh.get(pre + "beta")
            mu, var = sh.get(pre + "moving_mean"), sh.get(pre + "moving_variance")
            return (_t(incoming) - mu) / torch.sqrt(var + BN_EPS) * g + b
        tl.batch_normalization = batch_normalization

        def conv_2d(incoming, nb_filter, filter_size, strides=1, padding="same", activation="linear", bias=True,
                    weights_init=None, bias_init=None, regularizer=None, weight_decay=0.001, trainable=True,
                    restore=True, reuse=False, scope=None, name="Conv2D"):
            import torch.nn.functional as F
            assert padding == "same"
            x = _t(incoming)                                    # NHWC
            st = strides if isinstance(strides, int) else strides[1]
            assert isinstance(strides, int) or (strides[0] == 1 and strides[3] == 1 and strides[1] == strides[2])
            k = filter_size
            W = sh.get(scope.name + "/W")                       # [k, k, c_in, nb_filter]
            assert W.shape == (k, k, x.shape[3], nb_filter), (scope.name, tuple(W.shape), (k, k, x.shape[3], nb_filter))
            pads = []
            for size in (x.shape[2], x.shape[1]):               # F.pad order: (W_before, W_after, H_before, H_after)
                out = -(-size // st)
                tot = max((out - 1) * st + k - size, 0)
                pads += [tot // 2, tot - tot // 2]
            b = None
            if bias:
                b = sh.get(scope.name + "/b")
            else:
                assert scope.name + "/b" not in sh.vars, scope.name + " is bias-free in the reference"
            y = F.conv2d(F.pad(x.permute(0, 3, 1, 2), pads), W.permute(3, 2, 0, 1), b, stride=st).permute(0, 2, 3, 1)
            if activation == "relu":
                y = torch.relu(y)
            else:
                assert activation == "linear", activation
            return y
        tl.conv_2d = conv_2d
        tl.activations = types.SimpleNamespace(
            leaky_relu=lambda x, alpha=0.1: torch.relu(_t(x)) - alpha * torch.relu(-_t(x)))
        tl.is_training = lambda flag: None
        return tl


def variables_from_params(p, bnvars=None, prefix=""):
    """PicnnParams -> {tensorflow variable name: array}, the naming of the reference's variable scopes
    (multi-label-cls/icnn_ebundle.py:341,353,356,363,366,372; RL/src/icnn.py:346,361,366,373,377,384)."""
    v = {}
    for i in range(p.L):
        v["%su%d/W" % (prefix, i)] = p.Wu[i]
        v["%su%d/b" % (prefix, i)] = p.bu[i]
        if bnvars is not None and i < p.L - 1:
            for nm, a in zip(("gamma", "beta", "moving_mean", "moving_variance"), bnvars[i]):
                v["%su%d/bn/%s" % (prefix, i, nm)] = a
    for i in range(p.L + 1):
        if i > 0:
            v["%sz%d_zu_u/W" % (prefix, i)] = p.Wzu[i]
            v["%sz%d_zu_u/b" % (prefix, i)] = p.bzu[i]
            v["%sz%d_zu_proj/W" % (prefix, i)] = p.Wz[i]
        v["%sz%d_yu_u/W" % (prefix, i)] = p.Wyu[i]
        v["%sz%d_yu_u/b" % (prefix, i)] = p.byu[i]
        v["%sz%d_yu/W" % (prefix, i)] = p.Wy[i]
        v["%sz%d_u/W" % (prefix, i)] = p.Wzx[i]
        v["%sz%d_u/b" % (prefix, i)] = p.bzx[i]
    return v
