"""A minimal *eager* stand-in for the TensorFlow-1.x API surface the reference touches on the
hot path, so that the reference's own Python (lib/ops.py, lib/frvsr.py, lib/Teco.py of a
reference checkout) can be executed without TensorFlow to produce golden vectors.

Scope and honesty: TensorFlow itself is not installable here, so the *primitive* semantics
(SAME padding, conv2d_transpose alignment, legacy resize, dense_image_warp, fused BN) come
from tests/golden/tf_ext_ref.py -- numpy written from the operators' published definitions,
sharing no code with oracle/teco_oracle.py.  The goldens therefore pin the reference's WIRING
(layer order, scopes/variable names, activations, channel orders, loss formulas, slicing) by the
reference's own code, and the [TF-ext] primitives by a derivation that is independent of the
oracle under test (they are still a restatement of TensorFlow, not TensorFlow).  Used only by
tests/golden/make_golden.py (never at test time on the GPU box, never by the product).

Tensors are float32 numpy arrays (subclass with get_shape/set_shape) because the reference
uses negative-step slicing, which torch tensors reject.
"""
import contextlib
import sys
import types

import numpy as np
import torch

from tests.golden import tf_ext_ref as X


class _Shape(tuple):
    def as_list(self):
        return list(self)


class TFArray(np.ndarray):
    def get_shape(self):
        return _Shape(self.shape)

    def set_shape(self, s):
        assert tuple(int(v) for v in s) == tuple(self.shape), (s, self.shape)


def A(x):
    return np.asarray(x, dtype=np.float32).view(TFArray) if not isinstance(x, TFArray) else x


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(x, dtype=np.float32)))


def _a(t):
    return t.detach().numpy().view(TFArray)


# ---------------------------------------------------------------- variable store / scopes
class Store:
    def __init__(self):
        self.params = {}
        self.scope = []
        self.used = []
        self.arg_scopes = []
        self.collections = {}


S = Store()


class _VS:
    def __init__(self, name):
        self.name = name


@contextlib.contextmanager
def variable_scope(name_or_scope=None, default_name=None, values=None, reuse=None):
    nm = name_or_scope if name_or_scope is not None else default_name
    if isinstance(nm, _VS):
        nm = nm.name
    S.scope.append(nm)
    try:
        yield _VS("/".join(S.scope))
    finally:
        S.scope.pop()


@contextlib.contextmanager
def _noop_ctx(*a, **k):
    yield (a[0] if a and isinstance(a[0], str) else None)


def _var(local):
    full = "/".join(S.scope + [local])
    if full not in S.params:
        raise KeyError("reference asked for variable %r which the oracle's name map lacks" % full)
    S.used.append(full)
    return S.params[full]


# ---------------------------------------------------------------- slim
def _argscope_kwargs(fn):
    kw = {}
    for d in S.arg_scopes:
        if fn in d:
            kw.update(d[fn])
    return kw


@contextlib.contextmanager
def arg_scope(fns, **kw):
    d = {f: dict(kw) for f in fns}
    S.arg_scopes.append(d)
    try:
        yield d
    finally:
        S.arg_scopes.pop()


def _collect(coll, alias, out):
    if coll is not None:
        S.collections.setdefault(coll, []).append((alias, out))


_DEFAULT = object()


def relu(x):
    return np.maximum(x, 0).view(TFArray)


def slim_conv2d(inputs, num_outputs, kernel_size, stride=1, padding='SAME', data_format='NHWC',
                activation_fn=_DEFAULT, weights_initializer=None, biases_initializer=_DEFAULT,
                weights_regularizer=None, scope=None, reuse=None, outputs_collections=None):
    kw = _argscope_kwargs(slim_conv2d)
    if outputs_collections is None:
        outputs_collections = kw.get('outputs_collections')
    if activation_fn is _DEFAULT:
        activation_fn = kw.get('activation_fn', relu)
    assert padding == 'SAME' and data_format == 'NHWC'
    k = kernel_size if isinstance(kernel_size, (list, tuple)) else [kernel_size, kernel_size]
    with variable_scope(scope, 'Conv') as sc:
        w = _var('weights')
        assert tuple(w.shape) == (k[0], k[1], inputs.shape[-1], num_outputs), (sc.name, w.shape)
        b = _var('biases') if biases_initializer is not None else None
        y = A(X.conv2d(inputs, w.numpy(), None if b is None else b.numpy(), stride, 'SAME'))
        if activation_fn is not None:
            y = activation_fn(y)
        _collect(outputs_collections, sc.name, y)
    return y


def slim_conv2d_transpose(inputs, num_outputs, kernel_size, stride=1, padding='SAME', data_format='NHWC',
                          activation_fn=_DEFAULT, weights_initializer=None, biases_initializer=_DEFAULT, scope=None):
    assert padding == 'SAME' and data_format == 'NHWC' and activation_fn is None
    k = kernel_size if isinstance(kernel_size, (list, tuple)) else [kernel_size, kernel_size]
    with variable_scope(scope, 'Conv2d_transpose') as sc:
        w = _var('weights')
        assert tuple(w.shape) == (k[0], k[1], num_outputs, inputs.shape[-1]), (sc.name, w.shape)
        b = _var('biases') if biases_initializer is not None else None
        return A(X.conv2d_transpose(inputs, w.numpy(), None if b is None else b.numpy(), stride))


def slim_batch_norm(inputs, decay=0.999, epsilon=0.001, updates_collections=None, scale=False, fused=None,
                    is_training=True, scope=None):
    assert is_training and not scale
    with variable_scope(scope, 'BatchNorm'):
        return A(X.batch_norm_train(inputs, _var('beta').numpy(), epsilon))


def slim_max_pool2d(inputs, kernel_size, stride=2, padding='VALID', scope=None, outputs_collections=None):
    assert list(kernel_size) == [2, 2] and stride == 2 and padding == 'VALID'
    return A(X.max_pool_2x2(inputs))


def slim_repeat(inputs, repetitions, layer, *args, **kwargs):
    scope = kwargs.pop('scope')
    with variable_scope(scope):
        net = inputs
        for i in range(repetitions):
            kwargs['scope'] = scope + '_' + str(i + 1)
            net = layer(net, *args, **kwargs)
    return net


def convert_collection_to_dict(coll):
    return dict(S.collections.get(coll, []))


# ---------------------------------------------------------------- tf.*
class Dense:
    def __init__(self, units, activation=None, kernel_initializer=None):
        self.units = units

    def apply(self, inputs):
        with variable_scope('dense'):
            self.kernel = _var('kernel')
            bias = _var('bias')
        return _a(_t(inputs) @ self.kernel + bias)


class LeakyReLU:
    def __init__(self, alpha):
        self.alpha = alpha

    def call(self, x):
        return A(X.leaky_relu(x, self.alpha))


def tf_shape(x):
    return np.array(x.shape)


def tf_reshape(x, shape):
    return np.reshape(x, [int(s) for s in shape]).view(TFArray)


def tf_transpose(x, perm):
    return np.transpose(x, perm).view(TFArray)


def tf_concat(vals, axis):
    return np.concatenate([np.asarray(v) for v in vals], axis=axis).view(TFArray)


def tf_stack(vals, axis=0):
    return np.stack([np.asarray(v) for v in vals], axis=axis).view(TFArray)


def resize_images(x, size):
    return A(X.resize_bilinear(x, int(size[0]), int(size[1])))


def dense_image_warp(image, flow):
    return A(X.dense_image_warp(image, flow))


def crop_to_bounding_box(x, oy, ox, th, tw):
    return x[:, oy:oy + th, ox:ox + tw, :]


def tf_pad(x, paddings, mode="CONSTANT"):
    pads = [tuple(int(v) for v in p) for p in np.asarray(paddings)]
    return np.pad(x, pads, mode={"CONSTANT": "constant", "SYMMETRIC": "symmetric"}[mode]).view(TFArray)


def reduce_mean(x, axis=None, keepdims=False):
    ax = tuple(axis) if isinstance(axis, (list, tuple)) else axis
    return np.mean(np.asarray(x, dtype=np.float32), axis=ax, keepdims=keepdims, dtype=np.float32).view(TFArray)


def reduce_sum(x, axis=None, keepdims=False):
    ax = tuple(axis) if isinstance(axis, (list, tuple)) else axis
    return np.sum(np.asarray(x, dtype=np.float32), axis=ax, keepdims=keepdims, dtype=np.float32).view(TFArray)


def nn_conv2d(x, filt, strides, padding, name=None):
    assert padding == "VALID"
    return A(X.conv2d(x, np.asarray(filt), None, strides[1], "VALID"))


class _Optimizer:
    def __init__(self, *a, **k):
        pass

    def compute_gradients(self, loss, var_list=None):
        return []

    def apply_gradients(self, gv):
        return None


class _EMA:
    def __init__(self, decay):
        pass

    def apply(self, vals):
        return None

    def average(self, v):
        return np.float32(0.0)


def install():
    """Put stub modules into sys.modules so that `from lib.Teco import *` of the reference works."""
    tf = types.ModuleType("tensorflow")
    tf.float32, tf.int32, tf.int64, tf.bool = np.float32, np.int32, np.int64, np.bool_
    tf.variable_scope = variable_scope
    tf.name_scope = _noop_ctx
    tf.device = _noop_ctx
    tf.control_dependencies = _noop_ctx
    tf.shape = tf_shape
    tf.reshape = tf_reshape
    tf.transpose = lambda x, perm=None: tf_transpose(x, perm)
    tf.concat = lambda values, axis: tf_concat(values, axis)
    tf.stack = tf_stack
    tf.identity = lambda x: x
    tf.stop_gradient = lambda x: x
    tf.zeros = lambda shape, dtype=np.float32: np.zeros([int(s) for s in shape], dtype=np.float32).view(TFArray)
    tf.zeros_like = lambda x: np.zeros_like(x).view(TFArray)
    tf.constant = lambda v, dtype=None, shape=None, name=None: (np.asarray(v, dtype=np.float32).view(TFArray)
                                                                 if dtype in (None, np.float32) else np.asarray(v))
    tf.abs = lambda x: np.abs(x)
    tf.square = lambda x: np.square(x)
    tf.sqrt = lambda x: np.sqrt(x)
    tf.log = lambda x: np.log(x)
    tf.tanh = lambda x: np.tanh(x)
    tf.minimum = lambda a, b: np.minimum(a, b)
    tf.maximum = lambda a, b: np.maximum(a, b)
    tf.cast = lambda x, dt: np.asarray(x).astype(dt)
    tf.less = lambda a, b: bool(a < b)
    tf.equal = lambda a, b: bool(a == b)
    tf.cond = lambda pred, t, f: t() if pred else f()
    tf.reduce_mean = reduce_mean
    tf.reduce_sum = reduce_sum
    tf.pad = tf_pad
    tf.space_to_depth = lambda x, bs: A(X.space_to_depth(x, bs))
    tf.assign = lambda ref, val: val
    tf.assign_add = lambda ref, val: ref + val
    tf.group = lambda *a: None
    tf.get_collection = lambda key, scope=None: []
    tf.add_to_collection = lambda name, value: None
    tf.get_variable = lambda *a, **k: np.int32(0)
    tf.zeros_initializer = lambda: None
    tf.GraphKeys = types.SimpleNamespace(MODEL_VARIABLES="mv", TRAINABLE_VARIABLES="tv", GLOBAL_VARIABLES="gv",
                                         UPDATE_OPS="uo", SUMMARIES="s")
    tf.nn = types.SimpleNamespace(relu=relu, sigmoid=lambda x: A(X.sigmoid(x)), conv2d=nn_conv2d)
    tf.image = types.SimpleNamespace(resize_images=resize_images, crop_to_bounding_box=crop_to_bounding_box)
    tf.layers = types.SimpleNamespace(Dense=Dense)
    tf.train = types.SimpleNamespace(
        get_or_create_global_step=lambda: np.int64(0),
        exponential_decay=lambda lr, gs, ds, dr, staircase=False: np.float32(lr),
        AdamOptimizer=_Optimizer, ExponentialMovingAverage=_EMA)

    slim = types.ModuleType("tensorflow.contrib.slim")
    slim.conv2d, slim.conv2d_transpose = slim_conv2d, slim_conv2d_transpose
    slim.batch_norm, slim.max_pool2d, slim.repeat, slim.arg_scope = slim_batch_norm, slim_max_pool2d, slim_repeat, arg_scope
    slim.fully_connected = object()
    slim.l2_regularizer = lambda w: None
    slim.utils = types.SimpleNamespace(convert_collection_to_dict=convert_collection_to_dict)

    contrib = types.ModuleType("tensorflow.contrib")
    contrib.slim = slim
    contrib.image = types.SimpleNamespace(dense_image_warp=dense_image_warp)
    contrib.layers = types.SimpleNamespace(xavier_initializer=lambda: None)
    tf.contrib = contrib

    tfpy = types.ModuleType("tensorflow.python")
    tfpy_ops = types.ModuleType("tensorflow.python.ops")
    tfpy_ops.summary_op_util = types.SimpleNamespace()
    keras = types.ModuleType("keras")
    keras.layers = types.SimpleNamespace(LeakyReLU=LeakyReLU)

    import scipy.signal
    if not hasattr(scipy.signal, "gaussian"):  # moved to scipy.signal.windows in new scipy
        scipy.signal.gaussian = scipy.signal.windows.gaussian

    sys.modules.update({"tensorflow": tf, "tensorflow.contrib": contrib, "tensorflow.contrib.slim": slim,
                        "tensorflow.python": tfpy, "tensorflow.python.ops": tfpy_ops, "keras": keras})
    return tf


def set_params(params):
    S.params = {k: v.to(torch.float32) for k, v in params.items()}
    S.used = []
    S.collections = {}
    S.scope = []
