"""A small static graph of layers — the stand-in for the TensorFlow graph a ModelHelper builds.

The reference's learners work by *editing* the graph a ModelHelper's ``forward_train`` emits:
they search Conv2D / MatMul / DepthwiseConv2dNative ops and activation ops and splice quantizers
in (learners/uniform_quantization/utils.py:51-134).  To keep that plugin contract, ``forward_*``
here also builds a graph (of ``Op`` nodes with TF op-type names and TF-style variable names) which
the learner edits (marks) and ``engine.Executor`` lowers to launches of libpf_b200.so kernels.
Shapes are static NHWC; there is no tracing compiler — the executor's launch list is replayed
through a CUDA graph.
"""
import contextlib
import math
from collections import OrderedDict

import numpy as np

_default_graph = []


class Variable:
    def __init__(self, name, shape, initializer, trainable=True):
        self.name = name                # e.g. 'model/resnet_model/conv2d/kernel:0'
        self.shape = tuple(int(s) for s in shape)
        self.initializer = initializer  # callable(rng, shape) -> np.float32 array
        self.trainable = trainable
        self.numel = int(np.prod(self.shape)) if self.shape else 1

    def __repr__(self):
        return 'Variable(%s, %s)' % (self.name, self.shape)


class Tensor:
    def __init__(self, op, shape, name):
        self.op = op
        self.shape = tuple(int(s) for s in shape)
        self.name = name
        self.consumers = []

    @property
    def numel(self):
        return int(np.prod(self.shape))

    def __add__(self, other):
        return add(self, other)

    def __repr__(self):
        return 'Tensor(%s, %s)' % (self.name, self.shape)


class Op:
    def __init__(self, graph, type_, name, inputs, variables, attrs, out_shape):
        self.graph = graph
        self.type = type_
        self.name = name
        self.inputs = list(inputs)
        self.vars = dict(variables)       # role -> Variable  ('kernel', 'bias', 'gamma', ...)
        self.attrs = dict(attrs)
        self.output = Tensor(self, out_shape, name + ':0')
        for t in self.inputs:
            t.consumers.append(self)

    def get_attr(self, k):
        return self.attrs[k]

    def __repr__(self):
        return 'Op(%s, %s)' % (self.type, self.name)


class Graph:
    def __init__(self):
        self.ops = []
        self.variables = OrderedDict()
        self._scopes = []
        self._names = {}
        self.placeholders = OrderedDict()

    @contextlib.contextmanager
    def as_default(self):
        _default_graph.append(self)
        try:
            yield self
        finally:
            _default_graph.pop()

    # -- naming (TF-style: conv2d, conv2d_1, ...)
    def scope_prefix(self):
        return '/'.join(self._scopes) + ('/' if self._scopes else '')

    def unique_name(self, base):
        full = self.scope_prefix() + base
        n = self._names.get(full, 0)
        self._names[full] = n + 1
        return full if n == 0 else '%s_%d' % (full, n)

    def add_op(self, type_, base, inputs, variables, attrs, out_shape, name=None):
        op = Op(self, type_, name or self.unique_name(base), inputs, variables, attrs, out_shape)
        self.ops.append(op)
        return op

    def get_variable(self, name, shape, initializer, trainable=True):
        full = name + ':0'
        if full in self.variables:
            return self.variables[full]
        v = Variable(full, shape, initializer, trainable)
        self.variables[full] = v
        return v

    def get_operations(self):
        return list(self.ops)

    def vars_in_scope(self, scope, trainable_only=False):
        return [v for v in self.variables.values()
                if v.name.startswith(scope + '/') and (v.trainable or not trainable_only)]


def get_default_graph():
    if not _default_graph:
        raise RuntimeError('no default graph: use `with Graph().as_default():`')
    return _default_graph[-1]


@contextlib.contextmanager
def variable_scope(name):
    g = get_default_graph()
    g._scopes.append(name)
    try:
        yield
    finally:
        g._scopes.pop()


def placeholder(shape, name):
    g = get_default_graph()
    op = g.add_op('Placeholder', name, [], {}, {}, shape, name=g.scope_prefix() + name)
    g.placeholders[op.name] = op.output
    return op.output


# ------------------------------------------------------------------------------ initializers
def variance_scaling_initializer(scale=1.0, mode='fan_in', distribution='truncated_normal'):
    """tf.variance_scaling_initializer() defaults (utils/external/resnet_model.py:102)."""
    def init(rng, shape):
        if len(shape) == 4:
            fan_in, fan_out = shape[0] * shape[1] * shape[2], shape[0] * shape[1] * shape[3]
        else:
            fan_in, fan_out = shape[0], shape[-1]
        n = {'fan_in': fan_in, 'fan_out': fan_out, 'fan_avg': (fan_in + fan_out) / 2.0}[mode]
        std = math.sqrt(scale / max(1.0, n))
        if distribution == 'truncated_normal':
            std /= 0.87962566103423978
            x = rng.standard_normal(size=shape)
            bad = np.abs(x) > 2
            while bad.any():
                x[bad] = rng.standard_normal(size=int(bad.sum()))
                bad = np.abs(x) > 2
            return (x * std).astype(np.float32)
        return (rng.standard_normal(size=shape) * std).astype(np.float32)
    return init


def glorot_uniform_initializer():
    """tf.layers.conv2d / dense default kernel initializer."""
    def init(rng, shape):
        if len(shape) == 4:
            fan_in, fan_out = shape[0] * shape[1] * shape[2], shape[0] * shape[1] * shape[3]
        else:
            fan_in, fan_out = shape[0], shape[-1]
        lim = math.sqrt(6.0 / (fan_in + fan_out))
        return rng.uniform(-lim, lim, size=shape).astype(np.float32)
    return init


def constant_initializer(v):
    return lambda rng, shape: np.full(shape, v, dtype=np.float32)


# ------------------------------------------------------------------------------ layers
def _pads(padding, k, s, size):
    """Leading pad and output size for TF 'SAME'/'VALID' or an explicit (begin, end) pair."""
    if isinstance(padding, str):
        p = padding.upper()
        if p == 'VALID':
            return 0, (size - k) // s + 1
        if p == 'SAME':
            out = -(-size // s)
            total = max((out - 1) * s + k - size, 0)
            return total // 2, out
        raise ValueError('unknown padding: ' + padding)
    beg, end = padding
    return beg, (size + beg + end - k) // s + 1


def conv2d(inputs, filters, kernel_size, strides=1, padding='valid', use_bias=True,
           kernel_initializer=None, name=None, kernel_name='kernel', bias_name='bias', exact_name=False):
    """tf.layers.conv2d / slim.conv2d, NHWC x HWIO.  `padding`: 'same' | 'valid' | ((top,bottom),(left,right)).
    slim layers pass kernel_name='weights', bias_name='biases', exact_name=True (scope given by the caller)."""
    g = get_default_graph()
    n, h, w, c = inputs.shape
    kh, kw = (kernel_size, kernel_size) if isinstance(kernel_size, int) else kernel_size
    sh, sw = (strides, strides) if isinstance(strides, int) else strides
    ph, pw = (padding, padding) if isinstance(padding, str) else padding
    pt, p = _pads(ph, kh, sh, h)
    pl, q = _pads(pw, kw, sw, w)
    lname = (g.scope_prefix() + name) if exact_name else g.unique_name(name or 'conv2d')
    kernel = g.get_variable(lname + '/' + kernel_name, (kh, kw, c, filters),
                            kernel_initializer or glorot_uniform_initializer())
    vs = {'kernel': kernel}
    if use_bias:
        vs['bias'] = g.get_variable(lname + '/' + bias_name, (filters,), constant_initializer(0.0))
    op = g.add_op('Conv2D', 'Conv2D', [inputs], vs,
                  dict(strides=(sh, sw), pad=(pt, pl), padding=padding, ksize=(kh, kw)),
                  (n, p, q, filters), name=lname + '/Conv2D')
    return op.output


def depthwise_conv2d(inputs, kernel_size, strides=1, padding='same', kernel_initializer=None, name=None,
                     exact_name=False):
    """slim.separable_conv2d(num_outputs=None) depthwise part, depth_multiplier 1; kernel [kh,kw,C,1]."""
    g = get_default_graph()
    n, h, w, c = inputs.shape
    kh = kw = kernel_size
    sh = sw = strides
    pt, p = _pads(padding, kh, sh, h)
    pl, q = _pads(padding, kw, sw, w)
    lname = (g.scope_prefix() + name) if exact_name else g.unique_name(name or 'depthwise')
    kernel = g.get_variable(lname + '/depthwise_weights', (kh, kw, c, 1),
                            kernel_initializer or glorot_uniform_initializer())
    op = g.add_op('DepthwiseConv2dNative', 'depthwise', [inputs], {'kernel': kernel},
                  dict(strides=(sh, sw), pad=(pt, pl), padding=padding, ksize=(kh, kw)),
                  (n, p, q, c), name=lname + '/depthwise')
    return op.output


def dense(inputs, units, use_bias=True, kernel_initializer=None, name=None):
    g = get_default_graph()
    n, c = inputs.shape
    lname = g.unique_name(name or 'dense')
    kernel = g.get_variable(lname + '/kernel', (c, units), kernel_initializer or glorot_uniform_initializer())
    vs = {'kernel': kernel}
    if use_bias:
        vs['bias'] = g.get_variable(lname + '/bias', (units,), constant_initializer(0.0))
    op = g.add_op('MatMul', 'MatMul', [inputs], vs, {}, (n, units), name=lname + '/MatMul')
    return op.output


def batch_normalization(inputs, training, momentum=0.99, epsilon=1e-3, name=None, exact_name=False):
    """tf.layers.batch_normalization / slim.batch_norm (fused).  Variables: gamma, beta, moving_mean,
    moving_variance."""
    g = get_default_graph()
    c = inputs.shape[-1]
    lname = (g.scope_prefix() + name) if exact_name else g.unique_name(name or 'batch_normalization')
    vs = {'gamma': g.get_variable(lname + '/gamma', (c,), constant_initializer(1.0)),
          'beta': g.get_variable(lname + '/beta', (c,), constant_initializer(0.0)),
          'moving_mean': g.get_variable(lname + '/moving_mean', (c,), constant_initializer(0.0), trainable=False),
          'moving_variance': g.get_variable(lname + '/moving_variance', (c,), constant_initializer(1.0),
                                            trainable=False)}
    op = g.add_op('FusedBatchNorm', 'FusedBatchNorm', [inputs], vs,
                  dict(training=bool(training), momentum=float(momentum), epsilon=float(epsilon)),
                  inputs.shape, name=lname + '/FusedBatchNorm')
    return op.output


def relu(inputs, name=None):
    g = get_default_graph()
    return g.add_op('Relu', name or 'Relu', [inputs], {}, {}, inputs.shape).output


def relu6(inputs, name=None):
    g = get_default_graph()
    return g.add_op('Relu6', name or 'Relu6', [inputs], {}, {}, inputs.shape).output


def max_pooling2d(inputs, pool_size, strides, padding='valid', name=None):
    g = get_default_graph()
    n, h, w, c = inputs.shape
    kh, kw = (pool_size, pool_size) if isinstance(pool_size, int) else pool_size
    sh, sw = (strides, strides) if isinstance(strides, int) else strides
    pt, p = _pads(padding, kh, sh, h)
    pl, q = _pads(padding, kw, sw, w)
    op = g.add_op('MaxPool', name or 'max_pooling2d', [inputs], {},
                  dict(ksize=(kh, kw), strides=(sh, sw), pad=(pt, pl)), (n, p, q, c))
    return op.output


def reduce_mean_hw(inputs, name=None, keepdims=False):
    """tf.reduce_mean(x, [1, 2]) (+ squeeze unless keepdims) -> [N, C] or [N, 1, 1, C]."""
    g = get_default_graph()
    n, h, w, c = inputs.shape
    return g.add_op('Mean', name or 'Mean', [inputs], {}, {}, (n, 1, 1, c) if keepdims else (n, c)).output


def squeeze_hw(inputs, name=None):
    """tf.squeeze(x, [1, 2]) on [N,1,1,C]."""
    g = get_default_graph()
    n, h, w, c = inputs.shape
    assert h == 1 and w == 1
    return g.add_op('Reshape', name or 'SpatialSqueeze', [inputs], {}, {}, (n, c)).output


def truncated_normal_initializer(stddev):
    def init(rng, shape):
        x = rng.standard_normal(size=shape)
        bad = np.abs(x) > 2
        while bad.any():
            x[bad] = rng.standard_normal(size=int(bad.sum()))
            bad = np.abs(x) > 2
        return (x * stddev).astype(np.float32)
    init.stddev = stddev
    return init


def flatten(inputs, name=None):
    g = get_default_graph()
    n = inputs.shape[0]
    return g.add_op('Reshape', name or 'flatten', [inputs], {}, {}, (n, int(np.prod(inputs.shape[1:])))).output


def add(a, b, name=None):
    g = get_default_graph()
    if a.shape != b.shape:
        raise ValueError('add: shape mismatch %s vs %s' % (a.shape, b.shape))
    return g.add_op('Add', name or 'add', [a, b], {}, {}, a.shape).output


def softmax(inputs, name=None):
    g = get_default_graph()
    return g.add_op('Softmax', name or 'Softmax', [inputs], {}, {}, inputs.shape).output


def identity(inputs, name):
    g = get_default_graph()
    return g.add_op('Identity', name, [inputs], {}, {}, inputs.shape).output


def dropout(inputs, keep_prob, is_training, name=None):
    """slim.dropout: y = (x / keep_prob) * floor(keep_prob + u), u ~ U[0, 1), in a training-mode forward pass; the
    identity otherwise (and always when is_training is False)."""
    g = get_default_graph()
    return g.add_op('Dropout', name or 'Dropout', [inputs], {},
                    dict(keep_prob=float(keep_prob), training=bool(is_training)), inputs.shape).output


# ------------------------------------------------------------------------------ losses / metrics
class LossSpec:
    """Symbolic scalar loss: hard CE + sum_i coeff_i * l2_loss(var_i) (+ distillation).

    What ModelHelper.calc_loss returns in place of a TF scalar; supports `+` and `*` by floats so
    the reference's `loss += FLAGS.loss_w_dcy * tf.add_n([...])` idiom carries over."""

    def __init__(self):
        self.ce = None            # (labels Tensor, logits Tensor, weight)
        self.l2 = OrderedDict()   # Variable -> coefficient
        self.dst = None           # (student logits Tensor, teacher logits Tensor, w, T)
        self.scale = 1.0

    def copy(self):
        o = LossSpec()
        o.ce, o.dst = self.ce, self.dst
        o.l2 = OrderedDict(self.l2)
        return o

    def __add__(self, other):
        if other == 0:
            return self
        o = self.copy()
        if other.ce is not None:
            if o.ce is not None:
                raise ValueError('only one cross-entropy term is supported')
            o.ce = other.ce
        if other.dst is not None:
            o.dst = other.dst
        for v, c in other.l2.items():
            o.l2[v] = o.l2.get(v, 0.0) + c
        return o

    __radd__ = __add__

    def __mul__(self, f):
        f = float(f)
        o = self.copy()
        if o.ce is not None:
            o.ce = (o.ce[0], o.ce[1], o.ce[2] * f)
        if o.dst is not None:
            o.dst = (o.dst[0], o.dst[1], o.dst[2] * f, o.dst[3])
        o.l2 = OrderedDict((v, c * f) for v, c in o.l2.items())
        return o

    __rmul__ = __mul__


def softmax_cross_entropy(onehot_labels, logits):
    """tf.losses.softmax_cross_entropy (batch mean)."""
    s = LossSpec()
    s.ce = (onehot_labels, logits, 1.0)
    return s


def l2_loss(var):
    s = LossSpec()
    s.l2[var] = 1.0
    return s


def add_n(terms):
    out = 0
    for t in terms:
        out = out + t
    return out


def distillation_cross_entropy(logits_pri, logits_dst, w, tempr):
    s = LossSpec()
    s.dst = (logits_pri, logits_dst, float(w), float(tempr))
    return s


class Metric:
    """Symbolic metric: 'top1' / 'top5' accuracy of outputs vs one-hot labels."""

    def __init__(self, kind, labels, outputs):
        self.kind, self.labels, self.outputs = kind, labels, outputs


def accuracy(labels, outputs):
    return Metric('top1', labels, outputs)


def in_top_k_accuracy(labels, outputs, k=5):
    if k != 5:
        raise NotImplementedError('only top-5 is implemented')
    return Metric('top5', labels, outputs)
