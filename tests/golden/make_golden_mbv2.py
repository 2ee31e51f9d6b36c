"""MobileNet-v2 as the REFERENCE'S OWN code builds it, recorded by running it in this container under a stub of
TensorFlow / tf.contrib.slim (TensorFlow 1.x cannot be imported here).

  python tests/golden/make_golden_mbv2.py        ->  tests/golden/ref_executed_mbv2_v1.json

What runs is /root/reference's nets/mobilenet_at_ilsvrc12.py (forward_fn with --mobilenet_version 2, and
ModelHelper.setup_lrn_rate), utils/external/{mobilenet_v2,mobilenet,conv_blocks}.py, utils/lrn_rate_utils.py and
learners/weight_sparsification/utils.py, unmodified.  The stub extends the slim-stub recorder of
make_golden_from_reference.py (whose helpers `Flags`, `make_tf_stub` and `load` are imported, not changed) with what v2
touches: slim.add_arg_scope / arg_scope with slim's semantics (per-function defaults, explicit arguments win, a scope
dict re-entered by `with slim.arg_scope(sc)`), tf.variable_scope default names uniquified per parent scope
(`expanded_conv`, `expanded_conv_1`, ..., `Conv`, `Conv_1`), tf.identity, tf.nn.avg_pool, tf.zeros_initializer,
shape-tracking tensors with get_shape().as_list(), and `net += input_tensor`.  Recorded per layer, in call order:

  conv     [scope, filters, kernel, stride, padding, weights stddev, bias]
  dwconv   [scope, kernel, stride, padding, depth multiplier, weights stddev]
  bn       [scope, decay, epsilon, center, scale, is_training]
  act      [name]               (relu6; `identity` is the linear projection)
  add      []                   (the residual `net += input_tensor`)
  avgpool  [kernel h, kernel w, padding]
  dropout  [keep_prob, is_training]

plus the v2 learning-rate schedule (the arguments setup_lrn_rate hands tf.train.exponential_decay, and the number of
iterations), the reference's get_maskable_vars on this repo's v2 variable names, and the mobilenet flag defaults."""
import json
import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
from make_golden_from_reference import Flags, load, make_tf_stub  # noqa: E402

OUT = os.path.join(HERE, 'ref_executed_mbv2_v1.json')
MULTIPLIERS = [1.0, 1.4, 0.75, 0.5, 0.35]


class T4(object):
    """a symbolic NHWC tensor: shape and name"""

    def __init__(self, shape, name='t:0', rec=None):
        self.shape4, self.name, self._rec = list(shape), name, rec
        self.graph = types.SimpleNamespace(get_operations=lambda: [])

    @property
    def shape(self):
        return list(self.shape4)

    def get_shape(self):
        return types.SimpleNamespace(as_list=lambda: list(self.shape4))

    def set_shape(self, shape):
        pass

    def __add__(self, other):
        assert self.shape4 == other.shape4
        self._rec.append(('add',))
        return T4(self.shape4, self.name, self._rec)

    __iadd__ = __add__


def build_stub(flags, rec):
    tf = make_tf_stub(flags)
    scope_stack = [{}]
    names = [[]]                       # current variable-scope path
    used = {}                          # parent path -> {default name: count}, per graph

    def add_arg_scope(fn):
        def wrapper(*a, **kw):
            merged = dict(scope_stack[-1].get(wrapper, {}))
            merged.update(kw)
            return fn(*a, **merged)
        wrapper.__name__ = fn.__name__
        return wrapper

    class ArgScope(object):
        def __init__(self, funcs_or_scope, kw):
            if isinstance(funcs_or_scope, dict):
                cur = {k: dict(v) for k, v in funcs_or_scope.items()}
            else:
                cur = {k: dict(v) for k, v in scope_stack[-1].items()}
                for f in funcs_or_scope:
                    cur.setdefault(f, {}).update(kw)
            self.scope = cur

        def __enter__(self):
            scope_stack.append(self.scope)
            return self.scope

        def __exit__(self, *a):
            scope_stack.pop()
            return False

    class VarScope(object):
        def __init__(self, name_or_scope, default_name=None, values=None, reuse=None):
            if isinstance(name_or_scope, VarScope):
                self.path = list(name_or_scope.path)
            elif name_or_scope is not None:
                self.path = names[-1] + [name_or_scope]
            else:
                key = '/'.join(names[-1])
                cnt = used.setdefault(key, {})
                n = cnt.get(default_name, 0)
                cnt[default_name] = n + 1
                self.path = names[-1] + [default_name if n == 0 else '%s_%d' % (default_name, n)]
            self.name = self.original_name_scope = '/'.join(self.path)

        def __enter__(self):
            names.append(self.path)
            return self

        def __exit__(self, *a):
            names.pop()
            return False

    class NoOp(object):
        def __enter__(self):
            return None

        def __exit__(self, *a):
            return False

    def cur(name):
        return '/'.join(names[-1] + [name])

    def out_hw(h, k, s, padding):
        return -(-h // s) if padding == 'SAME' else (h - k) // s + 1

    def relu(x, name=None):
        return x

    def relu6(x, name=None):
        return x

    def identity(x, name=None):
        return T4(x.shape4, cur(name or 'Identity') + ':0', rec)

    def _finish(net, normalizer_fn, normalizer_params, activation_fn):
        if normalizer_fn is not None:
            net = normalizer_fn(net, **(normalizer_params or {}))
        if activation_fn is not None:
            rec.append(('act', activation_fn.__name__))
            net = activation_fn(net)
        return net

    def _stddev(init):
        return init[1] if isinstance(init, tuple) and init[0] == 'tn' else str(init)

    @add_arg_scope
    def conv2d(inputs, num_outputs, kernel_size, stride=1, padding='SAME', rate=1, activation_fn=relu,
               normalizer_fn=None, normalizer_params=None, weights_initializer=None, weights_regularizer=None,
               biases_initializer=('zeros',), scope=None, **kw):
        assert rate == 1
        n, h, w, c = inputs.shape4
        k = kernel_size if isinstance(kernel_size, int) else kernel_size[0]
        with VarScope(scope, default_name='Conv'):
            rec.append(('conv', '/'.join(names[-1]), int(num_outputs), int(k), int(stride), padding,
                        _stddev(weights_initializer), normalizer_fn is None and biases_initializer is not None))
            net = T4([n, out_hw(h, k, stride, padding), out_hw(w, k, stride, padding), int(num_outputs)], cur('Conv2D'), rec)
            return _finish(net, normalizer_fn, normalizer_params, activation_fn)

    @add_arg_scope
    def separable_conv2d(inputs, num_outputs, kernel_size, depth_multiplier=1, stride=1, rate=1, padding='SAME',
                         activation_fn=relu, normalizer_fn=None, normalizer_params=None, weights_initializer=None,
                         weights_regularizer=None, scope=None, **kw):
        assert num_outputs is None and rate == 1
        n, h, w, c = inputs.shape4
        k = kernel_size if isinstance(kernel_size, int) else kernel_size[0]
        with VarScope(scope, default_name='SeparableConv2d'):
            rec.append(('dwconv', '/'.join(names[-1]), int(k), int(stride), padding, int(depth_multiplier),
                        _stddev(weights_initializer)))
            net = T4([n, out_hw(h, k, stride, padding), out_hw(w, k, stride, padding), c * depth_multiplier],
                     cur('depthwise'), rec)
            return _finish(net, normalizer_fn, normalizer_params, activation_fn)

    @add_arg_scope
    def batch_norm(inputs, decay=0.999, center=True, scale=False, epsilon=0.001, is_training=True, scope=None, **kw):
        with VarScope(scope, default_name='BatchNorm'):
            rec.append(('bn', '/'.join(names[-1]), float(decay), float(epsilon), bool(center), bool(scale),
                        bool(is_training)))
        return inputs

    @add_arg_scope
    def dropout(inputs, keep_prob=0.5, is_training=True, scope=None, **kw):
        rec.append(('dropout', float(keep_prob), bool(is_training)))
        return inputs

    @add_arg_scope
    def fully_connected(*a, **k):
        raise AssertionError('MobileNet-v2 has no fully connected layer')

    def avg_pool(value, ksize, strides, padding, name=None):
        rec.append(('avgpool', int(ksize[1]), int(ksize[2]), padding))
        n, h, w, c = value.shape4
        return T4([n, out_hw(h, ksize[1], strides[1], padding), out_hw(w, ksize[2], strides[2], padding), c],
                  cur('AvgPool'), rec)

    slim = types.SimpleNamespace(
        add_arg_scope=add_arg_scope, arg_scope=lambda f, **kw: ArgScope(f, kw), conv2d=conv2d,
        separable_conv2d=separable_conv2d, batch_norm=batch_norm, dropout=dropout, fully_connected=fully_connected,
        softmax=lambda logits, scope=None: logits, l2_regularizer=lambda wd: ('l2', wd),
        initializers=types.SimpleNamespace(xavier_initializer=lambda: ('xavier',)))
    contrib = types.ModuleType('tensorflow.contrib')
    contrib.slim = slim
    tf.contrib = contrib
    tf.nn = types.SimpleNamespace(relu6=relu6, relu=relu, avg_pool=avg_pool)
    tf.identity = identity
    tf.variable_scope = VarScope
    tf.name_scope = lambda *a, **k: NoOp()
    tf.truncated_normal_initializer = lambda stddev=1.0: ('tn', float(stddev))
    tf.zeros_initializer = lambda: ('zeros',)
    tf.squeeze = lambda x, axis=None, name=None: T4([x.shape4[0], x.shape4[3]], cur('Squeeze'), rec)
    tf.convert_to_tensor = lambda x: x
    tf.shape = lambda x: x.shape4
    tf.GraphKeys = types.SimpleNamespace(UPDATE_OPS='update_ops')
    tf.int32 = 'int32'
    tf.cast = lambda x, dt: x
    tf.train.exponential_decay = lambda lr, step, decay_steps, rate, staircase=False: (
        'exponential_decay', float(lr), int(decay_steps), float(rate), bool(staircase))
    return tf, contrib, slim, used


def record():
    flags, rec = Flags(), []
    tf, contrib, slim, used = build_stub(flags, rec)
    blank = lambda **kw: types.SimpleNamespace(**kw)     # noqa: E731
    stubs = {'tensorflow': tf, 'tensorflow.contrib': contrib, 'tensorflow.contrib.slim': slim}
    cb = load('utils/external/conv_blocks.py', 'ref_conv_blocks', stubs)
    lib = load('utils/external/mobilenet.py', 'ref_mobilenet', stubs)
    ext = types.ModuleType('utils.external')
    ext.conv_blocks, ext.mobilenet = cb, lib
    stubs.update({'utils': types.ModuleType('utils'), 'utils.external': ext, 'utils.external.conv_blocks': cb,
                  'utils.external.mobilenet': lib})
    mv2 = load('utils/external/mobilenet_v2.py', 'ref_mobilenet_v2', stubs)
    ext.mobilenet_v2, ext.mobilenet_v1 = mv2, types.ModuleType('mv1')
    mgw = types.SimpleNamespace(size=lambda: 1, rank=lambda: 0)
    lru = load('utils/lrn_rate_utils.py', 'ref_lrn_rate_utils', stubs)
    stubs.update({'utils.external.mobilenet_v2': mv2, 'utils.external.mobilenet_v1': ext.mobilenet_v1,
                  'nets': types.ModuleType('nets'), 'nets.abstract_model_helper': blank(AbstractModelHelper=object),
                  'datasets': types.ModuleType('datasets'), 'datasets.ilsvrc12_dataset': blank(Ilsvrc12Dataset=object),
                  'utils.lrn_rate_utils': lru, 'utils.multi_gpu_wrapper': blank(MultiGpuWrapper=mgw)})
    net = load('nets/mobilenet_at_ilsvrc12.py', 'ref_mobilenet_at_ilsvrc12', stubs)
    gold = {'source': '/root/reference nets/mobilenet_at_ilsvrc12.py + utils/external/{mobilenet_v2,mobilenet,conv_blocks}.py '
                      'executed under a stub of tensorflow / tf.contrib.slim',
            'flag_defaults': {k: getattr(flags, k) for k in ('mobilenet_version', 'mobilenet_depth_mult', 'nb_epochs_rat',
                                                             'lrn_rate_init', 'batch_size_norm', 'momentum', 'loss_w_dcy')},
            'architecture': [], 'lrn_rate': [], 'maskable_vars': []}
    flags.mobilenet_version, flags.nb_classes = 2, 1001
    for dm in MULTIPLIERS:
        for is_train in (True, False):
            flags.mobilenet_depth_mult = dm
            del rec[:]
            used.clear()                               # every forward_fn call builds a fresh graph
            logits = net.forward_fn(T4([2, 224, 224, 3], 'input:0', rec), is_train)
            gold['architecture'].append(dict(depth_mult=dm, is_train=is_train, logits_shape=list(logits.shape4),
                                             layers=[list(r) for r in rec]))
    # the v2 schedule: the arguments of tf.train.exponential_decay and the iteration count, from the reference's own
    # ModelHelper.setup_lrn_rate
    flags.enbl_multi_gpu, flags.nb_smpls_train = False, 1281167
    for bs, rat in ((96, 1.0), (128, 1.0), (256, 0.5)):
        flags.batch_size, flags.nb_epochs_rat = bs, rat
        lr, nb_iters = net.ModelHelper.setup_lrn_rate(types.SimpleNamespace(), 'global_step')
        _, lr_init, decay_steps, rate, staircase = lr
        gold['lrn_rate'].append(dict(batch_size=bs, nb_epochs_rat=rat, lrn_rate_init=lr_init, decay_steps=decay_steps,
                                     decay_rate=rate, staircase=staircase, nb_iters=int(nb_iters)))
    flags.nb_epochs_rat = 1.0
    # get_maskable_vars on this repo's v2 variable names
    wsu = load('learners/weight_sparsification/utils.py', 'ref_ws_utils', stubs)
    from pocketflow_b200 import graph as G
    from pocketflow_b200.nets import mobilenet_v2 as M2
    for dm in (1.0, 0.35):
        g = G.Graph()
        with g.as_default():
            x = G.placeholder((2, 224, 224, 3), 'x')
            with G.variable_scope('model'):
                M2.mobilenet_v2(x, num_classes=1001, is_training=True, depth_multiplier=dm)
        tv = [types.SimpleNamespace(name=v.name) for v in g.variables.values() if v.trainable]
        gold['maskable_vars'].append(dict(depth_mult=dm, n_trainable=len(tv),
                                          maskable=[v.name for v in wsu.get_maskable_vars(tv)]))
    return gold


if __name__ == '__main__':
    gold = record()
    with open(OUT, 'w') as f:
        json.dump(gold, f, indent=0, sort_keys=True)
        f.write('\n')
    print('wrote', OUT, {k: len(v) for k, v in gold.items() if isinstance(v, list)})
