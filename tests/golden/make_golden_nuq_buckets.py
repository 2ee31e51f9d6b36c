"""Golden values of the BUCKETED codebook quantizer, produced by the reference's own code: NonUniformQuantization.
__bucket_quantize (learners/nonuniform_quantization/utils.py:196-243) with __split_bucket / __channel_bucket, __scale,
__quantile_init, __build_bucket_norm_quant_point, __inv_scale and __updt_bucket_storage, executed from /root/reference
on numpy-backed stub tensors (TensorFlow 1.x cannot be imported here), in the stub style of make_golden_from_reference.py.

  python tests/golden/make_golden_nuq_buckets.py        ->  tests/golden/ref_executed_nuq_buckets_v1.json

Every stub op maps one-to-one onto the numpy float32 op (each individually rounded).  tf.contrib.distributions.percentile
is not available: the stub calls the oracle's percentile_nearest (axis=0), as the existing generators do.  The codebook
is captured where the reference creates its `clusters` variable, the centroid indices where it takes the argmin.
The reference's bucketed 'uniform' init is recorded as the error it raises."""
import builtins
import hashlib
import importlib.util
import json
import os
import sys
import types

import numpy as np

REF = '/root/reference'
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, 'ref_executed_nuq_buckets_v1.json')
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import pf_oracle as ORC  # noqa: E402

# (shape, bucket_type, bucket_size): split with numel % size != 0, == 0 and numel < size; channel on conv, dense and
# depthwise kernels
LAYOUTS = [((3, 3, 8, 16), 'split', 100), ((3, 3, 8, 16), 'split', 64), ((1, 1, 8, 5), 'split', 64),
           ((5, 5, 3, 7), 'split', 256), ((3, 3, 8, 16), 'channel', 0), ((64, 10), 'channel', 0),
           ((3, 3, 12, 1), 'channel', 0), ((1, 1, 30, 6), 'channel', 0)]
BITS = (1, 2, 4, 8)


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


class Dim(object):
    def __init__(self, v):
        self.value = int(v)


class Shape(list):
    pass


class T(object):
    def __init__(self, a):
        self.a = np.asarray(a, dtype=np.float32)

    def get_shape(self):
        return Shape(Dim(d) for d in self.a.shape)

    @property
    def shape(self):
        return tuple(self.a.shape)

    def __getitem__(self, i):
        return T(self.a[i])

    @staticmethod
    def _v(o):
        return o.a if isinstance(o, T) else np.float32(o)

    def __add__(self, o):
        return T(self.a + T._v(o))

    def __radd__(self, o):
        return T(T._v(o) + self.a)

    def __sub__(self, o):
        return T(self.a - T._v(o))

    def __rsub__(self, o):
        return T(T._v(o) - self.a)

    def __mul__(self, o):
        return T(self.a * T._v(o))

    def __rmul__(self, o):
        return T(T._v(o) * self.a)

    def __truediv__(self, o):
        return T(self.a / T._v(o))


class Ctx(object):
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


def make_tf(record):
    tf = types.ModuleType('tensorflow')
    tf.int64, tf.int32, tf.float32 = 'int64', 'int32', 'float32'
    tf.variable_scope = lambda *a, **k: Ctx()
    tf.get_variable_scope = lambda: types.SimpleNamespace(name='scope')
    tf.reduce_max = lambda w, axis=None: T(np.max(w.a, axis=axis))
    tf.reduce_min = lambda w, axis=None: T(np.min(w.a, axis=axis))
    tf.stop_gradient = lambda x: x
    tf.constant = lambda value=0, dtype=None: T(value) if dtype == 'float32' else int(value)
    tf.cast = lambda x, dtype=None: int(x) if dtype == 'int64' else (x if isinstance(x, T) else T(np.float32(x)))
    tf.reshape = lambda t, shape: T(t.a.reshape([d.value if isinstance(d, Dim) else int(d) for d in shape]))
    tf.ones = lambda n, dtype=None: [1] * int(n) if dtype == 'int64' else T(np.ones(int(n), np.float32))
    tf.concat = lambda ts, axis=0: ([int(v) for part in ts for v in part] if isinstance(ts[0], list)
                                    else T(np.concatenate([t.a for t in ts], axis=axis)))
    tf.range = lambda n: list(range(int(n)))
    tf.map_fn = lambda fn, elems, dtype=None: T(np.stack([np.asarray(T._v(fn(e)), np.float32) for e in elems]))
    tf.expand_dims = lambda x, axis: T(np.expand_dims(x.a, axis))
    tf.tile = lambda x, reps: T(np.tile(x.a, np.asarray(reps, np.int64)))
    tf.transpose = lambda x, perm=None: T(np.transpose(x.a, perm))
    tf.abs = lambda x: T(np.abs(x.a))
    tf.sign = lambda x: T(np.sign(x.a))
    tf.gather = lambda c, idx: T(c.a[idx])
    tf.linspace = lambda start, stop, num: T(np.linspace(start, stop, num))

    def argmin(x, axis=-1):
        record['idx'] = np.argmin(x.a, axis=axis)
        return record['idx']

    def get_variable(name, validate_shape=True, initializer=None, trainable=True):
        record['clusters'] = np.array(initializer.a, np.float32)
        return T(record['clusters'])
    tf.argmin = argmin
    tf.get_variable = get_variable
    contrib = types.SimpleNamespace(
        distributions=types.SimpleNamespace(
            percentile=lambda x, q, axis=None: T(ORC.percentile_nearest(x.a, float(q), axis=axis))),
        graph_editor=types.ModuleType('ge'))
    tf.contrib = contrib
    return tf


def load(tf):
    stubs = {'tensorflow': tf, 'tensorflow.contrib': tf.contrib, 'tensorflow.contrib.graph_editor': tf.contrib.graph_editor}
    saved = {k: sys.modules.get(k) for k in stubs}
    sys.modules.update(stubs)
    try:
        spec = importlib.util.spec_from_file_location('ref_nuq_bucket_utils',
                                                      os.path.join(REF, 'learners/nonuniform_quantization/utils.py'))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        return mod
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def main():
    record = {}
    tf = make_tf(record)
    mod = load(tf)
    cls = mod.NonUniformQuantization
    quant = getattr(cls, '_NonUniformQuantization__bucket_quantize')
    sess = types.SimpleNamespace(graph=types.SimpleNamespace(gradient_override_map=lambda m: Ctx()))
    gold = {'source': 'NonUniformQuantization.__bucket_quantize of /root/reference executed under a stub tensorflow '
                      'module (percentile = oracle.pf_oracle.percentile_nearest)',
            'cases': [], 'bucket_storage': [], 'uniform_init': []}
    _print = builtins.print
    builtins.print = lambda *a, **k: None                      # the reference prints "Quantized: ..." per call
    try:
        ci = 0
        for shape, btype, bsize in LAYOUTS:
            for bits in BITS:
                rng = np.random.default_rng(6000 + ci)
                x = (rng.standard_normal(shape) * rng.choice([1e-2, 1.0, 9.0])).astype(np.float32)
                if ci % 9 == 4:
                    x.reshape(-1)[: x.size // 3] = x.reshape(-1)[0]     # runs of equal weights: argmin ties
                if ci % 11 == 7:
                    x[...] = x.reshape(-1)[0]                             # constant tensor: alpha = 1e-10
                obj = cls(sess, bsize, True, 'quantile', btype)
                record.clear()
                q = quant(obj, T(x), bits, 'weight', 'p')
                out = np.ascontiguousarray(q.a, np.float32)
                assert out.shape == tuple(shape)
                idx = np.asarray(record['idx']).reshape(-1)[:x.size].astype(np.int64)
                gold['cases'].append(dict(seed=6000 + ci, shape=list(shape), bucket_type=btype, bucket_size=bsize,
                                          bits=bits, tie_runs=(ci % 9 == 4), constant=(ci % 11 == 7),
                                          clusters_shape=list(record['clusters'].shape),
                                          qx=sha(out), clusters=sha(record['clusters']), idx=sha(idx),
                                          bucket_storage=int(obj.bucket_storage), first=[float(v) for v in out.reshape(-1)[:3]]))
                ci += 1
        # bucket storage over a list of kernels quantized by one NonUniformQuantization (sum of nb * 64)
        for btype, bsize in (('split', 256), ('split', 100), ('channel', 0)):
            obj = cls(sess, bsize, True, 'quantile', btype)
            shapes = [(3, 3, 16, 16), (1, 1, 16, 32), (3, 3, 32, 1), (32, 10)]
            for s in shapes:
                quant(obj, T(np.random.default_rng(7000).standard_normal(s).astype(np.float32)), 2, 'weight', 'p')
            gold['bucket_storage'].append(dict(bucket_type=btype, bucket_size=bsize, shapes=[list(s) for s in shapes],
                                               bits=int(obj.bucket_storage)))
        # --nuql_init_style uniform with buckets: __uniform_init(x_normalized, k) against (nb_clusters, bucket_num)
        for btype, bsize in (('split', 64), ('channel', 0)):
            obj = cls(sess, bsize, True, 'uniform', btype)
            try:
                quant(obj, T(np.ones((3, 3, 4, 8), np.float32)), 2, 'weight', 'p')
                err = None
            except Exception as e:  # noqa: BLE001  (what the reference raises is the record)
                err = type(e).__name__
            gold['uniform_init'].append(dict(bucket_type=btype, bucket_size=bsize, raises=err))
    finally:
        builtins.print = _print
    with open(OUT, 'w') as f:
        json.dump(gold, f, indent=1, sort_keys=True)
        f.write('\n')
    print('wrote', OUT, len(gold['cases']), 'cases')


if __name__ == '__main__':
    main()
