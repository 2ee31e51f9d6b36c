"""Host side of the u8 depthwise layers of the integer inference model (int8.select / IntModel with
cfg['int8_depthwise']): which depthwise layers of MobileNet-v1 and -v2 run on u8 levels and why the others do not, that
the option changes nothing else, the depthwise weight levels against the oracle's fake quantizer, and the sidecar's
versions."""
import importlib
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import pf_oracle as O  # noqa: E402
from pocketflow_b200 import compact, int8, ops  # noqa: E402

NOT_Q = 'weights not quantized (first / last layer)'
NOT_RELU = 'input is not a quantized batch norm + ReLU output'


def _graph(net, qall, **flags):
    from pocketflow_b200.flags import FLAGS
    mod = importlib.import_module('pocketflow_b200.nets.' + net)
    import pocketflow_b200.learners.uniform_quantization.learner  # noqa: F401
    FLAGS.reset()
    for k, v in flags.items():
        setattr(FLAGS, k, v)
    FLAGS.uql_weight_bits, FLAGS.uql_activation_bits = 8, 8
    FLAGS.uql_use_buckets, FLAGS.uql_bucket_type = True, 'channel'
    FLAGS.uql_quantize_all_layers = qall
    g, images, lg = compact.build_eval_graph(mod.ModelHelper(), 8)
    return g, images, lg, int8.config_from_flags()


def _short(sel):
    return [(n.split('/')[-2], w) for n, w in sel]


@pytest.mark.parametrize('qall', [False, True])
def test_select_mobilenet_v1_depthwise(qall):
    """every Conv2d_i_depthwise reads a batch norm + ReLU6 output of 32 .. 1024 channels (powers of two) with one
    consumer, and is a 3 x 3 layer of stride 1 or 2: all 13 run on u8 levels.  The rest is test_int8_cpu's selection."""
    g, _, lg, cfg = _graph('mobilenet_at_ilsvrc12', qall)
    want = [('Conv2d_0', NOT_RELU if qall else NOT_Q)]
    for i in range(1, 14):
        want.append(('Conv2d_%d_depthwise' % i, None))
        want.append(('Conv2d_%d_pointwise' % i, 'shape 32 -> 64 channels (the u8 kernel needs multiples of 64)'
                     if i == 1 else None))
    want.append(('Conv2d_1c_1x1', NOT_RELU if qall else NOT_Q))
    sel = int8.select(g, lg, dict(cfg, int8_depthwise=True))
    assert _short(sel) == want
    # the graph agrees: each depthwise input is a Relu6 of a FusedBatchNorm with power-of-two channels >= 16
    byname = {op.name: op for op in compact.reachable_ops(g, lg)}
    for name, why in sel:
        op = byname[name]
        if op.type == 'DepthwiseConv2dNative':
            x = op.inputs[0]
            assert x.op.type == 'Relu6' and x.op.inputs[0].op.type == 'FusedBatchNorm'
            c = x.shape[-1]
            assert c >= 16 and not c & (c - 1) and tuple(op.attrs['ksize']) == (3, 3)
    lines = int8.report_lines(sel)
    assert lines[-1] == '25 of 28 layers run as integers'
    assert sum('u8 depthwise (CUDA cores)' in ln for ln in lines) == 13


def _v2_reason(c):
    return 'input channels %d: the level producer needs a power of two >= 16' % c


def test_select_mobilenet_v2_depthwise():
    """MobileNet-v2's expanded depthwise inputs have 96 .. 960 channels, not powers of two, so the level producer
    cannot write them; only the first block's depthwise layer (the stem's 32 channels) runs on u8 levels"""
    g, _, lg, cfg = _graph('mobilenet_at_ilsvrc12', False, mobilenet_version=2)
    base = int8.select(g, lg, cfg)
    sel = int8.select(g, lg, dict(cfg, int8_depthwise=True))
    byname = {op.name: op for op in compact.reachable_ops(g, lg)}
    chans = [32, 96, 144, 144, 192, 192, 192, 384, 384, 384, 384, 576, 576, 576, 960, 960, 960]
    dws = [(n, w) for n, w in sel if byname[n].type == 'DepthwiseConv2dNative']
    assert [n.split('/')[-3] for n, _ in dws] == ['expanded_conv'] + ['expanded_conv_%d' % i for i in range(1, 17)]
    assert [w for _, w in dws] == [None] + [_v2_reason(c) for c in chans[1:]]
    assert [byname[n].inputs[0].shape[-1] for n, _ in dws] == chans
    # every other layer as without the option
    assert [e for e in sel if byname[e[0]].type != 'DepthwiseConv2dNative'] == \
        [e for e in base if byname[e[0]].type != 'DepthwiseConv2dNative']


@pytest.mark.parametrize('net,flags', [('resnet_at_cifar10', dict(resnet_size=20)),
                                       ('resnet_at_ilsvrc12', dict(resnet_size=50)),
                                       ('mobilenet_at_ilsvrc12', dict())], ids=['rn20', 'rn50', 'mbv1'])
@pytest.mark.parametrize('qall', [False, True])
def test_select_without_the_option_is_unchanged(net, flags, qall):
    g, _, lg, cfg = _graph(net, qall, **flags)
    assert 'int8_depthwise' not in cfg                     # config_from_flags does not set it
    base = int8.select(g, lg, cfg)
    assert int8.select(g, lg, dict(cfg, int8_depthwise=False)) == base
    byname = {op.name: op for op in compact.reachable_ops(g, lg)}
    on = int8.select(g, lg, dict(cfg, int8_depthwise=True))
    for (n, w), (n2, w2) in zip(base, on):
        assert n == n2 and (w == w2 or byname[n].type == 'DepthwiseConv2dNative')
    for n, w in base:
        if byname[n].type == 'DepthwiseConv2dNative':
            assert w == 'depthwise convolution' or w == NOT_Q


def test_select_depthwise_refusals():
    """the conditions of a Conv2D apply to a depthwise layer too: bucket type, weight and activation bits"""
    g, _, lg, cfg = _graph('mobilenet_at_ilsvrc12', False)
    cfg = dict(cfg, int8_depthwise=True)
    byname = {op.name: op for op in compact.reachable_ops(g, lg)}
    for change, why in ((dict(bucket_type='split'), 'split buckets'), (dict(weight_bits=16), 'weight bits 16 > 8'),
                        (dict(activation_bits=32), 'activation bits 32 > 8')):
        sel = int8.select(g, lg, dict(cfg, **change))
        assert [w for n, w in sel if byname[n].type == 'DepthwiseConv2dNative'] == [why] * 13


def test_depthwise_kernel_support():
    """pf_dwconv_u8_supported: depth multiplier 1, C % 16 == 0, <= 9 taps, strides 1 or 2"""
    ok = ops.conv_desc(256, 112, 112, 32, 32, 3, 3, 112, 112, 1, 1, 1, 1)
    assert ops.dwconv_u8_supported(ok)
    assert ops.dwconv_u8_supported(ops.conv_desc(256, 14, 14, 1024, 1024, 3, 3, 7, 7, 2, 2, 0, 0))
    assert ops.dwconv_u8_supported(ops.conv_desc(8, 20, 20, 48, 48, 1, 9, 20, 20, 1, 1, 0, 4))
    for bad in (ops.conv_desc(8, 14, 14, 40, 40, 3, 3, 14, 14, 1, 1, 1, 1),       # C % 16
                ops.conv_desc(8, 14, 14, 32, 64, 3, 3, 14, 14, 1, 1, 1, 1),       # depth multiplier 2
                ops.conv_desc(8, 14, 14, 32, 32, 5, 5, 14, 14, 1, 1, 2, 2),       # 25 taps
                ops.conv_desc(8, 14, 14, 32, 32, 3, 3, 5, 5, 3, 3, 1, 1)):        # stride 3
        assert not ops.dwconv_u8_supported(bad)


@pytest.mark.parametrize('bits', [2, 4, 8])
@pytest.mark.parametrize('per_channel', [False, True])
@pytest.mark.parametrize('c', [32, 1024])
def test_depthwise_levels_reproduce_fake_quant(c, per_channel, bits):
    """a [3, 3, C, 1] kernel: alpha * (q / k) + beta from the levels equals uniform_quantize's weight bit for bit;
    with channel buckets the kernel's one output channel is one bucket (uq_bucket_layout)"""
    shape = (3, 3, c, 1)
    assert ops.uq_bucket_layout(shape, True, 'channel', 0)[0] == 1
    rng = np.random.default_rng(c + bits * 7 + per_channel)
    w = (rng.standard_normal(shape) * rng.uniform(0.01, 0.5)).astype(np.float32)
    lv, alpha, beta = int8.weight_levels(w, bits, per_channel)
    assert lv.dtype == np.uint8 and lv.shape == shape and int(lv.max()) <= 2 ** bits - 1
    assert alpha.shape == beta.shape == (1,)
    ref, ra, rb = O.uniform_quantize(w, bits, use_buckets=per_channel, bucket_type='channel', return_scales=True)
    assert np.array_equal(alpha, np.atleast_1d(ra)) and np.array_equal(beta, np.atleast_1d(rb))
    got = int8.dequantize(lv, alpha, beta, bits)
    assert got.dtype == np.float32 and np.array_equal(got.view(np.uint32), ref.view(np.uint32))


class _Probe(int8.IntModel):
    """IntModel without the executor: what load() hands the constructor, and what export() writes"""

    def __init__(self, graph, images, logits, cfg, state, wlevels, device=None):
        self.graph, self.images, self.logits, self.cfg = graph, images, logits, dict(cfg)
        self.sel = int8.select(graph, logits, cfg)
        self.state, self.wlevels = dict(state), wlevels


def _probe(g, images, lg, cfg):
    byname = {op.name: op for op in compact.reachable_ops(g, lg)}
    wl = {}
    for n, why in int8.select(g, lg, cfg):
        if why is None:
            shape = byname[n].vars['kernel'].shape
            wl[n] = (np.zeros(shape, np.uint8), np.ones(1, np.float32), np.zeros(1, np.float32))
    return _Probe(g, images, lg, cfg, {'other/var': np.ones(3, np.float32)}, wl)


def test_sidecar_versions(tmp_path):
    g, images, lg, cfg = _graph('mobilenet_at_ilsvrc12', False)
    # without the option: version 1 and the same config keys as before
    old = str(tmp_path / 'old')
    _probe(g, images, lg, cfg).export(old)
    rec = json.load(open(old + '.int8.json'))
    assert rec['version'] == 1 and 'int8_depthwise' not in rec['config']
    p = _Probe.load(g, images, lg, old)
    assert p.cfg == cfg and not any('depthwise' in n for n in p.wlevels) and len(p.wlevels) == 12
    # with depthwise integer layers: version 2, the option recorded, and loaded back with it
    new = str(tmp_path / 'new')
    _probe(g, images, lg, dict(cfg, int8_depthwise=True)).export(new)
    rec = json.load(open(new + '.int8.json'))
    assert rec['version'] == int8.SIDECAR_VERSION == 2 and rec['config']['int8_depthwise'] is True
    p = _Probe.load(g, images, lg, new)
    assert p.cfg == dict(cfg, int8_depthwise=True) and len(p.wlevels) == 25
    assert sum(n.endswith('/depthwise') for n in p.wlevels) == 13
    # any other version is refused with a message
    for v in (0, 3, None):
        rec['version'] = v
        with open(new + '.int8.json', 'w') as f:
            json.dump(rec, f)
        with pytest.raises(ValueError, match='unsupported sidecar version'):
            _Probe.load(g, images, lg, new)
