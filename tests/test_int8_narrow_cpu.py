"""Host side of the narrow and non-power-of-two integer layers (int8.select / IntModel with cfg['int8_narrow']): which
layers of ResNet-20 and MobileNet-v2 run on u8 levels and why the others do not, that the option changes nothing
without it, the wider shape query of pf_conv2d_u8_fwd, and the sidecar round trip with the option."""
import importlib
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

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


@pytest.mark.parametrize('qall', [False, True])
def test_select_resnet20_narrow(qall):
    """every inner convolution of ResNet-20 (16, 32 and 64 channels, the strided 1x1 projections included) reads a
    quantized batch norm + ReLU output: with the option all 21 run on u8 levels"""
    g, _, lg, cfg = _graph('resnet_at_cifar10', qall, resnet_size=20)
    sel = int8.select(g, lg, dict(cfg, int8_narrow=True))
    want = [('conv2d', NOT_RELU if qall else NOT_Q)] + [('conv2d_%d' % i, None) for i in range(1, 22)]
    want += [('dense', 'dense layer' if qall else NOT_Q)]
    assert [(n.split('/')[-2], w) for n, w in sel] == want
    assert int8.report_lines(sel)[-1] == '21 of 23 layers run as integers'
    # the 16- and 32-channel layers are the ones the TMA-fed kernel does not take
    byname = {op.name: op for op in compact.reachable_ops(g, lg)}
    narrow = [n for n, w in sel if w is None and not ops.conv2d_u8_supported(int8._conv_desc(byname[n]))]
    assert len(narrow) == 16


def _v2(cfg_extra):
    g, _, lg, cfg = _graph('mobilenet_at_ilsvrc12', False, mobilenet_version=2)
    byname = {op.name: op for op in compact.reachable_ops(g, lg)}
    return g, lg, cfg, byname, int8.select(g, lg, dict(cfg, **cfg_extra))


def test_select_mobilenet_v2_narrow():
    """with both options: all 17 depthwise layers (32 .. 960 channels) and every projection whose Cout % 16 == 0; the
    96 -> 24 and 144 -> 24 projections name their channel counts; the expansion convolutions and Conv_1 read a linear
    bottleneck (no ReLU), the stem and the logits are not quantized"""
    g, lg, cfg, byname, sel = _v2(dict(int8_depthwise=True, int8_narrow=True))
    kinds = {}
    for n, w in sel:
        kinds.setdefault(n.split('/')[-2] if byname[n].type == 'Conv2D' else 'depthwise', []).append(w)
    assert kinds['depthwise'] == [None] * 17
    shape = 'shape %d -> 24 channels (the u8 kernels need multiples of 16)'
    assert kinds['project'] == [None, shape % 96, shape % 144] + [None] * 14
    assert kinds['expand'] == [NOT_RELU] * 16
    assert kinds['Conv'] == [NOT_Q] and kinds['Conv_1'] == [NOT_RELU] and kinds['Conv2d_1c_1x1'] == [NOT_Q]
    assert int8.report_lines(sel)[-1] == '32 of 53 layers run as integers'
    for n, w in sel:
        op = byname[n]
        if w is None and op.type == 'Conv2D':
            assert ops.conv2d_u8_narrow_supported(int8._conv_desc(op))
            assert op.inputs[0].shape[-1] % 16 == 0 and op.output.shape[-1] % 16 == 0


def test_select_mobilenet_v2_narrow_without_depthwise():
    """int8_narrow alone: the projections as above, every depthwise layer keeps fake-quant"""
    _, _, _, byname, both = _v2(dict(int8_depthwise=True, int8_narrow=True))
    _, _, _, _, sel = _v2(dict(int8_narrow=True))
    for (n, w), (n2, w2) in zip(sel, both):
        assert n == n2
        assert w == (w2 if byname[n].type == 'Conv2D' else 'depthwise convolution')


@pytest.mark.parametrize('net,flags', [('resnet_at_cifar10', dict(resnet_size=20)),
                                       ('mobilenet_at_ilsvrc12', dict(mobilenet_version=2)),
                                       ('resnet_at_ilsvrc12', dict(resnet_size=50)),
                                       ('mobilenet_at_ilsvrc12', dict())], ids=['rn20', 'mbv2', 'rn50', 'mbv1'])
def test_select_without_the_option_is_unchanged(net, flags):
    """int8_narrow False or absent selects what the parent selected, and the option only adds layers; on ResNet-50,
    whose layers all have the channel counts of the TMA-fed kernel, nothing, on MobileNet-v1 its 32 -> 64 pointwise"""
    g, _, lg, cfg = _graph(net, False, **flags)
    assert 'int8_narrow' not in cfg
    for extra in (dict(), dict(int8_depthwise=True)):
        base = int8.select(g, lg, dict(cfg, **extra))
        assert int8.select(g, lg, dict(cfg, int8_narrow=False, **extra)) == base
        on = int8.select(g, lg, dict(cfg, int8_narrow=True, **extra))
        assert [n for n, _ in on] == [n for n, _ in base]
        for (n, w), (_, w2) in zip(base, on):
            if w is None:
                assert w2 is None, n
        added = [n.split('/')[-2] for (n, w), (_, w2) in zip(base, on) if w is not None and w2 is None]
        if net == 'resnet_at_ilsvrc12':
            assert added == []
        elif net == 'mobilenet_at_ilsvrc12' and not flags:
            assert added == ['Conv2d_1_pointwise']


def test_narrow_support_query():
    """pf_conv2d_u8_narrow_supported: every shape pf_conv2d_u8_supported takes, plus Cin and Cout multiples of 16 with
    R*S*Cin <= 32768; pf_conv2d_u8_supported keeps its answer"""
    d = ops.conv_desc
    tma = [d(128, 56, 56, 64, 64, 3, 3, 56, 56, 1, 1, 1, 1), d(128, 7, 7, 2048, 512, 1, 1, 7, 7, 1, 1, 0, 0)]
    narrow = [d(128, 32, 32, 16, 16, 3, 3, 32, 32, 1, 1, 1, 1), d(128, 32, 32, 16, 32, 1, 1, 16, 16, 2, 2, 0, 0),
              d(128, 16, 16, 32, 64, 3, 3, 8, 8, 2, 2, 0, 0), d(8, 14, 14, 576, 160, 1, 1, 14, 14, 1, 1, 0, 0),
              d(8, 7, 7, 960, 160, 1, 1, 7, 7, 1, 1, 0, 0), d(8, 112, 112, 32, 16, 1, 1, 112, 112, 1, 1, 0, 0),
              d(8, 20, 20, 16, 48, 5, 7, 20, 20, 1, 1, 2, 3), d(8, 9, 9, 2048, 16, 4, 4, 9, 9, 1, 1, 1, 1)]
    bad = [d(8, 56, 56, 96, 24, 1, 1, 56, 56, 1, 1, 0, 0),      # Cout % 16
           d(8, 32, 32, 3, 16, 3, 3, 32, 32, 1, 1, 1, 1),       # Cin % 16
           d(8, 32, 32, 24, 32, 1, 1, 32, 32, 1, 1, 0, 0),      # Cin % 16
           d(8, 9, 9, 2064, 16, 4, 4, 9, 9, 1, 1, 1, 1)]        # R*S*Cin = 33024 > 32768
    for x in tma:
        assert ops.conv2d_u8_supported(x) and ops.conv2d_u8_narrow_supported(x)
    for x in narrow:
        assert not ops.conv2d_u8_supported(x) and ops.conv2d_u8_narrow_supported(x), (x.c, x.k)
    for x in bad:
        assert not ops.conv2d_u8_supported(x) and not ops.conv2d_u8_narrow_supported(x), (x.c, x.k)


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


def test_sidecar_round_trip_narrow(tmp_path):
    """the option is recorded in the config and read back; the version stays 1 without depthwise integer layers and 2
    with them; a loader that drops the option selects fewer layers and refuses the file with the coverage error"""
    g, images, lg, cfg = _graph('resnet_at_cifar10', False, resnet_size=20)
    path = str(tmp_path / 'rn20')
    _probe(g, images, lg, dict(cfg, int8_narrow=True)).export(path)
    rec = json.load(open(path + '.int8.json'))
    assert rec['version'] == 1 and rec['config']['int8_narrow'] is True
    p = _Probe.load(g, images, lg, path)
    assert p.cfg == dict(cfg, int8_narrow=True) and len(p.wlevels) == 21
    # what a loader that does not know the option rebuilds: the selection without it, which int8.IntModel checks the
    # levels against before it builds anything
    sel_old = int8.select(g, lg, cfg)
    assert sorted(n for n, w in sel_old if w is None) != sorted(p.wlevels)
    with pytest.raises(ValueError, match='do not cover the integer layers'):
        int8.IntModel(g, images, lg, cfg, p.state, p.wlevels)

    g2, images2, lg2, cfg2 = _graph('mobilenet_at_ilsvrc12', False, mobilenet_version=2)
    path2 = str(tmp_path / 'mbv2')
    both = dict(cfg2, int8_depthwise=True, int8_narrow=True)
    _probe(g2, images2, lg2, both).export(path2)
    rec = json.load(open(path2 + '.int8.json'))
    assert rec['version'] == int8.SIDECAR_VERSION == 2
    assert rec['config']['int8_narrow'] is True and rec['config']['int8_depthwise'] is True
    p = _Probe.load(g2, images2, lg2, path2)
    assert p.cfg == both and len(p.wlevels) == 32
