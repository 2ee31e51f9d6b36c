"""Host side of the integer inference path (pocketflow_b200/int8.py): the export's weight levels and scales against the
oracle's fake quantizer, and which layers of ResNet-20, ResNet-50 and MobileNet-v1 run on the u8 kernel."""
import importlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import pf_oracle as O  # noqa: E402
from pocketflow_b200 import compact, int8  # noqa: E402


@pytest.mark.parametrize('bits', [2, 4, 8])
@pytest.mark.parametrize('per_channel', [False, True])
@pytest.mark.parametrize('shape', [(3, 3, 64, 64), (1, 1, 256, 1024), (3, 3, 128, 128)])
def test_levels_reproduce_fake_quant(shape, per_channel, bits):
    """alpha * (q / k) + beta in fp32 from the exported levels equals uniform_quantize's weight bit for bit"""
    rng = np.random.default_rng(bits * 7 + per_channel)
    w = (rng.standard_normal(shape) * rng.uniform(0.01, 0.5)).astype(np.float32)
    lv, alpha, beta = int8.weight_levels(w, bits, per_channel)
    assert lv.dtype == np.uint8 and lv.shape == w.shape and int(lv.max()) <= 2 ** bits - 1
    ref, ra, rb = O.uniform_quantize(w, bits, use_buckets=per_channel, bucket_type='channel', return_scales=True)
    assert np.array_equal(alpha, np.atleast_1d(ra)) and np.array_equal(beta, np.atleast_1d(rb))
    got = int8.dequantize(lv, alpha, beta, bits)
    assert got.dtype == np.float32 and np.array_equal(got.view(np.uint32), ref.view(np.uint32))


def _select(net, qall, **flags):
    from pocketflow_b200.flags import FLAGS
    mod = importlib.import_module('pocketflow_b200.nets.' + net)
    import pocketflow_b200.learners.uniform_quantization.learner  # noqa: F401
    FLAGS.reset()
    for k, v in flags.items():
        setattr(FLAGS, k, v)
    FLAGS.uql_weight_bits, FLAGS.uql_activation_bits = 8, 8
    FLAGS.uql_use_buckets, FLAGS.uql_bucket_type = True, 'channel'
    FLAGS.uql_quantize_all_layers = qall
    g, _, lg = compact.build_eval_graph(mod.ModelHelper(), 8)
    return [(n.split('/')[-2], w) for n, w in int8.select(g, lg, int8.config_from_flags())]


NOT_Q = 'weights not quantized (first / last layer)'
NOT_RELU = 'input is not a quantized batch norm + ReLU output'


def _shape(c, k):
    return 'shape %d -> %d channels (the u8 kernel needs multiples of 64)' % (c, k)


@pytest.mark.parametrize('qall', [False, True])
def test_select_resnet20(qall):
    # ResNet-20 v2: stem 3 -> 16, stages of 16, 32 and 64 channels (3 blocks of two 3x3 convs, a 1x1 projection at the
    # first block of stages 2 and 3); only the 64 -> 64 convolutions have channel counts the u8 kernel takes
    chans = [(16, 16)] * 7 + [(16, 32)] * 2 + [(32, 32)] * 5 + [(32, 64)] * 2 + [(64, 64)] * 5
    want = [('conv2d', NOT_RELU if qall else NOT_Q)]
    want += [('conv2d_%d' % i, None if c == 64 else _shape(c, k)) for i, (c, k) in enumerate(chans, 1)]
    want += [('dense', 'dense layer' if qall else NOT_Q)]
    assert _select('resnet_at_cifar10', qall, resnet_size=20) == want


@pytest.mark.parametrize('qall', [False, True])
def test_select_resnet50(qall):
    # every bottleneck convolution of ResNet-50 v2 reads a batch norm + ReLU output and has Cin, Cout % 64 == 0
    want = [('conv2d', NOT_RELU if qall else NOT_Q)] + [('conv2d_%d' % i, None) for i in range(1, 53)]
    want += [('dense', 'dense layer' if qall else NOT_Q)]
    assert _select('resnet_at_ilsvrc12', qall, resnet_size=50) == want


@pytest.mark.parametrize('qall', [False, True])
def test_select_mobilenet_v1(qall):
    # the depthwise halves stay; the first pointwise layer has 32 input channels; the logits read the pooled features
    want = [('Conv2d_0', NOT_RELU if qall else NOT_Q)]
    for i in range(1, 14):
        want.append(('Conv2d_%d_depthwise' % i, 'depthwise convolution'))
        want.append(('Conv2d_%d_pointwise' % i, _shape(32, 64) if i == 1 else None))
    want.append(('Conv2d_1c_1x1', NOT_RELU if qall else NOT_Q))
    assert _select('mobilenet_at_ilsvrc12', qall) == want


def test_select_refuses_split_buckets_and_wide_bits():
    from pocketflow_b200.flags import FLAGS
    mod = importlib.import_module('pocketflow_b200.nets.resnet_at_ilsvrc12')
    import pocketflow_b200.learners.uniform_quantization.learner  # noqa: F401
    FLAGS.reset()
    FLAGS.resnet_size = 50
    g, _, lg = compact.build_eval_graph(mod.ModelHelper(), 2)
    base = dict(weight_bits=8, activation_bits=8, quantize_all_layers=False, use_buckets=True, bucket_type='channel',
                bucket_size=256)
    for change, why in ((dict(bucket_type='split'), 'split buckets'), (dict(weight_bits=16), 'weight bits 16 > 8'),
                        (dict(activation_bits=32), 'activation bits 32 > 8')):
        sel = int8.select(g, lg, dict(base, **change))
        assert [w for _, w in sel[1:-1]] == [why] * 52
    lines = int8.report_lines(int8.select(g, lg, base))
    assert lines[-1] == '52 of 54 layers run as integers'
