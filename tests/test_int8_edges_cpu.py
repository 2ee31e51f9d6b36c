"""The shape inventory of the integer inference models: every integer layer of ResNet-20 with `int8_narrow`,
ResNet-50, MobileNet-v1 with `int8_depthwise` and MobileNet-v2 with both, with the kernel it runs on, as
support.INT8_LAYERS pins it.  The kernel tests of tests/test_int8_edges_gpu.py parametrize over those lists, so a layer
shape the graphs gain cannot skip them: this checks the lists against int8.select on the graphs."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from support import INT8_LAYERS, INT8_MODELS, int8_graph  # noqa: E402


def _inventory(key):
    """the integer layers int8.select picks on the model's graph, as INT8_LAYERS entries in graph order"""
    from pocketflow_b200 import compact, int8, ops
    g, _, lg, cfg = int8_graph(key, 1)
    byname = {op.name: op for op in compact.reachable_ops(g, lg)}
    out = {}
    for name, why in int8.select(g, lg, cfg):
        if why is not None:
            continue
        op = byname[name]
        d = int8._conv_desc(op)
        assert d.stride_h == d.stride_w, name
        if op.type == 'Conv2D':
            kernel = 'tma' if ops.conv2d_u8_supported(d) else 'cp.async'
            assert ops.conv2d_u8_narrow_supported(d), name
            kind = 'conv'
        else:
            assert op.type == 'DepthwiseConv2dNative' and ops.dwconv_u8_supported(d), name
            # pf_dwconv_u8_fwd: the row-blocked kernel takes 3 x 3 filters at equal strides with >= 2 output rows
            kernel = 'rows' if d.r == 3 and d.s == 3 and d.stride_h == d.stride_w and d.p >= 2 else 'pixel'
            kind = 'dw'
        s = (kind, d.h, d.w, d.c, d.k, d.r, d.s, d.stride_h, d.pad_t, d.pad_l, d.p, d.q, kernel)
        out[s] = out.get(s, 0) + 1
    return [s + (n,) for s, n in out.items()]


@pytest.mark.parametrize('key', sorted(INT8_MODELS))
def test_int8_layers_are_the_graphs(key):
    assert _inventory(key) == INT8_LAYERS[key]


def test_int8_layer_counts():
    """the integer layer counts the whole-model tests assert: 21 (ResNet-20), 52 of ResNet-50's 53 convolutions (all
    but the stem), 13 depthwise + 12 pointwise (MobileNet-v1), 17 depthwise + 15 projections (MobileNet-v2)"""
    n = {k: sum(s[-1] for s in v) for k, v in INT8_LAYERS.items()}
    assert n == {'resnet20_narrow': 21, 'resnet50': 52, 'mobilenet_v1_depthwise': 25,
                 'mobilenet_v2_depthwise_narrow': 32}
    dw = {k: sum(s[-1] for s in v if s[0] == 'dw') for k, v in INT8_LAYERS.items()}
    assert dw == {'resnet20_narrow': 0, 'resnet50': 0, 'mobilenet_v1_depthwise': 13, 'mobilenet_v2_depthwise_narrow': 17}
