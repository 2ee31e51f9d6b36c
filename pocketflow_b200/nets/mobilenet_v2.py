"""MobileNet-v2 graph builder — the slim model the reference vendors (/root/reference/utils/external/mobilenet_v2.py:42-160,
mobilenet.py:62-106, 149-296, 305-470, conv_blocks.py:158-314), re-expressed on pocketflow_b200.graph with slim's
variable names (MobilenetV2/Conv/weights, MobilenetV2/expanded_conv_3/expand/BatchNorm/gamma,
.../depthwise/depthwise_weights, .../project/weights, MobilenetV2/Logits/Conv2d_1c_1x1/{weights,biases}), so the
reference's name filters and a TF-slim v2 checkpoint work unchanged.

Each expanded_conv block is expand 1x1 (BN + ReLU6; only when the expanded width exceeds the input width) ->
depthwise 3x3 (BN + ReLU6) -> project 1x1 (BN, no activation: the linear bottleneck) -> + input when the stride is 1
and the widths match.  The head is a global average pool, dropout (keep 0.8 in training) and a 1x1 conv with biases."""
from collections import namedtuple

from .. import graph as G

Conv = namedtuple('Conv', ['kernel', 'stride', 'depth'])
ExpandedConv = namedtuple('ExpandedConv', ['stride', 'depth', 'expansion', 'divisible_by'])

# V2_DEF['spec'] (mobilenet_v2.py:58-80): the first block expands by 1 (divisible_by 1), every other one by 6
V2_CONV_DEFS = [Conv(kernel=3, stride=2, depth=32), ExpandedConv(1, 16, 1, 1)] + \
    [ExpandedConv(s, d, 6, 8) for s, d in [(2, 24), (1, 24), (2, 32), (1, 32), (1, 32), (2, 64), (1, 64), (1, 64),
                                           (1, 64), (1, 96), (1, 96), (1, 96), (2, 160), (1, 160), (1, 160), (1, 320)]] + \
    [Conv(kernel=1, stride=1, depth=1280)]

BATCH_NORM_DECAY = 0.997        # training_scope(bn_decay=0.997), mobilenet.py:419
BATCH_NORM_EPSILON = 0.001      # slim.batch_norm's default
WEIGHTS_STDDEV = 0.09
DROPOUT_KEEP_PROB = 0.8


def make_divisible(v, divisor, min_value=None):
    """mobilenet.py:62-69 / conv_blocks.py:50-57"""
    if min_value is None:
        min_value = divisor
    new_v = max(min_value, int(v + divisor / 2) // divisor * divisor)
    if new_v < 0.9 * v:
        new_v += divisor
    return new_v


def _conv_bn(net, depth, kernel, stride, is_training, init, scope, act=True):
    """slim.conv2d(normalizer_fn=batch_norm, activation_fn=relu6 | None) under `scope`"""
    net = G.conv2d(net, depth, kernel, stride, 'same', use_bias=False, kernel_initializer=init, name=scope,
                   kernel_name='weights', exact_name=True)
    return _bn(net, is_training, scope, act)


def _bn(net, is_training, scope, act=True):
    with G.variable_scope(scope):
        net = G.batch_normalization(net, is_training, momentum=BATCH_NORM_DECAY, epsilon=BATCH_NORM_EPSILON,
                                    name='BatchNorm', exact_name=True)
        return G.relu6(net, name='Relu6') if act else net


def _expanded_conv(net, d, depth, is_training, init, scope):
    """conv_blocks.expanded_conv with depthwise_location 'expansion', split_expansion = split_projection = 1"""
    prev = net.shape[-1]
    inner = make_divisible(prev * d.expansion, d.divisible_by)
    x = net
    with G.variable_scope(scope):
        if inner > prev:
            net = _conv_bn(net, inner, 1, 1, is_training, init, 'expand')
        net = G.depthwise_conv2d(net, 3, d.stride, 'same', kernel_initializer=init, name='depthwise', exact_name=True)
        net = _bn(net, is_training, 'depthwise')
        net = _conv_bn(net, depth, 1, 1, is_training, init, 'project', act=False)
        if d.stride == 1 and depth == prev:
            net = G.add(net, x, name='add')
    return net


def mobilenet_v2(inputs, num_classes=1001, is_training=True, depth_multiplier=1.0, min_depth=8, divisible_by=8):
    """Returns logits [N, num_classes]."""
    if depth_multiplier <= 0:
        raise ValueError('multiplier is not greater than zero.')
    depth = lambda d: make_divisible(d * depth_multiplier, divisible_by, min_depth)
    init = G.truncated_normal_initializer(WEIGHTS_STDDEV)
    n_blocks = 0
    with G.variable_scope('MobilenetV2'):
        net = inputs
        for i, conv_def in enumerate(V2_CONV_DEFS):
            if isinstance(conv_def, Conv):
                net = _conv_bn(net, depth(conv_def.depth), conv_def.kernel, conv_def.stride, is_training, init,
                               'Conv' if i == 0 else 'Conv_1')
            else:
                scope = 'expanded_conv' if n_blocks == 0 else 'expanded_conv_%d' % n_blocks
                net = _expanded_conv(net, conv_def, depth(conv_def.depth), is_training, init, scope)
                n_blocks += 1
        with G.variable_scope('Logits'):
            net = G.reduce_mean_hw(net, name='AvgPool', keepdims=True)
            net = G.dropout(net, DROPOUT_KEEP_PROB, is_training, name='Dropout')
            logits = G.conv2d(net, num_classes, [1, 1], 1, 'same', use_bias=True, kernel_initializer=init,
                              name='Conv2d_1c_1x1', kernel_name='weights', bias_name='biases', exact_name=True)
            logits = G.squeeze_hw(logits, name='Squeeze')
    return logits
