"""Compact (channel-pruned) inference graphs, CPU side: pocketflow_b200/compact.py.

* Each conv's input set equals the `nnzs` of the reference's own export tool (insert_alt_routines, executed under a stub
  tensorflow by tests/golden/make_golden_chn_export.py) on masked kernels of ResNet-20 / -50, MobileNet-v1 / -v2 and
  LeNet, and its fake pruning draws the same channels for the same seed.
* Liveness: a float64 numpy forward of the compact graph equals the masked full-width forward on small nets (depthwise,
  BN, max-pool, residual Add, a layer whose whole input is dead).
* The executor plans a compact graph with every full-width tensor-core conv still on the tensor cores, and fuses the
  gathers into the inference-mode BN apply where that BN has no other reader."""
import json
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'golden'))

from pocketflow_b200 import compact as C  # noqa: E402
from pocketflow_b200 import graph as G  # noqa: E402
from pocketflow_b200.engine import Executor  # noqa: E402

GOLD = json.load(open(os.path.join(HERE, 'golden', 'ref_executed_chn_export_v1.json')))


def _gold_module():
    import make_golden_chn_export as M
    return M


@pytest.mark.parametrize('net', sorted(GOLD['nets']))
def test_conv_input_sets_equal_the_reference_nnzs(net):
    M = _gold_module()
    g, im, lg = M.eval_graph(net)
    convs = M.kernels(net)
    state = {}
    rng = np.random.default_rng(0)
    for op in C.reachable_ops(g, lg):
        for v in op.vars.values():
            state[v.name] = v.initializer(rng, v.shape)
    for op, k in convs:
        state[op.vars['kernel'].name] = k
    rec = C.plan(g, lg, state)
    cg, ci, cl = C.build_graph(g, im, lg, rec)
    cstate = C.slice_state(g, lg, rec, state)
    cops = {op.name: op for op in cg.ops}
    gold = GOLD['nets'][net]['convs']
    assert [r['conv'] for r in gold] == [op.name for op, _ in convs]
    for r, (op, k) in zip(gold, convs):
        assert rec['convs'][op.name] == r['nnzs'], op.name
        assert list(k[:, :, r['nnzs'], :].shape) == r['kernel_shrk']
        lin = C._input_layouts(op, rec)[0]
        lout = rec['tensors'][op.output.name]
        if op.inputs[0].op.type == 'Placeholder':
            assert lin == list(range(op.inputs[0].shape[-1]))       # the image is never narrowed
        else:
            assert sorted(c for c in lin if c >= 0) == r['nnzs']
            assert len(lin) == C.padded_width(len(r['nnzs']), op.inputs[0].shape[-1])
        # the compact kernel is kernel_shrk at the kept output channels, zero rows / columns at the padding
        ck = cstate[op.vars['kernel'].name]
        assert ck.shape == op.vars['kernel'].shape[:2] + (len(lin), len(lout))
        assert cops[op.name].vars['kernel'].shape == ck.shape
        rows = [j for j, c in enumerate(lin) if c >= 0]
        cols = [j for j, c in enumerate(lout) if c >= 0]
        ref = k[:, :, [lin[j] for j in rows], :][:, :, :, [lout[j] for j in cols]]
        assert np.array_equal(ck[:, :, rows, :][:, :, :, cols], ref)
        assert not np.any(np.delete(ck, rows, axis=2)) and not np.any(np.delete(ck, cols, axis=3))


@pytest.mark.parametrize('net', sorted(GOLD['nets']))
def test_fake_prune_draws_the_reference_channels(net):
    M = _gold_module()
    g, im, lg = M.eval_graph(net)
    convs = [op for op in C.reachable_ops(g, lg) if op.type == 'Conv2D']
    ones = {op.vars['kernel'].name: np.ones(op.vars['kernel'].shape, np.float32) for op in convs}
    for ent in GOLD['nets'][net]['fake']:
        st = C.fake_prune(g, lg, ones, ent['ratio'], ent['seed'])
        got = [sorted(int(c) for c in np.nonzero(np.all(st[op.vars['kernel'].name] == 0, axis=(0, 1, 3)))[0])
               for op in convs]
        assert got == ent['pruned']


# ------------------------------------------------------------------ float64 numpy forward (the statement of liveness)
def _conv(x, k, op, depthwise=False):
    n, h, w, c = x.shape
    (kh, kw), (sh, sw), (pt, pl) = op.attrs['ksize'], op.attrs['strides'], op.attrs['pad']
    p, q = op.output.shape[1:3]
    xp = np.zeros((n, (p - 1) * sh + kh, (q - 1) * sw + kw, c))
    hh, ww = min(h, xp.shape[1] - pt), min(w, xp.shape[2] - pl)
    xp[:, pt:pt + hh, pl:pl + ww] = x[:, :hh, :ww]
    y = 0.0
    for r in range(kh):
        for s in range(kw):
            win = xp[:, r:r + sh * (p - 1) + 1:sh, s:s + sw * (q - 1) + 1:sw, :]
            y = y + (win * k[r, s, :, 0] if depthwise else win @ k[r, s])
    return y


def _maxpool(x, op):
    n, h, w, c = x.shape
    (kh, kw), (sh, sw), (pt, pl) = op.attrs['ksize'], op.attrs['strides'], op.attrs['pad']
    p, q = op.output.shape[1:3]
    xp = np.full((n, (p - 1) * sh + kh, (q - 1) * sw + kw, c), -np.inf)
    hh, ww = min(h, xp.shape[1] - pt), min(w, xp.shape[2] - pl)
    xp[:, pt:pt + hh, pl:pl + ww] = x[:, :hh, :ww]
    y = np.full((n, p, q, c), -np.inf)
    for r in range(kh):
        for s in range(kw):
            y = np.maximum(y, xp[:, r:r + sh * (p - 1) + 1:sh, s:s + sw * (q - 1) + 1:sw, :])
    return y


def np_forward(graph, images, logits, state, x):
    v = {images: np.asarray(x, np.float64)}
    for op in C.reachable_ops(graph, logits):
        if op.type == 'Placeholder':
            continue
        a = v[op.inputs[0]]
        P = {role: np.asarray(state[var.name], np.float64) for role, var in op.vars.items()}
        if op.type == 'Conv2D':
            y = _conv(a, P['kernel'], op) + P.get('bias', 0.0)
        elif op.type == 'DepthwiseConv2dNative':
            y = _conv(a, P['kernel'], op, depthwise=True)
        elif op.type == 'MatMul':
            y = a @ P['kernel'] + P.get('bias', 0.0)
        elif op.type == 'FusedBatchNorm':
            y = (a - P['moving_mean']) / np.sqrt(P['moving_variance'] + op.attrs['epsilon']) * P['gamma'] + P['beta']
        elif op.type == 'Relu':
            y = np.maximum(a, 0.0)
        elif op.type == 'Relu6':
            y = np.minimum(np.maximum(a, 0.0), 6.0)
        elif op.type == 'MaxPool':
            y = _maxpool(a, op)
        elif op.type == 'Mean':
            y = a.mean(axis=(1, 2)).reshape(op.output.shape)
        elif op.type in ('Reshape', 'Identity', 'Dropout'):
            y = a.reshape(op.output.shape)
        elif op.type == 'Add':
            y = a + v[op.inputs[1]]
        elif op.type == 'Softmax':
            e = np.exp(a - a.max(axis=1, keepdims=True))
            y = e / e.sum(axis=1, keepdims=True)
        elif op.type == 'GatherChannels':
            idx = op.attrs['index']
            y = np.where(idx >= 0, a[..., np.maximum(idx, 0)], 0.0)
        else:
            raise NotImplementedError(op.type)
        v[op.output] = y
    return v[logits]


def _toy_graph():
    """depthwise chain, max-pool, a residual Add whose shortcut is narrowed, a layer whose whole input is dead"""
    g = G.Graph()
    with g.as_default():
        x = G.placeholder((2, 9, 9, 16), 'images')
        with G.variable_scope('model'):
            c0 = G.conv2d(x, 32, 3, padding='same', use_bias=False, name='c0')
            b0 = G.relu6(G.batch_normalization(c0, False, name='bn0'))
            d0 = G.depthwise_conv2d(b0, 3, name='dw0')
            b1 = G.relu6(G.batch_normalization(d0, False, name='bn1'))
            c1 = G.conv2d(b1, 32, 1, padding='same', use_bias=False, name='c1')
            p1 = G.max_pooling2d(c1, 3, 2, padding='same')
            b2 = G.relu(G.batch_normalization(p1, False, name='bn2'))
            c2 = G.conv2d(b2, 32, 3, padding='same', use_bias=False, name='c2')
            s = G.add(p1, c2)
            b3 = G.relu(G.batch_normalization(s, False, name='bn3'))
            c3 = G.conv2d(b3, 32, 1, padding='same', use_bias=True, name='dead')
            b4 = G.relu(G.batch_normalization(c3, False, name='bn4'))
            c4 = G.conv2d(b4, 48, 1, padding='same', use_bias=False, name='c4')
            s2 = G.add(c4, G.conv2d(p1, 48, 1, padding='same', use_bias=False, name='proj'))
            logits = G.dense(G.reduce_mean_hw(s2), 10, name='fc')
    return g, x, logits


def _random_masked_state(g, lg, rng, ratio=0.4, dead=()):
    st = {}
    for op in C.reachable_ops(g, lg):
        for role, v in op.vars.items():
            a = v.initializer(rng, v.shape)
            if role == 'moving_variance':
                a = rng.uniform(0.5, 2.0, v.shape).astype(np.float32)
            elif role in ('gamma', 'beta', 'moving_mean', 'bias'):
                a = rng.standard_normal(v.shape).astype(np.float32)
            elif op.type == 'Conv2D' and op.inputs[0].op.type != 'Placeholder':
                a[:, :, rng.random(v.shape[2]) < ratio, :] = 0.0
                if any(d in op.name for d in dead):
                    a[:] = 0.0
            st[v.name] = a
    return st


@pytest.mark.parametrize('case', ['toy', 'resnet20', 'lenet'])
def test_compact_forward_equals_masked_full_width_in_float64(case):
    rng = np.random.default_rng(3)
    if case == 'toy':
        g, im, lg = _toy_graph()
        st = _random_masked_state(g, lg, rng, dead=('dead',))
    else:
        g, im, lg = _gold_module().eval_graph(case)
        st = _random_masked_state(g, lg, rng, ratio=0.7 if case == 'lenet' else 0.4)
    rec = C.plan(g, lg, st)
    if case == 'toy':
        assert rec['convs']['model/dead/Conv2D'] == []
        assert rec['tensors']['model/dead/Conv2D:0'] != list(range(32))
        assert any(k.startswith('model/add') for k in rec['gathers'])         # a narrowed residual operand
    cg, ci, cl = C.build_graph(g, im, lg, rec)
    cst = C.slice_state(g, lg, rec, st)
    assert sum(a.size for a in cst.values()) < sum(a.size for a in st.values())
    x = rng.standard_normal(im.shape)
    ref = np_forward(g, im, lg, st, x)
    got = np_forward(cg, ci, cl, cst, x)
    assert got.shape == ref.shape
    assert np.max(np.abs(got - ref)) <= 1e-12 * np.max(np.abs(ref))


def test_checkpoint_scope_is_mapped_and_an_unmatched_variable_is_refused():
    g, im, lg = _toy_graph()
    st = _random_masked_state(g, lg, np.random.default_rng(0))
    ops_ = C.reachable_ops(g, lg)
    pruned = {'pruned_model/' + k.split('/', 1)[1]: v for k, v in st.items()}
    pruned['model/c0/kernel:0'] = np.zeros(1)              # the full model's scope is ignored when both are present
    got = C.map_state(g, ops_, pruned)
    assert set(got) == set(st) and all(np.array_equal(got[k], st[k]) for k in st)
    pruned.pop('pruned_model/bn2/moving_mean:0')
    with pytest.raises(KeyError, match='bn2/moving_mean'):
        C.map_state(g, ops_, pruned)


@pytest.mark.parametrize('net', ['resnet50', 'mobilenet_v1', 'resnet20'])
def test_executor_keeps_tensor_core_convs_and_fuses_gathers_into_bn(net):
    g, im, lg = _gold_module().eval_graph(net)
    st = {}
    rng = np.random.default_rng(0)
    for op in C.reachable_ops(g, lg):
        for v in op.vars.values():
            st[v.name] = v.initializer(rng, v.shape)
    st = C.fake_prune(g, lg, st, 0.5, 1)
    rec = C.plan(g, lg, st)
    cg, ci, cl = C.build_graph(g, im, lg, rec)
    cpu = torch.device('cpu')
    full, comp = Executor(g, im, lg, cpu, train=False), Executor(cg, ci, cl, cpu, train=False)
    tc_full = {op.name for op in full.ops if op in full.tc or op in full.im2col}
    tc_comp = {op.name for op in comp.ops if op in comp.tc or op in comp.im2col}
    assert tc_full <= tc_comp
    gathers = [op for op in comp.ops if op.type == 'GatherChannels']
    if net == 'mobilenet_v1':
        assert not gathers                              # every narrowed tensor has a single consumer chain
    else:
        assert gathers and comp.bn_gather
        for op in gathers:
            # a gather feeding only tensor-core convs writes their operand planes and no fp32 copy
            if all(c in comp.tc for c in comp._consumers(op.output)):
                assert op in comp.xplanes and not comp.bn_need_f32[op]
