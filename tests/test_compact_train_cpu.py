"""Fine-tuning channel-pruned models at their pruned width, CPU side: pocketflow_b200/compact.py on TRAINING graphs.

* Plans of the training graphs of LeNet, ResNet-20 / -50 and MobileNet-v1 / -v2 under fake pruning: layouts, gather
  positions, and the slice / expand round trip on parameters, optimizer slots and masks.
* The executor plans the compact training graph: gathers fused into the training-mode BN apply, an inverse table per
  gather for its backward.
* The float64 restatement (oracle/compact_oracle.py): the compact step equals the masked full-width step on every kept
  entry, and padding stays zero.
* --enbl_compact_ft is known to the four run scripts and off by default."""
import importlib
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'golden'))

from oracle import compact_oracle as CO  # noqa: E402
from pocketflow_b200 import compact as C  # noqa: E402
from pocketflow_b200 import graph as G  # noqa: E402
from pocketflow_b200 import ops  # noqa: E402
from pocketflow_b200.engine import Executor  # noqa: E402
from pocketflow_b200.flags import FLAGS  # noqa: E402
from support import seed_state, train_graph  # noqa: E402

NETS = ['lenet', 'resnet20', 'resnet50', 'mobilenet_v1', 'mobilenet_v2']


@pytest.mark.parametrize('ratio', [0.3, 0.5])
@pytest.mark.parametrize('net', NETS)
def test_training_graph_plan_and_state_round_trip(net, ratio):
    g, im, lg = train_graph(net)
    rng = np.random.default_rng(0)
    st = C.fake_prune(g, lg, seed_state(g, lg, rng), ratio, 1)
    rec = C.plan(g, lg, st)
    cg, ci, cl = C.build_graph(g, im, lg, rec)
    C.check_widths(cg, cl)
    ops_full = {op.name: op for op in C.reachable_ops(g, lg)}
    assert any(op.type == 'FusedBatchNorm' and op.attrs['training'] for op in cg.ops) or net == 'lenet'
    gathers = [op for op in cg.ops if op.type == 'GatherChannels']
    if net == 'mobilenet_v1':
        assert not gathers
    for op in cg.ops:
        if op.type == 'GatherChannels':
            # positions point into the producer's layout; every kept position is used at most once
            idx, src = op.attrs['index'], rec['tensors'][op.inputs[0].name]
            assert len(idx) == op.output.shape[-1] and idx.max() < len(src)
            kept = idx[idx >= 0]
            assert len(set(kept.tolist())) == len(kept) and all(src[j] >= 0 for j in kept)
            inv = ops.scatter_table(idx, len(src))
            assert np.array_equal(inv[kept], np.nonzero(idx >= 0)[0]) and (inv >= 0).sum() == len(kept)
            continue
        lay = rec['tensors'][op.output.name]
        assert len(lay) == op.output.shape[-1] <= ops_full[op.name].output.shape[-1]
        if op.type == 'Conv2D' and op.inputs[0].op.type != 'Placeholder':
            lin = C._input_layouts(ops_full[op.name], rec)[0]
            assert sorted(c for c in lin if c >= 0) == rec['convs'][op.name]
            assert op.vars['kernel'].shape[2] == len(lin) <= ops_full[op.name].vars['kernel'].shape[2]
    # parameters, an optimizer slot (any values), and the masks of the conv kernels alone
    cst = C.slice_state(g, lg, rec, st)
    assert {k: v.shape for k, v in cst.items()} == {v.name: v.shape for op in cg.ops for v in op.vars.values()}
    slot = {k: rng.standard_normal(v.shape).astype(np.float32) for k, v in st.items()}
    masks = {op.vars['kernel'].name: (st[op.vars['kernel'].name] != 0).astype(np.float32)
             for op in ops_full.values() if op.type == 'Conv2D'}
    for full, partial in ((st, False), (slot, False), (masks, True)):
        comp = C.slice_state(g, lg, rec, full, partial=partial)
        assert set(comp) == (set(full) if partial else set(cst))
        back = C.expand_state(g, lg, rec, comp, full)
        assert all(np.array_equal(back[k], full[k]) for k in full)
        # the kept entries really come from the compact state, everything else from the full one
        other = {k: np.full_like(v, 7.0) for k, v in full.items()}
        mixed = C.expand_state(g, lg, rec, comp, other)
        again = C.slice_state(g, lg, rec, mixed, partial=partial)
        for k in comp:
            pad = C.slice_state(g, lg, rec, {k: np.ones_like(full[k])}, partial=True)[k] == 0
            if k.endswith('moving_variance:0'):
                pad = C.slice_state(g, lg, rec, {k: np.full_like(full[k], 3.0)}, partial=True)[k] == 1.0
            assert np.array_equal(again[k][~pad], comp[k][~pad]), k
        assert sum(int((mixed[k] != 7.0).sum()) for k in mixed) <= sum(v.size for v in comp.values())
    # a sliced mask is zero on every padding row / column
    cm = C.slice_state(g, lg, rec, masks, partial=True)
    for op in cg.ops:
        if op.type == 'Conv2D' and op.inputs[0].op.type != 'Placeholder':
            lin = np.asarray(C._input_layouts(ops_full[op.name], rec)[0])
            lout = np.asarray(rec['tensors'][op.output.name])
            m = cm[op.vars['kernel'].name]
            assert not m[:, :, lin < 0, :].any() and not m[:, :, :, lout < 0].any()


@pytest.mark.parametrize('net', ['resnet20', 'resnet50', 'mobilenet_v1'])
def test_executor_plans_the_compact_training_graph(net):
    g, im, lg = train_graph(net)
    st = C.fake_prune(g, lg, seed_state(g, lg, np.random.default_rng(0)), 0.5, 1)
    rec = C.plan(g, lg, st)
    cg, ci, cl = C.build_graph(g, im, lg, rec)
    cpu = torch.device('cpu')
    full, comp = Executor(g, im, lg, cpu, train=True), Executor(cg, ci, cl, cpu, train=True)
    assert {op.name for op in full.ops if op in full.tc} <= {op.name for op in comp.ops if op in comp.tc}
    assert comp.G.numel() < full.G.numel()
    gathers = [op for op in comp.ops if op.type == 'GatherChannels']
    assert set(comp.scatter_inv) == set(gathers)
    if net == 'mobilenet_v1':
        assert not gathers
        return
    assert comp.bn_gather and all(bn.attrs['training'] for bn in comp.bn_gather)
    for bn, op in comp.bn_gather.items():
        assert comp._consumers(op.inputs[0]) == [op]
    # an inference executor of the same training-mode graph keeps the BN apply and the gather apart
    assert not Executor(cg, ci, cl, cpu, train=False).bn_gather


def test_a_layer_whose_whole_input_is_dead_keeps_one_padding_group():
    g = G.Graph()
    with g.as_default():
        x = G.placeholder((2, 8, 8, 16), 'images')
        with G.variable_scope('model'):
            c0 = G.conv2d(x, 32, 3, padding='same', use_bias=False, name='c0')
            b0 = G.relu(G.batch_normalization(c0, True, name='bn0'))
            c1 = G.conv2d(b0, 32, 1, padding='same', use_bias=True, name='dead')
            b1 = G.relu(G.batch_normalization(c1, True, name='bn1'))
            logits = G.dense(G.reduce_mean_hw(G.conv2d(b1, 32, 1, use_bias=False, name='c2')), 10, name='fc')
    st = seed_state(g, logits, np.random.default_rng(1))
    st['model/dead/kernel:0'][:] = 0.0
    rec = C.plan(g, logits, st)
    assert rec['convs']['model/dead/Conv2D'] == [] and rec['tensors']['model/c0/Conv2D:0'] == [-1] * 16
    cg, ci, cl = C.build_graph(g, x, logits, rec)
    cst = C.slice_state(g, logits, rec, st)
    assert cst['model/c0/kernel:0'].shape == (3, 3, 16, 16) and not cst['model/c0/kernel:0'].any()
    assert not cst['model/bn0/gamma:0'].any() and not cst['model/bn0/beta:0'].any()
    back = C.expand_state(g, logits, rec, cst, st)
    assert all(np.array_equal(back[k], st[k]) for k in st)


def test_a_width_the_kernels_cannot_run_is_refused_by_name():
    g = G.Graph()
    with g.as_default():
        x = G.placeholder((2, 4, 4, 8), 'images')
        with G.variable_scope('model'):
            b = G.relu(G.batch_normalization(G.conv2d(x, 6, 1, use_bias=False, name='c0'), True, name='bn0'))
            logits = G.dense(G.reduce_mean_hw(G.conv2d(b, 8, 1, use_bias=False, name='c1')), 10, name='fc')
    with pytest.raises(ValueError, match='model/bn0/FusedBatchNorm'):
        C.check_widths(g, logits)
    with pytest.raises(ValueError, match='at most once'):
        ops.scatter_table([0, 2, 2, -1], 4)


def test_compact_step_equals_the_masked_step_on_every_kept_entry_in_float64():
    rng = np.random.default_rng(5)
    n, cin, c, k = 12, 7, 16, 5
    keep = np.array([1, 4, 5, 9, 14])                       # the consumer's input set
    lay1 = list(keep) + [-1] * 3                            # layout of the producer's output, padded to 8
    idx = np.array([0, 1, 2, 3, 4, -1, -1, -1])             # the consumer gathers every kept position (+ padding)
    x, t = rng.standard_normal((n, cin)), rng.standard_normal((n, k))
    w1, w2 = rng.standard_normal((cin, c)), rng.standard_normal((c, k))
    mask2 = np.zeros((c, k))
    mask2[keep] = 1.0
    w2 = w2 * mask2
    a1, a2 = rng.standard_normal(w1.shape), rng.standard_normal(w2.shape) * mask2
    lr, mom, wd = 0.1, 0.9, 1e-2
    # compact state: slices of the full one, zero padding
    w1c = np.where(np.array(lay1) >= 0, w1[:, np.maximum(lay1, 0)], 0.0)
    a1c = np.where(np.array(lay1) >= 0, a1[:, np.maximum(lay1, 0)], 0.0)
    rows = np.array(lay1)[np.maximum(idx, 0)]
    w2c = np.where((idx >= 0)[:, None], w2[np.maximum(rows, 0)], 0.0)
    a2c = np.where((idx >= 0)[:, None], a2[np.maximum(rows, 0)], 0.0)
    m2c = np.where((idx >= 0)[:, None], mask2[np.maximum(rows, 0)], 0.0)
    for _ in range(3):
        y, g1, g2 = CO.two_layer_grads(x, w1, w2, t)
        yc, g1c, g2c = CO.two_layer_grads(x, w1c, w2c, t, idx)
        assert np.abs(y - yc).max() <= 1e-13 * np.abs(y).max()
        assert np.abs(g1[:, keep] - g1c[:, :5]).max() <= 1e-12 * np.abs(g1).max()
        assert np.abs(g2[keep] - g2c[:5]).max() <= 1e-12 * np.abs(g2).max()
        dead = np.setdiff1d(np.arange(c), keep)
        assert not g1[:, dead].any()                        # a dead producer channel only ever decays
        assert not g1c[:, 5:].any() and not g2c[5:].any()   # padding: zero gradients
        w1, a1 = CO.momentum_step(w1, a1, g1, 1.0, lr, mom, wd)
        w2, a2 = CO.momentum_step(w2, a2, g2, mask2, lr, mom, wd)
        w1c, a1c = CO.momentum_step(w1c, a1c, g1c, 1.0, lr, mom, wd)
        w2c, a2c = CO.momentum_step(w2c, a2c, g2c, m2c, lr, mom, wd)
        assert np.abs(w1[:, keep] - w1c[:, :5]).max() <= 1e-12 and np.abs(w2[keep] - w2c[:5]).max() <= 1e-12
        assert np.abs(a1[:, keep] - a1c[:, :5]).max() <= 1e-12 and np.abs(a2[keep] - a2c[:5]).max() <= 1e-12
        assert not w1c[:, 5:].any() and not w2c[5:].any() and not a1c[:, 5:].any() and not a2c[5:].any()
    # gather / scatter are adjoint: <gather(x), dy> == <x, scatter(dy)>
    h, dy = rng.standard_normal((n, 8)), rng.standard_normal((n, 8))
    assert abs((CO.gather(h, idx) * dy).sum() - (h * CO.scatter(dy, idx, 8)).sum()) <= 1e-12


@pytest.mark.parametrize('script', ['lenet_at_cifar10_run', 'resnet_at_cifar10_run', 'resnet_at_ilsvrc12_run',
                                    'mobilenet_at_ilsvrc12_run'])
def test_the_flag_is_known_to_every_run_script_and_off_by_default(script):
    importlib.import_module('pocketflow_b200.nets.' + script)
    FLAGS.reset()
    assert FLAGS._defaults['enbl_compact_ft'] is False and FLAGS.enbl_compact_ft is False
    FLAGS.parse(['--enbl_compact_ft', '--learner', 'chn-pruned-rmt'])
    assert FLAGS.enbl_compact_ft is True
    FLAGS.reset()


def test_a_learner_that_cannot_honour_the_flag_refuses_it():
    from pocketflow_b200.learners.learner_utils import create_learner
    importlib.import_module('pocketflow_b200.nets.resnet_at_cifar10_run')
    FLAGS.reset()
    FLAGS.learner, FLAGS.enbl_compact_ft = 'full-prec', True
    with pytest.raises(ValueError, match='enbl_compact_ft applies to the channel-pruning learners'):
        create_learner(None, None)
    FLAGS.reset()
