"""Pruned-width fine-tuning of MobileNet-v2 and LeNet, CPU side.

* The compact training plans of MobileNet-v2 at every multiplier and pruning ratio: the kernels run every narrowed
  width (check_widths), each Dropout carries its layout and full width, and at x1.0 / 0.5 the plan has the gathers,
  fused BN + Adds with gathered shortcuts and the narrowed Dropout that tests/test_compact_nets_gpu.py relies on.
* CompactTrainer.pull / push carry the dropout step counters both ways.
* The numpy statement of the channel-mapped Philox draw (pf_dropout_fwd_mapped) equals the full-width draw
  (pf_dropout_fwd) gathered by the layout, padding 0."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'golden'))

from pocketflow_b200 import compact as C  # noqa: E402
from pocketflow_b200.engine import Executor  # noqa: E402
from pocketflow_b200.flags import FLAGS  # noqa: E402
from support import mapped_mask, ref_mask, seed_state, train_graph  # noqa: E402

V2_MULTS = [0.35, 0.75, 1.0, 1.4]
RATIOS = [0.3, 0.5, 0.7]


def v2_train_graph(mult):
    g, im, lg = train_graph('mobilenet_v2')      # sets FLAGS for v2; the multiplier is read when the net is built
    if mult == 1.0:
        return g, im, lg
    import importlib
    import make_golden_chn_export as M
    mod, flags = M.NETS['mobilenet_v2']
    FLAGS.reset()
    for k, v in dict(flags, mobilenet_depth_mult=mult).items():
        setattr(FLAGS, k, v)
    mh = importlib.import_module('pocketflow_b200.nets.' + mod).ModelHelper()
    return C.build_train_graph(mh, 2)


def compact_plan(g, im, lg, ratio, seed=1):
    st = C.fake_prune(g, lg, seed_state(g, lg, np.random.default_rng(0)), ratio, seed)
    rec = C.plan(g, lg, st)
    cg, ci, cl = C.build_graph(g, im, lg, rec)
    return st, rec, cg, ci, cl


@pytest.mark.parametrize('ratio', RATIOS)
@pytest.mark.parametrize('mult', V2_MULTS)
def test_v2_compact_plans_run_at_every_multiplier_and_ratio(mult, ratio):
    g, im, lg = v2_train_graph(mult)
    st, rec, cg, ci, cl = compact_plan(g, im, lg, ratio)
    C.check_widths(cg, cl)
    full = {op.name: op for op in C.reachable_ops(g, lg)}
    drops = [op for op in cg.ops if op.type == 'Dropout']
    assert len(drops) == 1
    for op in drops:
        lay = op.attrs['layout']
        assert lay.dtype == np.int32 and lay.tolist() == rec['tensors'][op.output.name]
        assert op.attrs['full_width'] == full[op.name].output.shape[-1] and len(lay) == op.output.shape[-1]
        # the logits conv's pruned input channels are dropped before the Dropout: it narrows
        assert op.output.shape[-1] < op.attrs['full_width']
        kept = lay[lay >= 0]
        assert sorted(kept.tolist()) == rec['convs'][op.output.consumers[0].name]
    # the full-width graph's Dropout has no map
    assert not any('layout' in op.attrs for op in full.values())


def test_v2_x1_plan_has_the_paths_the_gpu_tests_need():
    """x1.0, ratio 0.5, batch 2: 20 gathers, none fused into a BN; 10 fused BN + Adds whose shortcut is a gather's
    output; 10 gathers that read the output of 5 of those fused Adds; the Dropout narrowed 1280 -> 640"""
    g, im, lg = v2_train_graph(1.0)
    st, rec, cg, ci, cl = compact_plan(g, im, lg, 0.5)
    ex = Executor(cg, ci, cl, torch.device('cpu'), train=True)
    gathers = [op for op in ex.ops if op.type == 'GatherChannels']
    assert len(gathers) == 20 and not ex.bn_gather and set(ex.scatter_inv) == set(gathers)
    assert len(ex.bn_add) == 10
    adds = [op for op in ex.ops if op.type == 'Add']
    assert all(any(x.op.type == 'GatherChannels' for x in op.inputs) for op in adds)
    fused = {add for add, _ in ex.bn_add.values()}
    from_add = [op for op in gathers if op.inputs[0].op.type == 'Add']
    assert len(from_add) == 10 and len({op.inputs[0].op for op in from_add}) == 5
    assert all(op.inputs[0].op in fused for op in from_add)
    drop, = [op for op in ex.ops if op.type == 'Dropout']
    assert (drop.attrs['full_width'], drop.output.shape[-1]) == (1280, 640)
    assert drop in ex.drop_layout and ex.drop_layout[drop].tolist() == drop.attrs['layout'].tolist()
    assert ex.dropout[drop].numel() == 2 * 640


def test_lenet_compact_plan_narrows_the_conv_in_front_of_the_flatten():
    g, im, lg = train_graph('lenet')
    st, rec, cg, ci, cl = compact_plan(g, im, lg, 0.5)
    C.check_widths(cg, cl)
    full = {op.name: op for op in C.reachable_ops(g, lg)}
    # a MatMul needs every input channel, so the flatten -> dense keeps its width; the convs in front narrow
    convs = [op for op in cg.ops if op.type == 'Conv2D']
    assert any(op.vars['kernel'].shape[2] < full[op.name].vars['kernel'].shape[2] for op in convs)
    assert any(op.type == 'MaxPool' for op in cg.ops) and any(op.type == 'MatMul' for op in cg.ops)


def _v2_trainer():
    import make_plan_snapshot as SNAP
    ex = SNAP.build('mobilenet_at_ilsvrc12', dict(batch_size=2, mobilenet_version=2))
    st = C.fake_prune(ex.g, ex.logits_t, ex.store.state_dict(), 0.5, 1)
    ex.store.load_state_dict(st, strict=True)
    return ex, C.CompactTrainer(ex)


def test_pull_and_push_carry_the_dropout_step_counters():
    ex, ct = _v2_trainer()
    cex = ct.ex
    assert ex.drop_state.shape == cex.drop_state.shape == (1, 2)
    (fop, i), = ex.drop_stream.items()
    (cop, j), = cex.drop_stream.items()
    assert fop.name == cop.name and i == j == 0 and cop in cex.drop_layout and fop not in ex.drop_layout
    ex.drop_state[0, 0] = 7
    ct.pull()
    assert cex.drop_state.tolist() == [[7, 0]]
    cex.drop_state[0, 0] = 12
    ct.push()
    assert ex.drop_state.tolist() == [[12, 0]]


@pytest.mark.parametrize('rows,cfull,layout', [
    (3, 1280, 'half'),                                         # MobileNet-v2 x1.0 at 0.5
    (5, 7, [6, 0, -1, 3]),                                     # unsorted, padding, cfull % 4 != 0
    (2, 9, [8, 7, 6, 5, 4, 3, 2, 1, 0]),                       # every channel, reversed
    (1, 16, [-1, -1, -1, -1]),                                 # only padding
])
@pytest.mark.parametrize('step,stream', [(0, 0), (3, 1), (2 ** 32 + 5, 2)])
def test_mapped_draw_is_the_full_width_draw_gathered(rows, cfull, layout, step, stream):
    if layout == 'half':
        layout = sorted(np.random.RandomState(0).permutation(cfull)[:cfull // 2].tolist())
    lay = np.asarray(layout)
    full = ref_mask(rows * cfull, 0.8, 1234, 3, step, stream).reshape(rows, cfull)
    want = np.where(lay[None, :] >= 0, full[:, np.maximum(lay, 0)], 0.0)
    got = mapped_mask(rows, layout, cfull, 0.8, 1234, 3, step, stream)
    assert np.array_equal(got, want)
    # the identity layout is the full-width draw itself
    assert np.array_equal(mapped_mask(rows, list(range(cfull)), cfull, 0.8, 1234, 3, step, stream), full)
