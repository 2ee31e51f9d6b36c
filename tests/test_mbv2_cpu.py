"""MobileNet-v2 (`--mobilenet_version 2`) on the CPU: the graph builder, the schedule, the maskable variables and the flag
defaults against what the reference's own code produced (tests/golden/ref_executed_mbv2_v1.json, recorded by
tests/golden/make_golden_mbv2.py); the planner's lowering of linear bottlenecks and dropout; and the launch plans of the
benchmarked networks against the snapshot tests/golden/plans_v1.json (tests/golden/make_plan_snapshot.py) — the fusion
must leave them untouched."""
import importlib.util
import json
import os
import subprocess
import sys

import pytest

from pocketflow_b200 import graph as G
from pocketflow_b200.flags import FLAGS
from pocketflow_b200.nets import mobilenet_v2 as M2
from support import expected_contributions, grad_inputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location('make_plan_snapshot',
                                               os.path.join(ROOT, 'tests', 'golden', 'make_plan_snapshot.py'))
SNAP = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(SNAP)

GOLD = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'ref_executed_mbv2_v1.json')))
MULTIPLIERS = [1.0, 1.4, 0.75, 0.5, 0.35]


def v2_graph(dm, is_training=True, batch=2):
    g = G.Graph()
    with g.as_default():
        x = G.placeholder((batch, 224, 224, 3), 'x')
        logits = M2.mobilenet_v2(x, num_classes=1001, is_training=is_training, depth_multiplier=dm)
    return g, logits


def layer_table(g):
    """this repo's graph in the recorder's terms (tests/golden/make_golden_mbv2.py): conv / dwconv / bn / act / add /
    avgpool / dropout rows in op order; a BN not followed by ReLU6 is slim's linear projection (`identity`)"""
    rows = []
    for op in g.ops:
        a = op.attrs
        if op.type == 'Conv2D':
            k = op.vars['kernel']
            rows.append(['conv', op.name[:-len('/Conv2D')], op.output.shape[-1], a['ksize'][0], a['strides'][0],
                         a['padding'].upper(), k.initializer.stddev, 'bias' in op.vars])
        elif op.type == 'DepthwiseConv2dNative':
            k = op.vars['kernel']
            rows.append(['dwconv', op.name[:-len('/depthwise')], a['ksize'][0], a['strides'][0], a['padding'].upper(),
                         k.shape[3], k.initializer.stddev])
        elif op.type == 'FusedBatchNorm':
            rows.append(['bn', op.name[:-len('/FusedBatchNorm')], a['momentum'], a['epsilon'], 'beta' in op.vars,
                         'gamma' in op.vars, a['training']])
            acts = [c.type for c in op.output.consumers if c.type in ('Relu', 'Relu6')]
            rows.append(['act', acts[0].lower() if acts else 'identity'])
        elif op.type == 'Add':
            rows.append(['add'])
        elif op.type == 'Mean':
            rows.append(['avgpool', op.inputs[0].shape[1], op.inputs[0].shape[2], 'VALID'])
        elif op.type == 'Dropout':
            rows.append(['dropout', a['keep_prob'], a['training']])
    return rows


@pytest.mark.parametrize('case', GOLD['architecture'], ids=lambda c: '%s-%s' % (c['depth_mult'], c['is_train']))
def test_v2_graph_equals_the_reference_recorded_architecture(case):
    """forward_fn of the reference's nets/mobilenet_at_ilsvrc12.py, run under a slim stub, at all five multipliers in
    train and eval: the same layers in the same order with the same scopes, widths, kernels, strides, padding,
    initializer, BN arguments, activations, residual adds, pool, dropout and logits bias"""
    g, logits = v2_graph(case['depth_mult'], case['is_train'])
    assert list(logits.shape) == case['logits_shape']
    assert len(GOLD['architecture']) == 2 * len(MULTIPLIERS)
    got, want = layer_table(g), case['layers']
    for i, (a, b) in enumerate(zip(got, want)):
        assert a == b, (i, a, b)
    assert len(got) == len(want)


def test_v2_parameter_count_at_depth_1():
    g, _ = v2_graph(1.0)
    # 3,504,872 weights of the 1000-class network + 1,281 for the 1001st class
    assert sum(v.numel for v in g.variables.values() if v.trainable) == 3506153


def helper(version=2, **flags):
    import importlib
    FLAGS.reset()
    import pocketflow_b200.datasets.ilsvrc12_dataset as D
    importlib.reload(D)
    from pocketflow_b200.nets import mobilenet_at_ilsvrc12 as M
    M = importlib.reload(M)
    FLAGS.mobilenet_version = version
    for k, v in flags.items():
        setattr(FLAGS, k, v)
    return M


def test_flag_defaults_match_the_reference_and_other_versions_are_rejected():
    M = helper(version=1)
    FLAGS.reset()
    for k, v in GOLD['flag_defaults'].items():
        assert getattr(FLAGS, k) == v, k
    FLAGS.mobilenet_version = 3
    g = G.Graph()
    with g.as_default():
        x = G.placeholder((1, 224, 224, 3), 'x')
        with pytest.raises(ValueError):
            M.forward_fn(x, True)


@pytest.mark.parametrize('case', GOLD['lrn_rate'], ids=lambda c: 'bs%d' % c['batch_size'])
def test_v2_schedule_equals_the_reference_setup_lrn_rate(case):
    """the reference's setup_lrn_rate hands tf.train.exponential_decay(lr_init, step, decay_steps, rate,
    staircase=True): lr = lr_init * rate ** (step // decay_steps), evaluated at corner steps"""
    M = helper(version=2, batch_size=case['batch_size'], nb_epochs_rat=case['nb_epochs_rat'])
    lr, nb_iters = M.ModelHelper().setup_lrn_rate(None)
    assert nb_iters == case['nb_iters'] and case['staircase']
    ds = case['decay_steps']
    for step in (0, ds - 1, ds, 2 * ds + 7, 10 * ds, nb_iters - 1):
        assert lr(step) == case['lrn_rate_init'] * case['decay_rate'] ** (step // ds), step


def test_v1_schedule_unchanged():
    M = helper(version=1, batch_size=96)
    lr, nb_iters = M.ModelHelper().setup_lrn_rate(None)
    per_epoch = 1281167 / 96
    assert nb_iters == int(1281167 * 100 / 96)
    init = 0.045 * 96 / 96
    assert lr(0) == init and lr(int(per_epoch * 30)) == init and lr(int(per_epoch * 30) + 1) == init * 0.1
    assert lr(nb_iters) == init * 0.0001


@pytest.mark.parametrize('case', GOLD['maskable_vars'], ids=lambda c: str(c['depth_mult']))
def test_maskable_vars_equal_the_reference_filter(case):
    """the reference's get_maskable_vars on this repo's v2 names keeps only the logits conv; so must this repo's"""
    from pocketflow_b200.learners.weight_sparsification.utils import get_maskable_vars
    g = G.Graph()
    with g.as_default():
        x = G.placeholder((2, 224, 224, 3), 'x')
        with G.variable_scope('model'):
            M2.mobilenet_v2(x, num_classes=1001, is_training=True, depth_multiplier=case['depth_mult'])
    tv = [v for v in g.variables.values() if v.trainable]
    assert len(tv) == case['n_trainable']
    assert [v.name for v in get_maskable_vars(tv)] == case['maskable']


# ------------------------------------------------------------------------------------------------ planning
def v2_executor(dm, batch=4):
    return SNAP.build('mobilenet_at_ilsvrc12', dict(batch_size=batch, mobilenet_version=2, mobilenet_depth_mult=dm))


@pytest.mark.parametrize('dm', MULTIPLIERS)
def test_v2_plan_fuses_every_linear_bottleneck(dm):
    ex = v2_executor(dm)
    bns = [op.inputs[0].op for op in ex.ops if op.type == 'Add']
    assert len(bns) == 10 and set(ex.bn_add) == set(bns)
    for bn, (add, other) in ex.bn_add.items():
        assert add in ex.add_fused and ex.buf[bn.output] is ex.buf[add.output] and bn not in ex.fused_act
        readers = ex._consumers(add.output)
        tc_readers = [c for c in readers if c in ex.tc and c not in ex.im2col]
        if tc_readers:
            # planes when a tensor-core conv reads the sum; the fp32 copy only when something else reads it too
            assert add in ex.xplanes
            assert ex.bn_need_f32[add] == any(c not in ex.tc_wgrad for c in readers)
            for c in tc_readers:
                assert ex.planes_of(c.inputs[0]) is ex.xplanes[add]
        else:
            assert add not in ex.xplanes
        # the backward needs no new kernel: the BN reads the Add's gradient buffer
        assert ex.gkey(bn.output) is ex.gkey(add.output)
    drops = [op for op in ex.ops if op.type == 'Dropout']
    assert len(drops) == 1 and drops[0] in ex.dropout
    assert ex.dropout[drops[0]].numel() == 4 * M2.make_divisible(1280 * dm, 8)
    assert ex.drop_state is not None and ex.drop_state.numel() == 2


def test_v2_plan_at_depth_1_keeps_fp32_copies_only_for_shortcuts():
    ex = v2_executor(1.0)
    planes_only = sorted(a.name.split('/')[2] for a in ex.xplanes if a.type == 'Add' and not ex.bn_need_f32[a])
    assert planes_only == ['expanded_conv_12', 'expanded_conv_15', 'expanded_conv_5', 'expanded_conv_9']
    assert not [a for a in ex.xplanes if a.type == 'Add' and a.name.split('/')[2] == 'expanded_conv_2']


def test_v2_inference_graph_dropout_is_an_alias():
    ex = SNAP.build('mobilenet_at_ilsvrc12', dict(batch_size=2, mobilenet_version=2), train=False)
    drop = [op for op in ex.ops if op.type == 'Dropout'][0]
    assert not ex.dropout and ex.alias[drop.output] is drop.inputs[0]


def test_v2_gradient_buffers_hold_exactly_the_consumers_contributions():
    ex = v2_executor(1.0)
    memo, state = {}, {ex.gkey(ex.loss.ce[1]): {'loss'}}
    for op in reversed(ex.ops):
        if op.type == 'Placeholder' or ex.gkey(op.output) not in state:
            continue
        if not (op.type in ('Reshape', 'Identity') or op in ex.fused_into):
            assert state[ex.gkey(op.output)] == expected_contributions(ex, op.output, memo), op.name
        for t in grad_inputs(ex, op):
            k = ex.gkey(t)
            state[k] = (state[k] | {op}) if k in state else {op}


def test_existing_bench_networks_plan_exactly_as_before():
    """planned in a child process that sees no CUDA device, as the snapshot was: the split-K partition of a weight
    gradient (wg_part) follows the SM count of the current device, so on a GPU host the plans differ there"""
    want = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'plans_v1.json')))
    code = ('import json, sys; sys.path.insert(0, %r); import make_plan_snapshot as S; print(json.dumps(S.snapshot()))'
            % os.path.join(ROOT, 'tests', 'golden'))
    argv = [sys.executable, '-B'] + (['-s'] if sys.flags.no_user_site else []) + ['-c', code]
    out = subprocess.run(argv, cwd=ROOT, env=dict(os.environ, CUDA_VISIBLE_DEVICES=''), capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
    got = json.loads(out.stdout.strip().splitlines()[-1])
    assert sorted(got) == sorted(want)
    for key in want:
        assert got[key] == want[key], key
