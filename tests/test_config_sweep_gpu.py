"""The networks, widths and quantizer modes that bench.py does not run, layer by layer against float64.

The planner picks each layer's lowering from its channel counts, bit-widths and bucket mode, so the default networks of
the learners (ResNet-18 / 34 on ILSVRC-12, the uniform learner's W4 per-layer A32 defaults), split buckets, mixed
bit-widths set through Executor.set_quant_bits, quantized stems and logits, codebook training and MobileNet widths whose
channel counts are not multiples of 16 or 64 reach plan branches the benchmarked steps never take.  Per configuration
(CONFIGS), from one learner built with the product's own flags:
  * REPLAY: one step replayed from a captured CUDA graph gives bit for bit the P, O, S1, S2 and losses of one eager step
    from the same state and batch;
  * BACKWARD: tests/test_backward_parity_gpu.run_parity, unchanged — every backward op teacher-forced against float64,
    every trainable variable's gradient (trained codebooks included: Parity.codebook_terms), the optimizer update;
  * TRAINING FORWARD: that step's forward, layer-local against StepOracle (test_bench_configs_gpu.local_parity): every
    conv / depthwise / pool / Add / Mean output within 2e-5 of its scale, at most 1e-4 of the quantized activation
    elements on a neighbouring level; the quantized kernels in ex.QW bit-exact against oracle.pf_oracle for the
    configuration's quantizer (per-layer, per-channel, split buckets, mixed bits, codebooks + the device's index);
  * INFERENCE FORWARD: ex.forward(training=False), what evaluate() runs, layer-local against the oracle in inference
    mode at the same bars; with distillation also the teacher's executor (BN folded into its convolutions' epilogues)
    against its own oracle;
  * COVERAGE: each configuration records the plan branches its executor took (branches()); the last test fails when a
    branch in REQUIRED was never reached;
  * CONTROLS: the codebook gradient against a reference whose centroid indices are shifted by one, and the inference
    forward against a reference that uses the batch statistics, each miss their bar by more than 10x.
Worst errors, runtime and peak device memory go to parity_flips.json in $PF_PARITY_DIR (default: the system temp
directory); DESIGN.md §4 quotes them."""
import time

import numpy as np
import pytest
import torch

from oracle import pf_oracle as O
from oracle.mbv2_oracle import DropoutStepOracle
from oracle.step_oracle import StepOracle
from pocketflow_b200 import engine
from support import BAR_FWD, BAR_W, QUIET, free, local_parity, make, record, run_parity, snapshot

pytestmark = pytest.mark.gpu
F32 = np.float32

# Of the output's (the gradient's) max|float64|.  DESIGN.md §6 holds a convolution with a split-bf16 operand to 2e-5;
# ResNet-18 / 34's last stage (3x3x512, a 4608-long reduction) with both operands split — the teacher, inference passes,
# codebook weights, dgrad — measured up to 3.3e-5 (outputs) and 2.1e-5 (dx) on an H100, so this sweep's bars are 4e-5
# and 3e-5 (DESIGN.md §4, "Open": the error of a split operand scales with the sum of |terms|, not with max|output|).
BAR_DX = 3e-5
BAR_FLIPS = 1e-4        # of the quantized activation elements

UQ8 = dict(uql_weight_bits=8, uql_activation_bits=8, uql_use_buckets=True, uql_bucket_type='channel')
R18 = ('resnet_at_ilsvrc12', dict(resnet_size=18))

# (id, net module, learner, batch, flags, what else the configuration does)
CONFIGS = [
    ('resnet18_uq8_dst_b128', R18, 'uniform', 128, dict(UQ8, enbl_dst=True), {}),
    ('resnet34_uq_defaults', ('resnet_at_ilsvrc12', dict(resnet_size=34)), 'uniform', 2, {}, {}),
    ('resnet18_uq_w4a4_layer', R18, 'uniform', 2, dict(uql_weight_bits=4, uql_activation_bits=4), {}),
    ('resnet18_uq8_split', R18, 'uniform', 2, dict(UQ8, uql_bucket_type='split'), {}),
    ('resnet18_uq8_all_layers', R18, 'uniform', 2, dict(UQ8, uql_quantize_all_layers=True), {}),
    ('resnet18_uq_mixed_bits', R18, 'uniform', 2, dict(UQ8), {'mixed_bits': True}),
    ('resnet18_nuq4_both', R18, 'non-uniform', 2, dict(nuql_weight_bits=4, nuql_opt_mode='both'), {}),
    ('resnet18_nuq4_cluster', R18, 'non-uniform', 2, dict(nuql_weight_bits=4, nuql_opt_mode='cluster'), {}),
    ('resnet18_full_prec', R18, 'full-prec', 2, {}, {'eval_control': True}),
    ('resnet18_ws50', R18, 'weight-sparse', 2, dict(ws_prune_ratio=0.5, ws_prune_ratio_prtl='uniform', enbl_dst=False),
     {}),
    ('mobilenet_v1_x0.25_uq8', ('mobilenet_at_ilsvrc12', dict(mobilenet_depth_mult=0.25)), 'uniform', 2, dict(UQ8), {}),
    ('mobilenet_v1_x0.75_uq8', ('mobilenet_at_ilsvrc12', dict(mobilenet_depth_mult=0.75)), 'uniform', 2, dict(UQ8), {}),
    ('mobilenet_v1_x0.5_cpg50', ('mobilenet_at_ilsvrc12', dict(mobilenet_depth_mult=0.5)), 'chn-pruned-gpu', 2,
     dict(cpg_prune_ratio=0.5), {'choose_channels': True}),
    ('mobilenet_v2_x0.35_uq8', ('mobilenet_at_ilsvrc12', dict(mobilenet_version=2, mobilenet_depth_mult=0.35)),
     'uniform', 2, dict(UQ8), {}),
    ('mobilenet_v2_x1.4_full_prec', ('mobilenet_at_ilsvrc12', dict(mobilenet_version=2, mobilenet_depth_mult=1.4)),
     'full-prec', 2, {}, {}),
]

# Plan branches the configurations above must reach between them (branches() reads them from the executors).
REQUIRED = frozenset([
    'levels: per-channel weight levels',
    'levels: per-layer weight levels',
    'levels: activations against split-bf16 weights',
    'levels: weights below 8 bits',
    'levels: an activation above 8 bits',
    'residual fused into a 3x3 level-operand conv',
    'per-layer weight quantization',
    'split buckets',
    'mixed bit-widths (set_quant_bits)',
    'quantized stem',
    'quantized logits MatMul',
    'codebook training',
    'stem: CUDA cores',
    'stem: im2col, no pixel pairing',
    'conv: CUDA cores between tensor-core convs',
    'conv: tensor-core fwd / dgrad, CUDA-core wgrad',
    'depthwise: generic kernels',
    'fp32 copy beside operand planes',
    'dy planes from a BN backward',
    'dy planes in the gradient buffer',
    'Add alias of an input gradient',
    'teacher: BN folded into conv epilogues',
])
SEEN = {}                       # branch -> first configuration that reached it
RAN = set()


@pytest.fixture(autouse=True)
def _reset_flags():
    yield
    from pocketflow_b200.flags import FLAGS
    FLAGS.reset()


# ------------------------------------------------------------------------------------------ plan branches
def _dw_generic(c):
    """pf_dwconv.cu dw_is3x3: the 3x3 kernels need a 256-thread block to be a multiple of C / 4"""
    return c % 4 == 0 and 256 % (c // 4) != 0


def branches(ex):
    seen = set()
    wq = ex.weight_quant
    if wq and wq.get('kind', 'uniform') == 'uniform':
        seen.add('per-layer weight quantization' if not wq.get('use_buckets', False) else
                 '%s buckets' % wq.get('bucket_type', 'channel'))
    if ex.train_clusters:
        seen.add('codebook training')
    for op, lo in ex.conv.items():
        stem = op.type == 'Conv2D' and op.inputs[0].op.type == 'Placeholder'
        if stem and op in ex.qvars:
            seen.add('quantized stem')
        if op.type == 'MatMul' and op in ex.qvars:
            seen.add('quantized logits MatMul')
        if stem and type(lo) is engine._ConvLowering:
            seen.add('stem: CUDA cores')
        if stem and isinstance(lo, engine._StemConv) and lo.im['mode'] == 'im2col' and 'pair' not in lo.im:
            seen.add('stem: im2col, no pixel pairing')
        if not stem and op.type == 'Conv2D' and type(lo) is engine._ConvLowering and ex.tc:
            seen.add('conv: CUDA cores between tensor-core convs')
        if not stem and op in ex.tc and op not in ex.tc_wgrad:
            seen.add('conv: tensor-core fwd / dgrad, CUDA-core wgrad')
        if isinstance(lo, engine._TcConv) and lo.x_lv is not None:
            if lo.w_lv is None:
                seen.add('levels: activations against split-bf16 weights')
            else:
                seen.add('levels: per-layer weight levels' if lo.w_lv['ncols'] == 1 else 'levels: per-channel weight levels')
                if ex.wq.bits[lo.w_lv['index']] < 8:
                    seen.add('levels: weights below 8 bits')
            if op in ex.fused_add and tuple(op.attrs['ksize']) == (3, 3):
                seen.add('residual fused into a 3x3 level-operand conv')
    for bn in ex.act_lv:
        if int(ex.act_quant['bits'][ex._aq_of_bn(bn)]) > 8:
            seen.add('levels: an activation above 8 bits')
    for op in ex.ops:
        if op.type == 'DepthwiseConv2dNative' and _dw_generic(op.inputs[0].shape[-1]):
            seen.add('depthwise: generic kernels')
    if any(ex.bn_need_f32.values()):
        seen.add('fp32 copy beside operand planes')
    if ex.conv_dy_planes:
        seen.add('dy planes from a BN backward')
    if any(ex.bn_gplanes_only.values()):
        seen.add('dy planes in the gradient buffer')
    if any(t.op.type != 'Placeholder' and a is not ex.alias.get(t) and a.op.type == 'Add' for t, a in ex.galias.items()):
        seen.add('Add alias of an input gradient')
    if ex.teacher is not None and ex.teacher.bn_fold:
        seen.add('teacher: BN folded into conv epilogues')
    return seen


# ------------------------------------------------------------------------------------------ checks
def frozen_names(ex):
    """trainable variables the optimizer leaves alone (the non-uniform learner's codebooks or everything else)"""
    st = ex.store
    return tuple(v.name for v in st.train_vars if any(s <= st.offset[v] < e for s, e in st.frozen_ranges))


def check_quantized_weights(ex, state):
    """ex.QW bit-exact against the oracle's quantizer of the configuration, from `state` (the parameters the last
    forward read); for trained codebooks also the device's centroid index of every weight"""
    wq = ex.weight_quant
    for i, op in enumerate(ex.wq_ops):
        v, bits = op.vars['kernel'], int(wq['bits'][i])
        got = ex.store.view(v, ex.QW).cpu().numpy()
        if wq.get('kind', 'uniform') == 'uniform':
            ref = O.uniform_quantize(state[v.name], bits, use_buckets=wq.get('use_buckets', False),
                                     bucket_type=wq.get('bucket_type', 'channel'), bucket_size=wq.get('bucket_size', 256))
        else:
            assert not wq.get('use_buckets', False)
            ref, _, idx = O.nonuniform_quantize(state[v.name], bits, state[op.vars['clusters'].name][:1 << bits])
            if ex.wq.idx is not None:
                a = ex.wq.idx_offsets[i]
                dev_idx = ex.wq.idx[a:a + v.numel].cpu().numpy().astype(np.int64)
                assert np.array_equal(dev_idx, np.asarray(idx).reshape(-1)), (v.name, 'centroid index')
        assert np.array_equal(got.view(np.uint32), np.asarray(ref, F32).view(np.uint32)), (v.name, bits)
    return len(ex.wq_ops)


def oracle_of(ex, lrn, student=True):
    masks = {op.name: ex.dropout[op].view(op.output.shape).cpu().numpy() for op in ex.dropout}
    if not student:
        return StepOracle(ex.ops, ex.logits_t, lrn.images)
    kw = dict(weight_quant=ex.weight_quant, act_quant=ex.act_quant)
    if masks:
        return DropoutStepOracle(ex.ops, ex.logits_t, lrn.images, lrn.labels, ex.loss, masks=masks, **kw)
    return StepOracle(ex.ops, ex.logits_t, lrn.images, lrn.labels, ex.loss, **kw)


def forward_parity(tag, ex, orc, state, img, training):
    worst, where, flips, total, frac = local_parity(ex, orc, state, img, training)
    print('%s: worst %.2e (%s), %d of %d quantized activation elements on a neighbouring level, worst non-flip %.3f '
          'of a level' % (tag, worst, where, flips, total, frac))
    assert worst <= BAR_FWD, (tag, where, worst)
    assert flips <= BAR_FLIPS * max(total, 1), (tag, flips, total)
    return worst, flips, total


def _state(ex):
    s = snapshot(ex)
    s['drop'] = ex.drop_state.clone() if ex.drop_state is not None else None
    s['step'] = ex.step_count
    return s


def _restore(ex, s):
    ex.store.P.copy_(s['P'])
    ex.store.O.copy_(s['O'])
    ex.S1.copy_(s['S1'])
    if s['S2'] is not None:
        ex.S2.copy_(s['S2'])
    if s['drop'] is not None:
        ex.drop_state.copy_(s['drop'])
    ex.beta1_power, ex.beta2_power, ex.step_count = s['b1'], s['b2'], s['step']
    torch.cuda.synchronize()


def _outcome(ex):
    torch.cuda.synchronize()
    return [t.clone() for t in (ex.store.P, ex.store.O, ex.S1, ex.S2) if t is not None], ex.fetch_losses()


def check_replay(lrn):
    """one eager step and one replay of the captured step from the same state and batch: bit for bit the same"""
    ex = lrn.sess_train
    images, labels = lrn.iterator_train.next_batch()
    ex.buf[lrn.images].copy_(images)
    ex.buf[lrn.labels].copy_(labels)
    s0 = _state(ex)
    lr = lrn.lrn_rate(ex.step_count)
    ex.run_step(lr)
    eager = _outcome(ex)
    _restore(ex, s0)
    ex.capture()                               # its warm-up is one more eager step
    _restore(ex, s0)
    ex.run_step(lr)
    graph = _outcome(ex)
    ex._graph = None
    _restore(ex, s0)
    for a, b in zip(eager[0], graph[0]):
        assert torch.equal(a, b), 'captured step differs from the eager step'
    l0, l1 = eager[1], graph[1]
    assert all(F32(l0[k]).view(np.uint32) == F32(l1[k]).view(np.uint32) for k in l0), (l0, l1)


def mixed_bits(ex):
    """weights cycling through 2..8 bits, activations through 4..8 with one at 32 (the RL bit optimizer's lists)"""
    nw, na = len(ex.wq_ops), len(ex.aq_ops)
    a = [4 + i % 5 for i in range(na)]
    a[na // 2] = 32
    ex.set_quant_bits([2 + i % 7 for i in range(nw)], a)


@pytest.mark.parametrize('cfg', CONFIGS, ids=[c[0] for c in CONFIGS])
def test_config_matches_float64_layer_by_layer(cfg, monkeypatch):
    import support
    name, (net, net_flags), learner, batch, flags, extra = cfg
    monkeypatch.setenv('PF_POISON', '1')
    monkeypatch.setattr(support, 'BAR_DX', BAR_DX)
    free()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    lrn = make(net, learner, batch, **dict(dict(QUIET, nb_classes=1001, **net_flags), **flags))
    try:
        ex = lrn.sess_train
        if extra.get('choose_channels'):
            lrn.init_from_full()
            lrn.choose_channels(nb_iters_layer=2)
        seen = set()
        if extra.get('mixed_bits'):
            mixed_bits(ex)
            assert len(set(ex.weight_quant['bits'])) == 7 and 32 in ex.act_quant['bits']
            seen.add('mixed bit-widths (set_quant_bits)')
        seen |= branches(ex)
        for b in seen:
            SEEN.setdefault(b, name)

        check_replay(lrn)

        state0 = ex.store.state_dict()
        par = run_parity(name, lrn, frozen_names(ex))
        img = ex.buf[lrn.images].cpu().numpy()
        nq = check_quantized_weights(ex, state0)
        orc = oracle_of(ex, lrn)
        w_train = forward_parity(name + ' training forward', ex, orc, state0, img, True)

        cb_ctrl = None
        if ex.train_clusters:
            # negative control: the codebook gradient against centroid indices shifted by one
            worst = 0.0
            for op, (g, mag, idx, alpha, k) in par.codebooks.items():
                cv = op.vars['clusters']
                ref, m = par.codebook_ref(cv.shape, g, mag, (idx + 1) % k, alpha, k)
                got = ex.store.view(cv, ex.G).double()
                worst = max(worst, ((got - ref).abs().max() / m.max().clamp_min(1e-300)).item())
            cb_ctrl = worst / BAR_W
            print('%s: codebook gradient against shifted centroid indices: %.3g x the bar' % (name, cb_ctrl))
            assert cb_ctrl > 10.0, cb_ctrl

        state1 = ex.store.state_dict()
        with ex.standalone_forward():
            ex.forward(training=False)
        torch.cuda.synchronize()
        check_quantized_weights(ex, state1)
        w_eval = forward_parity(name + ' inference forward', ex, orc, state1, img, False)
        ev_ctrl = None
        if extra.get('eval_control'):
            # negative control: an inference reference that normalises with the batch statistics
            ev_ctrl = local_parity(ex, orc, state1, img, True)[0] / BAR_FWD
            print('%s: inference forward against a batch-statistics reference: %.3g x the bar' % (name, ev_ctrl))
            assert ev_ctrl > 10.0, ev_ctrl
        w_teacher = None
        if ex.teacher is not None:
            t = ex.teacher
            t.forward()
            torch.cuda.synchronize()
            w_teacher = forward_parity(name + ' teacher forward', t, oracle_of(t, lrn, student=False),
                                       t.store.state_dict(), img, False)[0]
        secs, peak = time.time() - t0, torch.cuda.max_memory_allocated() / 2 ** 30
        worst = {k: float('%.3g' % v) for k, v in par.worst.items()}
        dx = max([v for k, v in worst.items() if k.endswith(' dx') or ' dx ' in k] + [0.0])
        dw = max([v for k, v in worst.items() if k.startswith('dW ')] + [0.0])
        print('%s: %d backward ops, %d variables compared, %d quantized kernels bit-exact; worst forward %.2e '
              '(inference %.2e, teacher %s), dx %.2e, dW %.2e; level flips %d of %d; %.0f s, peak %.2f GiB' % (
                  name, len(par.checked_ops) - 1, len(ex.store.train_vars), nq, w_train[0], w_eval[0], w_teacher, dx,
                  dw, w_train[1], w_train[2], secs, peak))
        record('sweep_' + name, ops=len(par.checked_ops) - 1, variables=len(ex.store.train_vars), fwd=w_train[0],
               fwd_eval=w_eval[0], fwd_teacher=w_teacher, dx=dx, dw=dw, flips=w_train[1], elements=w_train[2],
               seconds=round(secs), peak_gib=round(peak, 2), codebook_control=cb_ctrl, eval_control=ev_ctrl,
               branches=sorted(seen))
        RAN.add(name)
    finally:
        del lrn
        free()


def test_every_plan_branch_was_reached():
    """Runs last: the configurations above reached every branch in REQUIRED (skipped when only part of them ran)."""
    if not {c[0] for c in CONFIGS} <= RAN:
        pytest.skip('only part of the sweep ran')
    print('plan branches reached: ' + ', '.join('%s (%s)' % kv for kv in sorted(SEEN.items())))
    missing = REQUIRED - set(SEEN)
    assert not missing, 'plan branches never reached: %s' % sorted(missing)
