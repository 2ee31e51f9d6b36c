"""Planner invariants of engine.Executor, checked symbolically on the CPU (no kernels run):

* gradient-buffer sharing through residual Adds (in-place accumulation through identity shortcuts): when an op's
  backward runs, the buffer holding the gradient of its output contains exactly the contributions of that output's
  consumers — no more (a foreign writer ran too early), no fewer (a reader ran too early);
* dy operand planes: the BatchNorm chosen to emit a conv's dy planes is the LAST writer of that gradient before the
  conv's backward, and what it leaves in the buffer is the conv output's complete gradient;
* x operand planes: a BN output's fp32 copy is dropped only when every consumer reads planes.
"""
import pytest
import torch

from pocketflow_b200 import graph as G
from pocketflow_b200.engine import Executor
from pocketflow_b200.flags import FLAGS
from support import expected_contributions, grad_inputs


def build(net, **flags):
    FLAGS.reset()
    import importlib
    mod = importlib.import_module('pocketflow_b200.nets.' + net)
    for k, v in flags.items():
        setattr(FLAGS, k, v)
    mh = mod.ModelHelper()
    g = G.Graph()
    with g.as_default():
        with G.variable_scope('data'):
            it = mh.build_dataset_train()
            im, lab = it.get_next()
        with G.variable_scope('model'):
            out = mh.forward_train(im)
            tv = [v for v in g.variables.values() if v.name.startswith('model/') and v.trainable]
            loss, _ = mh.calc_loss(lab, out, tv)
    return Executor(g, im, out, torch.device('cpu'), train=True, loss=loss, labels=lab,
                    optimizer=dict(kind='momentum', momentum=0.9))


@pytest.mark.parametrize('net,flags', [('resnet_at_cifar10', dict(resnet_size=20, batch_size=4)),
                                       ('resnet_at_ilsvrc12', dict(resnet_size=50, batch_size=2)),
                                       ('resnet_at_ilsvrc12', dict(resnet_size=18, batch_size=2)),
                                       ('mobilenet_at_ilsvrc12', dict(batch_size=2, nb_classes=1001)),
                                       ('lenet_at_cifar10', dict(batch_size=4))])
def test_gradient_buffers_hold_exactly_the_consumers_contributions(net, flags):
    ex = build(net, **flags)
    memo, state = {}, {}
    state[ex.gkey(ex.loss.ce[1])] = {'loss'}                             # softmax-CE writes dL/dlogits first
    ran = []
    dy_plane_state = {}
    for op in reversed(ex.ops):
        if op.type == 'Placeholder':
            continue
        k = ex.gkey(op.output)
        if k not in state:
            continue                                                     # no gradient flows here
        if not (op.type in ('Reshape', 'Identity') or op in ex.fused_into):
            want = expected_contributions(ex, op.output, memo)
            assert state[k] == want, '%s: buffer holds %s, expected %s' % (
                op.name, sorted(getattr(o, 'name', o) for o in state[k]), sorted(getattr(o, 'name', o) for o in want))
            if op in getattr(ex, 'conv_dy_planes', {}):
                # the planes were emitted by a BN backward that ran earlier: they must hold this same complete gradient
                bn = [b for b, pl in ex.bn_gplanes.items() if pl is ex.conv_dy_planes[op]][0]
                assert dy_plane_state[bn] == want, op.name
        for t in grad_inputs(ex, op):
            kk = ex.gkey(t)
            state[kk] = (state[kk] | {op}) if kk in state else {op}     # accumulate / first write
            if op.type == 'FusedBatchNorm' and op in getattr(ex, 'bn_gplanes', {}):
                dy_plane_state[op] = set(state[kk])                      # what the emitted planes contain
        ran.append(op)
    # every residual Add shares its buffer with all of its inputs (no copy kernels) in the ResNets
    adds = [op for op in ex.ops if op.type == 'Add']
    for a in adds:
        assert all(ex.gkey(t) is ex.gkey(a.output) for t in a.inputs), a.name


@pytest.mark.parametrize('net,flags', [('resnet_at_cifar10', dict(resnet_size=20, batch_size=4)),
                                       ('resnet_at_ilsvrc12', dict(resnet_size=50, batch_size=2)),
                                       ('mobilenet_at_ilsvrc12', dict(batch_size=2, nb_classes=1001))])
def test_fp32_copy_of_a_bn_output_is_dropped_only_when_every_consumer_reads_planes(net, flags):
    ex = build(net, **flags)
    assert ex.xplanes, 'no operand planes planned'
    for bn_op, planes in ex.xplanes.items():
        outs = [bn_op.output] + [c.output for c in ex._consumers(bn_op.output) if c in ex.fused_into]
        consumers = [c for t in outs for c in ex._consumers(t) if not (c in ex.fused_into and ex.fused_into[c] is bn_op)]
        all_planes = all(c in ex.tc_wgrad and c not in ex.im2col for c in consumers)
        assert ex.bn_need_f32[bn_op] == (not all_planes), bn_op.name
        assert planes.numel == bn_op.output.numel
    n_dy = len(ex.conv_dy_planes)
    assert n_dy > 0 and all(op in ex.tc_wgrad for op in ex.conv_dy_planes)


def test_unsafe_identity_sharing_is_refused():
    """A tensor that is consumed again AFTER the residual Add (so one of its gradient writers would run BEFORE the
    readers of the Add's gradient) must keep its own gradient buffer; the symbolic check still holds."""
    FLAGS.reset()
    import pocketflow_b200.datasets.cifar10_dataset  # noqa: F401  (flags)
    g = G.Graph()
    with g.as_default():
        im = G.placeholder((2, 8, 8, 64), 'images')
        lab = G.placeholder((2, 10), 'labels')
        with G.variable_scope('model'):
            a = G.conv2d(im, 64, 3, padding='same', use_bias=False)
            b = G.conv2d(G.relu(G.batch_normalization(a, training=True)), 64, 3, padding='same', use_bias=False)
            s = G.add(b, a)                                   # `a` feeds the BN, the Add ...
            c = G.conv2d(a, 64, 1, use_bias=False)            # ... and is consumed AGAIN later in forward order
            t = G.add(s, c)
            out = G.dense(G.reduce_mean_hw(G.relu(G.batch_normalization(t, training=True))), 10)
            loss = G.softmax_cross_entropy(lab, out)
    ex = Executor(g, im, out, torch.device('cpu'), train=True, loss=loss, labels=lab,
                  optimizer=dict(kind='momentum', momentum=0.9))
    add_s = s.op
    a_root = ex._root(a)
    assert ex.gkey(a_root) is not ex.gkey(add_s.output), 'unsafe in-place sharing was planned'
    assert ex.gkey(b) is ex.gkey(add_s.output)                # the single-consumer branch still shares
    # and the general invariant holds for this graph too
    memo, state = {}, {ex.gkey(ex.loss.ce[1]): {'loss'}}
    for op in reversed(ex.ops):
        if op.type == 'Placeholder' or ex.gkey(op.output) not in state:
            continue
        if not (op.type in ('Reshape', 'Identity') or op in ex.fused_into):
            assert state[ex.gkey(op.output)] == expected_contributions(ex, op.output, memo), op.name
        for x in grad_inputs(ex, op):
            kk = ex.gkey(x)
            state[kk] = (state[kk] | {op}) if kk in state else {op}


def test_param_store_frozen_ranges_and_checked_restores():
    """ParamStore: frozen variables (the optimizer's var_list excludes them — the non-uniform learner's modes) form
    their own ranges; a restore counts what it found and refuses checkpoints that match nothing / not everything."""
    import numpy as np
    from pocketflow_b200.engine import ParamStore
    init = lambda rng, shape: rng.standard_normal(shape).astype(np.float32)
    mk = lambda name, shape, trainable=True: G.Variable(name + ':0', shape, init, trainable)
    k1, k2, c1, c2 = mk('m/conv/kernel', (3, 3, 4, 8)), mk('m/conv_1/kernel', (1, 1, 8, 8)), \
        mk('m/conv/Conv2D/nonuniform_quantize/clusters', (16,)), mk('m/conv_1/Conv2D/nonuniform_quantize/clusters', (16,))
    gam, mm = mk('m/bn/gamma', (8,)), mk('m/bn/moving_mean', (8,), trainable=False)
    wd = {k1: 5e-4, k2: 5e-4, c1: 5e-4, c2: 5e-4}
    st = ParamStore([k1, c1, gam, k2, c2, mm], torch.device('cpu'), wd, frozen=[c1, c2])
    # kernels (wd, live) | codebooks (wd, frozen) | gamma (no wd): three ranges, the middle one skipped by the optimizer
    assert len(st.ranges) == 3 and len(st.frozen_ranges) == 1
    (s, e), = st.frozen_ranges
    assert {st.offset[c1], st.offset[c2]} == {s, s + 16} and e - s == 32
    assert all(not (s <= st.offset[v] < e) for v in (k1, k2, gam))
    assert [r for r in st.ranges if (r[0], r[1]) == (s, e)][0][3] == 5e-4        # still weight-decayed (loss term)
    state = st.state_dict()
    assert set(state) == {v.name for v in (k1, k2, c1, c2, gam, mm)}
    # checked restores
    assert st.load_state_dict(state, strict=True) == (5, 5)
    no_clusters = {k: v for k, v in state.items() if 'clusters' not in k}
    with pytest.raises(ValueError):
        st.load_state_dict(no_clusters, strict=False, require='all')
    assert st.load_state_dict(no_clusters, strict=False, require='all', optional=('/clusters',)) == (3, 3)
    with pytest.raises(ValueError):
        st.load_state_dict({'other/' + k: v for k, v in state.items()}, strict=False, require='any')
    with pytest.raises(ValueError):
        st.load_state_dict({k1.name: np.zeros(7, np.float32)}, strict=False)      # wrong size
    with pytest.raises(KeyError):
        st.load_state_dict(no_clusters, strict=True)


def test_nuq_graph_edit_creates_the_reference_cluster_variables():
    """NonUniformQuantization.insert_quant_op_for_weights: one trainable `clusters` variable per quantized op, under
    <model scope>/<op name without its scope>/nonuniform_quantize/ (learners/nonuniform_quantization/utils.py:180, :297),
    2^bits entries — or 2^cap when the RL bit search may change the bit-width."""
    FLAGS.reset()
    import importlib
    importlib.import_module('pocketflow_b200.learners.nonuniform_quantization.learner')
    from pocketflow_b200.learners.nonuniform_quantization.utils import NonUniformQuantization
    mod = importlib.import_module('pocketflow_b200.nets.resnet_at_cifar10')
    FLAGS.resnet_size = 8
    mh = mod.ModelHelper()
    for cap, size in ((None, 16), (6, 64)):
        g = G.Graph()
        with g.as_default():
            with G.variable_scope('data'):
                im, _ = mh.build_dataset_train().get_next()
            with G.variable_scope('model'):
                mh.forward_train(im)
                before = set(g.variables)
                nq = NonUniformQuantization(g, 256, False, 'quantile', 'split', codebook_bits_cap=cap)
                ops_ = nq.search_matmul_op(False)
                nq.insert_quant_op_for_weights({o.name: 4 for o in ops_})
        new = sorted(set(g.variables) - before)
        assert len(new) == len(ops_) == 9
        for o in ops_:
            v = o.vars['clusters']
            assert v.name == 'model/' + o.name.split('/', 1)[1] + '/nonuniform_quantize/clusters:0' and v.name in new
            assert v.trainable and v.shape == (size,)
        spec = nq.weight_quant_spec()
        assert spec['kind'] == 'nonuniform' and spec['bits'] == [4] * 9 and spec['train_clusters'] is False
    FLAGS.reset()


def test_channel_pruned_learner_builds_the_full_and_the_pruned_model_side_by_side(tmp_path):
    """ChannelPrunedGpuLearner's graph (learners/channel_pruning_gpu/learner.py:207-229, :347-352), on the CPU (planning
    only): the full model under 'model', the pruned one under 'pruned_model', their Conv2D ops paired by index, the
    maskable variables = the pruned model's Conv2D kernels (depthwise excluded), the per-layer ratios of both protocols."""
    import importlib
    FLAGS.reset()
    import pocketflow_b200.datasets.ilsvrc12_dataset as D
    importlib.reload(D)
    M = importlib.reload(importlib.import_module('pocketflow_b200.nets.mobilenet_at_ilsvrc12'))
    L = importlib.import_module('pocketflow_b200.learners.channel_pruning_gpu.learner')
    FLAGS.batch_size, FLAGS.nb_classes, FLAGS.cpg_prune_ratio = 2, 1001, 0.3
    lrn = L.ChannelPrunedGpuLearner(None, M.ModelHelper())
    assert lrn.model_scope == 'pruned_model' and lrn.nb_layers == 15
    assert len(lrn.conv_ops_full) == len(lrn.conv_ops_prnd) == 15
    for f, p in zip(lrn.conv_ops_full, lrn.conv_ops_prnd):
        assert f.name.startswith('model/') and p.name == 'pruned_' + f.name and f.output.shape == p.output.shape
        assert 'depthwise' not in p.name
    assert lrn.maskable_var_names == [op.vars['kernel'].name for op in lrn.conv_ops_prnd]
    assert lrn.prune_ratios == [0.0] + [0.3] * 13 + [0.0]                  # head and tail skipped (:452-454)
    # the training executor only holds the pruned model; the full model has its own store with the 'model/' names
    assert all(v.name.startswith('pruned_model/') for v in lrn.sess_train.store.train_vars)
    full_names = {v.name for v in lrn.store_full.train_vars + lrn.store_full.other_vars}
    assert full_names == {'model/' + v.name.split('/', 1)[1]
                          for v in lrn.sess_train.store.train_vars + lrn.sess_train.store.other_vars}
    assert not lrn.sess_train.fused_add and lrn.channels_chosen is False
    # 'list' protocol: one ratio per Conv2D layer from a file (:455-458)
    ratios = [0.0, 0.5, 0.25] + [0.1] * 12
    (tmp_path / 'r.txt').write_text(','.join(str(r) for r in ratios) + '\n')
    FLAGS.cpg_prune_ratio_type, FLAGS.cpg_prune_ratio_file = 'list', str(tmp_path / 'r.txt')
    assert L.ChannelPrunedGpuLearner(None, M.ModelHelper()).prune_ratios == ratios
    FLAGS.cpg_prune_ratio_type = 'bogus'
    with pytest.raises(ValueError):
        L.ChannelPrunedGpuLearner(None, M.ModelHelper())
    FLAGS.reset()


def test_learner_restore_helpers(tmp_path, capsys):
    """AbstractLearner.restore_model / restore_for_eval / eval_nb_iters against a CPU parameter store: the latest
    checkpoint beside the path is loaded and counted; evaluate() only restores under --exec_mode eval (while training, the
    executor already holds what was saved); the iteration count is the reference's ceil(nb_smpls_eval / batch_size_eval)."""
    import numpy as np
    from types import SimpleNamespace
    import pocketflow_b200.datasets.cifar10_dataset  # noqa: F401  (declares nb_smpls_eval / batch_size_eval)
    from pocketflow_b200.engine import ParamStore
    from pocketflow_b200.learners.abstract_learner import AbstractLearner, save_checkpoint
    FLAGS.reset()
    init = lambda rng, shape: rng.standard_normal(shape).astype(np.float32)
    vs = [G.Variable('model/a/kernel:0', (4, 4), init), G.Variable('model/a/bias:0', (4,), init)]
    st = ParamStore(vs, torch.device('cpu'))
    me = SimpleNamespace(sess_train=SimpleNamespace(store=st), iterator_train=SimpleNamespace(batch_size=32))
    me.restore_model = lambda path, **kw: AbstractLearner.restore_model(me, path, **kw)
    path = str(tmp_path / 'ck' / 'model.ckpt')
    with pytest.raises(ValueError, match='no checkpoint'):
        AbstractLearner.restore_model(me, path)
    want = {k: v + 1.0 for k, v in st.state_dict().items()}
    save_checkpoint(path, want, 7)
    fn = AbstractLearner.restore_model(me, path)
    assert fn.endswith('-7.npz') and '2 of 2 trainable variables' in capsys.readouterr().out
    assert all(np.array_equal(st.state_dict()[k], want[k]) for k in want)
    # restore_for_eval: a no-op while training, a restore under --exec_mode eval
    st.P.zero_()
    FLAGS.exec_mode = 'train'
    AbstractLearner.restore_for_eval(me, path)
    assert float(st.P.abs().sum()) == 0.0
    FLAGS.exec_mode = 'eval'
    AbstractLearner.restore_for_eval(me, path)
    assert all(np.array_equal(st.state_dict()[k], want[k]) for k in want)
    # iteration count
    FLAGS.nb_smpls_eval, FLAGS.batch_size_eval, FLAGS.data_dir_local = 10000, 96, None
    assert AbstractLearner.eval_nb_iters(me) == 105 and AbstractLearner.eval_nb_iters(me, 3) == 3
    FLAGS.data_dir_local = '/data'                                     # real data is read at the step's batch size
    assert AbstractLearner.eval_nb_iters(me) == 313
    FLAGS.reset()
