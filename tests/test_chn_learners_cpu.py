"""The three channel-pruning learners (`chn-pruned-gpu`, `chn-pruned-rmt`, `channel`) without a GPU: their two-model
graph (scopes, conv pairing, maskable kernels, which store holds which variables, the step executor's Add fusion), the
restore of the full model into the pruned one, the cached batches and selection executors, and what train() does, in
order, with the device work replaced by recorders: selection, barriers, restores, masks, saves with their paths,
evaluations, steps and the progress lines."""
import builtins
import importlib
import re

import numpy as np
import pytest

from pocketflow_b200.flags import FLAGS

BUILD = {'chn-pruned-gpu': ('channel_pruning_gpu', 'mobilenet_at_ilsvrc12', 'ilsvrc12_dataset', dict(nb_classes=1001)),
         'chn-pruned-rmt': ('channel_pruning_rmt', 'mobilenet_at_ilsvrc12', 'ilsvrc12_dataset', dict(nb_classes=1001)),
         'channel': ('channel_pruning', 'resnet_at_cifar10', 'cifar10_dataset',
                     dict(resnet_size=20, cp_prune_option='uniform'))}
SAVE_PATHS = ('save_path', 'cpg_save_path', 'cpr_save_path', 'cpr_save_path_eval', 'cpr_save_path_ws',
              'cp_channel_pruned_path')


def build(learner, tmp_path, **flags):
    """the learner as create_learner builds it at batch 2, every save path under tmp_path"""
    module, net, dataset, over = BUILD[learner]
    FLAGS.reset()
    importlib.import_module('pocketflow_b200.learners.%s.learner' % module)
    importlib.reload(importlib.import_module('pocketflow_b200.datasets.' + dataset))
    mod = importlib.reload(importlib.import_module('pocketflow_b200.nets.' + net))
    from pocketflow_b200.learners.learner_utils import create_learner
    FLAGS.learner, FLAGS.batch_size = learner, 2
    for name in SAVE_PATHS:
        setattr(FLAGS, name, str(tmp_path / name / 'model.ckpt'))
    for k, v in dict(over, **flags).items():
        setattr(FLAGS, k, v)
    return create_learner(None, mod.ModelHelper())


@pytest.fixture(autouse=True)
def reset_flags():
    yield
    FLAGS.reset()


@pytest.mark.parametrize('learner,nb_layers', [('chn-pruned-gpu', 15), ('chn-pruned-rmt', 15), ('channel', 22)])
def test_the_full_and_the_pruned_model_side_by_side(tmp_path, learner, nb_layers):
    lrn = build(learner, tmp_path)
    assert (lrn.model_scope_full, lrn.model_scope_prnd, lrn.model_scope) == ('model', 'pruned_model', 'pruned_model')
    assert lrn.nb_layers == nb_layers == len(lrn.conv_ops_full) == len(lrn.conv_ops_prnd)
    for f, p in zip(lrn.conv_ops_full, lrn.conv_ops_prnd):
        assert f.type == p.type == 'Conv2D' and f.name.startswith('model/') and p.name == 'pruned_' + f.name
        assert f.output.shape == p.output.shape
    assert lrn.maskable_vars == [op.vars['kernel'] for op in lrn.conv_ops_prnd]
    if learner == 'chn-pruned-gpu':
        assert lrn.maskable_var_names == [v.name for v in lrn.maskable_vars]
    assert lrn.logits_full.op.name.startswith('model/')
    assert lrn.images is lrn.iterator_train.images and lrn.labels is lrn.iterator_train.labels
    ex = lrn.sess_train
    assert all(v.name.startswith('pruned_model/') for v in ex.store.train_vars + ex.store.other_vars)
    assert ex.maskable == lrn.maskable_vars and ex.train and ex.teacher is None
    full = {v.name for v in lrn.store_full.train_vars + lrn.store_full.other_vars}
    assert full == {'model/' + v.name.split('/', 1)[1] for v in ex.store.train_vars + ex.store.other_vars}
    # only chn-pruned-gpu's step leaves every residual Add unfused (its selection regresses on the step's own outputs)
    assert ex.fuse_add is (learner != 'chn-pruned-gpu')
    assert lrn.compact is None and lrn.sess_step is ex
    assert len(lrn.prune_ratios) == nb_layers


def test_channel_refuses_list_groups_before_building_an_executor(tmp_path, monkeypatch):
    from pocketflow_b200 import engine
    built = []
    init = engine.Executor.__init__
    monkeypatch.setattr(engine.Executor, '__init__', lambda self, *a, **k: (built.append(1), init(self, *a, **k))[1])
    with pytest.raises(ValueError, match='cp_finetune'):
        build('channel', tmp_path, cp_finetune=True)
    with pytest.raises(ValueError, match='cp_list_group'):
        build('channel', tmp_path, cp_prune_option='list', cp_list_group=4)
    assert built == []
    build('channel', tmp_path)
    assert built


@pytest.mark.parametrize('learner', ['chn-pruned-gpu', 'chn-pruned-rmt', 'channel'])
def test_init_from_full_copies_the_full_model_into_the_pruned_one(tmp_path, capsys, learner):
    lrn = build(learner, tmp_path)
    ex = lrn.sess_train
    ex.store.P.mul_(2.0).add_(1.0)
    ex.store.O.add_(3.0)
    ex.step_count = 7
    if learner == 'chn-pruned-gpu':
        ex.MASK.zero_()
        lrn.channels_chosen = True
    lrn.init_from_full()
    assert capsys.readouterr().out == ('no pre-trained checkpoint in %s: the full model keeps its seed initialisation '
                                       '(synthetic run)\n' % (tmp_path / 'save_path'))
    full, prnd = lrn.store_full.state_dict(), ex.store.state_dict()
    assert len(full) == len(prnd)
    for k, v in full.items():
        assert np.array_equal(prnd['pruned_' + k], v), k
    if learner == 'chn-pruned-gpu':
        assert float(ex.MASK.min()) == float(ex.MASK.max()) == 1.0
        assert ex.step_count == 0 and lrn.channels_chosen is False
    else:
        assert ex.step_count == 7
    # with a pre-trained checkpoint the full model is restored from it first
    from pocketflow_b200.learners.abstract_learner import save_checkpoint
    want = {k: v + 0.5 for k, v in full.items()}
    save_checkpoint(FLAGS.save_path, want, 3)
    lrn.init_from_full()
    assert 'model restored from %s-3.npz' % FLAGS.save_path in capsys.readouterr().out
    prnd = ex.store.state_dict()
    for k, v in want.items():
        assert np.array_equal(lrn.store_full.state_dict()[k], v) and np.array_equal(prnd['pruned_' + k], v), k


@pytest.mark.parametrize('learner,flags,count', [('chn-pruned-rmt', dict(cpr_nb_smpls=5), 3),      # ceil(5 / 2)
                                                 ('channel', dict(cp_nb_batches=4), 4)])
def test_cached_batches_and_selection_executors(tmp_path, learner, flags, count):
    lrn = build(learner, tmp_path, **flags)
    cached = lrn.cache_batches()
    assert len(cached) == count and all(c.shape == tuple(lrn.images.shape) for c in cached)
    ex_f, ex_p = lrn.selection_executors()
    assert ex_f.store is lrn.store_full and ex_p.store is lrn.sess_train.store
    assert ex_f.buf[lrn.images] is ex_p.buf[lrn.images]
    for ex_ in (ex_f, ex_p):
        assert not ex_.train and not ex_.fuse_add and not ex_.update_moving_stats
    assert ex_f.logits_t is lrn.logits_full and ex_p.logits_t is lrn.logits_prnd


def run_train(lrn, tmp_path, monkeypatch):
    """train(nb_iters=5) at save_step = summ_step = 2 with the device work replaced by recorders"""
    FLAGS.save_step, FLAGS.summ_step = 2, 2
    ev, tmp = [], str(tmp_path)

    def step():
        ev.append('step')
        lrn.sess_train.step_count += 1
    for name in ('choose_channels', 'init_from_full', 'evaluate', 'auto_barrier', 'init_masks'):
        setattr(lrn, name, lambda *a, name=name, **k: ev.append(name))
    lrn.train_step = step
    lrn.restore_model = lambda path, **k: ev.append(('restore', path.replace(tmp, '<tmp>')))
    lrn.sess_train.fetch_losses = lambda: (ev.append('fetch_losses'), dict(loss=1.5))[1]

    def record_print(*args, **kw):
        s = ' '.join(str(a) for a in args).replace(tmp, '<tmp>')
        s = re.sub(r'speed = [0-9.]+', 'speed = <s>', s)
        ev.append(('print', re.sub(r'\(channel selection\): [0-9.]+', '(channel selection): <t>', s)))
    monkeypatch.setattr(builtins, 'print', record_print)
    lrn.train(nb_iters=5)
    monkeypatch.undo()
    return ev


def saved(path):
    return ('print', 'model saved to <tmp>/%s' % path)


def progress(it, lr, label):
    return ('print', 'iter #%d: lr = %s | loss = 1.5000e+00 | %s = 0.0000e+00 | speed = <s> pics / sec' % (it, lr, label))


def fine_tune(flag, label, lrs):
    """the steps of train(nb_iters=5) and what the primary worker does around them"""
    return ['step', 'step', 'fetch_losses', progress(2, lrs[0], label),
            saved('%s/model.ckpt-2.npz' % flag), 'evaluate', 'auto_barrier',
            'step', 'step', 'fetch_losses', progress(4, lrs[1], label),
            saved('%s/model.ckpt-4.npz' % flag), 'evaluate', 'auto_barrier',
            'step', saved('%s/model.ckpt-5.npz' % flag)]


MBV1_LR = ('9.3750e-04', '9.3750e-04')       # the nets' schedules at iterations 1 and 3, scaled to batch 2
RN20_LR = ('1.5625e-03', '1.5625e-03')


def test_cpg_train_selects_on_every_rank_then_saves_and_evaluates_before_the_first_step(tmp_path, monkeypatch):
    lrn = build('chn-pruned-gpu', tmp_path)
    ev = run_train(lrn, tmp_path, monkeypatch)
    want = ['init_from_full', 'choose_channels', saved('cpg_save_path/model.ckpt-0.npz'), 'evaluate', 'auto_barrier']
    want += fine_tune('cpg_save_path', 'pr_msk', MBV1_LR) + ['evaluate']
    assert ev == want


@pytest.mark.parametrize('warm', [False, True])
def test_cpr_train_restores_the_selection_and_writes_the_eval_checkpoint_last(tmp_path, monkeypatch, warm):
    lrn = build('chn-pruned-rmt', tmp_path, cpr_warm_start=warm)
    ev = run_train(lrn, tmp_path, monkeypatch)
    want = [] if warm else ['choose_channels', ('print', 'time (channel selection): <t> (s)'), 'auto_barrier']
    want += [('restore', '<tmp>/cpr_save_path_ws/model.ckpt'), 'init_masks',
             saved('cpr_save_path/model.ckpt-0.npz'), 'evaluate', 'auto_barrier']
    want += fine_tune('cpr_save_path', 'pr_krn', MBV1_LR)
    want += [saved('cpr_save_path_eval/model.ckpt.npz'), 'evaluate']
    assert ev == want


def test_channel_train_fine_tunes_straight_after_the_restored_selection(tmp_path, monkeypatch):
    lrn = build('channel', tmp_path)
    ev = run_train(lrn, tmp_path, monkeypatch)
    want = ['choose_channels', ('print', 'time (channel selection): <t> (s)'), 'auto_barrier',
            ('restore', '<tmp>/cp_channel_pruned_path/model.ckpt'), 'init_masks']
    want += fine_tune('save_path', 'pr_krn', RN20_LR) + ['evaluate']
    assert ev == want
