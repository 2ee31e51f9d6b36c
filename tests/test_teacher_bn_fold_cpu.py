"""Which inference-mode batch norms the executor folds into the epilogue of the tensor-core conv that produces their
input (Executor._plan_bn_fold), checked on the CPU: the plan is computed as a GPU executor computes it, no kernel runs.

The ResNet-50 teacher has 49 BNs: 48 read a tensor-core conv's output (32 directly, 16 through the residual Add fused
into conv3) and one reads the stem's max-pool.  Training executors fold nothing."""
import pytest
import torch

import bench
from pocketflow_b200 import graph as G
from pocketflow_b200.engine import Executor
from pocketflow_b200.flags import FLAGS


@pytest.fixture(autouse=True)
def _flags_back_to_defaults():
    """the workloads' flag settings do not leak into the tests that run after these"""
    yield
    FLAGS.reset()


def eval_executor(workload):
    mod = bench.setup_flags(workload, 1)
    mh = mod.ModelHelper()
    g = G.Graph()
    with g.as_default():
        with G.variable_scope('data'):
            im, _ = mh.build_dataset_train().get_next()
        with G.variable_scope('model'):
            out = mh.forward_eval(im)
    return Executor(g, im, out, torch.device('cpu'), train=False)


def fold_on_gpu(ex):
    """the fold set of the same plan on a GPU (the method only reads the plan)"""
    cpu = ex.device
    ex.device = torch.device('cuda')
    try:
        return ex._plan_bn_fold()
    finally:
        ex.device = cpu


def producer(ex, bn):
    """the tensor-core conv whose epilogue writes the BN's input, or None"""
    src = ex._root(bn.inputs[0]).op
    for conv, (add, _) in ex.fused_add.items():
        if add is src:
            return conv
    return src if src in ex.tc and src not in ex.im2col else None


@pytest.mark.parametrize('workload,n_bn,n_fold', [('resnet50_uq8_dst_b128', 49, 48),
                                                  ('resnet20_uq8_dst_b256', None, None),
                                                  ('mobilenet_cpg50_b256', None, None)])
def test_fold_set_of_the_eval_graphs(workload, n_bn, n_fold):
    ex = eval_executor(workload)
    assert ex.bn_fold == {}, 'an executor planned on the CPU folds nothing (golden plan snapshots)'
    fold = fold_on_gpu(ex)
    bns = [op for op in ex.ops if op.type == 'FusedBatchNorm']
    assert all(not bn.attrs['training'] for bn in bns)
    if n_bn is not None:
        assert (len(bns), len(fold)) == (n_bn, n_fold)
    assert len(set(fold.values())) == len(fold)
    for conv, bn in fold.items():
        assert producer(ex, bn) is conv, (conv.name, bn.name)
        assert bn not in ex.bn_add and bn not in ex.bn_gather
    # every BN left out has no tensor-core producer to fold into
    for bn in bns:
        if bn not in fold.values():
            assert producer(ex, bn) is None, bn.name
    assert fold, workload


def test_training_executors_fold_nothing():
    mod = bench.setup_flags('resnet20_uq8_dst_b256', 1)
    mh = mod.ModelHelper()
    g = G.Graph()
    with g.as_default():
        with G.variable_scope('data'):
            im, lab = mh.build_dataset_train().get_next()
        with G.variable_scope('model'):
            out = mh.forward_train(im)
            tv = [v for v in g.variables.values() if v.name.startswith('model/') and v.trainable]
            loss, _ = mh.calc_loss(lab, out, tv)
    ex = Executor(g, im, out, torch.device('cpu'), train=True, loss=loss, labels=lab,
                  optimizer=dict(kind='momentum', momentum=0.9))
    assert fold_on_gpu(ex) == {}
