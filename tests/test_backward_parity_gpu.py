"""The backward pass and the optimizer update of the benchmarked training steps, layer by layer, against float64.

The step tests compare gradients with a free-running oracle only where no activation level or ReLU gate differs
(test_bench_configs_gpu); at 8-bit activations that never happens, so the wiring of the backward pass — which dy planes
a dgrad reads, which levels a wgrad is fed, whether a residual gradient is accumulated, where the STE, the weight decay
and the momentum mask land — had no graph-level check.  Here one eager step runs with the executor's backward tapped
(no change to the engine: its `grad_of` / `grad_target` and the lowerings' wgrad / dgrad / BN backward are wrapped on
the instance), synchronising at every op boundary, and the backward is teacher-forced:
  * LOCAL: every op that has a gradient is rebuilt alone in float64 through autograd, with StepOracle's semantics for
    its type, from the device's own forward inputs as the op read them (operand planes as hi + lo, activation levels as
    scale x level, quantized weights from ex.QW) and the device's own upstream gradient as the op read it (the fp32
    gradient, or the dy planes of the BN backward where the lowering reads those).  Every discrete decision comes from
    the device: ReLU masks from the fp32 chain ((x - mean) * rstd) * gamma + beta on the saved statistics (bn_chain),
    ReLU masks of convolutions with a fused activation from their own output, the max-pool argmax, the dropout mask and
    the teacher's logits — so no flipped level or gate can make a difference and no comparison is gated on one.
    Bars: a gradient contribution to an activation within 2e-5 of max|float64|; a variable's gradient in ex.G after
    the step (split-K reduce, STE) within 2e-5 of the largest sum of |terms|; the dy operand a convolution's kernels
    read is bit for bit the gradient it was handed (times its ReLU mask), or the bf16 split of it.
  * CHAIN: the gradient each op read equals the sum of the contributions its output's consumers wrote, by the graph's
    semantics (Add / Reshape / Identity / a fused activation pass their gradient through), within 1e-6 of the sum of
    |terms| per element: this covers the plan-time Add aliases, the in-place shortcut accumulators, the dy planes that
    live in the fp32 gradient buffer's memory and the passthrough ops.
  * OPTIMIZER: given the device's final G and the state before the step, P, S1 and S2 are bit-exact per variable
    against oracle.pf_oracle.adam_step / momentum_step with the loss's own weight decay, the step's masks and the
    frozen codebooks; the BN moving statistics within 1e-6 of the float64 update from the device's batch statistics.
  * COVERAGE: every op of the executor that has a gradient is checked locally and every trainable variable's gradient
    is compared, except what EXEMPT lists with its reason.
  * CONTROLS (default workload, once): a dgrad referenced with the unquantized kernel, one convolution's gradient
    swapped with a same-shaped neighbour's and a dropped accumulate at a residual each miss their bar by more than 10x.
A second test checks that the multi-stream schedule does not change a bit of the benchmarked step (the tap above
synchronises, so it cannot see a side-stream race).
Worst errors go to parity_flips.json in $PF_PARITY_DIR (default: the system temp directory); DESIGN.md §4 quotes them.
"""

import numpy as np
import pytest
import torch

from support import free, run_parity

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
F32 = np.float32




def build(workload, batch, monkeypatch, **flags):
    import bench
    monkeypatch.setenv('PF_POISON', '1')
    if flags:
        net, size, learner, over, descr = bench.WORKLOADS[workload]
        monkeypatch.setitem(bench.WORKLOADS, workload, (net, size, learner, dict(over, **flags), descr))
    return bench.build_learner(workload, 1, batch)


@pytest.mark.parametrize('workload,batch,flags', [
    ('resnet50_uq8_dst_b128', 128, {}),
    ('resnet20_uq8_dst_b256', 256, {}),
    ('resnet50_uq8_dst_b128', 2, {'uql_activation_bits': 32}),
    ('resnet50_ws50_dst_b128', 2, {}),
    ('resnet50_nuq4_dst_b128', 2, {}),
    ('mobilenet_cpg50_b256', 2, {}),
    ('lenet_uq8_b128', 2, {}),
], ids=['resnet50_uq8_b128', 'resnet20_uq8_b256', 'resnet50_w8a32_b2', 'resnet50_ws50_b2', 'resnet50_nuq4_b2',
        'mobilenet_cpg50_b2', 'lenet_uq8_b2'])
def test_backward_and_update_match_float64_layer_by_layer(workload, batch, flags, monkeypatch):
    import bench
    lrn = build(workload, batch, monkeypatch, **flags)
    ex = lrn.sess_train
    frozen = ()
    if bench.WORKLOADS[workload][2] == 'non-uniform':
        frozen = tuple(op.vars['clusters'].name for op in ex.wq_ops if 'clusters' in op.vars)
        assert frozen and not ex.train_clusters
    name = '%s_b%d' % (workload.rsplit('_b', 1)[0], batch) + ''.join('_%s%s' % kv for kv in sorted(flags.items()))
    controls = workload == 'resnet50_uq8_dst_b128' and batch == 128 and not flags
    if controls:
        assert ex.act_lv and ex.w_lv and ex.bn_gplanes and any(ex.bn_gplanes_only.values())
    try:
        run_parity(name, lrn, frozen, controls)
    finally:
        del lrn, ex
        free()


def test_mobilenet_v2_uniform_backward_matches_float64_layer_by_layer(monkeypatch):
    """the linear-bottleneck BN + residual (bn_add) and dropout backward"""
    import importlib
    from pocketflow_b200.flags import FLAGS
    monkeypatch.setenv('PF_POISON', '1')
    FLAGS.reset()
    import pocketflow_b200.datasets.ilsvrc12_dataset as D
    importlib.reload(D)
    from pocketflow_b200.nets import mobilenet_at_ilsvrc12 as M
    importlib.reload(M)
    from pocketflow_b200.learners.learner_utils import create_learner
    import pocketflow_b200.learners.uniform_quantization.learner  # noqa: F401
    FLAGS.batch_size, FLAGS.learner, FLAGS.nb_classes, FLAGS.mobilenet_version = 2, 'uniform', 1001, 2
    FLAGS.uql_weight_bits, FLAGS.uql_activation_bits = 8, 8
    FLAGS.uql_use_buckets, FLAGS.uql_bucket_type = True, 'channel'
    lrn = create_learner(None, M.ModelHelper())
    ex = lrn.sess_train
    assert len(ex.bn_add) == 10 and len(ex.dropout) == 1
    try:
        run_parity('mobilenet_v2_uq8_b2', lrn)
    finally:
        del lrn, ex
        free()


def test_overlapped_step_is_bit_identical_to_serial_at_the_benchmarked_batch(monkeypatch):
    """resnet50_uq8_dst_b128 at batch 128: one eager step with PF_OVERLAP=0 and one with PF_OVERLAP=1 (teacher forward
    and weight gradients on side streams) from the same state and batch: P, O, S1, S2 and the losses bit for bit"""
    import bench
    out, start = [], None
    for overlap in ('0', '1'):
        monkeypatch.setenv('PF_OVERLAP', overlap)
        lrn = bench.build_learner('resnet50_uq8_dst_b128', 1, 128)
        ex = lrn.sess_train
        assert ex.overlap == (overlap == '1') and ex._graph is None
        if start is None:
            images, labels = lrn.iterator_train.next_batch()
            start = (ex.store.P.cpu(), ex.store.O.cpu(), ex.teacher.store.P.cpu(), ex.teacher.store.O.cpu(),
                     images.clone(), labels.clone())
        else:
            ex.store.P.copy_(start[0])
            ex.store.O.copy_(start[1])
            ex.teacher.store.P.copy_(start[2])
            ex.teacher.store.O.copy_(start[3])
            for f in ex.teacher.store.listeners:
                f()
        ex.buf[lrn.images].copy_(start[4])
        ex.buf[lrn.labels].copy_(start[5])
        ex.run_step(lrn.lrn_rate(0))
        torch.cuda.synchronize()
        out.append((ex.store.P.cpu(), ex.store.O.cpu(), ex.S1.cpu(), ex.S2.cpu(), ex.fetch_losses()))
        del lrn, ex                                   # one benchmarked learner on the device at a time
        free()
    (p0, o0, m0, v0, l0), (p1, o1, m1, v1, l1) = out
    assert torch.equal(p0, p1) and torch.equal(o0, o1) and torch.equal(m0, m1) and torch.equal(v0, v1)
    assert all(F32(l0[k]).view(np.uint32) == F32(l1[k]).view(np.uint32) for k in l0), (l0, l1)
