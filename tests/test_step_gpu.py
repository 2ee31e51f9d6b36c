"""Full-step parity: the learner-level CUDA step against the CPU oracle step (oracle/step_oracle.py)
from identical state on the same batch.  Bar (north star): per-step losses and updated weights
within 1e-5 relative fp32; quantized weights bit-exact."""
import numpy as np
import pytest
import torch

from oracle.step_oracle import StepOracle
from oracle import pf_oracle as O
from pocketflow_b200.flags import FLAGS
from support import rel

pytestmark = pytest.mark.gpu
F32 = np.float32


def make_uq_learner(resnet_size=8, batch=16, w_bits=8, a_bits=8, dst=True, buckets=True):
    FLAGS.reset()
    from pocketflow_b200.nets import resnet_at_cifar10 as R
    from pocketflow_b200.learners.uniform_quantization.learner import UniformQuantLearner
    FLAGS.resnet_size, FLAGS.batch_size = resnet_size, batch
    FLAGS.uql_weight_bits, FLAGS.uql_activation_bits = w_bits, a_bits
    FLAGS.uql_use_buckets, FLAGS.uql_bucket_type = buckets, 'channel'
    FLAGS.enbl_dst = dst
    return UniformQuantLearner(None, R.ModelHelper())


def oracle_for(learner):
    ex = learner.sess_train
    teacher = None
    if ex.teacher is not None:
        teacher = StepOracle(ex.teacher.ops, ex.teacher.logits_t, learner.images)
    return StepOracle(ex.ops, ex.logits_t, learner.images, learner.labels, ex.loss,
                      ex.weight_quant, ex.act_quant, teacher)


def relu_mask_mismatches(ex, orc, state, img):
    """# of ReLU outputs whose sign pattern differs between the CUDA forward and the oracle forward.
    ReLU'(0) is a derivative discontinuity: one element whose pre-activation is within fp32
    summation-order noise (1e-7) of zero flips the mask and moves every upstream gradient by ~1e-2 of
    its max-norm, so gradient parity is only meaningful on batches where no such element exists."""
    params = {k: torch.from_numpy(v.copy()) for k, v in state.items()}
    val = orc.forward(params, torch.from_numpy(img), True)
    bad = 0
    for op in ex.ops:
        if op.type in ('Relu', 'Relu6'):
            a = ex.T(op.output).cpu().numpy() > 0
            b = val[op.output.name].numpy() > 0
            bad += int((a != b).sum())
    return bad


@pytest.mark.parametrize('dst,buckets', [(True, True), (False, False)])
def test_uq_step_matches_oracle(dst, buckets, monkeypatch):
    """W8 (per-channel / per-layer), activations at the reference's default 32 bits (the quantizer
    chain still runs, SURVEY A.6-2): losses within 1e-5, quantized weights bit-exact, gradients and
    updated weights within 1e-4 / 1e-5 from identical state.  Runs the EXACT-fp32 conv path
    (PF_CONV_PATH=fp32): with fp32 accumulation-order noise of 1e-7 most batches have no ReLU element
    inside the noise band, so the backward pass can be compared tightly; the tensor-core path has its
    own test below."""
    monkeypatch.setenv('PF_CONV_PATH', 'fp32')
    lrn = make_uq_learner(dst=dst, buckets=buckets, a_bits=32)
    assert not lrn.sess_train.tc
    ex = lrn.sess_train
    orc = oracle_for(lrn)
    state = ex.store.state_dict()
    tstate = ex.teacher.store.state_dict() if ex.teacher is not None else None
    opt = dict(kind='adam', slots={})
    b1p, b2p = F32(0.9), F32(0.999)
    checked = 0
    for step in range(6):
        images, labels = lrn.iterator_train.next_batch()
        img, lab = images.numpy().copy(), labels.numpy().copy()
        ex.buf[lrn.images].copy_(images)
        ex.buf[lrn.labels].copy_(labels)
        lr = lrn.lrn_rate(step)
        ex.run_step(lr)
        got = ex.fetch_losses()
        flips = relu_mask_mismatches(ex, orc, state, img)
        ref, new_state, grads = orc.step(state, img, lab, opt, lr, teacher_state=tstate, beta_powers=(b1p, b2p))
        b1p, b2p = F32(b1p * F32(0.9)), F32(b2p * F32(0.999))
        for op, bits in zip(ex.wq_ops, ex.weight_quant['bits']):
            v = op.vars['kernel']
            qref = O.uniform_quantize(state[v.name], bits, use_buckets=buckets, bucket_type='channel')
            assert np.array_equal(ex.store.view(v, ex.QW).cpu().numpy(), qref), v.name
        for k in ('ce', 'l2', 'loss') + (('dst_loss',) if dst else ()):
            assert rel(got[k], ref[k]) <= 1e-5, (step, k, got[k], ref[k])     # north-star tolerance
        assert got['acc_top1'] == ref['acc_top1']
        if flips == 0:
            checked += 1
            for v in ex.store.train_vars:
                g_ref = grads[v.name]
                err = np.abs(ex.store.view(v, ex.G).cpu().numpy() - g_ref).max() / (np.abs(g_ref).max() + 1e-12)
                assert err <= 1e-4, (step, v.name, err)
            # Adam's first steps move every weight by ~lr regardless of |g|: compare the UPDATE
            for v in ex.store.train_vars:
                d_gpu = ex.store.view(v).cpu().numpy() - state[v.name]
                d_ref = new_state[v.name] - state[v.name]
                assert np.abs(ex.store.view(v).cpu().numpy() - new_state[v.name]).max() <= \
                    1e-5 * np.abs(new_state[v.name]).max() + 1e-9, v.name
                del d_gpu, d_ref
            for v in ex.store.other_vars:           # BN moving statistics
                np.testing.assert_allclose(ex.store.view(v).cpu().numpy(), new_state[v.name], rtol=2e-5, atol=1e-7)
        # step from the SAME state next time (state injected from the oracle, SURVEY §7 hard part 1)
        ex.store.load_state_dict(new_state)
        for v in ex.store.train_vars:
            ex.store.view(v, ex.S1).copy_(torch.from_numpy(opt['slots'][v.name + '/m']))
            ex.store.view(v, ex.S2).copy_(torch.from_numpy(opt['slots'][v.name + '/v']))
        state = new_state
        if checked >= 2:
            break
    assert checked >= 1, 'every batch had a ReLU element within fp32 noise of zero'


def test_uq_step_tensor_core_path_matches_oracle(monkeypatch):
    """Same step on the tensor-core split-bf16 conv path (the default): quantized weights bit-exact, every
    loss term within the north-star 1e-5, gradients within split-bf16 accuracy.  ReLU pre-activations
    within ~1e-6 of zero now flip in most batches (each flip perturbs upstream gradients by ~1e-2 of
    their max-norm in ANY two implementations), so the gradient check is directional + L2, not max-norm."""
    monkeypatch.setenv('PF_CONV_PATH', 'tc')
    lrn = make_uq_learner(dst=True, buckets=True, a_bits=32)
    ex = lrn.sess_train
    assert len(ex.tc) >= 8 and len(ex.tc_wgrad) >= 1 and len(ex.im2col) == 1
    orc = oracle_for(lrn)
    state, tstate = ex.store.state_dict(), ex.teacher.store.state_dict()
    images, labels = lrn.iterator_train.next_batch()
    ex.buf[lrn.images].copy_(images)
    ex.buf[lrn.labels].copy_(labels)
    ex.run_step(lrn.lrn_rate(0))
    got = ex.fetch_losses()
    ref, new_state, grads = orc.step(state, images.numpy(), labels.numpy(), dict(kind='adam', slots={}),
                                     lrn.lrn_rate(0), teacher_state=tstate)
    for k in ('ce', 'l2', 'dst_loss', 'loss'):
        assert rel(got[k], ref[k]) <= 1e-5, (k, got[k], ref[k])
    for op, bits in zip(ex.wq_ops, ex.weight_quant['bits']):
        v = op.vars['kernel']
        assert np.array_equal(ex.store.view(v, ex.QW).cpu().numpy(),
                              O.uniform_quantize(state[v.name], bits, use_buckets=True, bucket_type='channel'))
    for v in ex.store.train_vars:
        g, r = ex.store.view(v, ex.G).cpu().numpy().ravel().astype(np.float64), grads[v.name].ravel().astype(np.float64)
        cos = float(g @ r / (np.linalg.norm(g) * np.linalg.norm(r) + 1e-30))
        l2 = float(np.linalg.norm(g - r) / (np.linalg.norm(r) + 1e-30))
        assert cos >= 0.9995 and l2 <= 3e-2, (v.name, cos, l2)


def test_uq_w8a8_step_loss_parity():
    """8-bit ACTIVATION quantization makes the loss itself discontinuous in the activations: a value
    within 1e-7 of a rounding boundary lands on a different level (1/255 of the range) in any two
    fp32 implementations.  Measured on this net at batch 16: ~6e-5 relative on the loss; the bar
    here is 2e-4 (documented deviation from the 1e-5 that holds at the default 32-bit activations)."""
    lrn = make_uq_learner(dst=True, buckets=True, a_bits=8)
    ex = lrn.sess_train
    orc = oracle_for(lrn)
    state = ex.store.state_dict()
    tstate = ex.teacher.store.state_dict()
    images, labels = lrn.iterator_train.next_batch()
    ex.buf[lrn.images].copy_(images)
    ex.buf[lrn.labels].copy_(labels)
    ex.run_step(lrn.lrn_rate(0))
    got = ex.fetch_losses()
    ref, _, _ = orc.step(state, images.numpy(), labels.numpy(), dict(kind='adam', slots={}), lrn.lrn_rate(0),
                         teacher_state=tstate)
    for k in ('ce', 'dst_loss', 'loss'):
        assert rel(got[k], ref[k]) <= 2e-4, (k, got[k], ref[k])
    assert rel(got['l2'], ref['l2']) <= 1e-6
    for op, bits in zip(ex.wq_ops, ex.weight_quant['bits']):
        v = op.vars['kernel']
        assert np.array_equal(ex.store.view(v, ex.QW).cpu().numpy(),
                              O.uniform_quantize(state[v.name], bits, use_buckets=True, bucket_type='channel'))


def test_uq_step_cuda_graph_replay_matches_eager():
    lrn = make_uq_learner(dst=True)
    ex = lrn.sess_train
    images, labels = lrn.iterator_train.next_batch()
    ex.buf[lrn.images].copy_(images)
    ex.buf[lrn.labels].copy_(labels)
    P0, O0 = ex.store.P.clone(), ex.store.O.clone()
    ex.run_step(1e-3)
    eager = ex.fetch_losses()
    P1 = ex.store.P.clone()
    # rewind and replay through a captured graph
    ex.store.P.copy_(P0); ex.store.O.copy_(O0); ex.S1.zero_(); ex.S2.zero_()
    ex.beta1_power, ex.beta2_power = F32(0.9), F32(0.999)
    ex.capture()
    ex.store.P.copy_(P0); ex.store.O.copy_(O0); ex.S1.zero_(); ex.S2.zero_()
    ex.run_step(1e-3)
    replay = ex.fetch_losses()
    assert replay['loss'] == eager['loss']
    assert torch.equal(ex.store.P, P1)


def test_multi_stream_step_is_bit_identical_to_serial(monkeypatch):
    """The multi-stream schedule (teacher forward beside the student's, wgrad beside dgrad/BN-backward, input staging
    on a copy stream) must not change a single bit: three learner-level steps, serial vs overlapped vs overlapped +
    captured graph, from the same seeds."""
    results = []
    for overlap, graph in (('0', False), ('1', False), ('1', True)):
        monkeypatch.setenv('PF_OVERLAP', overlap)
        monkeypatch.setenv('PF_CONV_PATH', 'tc')
        lrn = make_uq_learner(resnet_size=20, batch=32, dst=True)
        ex = lrn.sess_train
        lrn.iterator_train.prefill()                      # fixed cycle of pre-generated batches
        if graph:
            P0, O0 = ex.store.P.clone(), ex.store.O.clone()
            lrn.feed(ex, lrn.iterator_train)              # capture runs the step twice: rewind afterwards
            ex.capture()
            ex.store.P.copy_(P0); ex.store.O.copy_(O0); ex.S1.zero_(); ex.S2.zero_()
            lrn.iterator_train.cursor = 0
            lrn.iterator_train._staging = None
        for _ in range(3):
            lrn.train_step()
        torch.cuda.synchronize()
        results.append((ex.store.P.clone(), ex.store.O.clone(), ex.fetch_losses()['loss']))
    for P, O_, loss in results[1:]:
        assert torch.equal(P, results[0][0]) and torch.equal(O_, results[0][1]) and loss == results[0][2]


def test_bucketed_gradient_exchange_covers_the_buffer_once_and_changes_nothing(monkeypatch):
    """The data-parallel step sums the flat gradient buffer in buckets issued from inside the backward pass (SURVEY §8e;
    engine._bucket_plan).  With a recording stand-in for the collective (world 1: the sum is the identity): every float of
    the buffer is handed to the collective exactly once, the early bucket holds the LAST layers' kernels and goes out
    before the backward pass has finished, and eager step, captured graph and the collective-free step agree bit for bit.
    (The NCCL path itself — pf_allreduce_flat at world 2 / 8 — is tools/mgpu_check.py and the N > 1 bench lines.)"""
    monkeypatch.setenv('PF_CONV_PATH', 'tc')
    lrn = make_uq_learner(resnet_size=20, batch=32, dst=True)
    ex = lrn.sess_train
    lrn.iterator_train.prefill()
    images, labels = lrn.iterator_train.next_batch()
    ex.buf[lrn.images].copy_(images)
    ex.buf[lrn.labels].copy_(labels)
    P0, O0 = ex.store.P.clone(), ex.store.O.clone()
    calls = []

    def collective(flat):
        assert flat.is_contiguous() and flat.dtype == torch.float32
        calls.append(((flat.data_ptr() - ex.G.data_ptr()) // 4, flat.numel(), torch.cuda.current_stream().cuda_stream))
        return flat

    def rewind():
        ex.store.P.copy_(P0)
        ex.store.O.copy_(O0)
        ex.reset_optimizer_state()

    lr = lrn.lrn_rate(0)
    ex.run_step(lr)                                        # no collective
    torch.cuda.synchronize()
    P_ref, G_ref = ex.store.P.clone(), ex.G.clone()
    rewind()
    ex.run_step(lr, collective)                            # eager, bucketed
    torch.cuda.synchronize()
    bk = ex._bucket_plan()
    assert bk is not None and 0 < bk['split'] < bk['end'] <= ex.G.numel()
    assert [c[:2] for c in calls][0] == (bk['split'], bk['end'] - bk['split'])          # the last layers' kernels first
    spans = sorted(c[:2] for c in calls)
    assert spans[0][0] == 0 and all(a[0] + a[1] == b[0] for a, b in zip(spans, spans[1:])) \
        and spans[-1][0] + spans[-1][1] == ex.G.numel()                                  # a partition of the buffer
    assert calls[0][2] != calls[-1][2]                                                   # on the communication stream
    assert (bk['end'] - bk['split']) >= 0.4 * bk['end']
    assert torch.equal(ex.store.P, P_ref) and torch.equal(ex.G, G_ref)
    # the captured graph carries the same schedule
    del calls[:]
    rewind()
    ex.capture(collective)
    rewind()
    ex.run_step(lr, collective)
    torch.cuda.synchronize()
    assert torch.equal(ex.store.P, P_ref) and torch.equal(ex.G, G_ref)
    # PF_AR_BUCKETS=1: one call for the whole buffer after the backward pass
    monkeypatch.setenv('PF_AR_BUCKETS', '1')
    lrn1 = make_uq_learner(resnet_size=20, batch=32, dst=True)
    ex1 = lrn1.sess_train
    assert ex1._bucket_plan() is None
    seen = []
    ex1.buf[lrn1.images].copy_(images)
    ex1.buf[lrn1.labels].copy_(labels)
    ex1.run_step(lr, lambda flat: seen.append(flat.numel()))
    assert seen == [ex1.G.numel()]


def test_lenet_uq_step_matches_oracle():
    FLAGS.reset()
    from pocketflow_b200.nets import lenet_at_cifar10 as Lnet
    from pocketflow_b200.learners.uniform_quantization.learner import UniformQuantLearner
    FLAGS.batch_size, FLAGS.uql_weight_bits, FLAGS.uql_activation_bits = 16, 8, 32
    FLAGS.loss_w_dcy, FLAGS.lrn_rate_init = 5e-4, 1e-2
    lrn = UniformQuantLearner(None, Lnet.ModelHelper())
    ex = lrn.sess_train
    assert [op.vars['kernel'].shape for op in ex.wq_ops] == [(5, 5, 32, 64), (1600, 256)]
    orc = oracle_for(lrn)
    state = ex.store.state_dict()
    images, labels = lrn.iterator_train.next_batch()
    ex.buf[lrn.images].copy_(images)
    ex.buf[lrn.labels].copy_(labels)
    ex.run_step(lrn.lrn_rate(0))
    got = ex.fetch_losses()
    ref, new_state, grads = orc.step(state, images.numpy(), labels.numpy(), dict(kind='adam', slots={}),
                                     lrn.lrn_rate(0), beta_powers=(F32(0.9), F32(0.999)))
    for k in ('ce', 'l2', 'loss'):
        assert rel(got[k], ref[k]) <= 1e-5, (k, got[k], ref[k])
    if relu_mask_mismatches(ex, orc, state, images.numpy()) == 0:
        for v in ex.store.train_vars:
            g_ref = grads[v.name]
            err = np.abs(ex.store.view(v, ex.G).cpu().numpy() - g_ref).max() / (np.abs(g_ref).max() + 1e-12)
            assert err <= 1e-4, (v.name, err)
