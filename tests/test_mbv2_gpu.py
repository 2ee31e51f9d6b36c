"""MobileNet-v2 on the GPU: the fused linear-bottleneck BN + residual kernel (pf_bn_apply_add / _eval), the dropout
kernels and their Philox stream, layer-local step parity of every learner on v2 at 224x224 against the oracle, the
benchmarked batch under PF_POISON=1 with its CUDA-graph replay, and a TF-slim-named checkpoint round trip."""

import numpy as np
import pytest
import torch

from oracle import pf_oracle as O
from oracle.mbv2_oracle import DropoutStepOracle
from pocketflow_b200 import ops
from pocketflow_b200.flags import FLAGS
from support import check_selection, ref_mask, rel

pytestmark = pytest.mark.gpu
F32 = np.float32
DEV = torch.device('cuda', 0)


def split_np(v):
    """hi / lo bf16 planes (as float32) of the split the kernels write: hi = bf16_rn(v), lo = bf16_rn(v - hi)"""
    t = torch.from_numpy(np.ascontiguousarray(v, F32))
    hi = t.to(torch.bfloat16)
    lo = (t - hi.float()).to(torch.bfloat16)
    return hi.float().numpy(), lo.float().numpy()


# ------------------------------------------------------------------------------------------------ BN apply + residual
@pytest.mark.parametrize('c', [24, 32, 96, 160])
@pytest.mark.parametrize('m', [1, 333, 12544 * 4 + 5])
@pytest.mark.parametrize('mode', ['train', 'eval'])
@pytest.mark.parametrize('out', ['f32', 'planes', 'both'])
def test_bn_apply_add_matches_the_fp32_op_chain(c, m, mode, out):
    """bn(x) + r in one pass against pf_bn_apply (act none) followed by pf_add, bit for bit; planes against the split of
    that fp32 sum.  m = 1 is one row; the largest case spans many BN splits with a ragged last one."""
    g = torch.Generator().manual_seed(c * 7 + m)
    x = (torch.randn(m, c, generator=g) * 3 + 1).to(DEV)
    r = torch.randn(m, c, generator=g).to(DEV)
    gamma, beta = (torch.rand(c, generator=g) + 0.5).to(DEV), torch.randn(c, generator=g).to(DEV)
    mean, var, rstd = (torch.empty(c, device=DEV) for _ in range(3))
    mm, mv = torch.randn(c, generator=g).to(DEV), (torch.rand(c, generator=g) + 0.1).to(DEV)
    ws = torch.empty(5 * c * ops.BN_MAX_SPLITS, device=DEV)
    ref = torch.full((m, c), float('nan'), device=DEV)
    if mode == 'train':
        ops.bn_train_stats(x, m, c, 1e-3, 1.0, mean, var, rstd, mm.clone(), mv.clone(), ws)
        ops.bn_apply(x, m, c, mean, rstd, gamma, beta, 0, ref)
    else:
        ops.bn_apply_eval(x, m, c, mm, mv, 1e-3, gamma, beta, 0, ref)
    ops.add(ref, r, ref)
    y = torch.full((m, c), float('nan'), device=DEV) if out != 'planes' else None
    pl = ops.Planes(m * c + (-(m * c)) % 8, DEV) if out != 'f32' else None
    if mode == 'train':
        ops.bn_apply_add(x, m, c, mean, rstd, gamma, beta, r, y, pl)
    else:
        ops.bn_apply_add_eval(x, m, c, mm, mv, 1e-3, gamma, beta, r, y, pl)
    want = ref.cpu().numpy()
    if y is not None:
        assert np.array_equal(y.cpu().numpy().view(np.uint32), want.view(np.uint32))
    if pl is not None:
        hi, lo = split_np(want.reshape(-1))
        assert np.array_equal(pl.hi[:m * c].float().cpu().numpy(), hi)
        assert np.array_equal(pl.lo[:m * c].float().cpu().numpy(), lo)


def test_bn_apply_add_with_one_block_grid(monkeypatch):
    """PF_BN_GRIDCAP=1: the grid is the smallest channel-stationary one, every thread walks many rows"""
    monkeypatch.setenv('PF_BN_GRIDCAP', '1')
    for c in (24, 160):
        test_bn_apply_add_matches_the_fp32_op_chain(c, 12544 * 4 + 5, 'train', 'both')
        test_bn_apply_add_matches_the_fp32_op_chain(c, 12544 * 4 + 5, 'eval', 'both')


# ------------------------------------------------------------------------------------------------ dropout


def test_dropout_stream_is_philox4x32_10_and_keeps_keep_prob():
    n, keep, seed, rank = 10_000_003, 0.8, 1234, 3
    x = torch.randn(n, device=DEV)
    y, mask = torch.empty_like(x), torch.empty(n, dtype=torch.uint8, device=DEV)
    state = torch.tensor([5, 0], dtype=torch.int64, device=DEV)
    ops.dropout_fwd(x, keep, seed, rank, state, y, mask)
    got = mask.cpu().numpy()
    assert np.array_equal(got.astype(np.float32), ref_mask(n, keep, seed, rank, 5))
    assert state.cpu().tolist() == [6, 0]
    kept = got.mean()
    assert abs(kept - keep) <= 5 * np.sqrt(keep * (1 - keep) / n), kept


def test_dropout_streams_of_two_ops_are_independent():
    """two Dropout ops of one graph pass their own stream index (and their own step counter): stream 3 at step 0 is
    Philox at counter word 3 = 3, not stream 0 at a later step; n % 4 == 0 here (vectorised path)"""
    n, keep = 64 * 1280, 0.8
    x = torch.randn(n, device=DEV)
    y, mask = torch.empty_like(x), torch.empty(n, dtype=torch.uint8, device=DEV)
    masks = {}
    for stream in (0, 3):
        state = torch.zeros(2, dtype=torch.int64, device=DEV)
        ops.dropout_fwd(x, keep, 11, 0, state, y, mask, stream_id=stream)
        masks[stream] = mask.cpu().numpy().copy()
        assert np.array_equal(masks[stream].astype(np.float32), ref_mask(n, keep, 11, 0, 0, stream))
    state = torch.tensor([1, 0], dtype=torch.int64, device=DEV)
    ops.dropout_fwd(x, keep, 11, 0, state, y, mask)
    for a, b in ((masks[0], masks[3]), (masks[3], mask.cpu().numpy())):
        assert abs(float(np.mean(a == b)) - (keep ** 2 + (1 - keep) ** 2)) < 0.01    # independent draws agree this often


def test_dropout_fwd_bwd_bit_exact_on_the_device_mask():
    n, keep = 256 * 1280, F32(0.8)
    x, dy = torch.randn(n, device=DEV) * 4, torch.randn(n, device=DEV)
    y, mask = torch.full_like(x, float('nan')), torch.empty(n, dtype=torch.uint8, device=DEV)
    state = torch.zeros(2, dtype=torch.int64, device=DEV)
    ops.dropout_fwd(x, keep, 1, 0, state, y, mask)
    m = mask.cpu().numpy().astype(F32)
    xn, dyn = x.cpu().numpy(), dy.cpu().numpy()
    assert set(np.unique(m)) <= {0.0, 1.0}
    assert np.array_equal(y.cpu().numpy().view(np.uint32), ((xn / keep) * m).view(np.uint32))
    dx = torch.full_like(x, float('nan'))
    ops.dropout_bwd(dy, mask, keep, dx)
    want = (dyn * m) / keep
    assert np.array_equal(dx.cpu().numpy().view(np.uint32), want.view(np.uint32))
    acc = torch.ones_like(x)
    ops.dropout_bwd(dy, mask, keep, acc, accumulate=True)
    assert np.array_equal(acc.cpu().numpy().view(np.uint32), (F32(1) + want).view(np.uint32))


def test_eager_steps_and_graph_replays_draw_the_same_masks():
    n, keep = 64 * 1280, 0.8
    x = torch.randn(n, device=DEV)
    y, mask = torch.empty_like(x), torch.empty(n, dtype=torch.uint8, device=DEV)
    state = torch.zeros(2, dtype=torch.int64, device=DEV)
    eager = []
    for _ in range(3):
        ops.dropout_fwd(x, keep, 7, 0, state, y, mask)
        eager.append(mask.cpu().numpy().copy())
    assert not np.array_equal(eager[0], eager[1])
    state.zero_()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        ops.dropout_fwd(x, keep, 7, 0, state, y, mask)
    torch.cuda.synchronize()
    assert state.cpu().tolist() == [0, 0]                  # capture launches nothing
    for i in range(3):
        graph.replay()
        torch.cuda.synchronize()
        assert np.array_equal(mask.cpu().numpy(), eager[i]), i


# ------------------------------------------------------------------------------------------------ learners on v2
def make_v2(learner, batch=2, **flags):
    import importlib
    FLAGS.reset()
    import pocketflow_b200.datasets.ilsvrc12_dataset as D
    importlib.reload(D)
    from pocketflow_b200.nets import mobilenet_at_ilsvrc12 as M
    importlib.reload(M)
    from pocketflow_b200.learners.learner_utils import create_learner
    import pocketflow_b200.learners.channel_pruning_gpu.learner  # noqa: F401
    import pocketflow_b200.learners.channel_pruning_rmt.learner  # noqa: F401
    import pocketflow_b200.learners.nonuniform_quantization.learner  # noqa: F401
    import pocketflow_b200.learners.uniform_quantization.learner  # noqa: F401
    import pocketflow_b200.learners.weight_sparsification.learner  # noqa: F401
    FLAGS.batch_size, FLAGS.learner, FLAGS.nb_classes, FLAGS.mobilenet_version = batch, learner, 1001, 2
    for k, v in flags.items():
        setattr(FLAGS, k, v)
    return create_learner(None, M.ModelHelper())


def device_value(ex, t):
    """a tensor as its consumers read it: fp32 buffer, or hi + lo of the operand planes when no fp32 copy is kept"""
    r = ex._root(t)
    pl = ex.xplanes.get(r.op) if r is not None else None
    if pl is not None and not ex.bn_need_f32.get(r.op, True) and r.op.type == 'Add':
        return (pl.hi.float() + pl.lo.float()).cpu().reshape(t.shape)
    if r is not None and r.op in ex.act_lv and ex._lv_on:
        hdr = ex.act_lv[r.op]['hdr'].cpu().numpy().view(ops.ACT_HDR)[0]
        if int(hdr['nplanes']) == 1:
            return (pl.hi.float() * float(hdr['scale'])).cpu().reshape(t.shape)
    if pl is not None and not ex.bn_need_f32[r.op]:
        return (pl.hi.float() + pl.lo.float()).cpu().reshape(t.shape)
    return ex.T(t).float().cpu().clone()


def layer_local(ex, orc, state, img, skip=()):
    """every oracle op applied to the device's own inputs: worst error of conv / depthwise / fused BN + add / pool /
    dropout outputs relative to the output scale (op types in `skip` excepted), and the activation elements on another
    quantizer level"""
    params = {k: torch.from_numpy(np.array(v, dtype=F32, copy=True)) for k, v in state.items()}
    force = {}
    for op in ex.ops:
        if op.type in ('Relu', 'Relu6', 'Add', 'Mean', 'Dropout') or \
                (op.type in ('Conv2D', 'DepthwiseConv2dNative') and op not in ex.fused_add):
            force[op.output.name] = device_value(ex, op.output)
    local = {}
    with torch.no_grad():
        orc.forward(params, torch.from_numpy(img), True, force=force, local_out=local)
    bits_of = dict(zip([o.name for o in ex.aq_ops], ex.act_quant['bits'])) if ex.aq_ops else {}
    worst, worst_op, flips, total = 0.0, None, 0, 0
    for op in ex.ops:
        name = op.output.name
        if name not in force:
            continue
        if op.type in skip:
            continue
        got, ref = force[name].numpy(), local[name].numpy()
        if op.name in bits_of:
            step = (float(ref.max()) - float(ref.min())) / float(2 ** int(bits_of[op.name]) - 1)
            if step > 0:
                flips += int((np.abs(got - ref) > 0.5 * step).sum())
                total += ref.size
            continue
        e = float(np.abs(got - ref).max() / (np.abs(ref).max() + 1e-30))
        if e > worst:
            worst, worst_op = e, op.name
    return worst, worst_op, flips, total


def relu6_flips(ex, orc, state, img):
    """elements whose ReLU6 gate (0 < y < 6) differs between the device step and the free-running oracle forward"""
    params = {k: torch.from_numpy(np.array(v, dtype=F32, copy=True)) for k, v in state.items()}
    with torch.no_grad():
        val = orc.forward(params, torch.from_numpy(img), True)
    bad = 0
    for op in ex.ops:
        if op.type == 'Relu6':
            g, r = device_value(ex, op.output).numpy(), val[op.output.name].numpy()
            bad += int((((g > 0) & (g < 6)) != ((r > 0) & (r < 6))).sum())
    return bad


def check_gradients(ex, orc, state, img, grads):
    """the backward pass (dropout backward, the projection BN-backward reading the Add's shared gradient, the dy planes
    it writes) against the oracle's autograd: direction of the whole gradient, and per variable within 1e-3 of its
    largest entry when no ReLU6 gate differs"""
    g_all = np.concatenate([ex.store.view(v, ex.G).cpu().numpy().ravel().astype(np.float64) for v in ex.store.train_vars])
    r_all = np.concatenate([grads[v.name].ravel().astype(np.float64) for v in ex.store.train_vars])
    cos = float(g_all @ r_all / (np.linalg.norm(g_all) * np.linalg.norm(r_all) + 1e-30))
    flips = relu6_flips(ex, orc, state, img)
    print('gradient cosine %.8f, ReLU6 gate flips %d' % (cos, flips))
    assert cos >= 0.99, cos
    if flips == 0:
        for v in ex.store.train_vars:
            g, r = ex.store.view(v, ex.G).cpu().numpy(), grads[v.name]
            assert np.abs(g - r).max() <= 1e-3 * (np.abs(r).max() + 1e-12), v.name


def run_and_check(lrn, optimizer, masks=None, e2e=True):
    ex = lrn.sess_train
    assert len(ex.bn_add) == 10 and len(ex.dropout) == 1
    state = ex.store.state_dict()
    images, labels = lrn.iterator_train.next_batch()
    img, lab = images.numpy().copy(), labels.numpy().copy()
    ex.buf[lrn.images].copy_(images)
    ex.buf[lrn.labels].copy_(labels)
    lr = lrn.lrn_rate(0)
    ex.run_step(lr)
    got = ex.fetch_losses()
    drop = {op.name: ex.dropout[op].cpu().numpy().astype(F32).reshape(op.output.shape) for op in ex.dropout}
    orc = DropoutStepOracle(ex.ops, ex.logits_t, lrn.images, lrn.labels, ex.loss, ex.weight_quant, ex.act_quant,
                            masks=drop)
    worst, worst_op, flips, total = layer_local(ex, orc, state, img)
    print('layer-local worst %.2e (%s), level flips %d of %d' % (worst, worst_op, flips, total))
    assert worst <= 2e-5, (worst_op, worst)
    assert flips <= 1e-4 * max(total, 1), (flips, total)
    ref, _, grads = orc.step(state, img, lab, optimizer, lr, masks=masks)
    assert rel(got['l2'], ref['l2']) <= 1e-6
    if e2e:
        for k in ('ce', 'loss'):
            assert rel(got[k], ref[k]) <= 3e-5, (k, got[k], ref[k])
        check_gradients(ex, orc, state, img, grads)
    return ex


@pytest.mark.parametrize('conv_path', ['tc', 'fp32'])
def test_v2_full_precision_step(monkeypatch, conv_path):
    """also on the exact-fp32 conv path, where the device and the oracle agree on every ReLU6 gate and the gradient of
    every variable is held to 1e-3 of its largest entry"""
    monkeypatch.setenv('PF_CONV_PATH', conv_path)
    run_and_check(make_v2('full-prec'), dict(kind='momentum', slots={}, momentum=0.9))


def test_v2_uniform_w8a8_step():
    lrn = make_v2('uniform', uql_weight_bits=8, uql_activation_bits=8, uql_use_buckets=True, uql_bucket_type='channel')
    ex = lrn.sess_train
    state = ex.store.state_dict()
    run_and_check(lrn, dict(kind='adam', slots={}), e2e=False)
    for op, bits in zip(ex.wq_ops, ex.weight_quant['bits']):
        v = op.vars['kernel']
        assert np.array_equal(ex.store.view(v, ex.QW).cpu().numpy(),
                              O.uniform_quantize(state[v.name], bits, use_buckets=True, bucket_type='channel')), v.name


def test_v2_weight_sparse_step():
    lrn = make_v2('weight-sparse', ws_prune_ratio=0.5, ws_prune_ratio_prtl='uniform')
    ex = lrn.sess_train
    masks = {v.name: ex.store.view(v, ex.MASK).cpu().numpy().copy() for v in lrn.maskable_vars}
    # get_maskable_vars matches only the logits conv on v2, as in the reference
    assert [v.name.split('/')[-2] for v in lrn.maskable_vars] == ['Conv2d_1c_1x1']
    run_and_check(lrn, dict(kind='momentum', slots={}, momentum=0.9), masks=masks)


def test_v2_nonuniform_step():
    """4-bit codebooks.  v2's depthwise kernels have no `clusters` variable, so the quantizer keeps every codebook in its
    private table: the kernels are checked bit for bit against those codebooks, and the step layer by layer with the
    oracle reading the same codebooks (StepOracle quantizes depthwise kernels only uniformly, so the depthwise outputs
    are left to the bit-exact kernel check and the full-precision test)."""
    lrn = make_v2('non-uniform', nuql_weight_bits=4)
    ex = lrn.sess_train
    state = ex.store.state_dict()
    images, labels = lrn.iterator_train.next_batch()
    ex.buf[lrn.images].copy_(images)
    ex.buf[lrn.labels].copy_(labels)
    ex.run_step(lrn.lrn_rate(0))
    assert ex.wq.clusters is not None
    books = {op.name: ex.wq.clusters[i, :1 << bits].cpu().numpy().copy()
             for i, (op, bits) in enumerate(zip(ex.wq_ops, ex.weight_quant['bits']))}
    for op in ex.wq_ops:
        v = op.vars['kernel']
        q_ref, _, _ = O.nonuniform_quantize(state[v.name], 4, books[op.name])
        assert np.array_equal(ex.store.view(v, ex.QW).cpu().numpy(), q_ref), v.name
    drop = {op.name: ex.dropout[op].cpu().numpy().astype(F32).reshape(op.output.shape) for op in ex.dropout}
    orc = DropoutStepOracle(ex.ops, ex.logits_t, lrn.images, lrn.labels, ex.loss, ex.weight_quant, ex.act_quant,
                            masks=drop)
    orc.clusters = books
    fwd_state = {k: v for k, v in state.items() if not k.endswith('/clusters:0')}
    worst, worst_op, _, _ = layer_local(ex, orc, fwd_state, images.numpy(), skip=('DepthwiseConv2dNative',))
    assert worst <= 2e-5, (worst_op, worst)


def test_v2_channel_pruned_gpu_masked_step():
    lrn = make_v2('chn-pruned-gpu', cpg_prune_ratio=0.5)
    ex = lrn.sess_train
    lrn.init_from_full()
    lrn.choose_channels(nb_iters_layer=2)
    masks = {v.name: ex.store.view(v, ex.MASK).cpu().numpy().copy() for v in lrn.maskable_vars}
    run_and_check(lrn, dict(kind='momentum', slots={}, momentum=0.9), masks=masks)


# ------------------------------------------------------------------------------------------------ benchmarked batch
def test_v2_batch128_poisoned_step_and_graph_replay(monkeypatch):
    monkeypatch.setenv('PF_POISON', '1')
    lrn = make_v2('full-prec', batch=128)
    ex = lrn.sess_train
    images, labels = lrn.iterator_train.next_batch()
    ex.buf[lrn.images].copy_(images)
    ex.buf[lrn.labels].copy_(labels)
    st0, s1_0 = ex.store.state_dict(), ex.S1.clone()
    lr = lrn.lrn_rate(0)
    ex.set_hyper(lr)
    ex.device_step()
    torch.cuda.synchronize()
    eager_losses = ex.fetch_losses()
    assert all(np.isfinite(float(v)) for v in eager_losses.values()), eager_losses
    eager = ex.store.state_dict()
    eager_mask = ex.dropout[next(iter(ex.dropout))].cpu().numpy().copy()
    ex.capture()                                           # (runs one eager warm-up step)

    def rewind():
        ex.store.load_state_dict(st0)
        ex.S1.copy_(s1_0)
        ex.drop_state.zero_()
    rewind()
    ex.set_hyper(lr)
    ex._graph.replay()
    torch.cuda.synchronize()
    assert np.array_equal(ex.dropout[next(iter(ex.dropout))].cpu().numpy(), eager_mask)
    replay = ex.store.state_dict()
    for k in eager:
        assert np.array_equal(eager[k], replay[k]), k
    assert ex.fetch_losses()['loss'] == eager_losses['loss']


# ------------------------------------------------------------------------------------------------ checkpoints
def test_v2_slim_named_bundle_warm_starts_every_variable(tmp_path):
    """a seeded v2 state written as a TF bundle under slim's names (with the model/ prefix) comes back in full through
    the uniform learner's train() under --enbl_warm_start"""
    from pocketflow_b200.learners.abstract_learner import save_checkpoint
    lrn = make_v2('uniform', ckpt_format='tf', enbl_warm_start=True, save_path=str(tmp_path / 'model.ckpt'),
                  uql_save_quant_model_path=str(tmp_path / 'uql' / 'model.ckpt'))
    ex = lrn.sess_train
    names = [v.name for v in ex.store.train_vars + ex.store.other_vars]
    assert 'model/MobilenetV2/Conv/weights:0' in names
    assert 'model/MobilenetV2/expanded_conv_3/expand/BatchNorm/gamma:0' in names
    assert 'model/MobilenetV2/expanded_conv_3/depthwise/depthwise_weights:0' in names
    assert 'model/MobilenetV2/expanded_conv_3/project/weights:0' in names
    assert 'model/MobilenetV2/Logits/Conv2d_1c_1x1/biases:0' in names
    rng = np.random.default_rng(5)
    seeded = {n: rng.standard_normal(ex.store.view(v).shape).astype(F32)
              for n, v in zip(names, ex.store.train_vars + ex.store.other_vars)}
    save_checkpoint(FLAGS.save_path, seeded, 3)
    lrn.evaluate = lambda *a, **k: None                  # (train() ends with a full evaluation pass)
    lrn.train(nb_iters=0)
    back = ex.store.state_dict()
    for n in names:
        assert np.array_equal(back[n], seeded[n]), n


def test_v2_channel_pruned_rmt_selection_and_masked_steps(tmp_path):
    """chn-pruned-rmt on v2: its selection executors sample conv inputs that the linear-bottleneck fusion may hold only as
    operand planes; every sampled patch x W must reproduce the full model's output (err < 1e-6), the kept counts meet
    their targets, and masked steps follow"""
    lrn = make_v2('chn-pruned-rmt', cpr_nb_smpls=4, cpr_nb_crops_per_smpl=4, cpr_ista_nb_iters=30, cpr_lstsq_nb_iters=5,
                  cpr_save_path_ws=str(tmp_path / 'ws' / 'model.ckpt'), summ_step=10 ** 9, save_step=10 ** 9)
    ex = lrn.sess_train
    assert len(ex.bn_add) == 10
    lrn.choose_channels()
    check_selection(lrn, lrn.store_full.state_dict())
    images, labels = lrn.iterator_train.next_batch()
    ex.buf[lrn.images].copy_(images)
    ex.buf[lrn.labels].copy_(labels)
    for i in range(2):
        ex.run_step(lrn.lrn_rate(i))
    assert np.isfinite(ex.fetch_losses()['loss'])
