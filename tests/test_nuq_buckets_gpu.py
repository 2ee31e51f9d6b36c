"""Bucketed codebooks on the GPU (pf_nuq_bucket_quant / pf_nuq_bucket_quantile_init / pf_nuq_bucket_cluster_grad and
the non-uniform learner with --nuql_use_buckets) against the bucketed oracle (oracle/nuq_bucket_oracle.py, itself pinned
to the reference's __bucket_quantize by tests/test_nuq_buckets_cpu.py)."""
import numpy as np
import pytest
import torch

from oracle import nuq_bucket_oracle as B
from oracle import pf_oracle as O
from pocketflow_b200 import ops
from pocketflow_b200.flags import FLAGS
from support import rel

pytestmark = pytest.mark.gpu
F32 = np.float32

# (shape, bucket_type, bucket_size): cout not a multiple of 4, dense, depthwise (one channel bucket of 9216 rows),
# ragged split tails, numel < bucket size, exact multiples
SHAPES = [((3, 3, 8, 7), 'channel', 0), ((3, 3, 16, 32), 'channel', 0), ((64, 10), 'channel', 0),
          ((3, 3, 1024, 1), 'channel', 0), ((1, 1, 30, 6), 'channel', 0),
          ((3, 3, 8, 7), 'split', 100), ((3, 3, 16, 32), 'split', 256), ((1, 1, 8, 5), 'split', 64),
          ((5, 5, 3, 7), 'split', 77), ((64, 10), 'split', 64)]


def _weights(shapes, seed):
    rng = np.random.default_rng(seed)
    ws = []
    for i, s in enumerate(shapes):
        w = (rng.standard_normal(s) * rng.choice([1e-2, 1.0, 9.0])).astype(F32)
        if i % 4 == 1:
            w.reshape(-1)[: w.size // 3] = w.reshape(-1)[0]          # runs of equal weights
        ws.append(w)
    return ws


def _quantizer(ws, bits, bucket_type, bucket_size, **kw):
    src = [torch.from_numpy(w).cuda() for w in ws]
    dst = [torch.empty_like(s) for s in src]
    q = ops.CodebookWeightQuantizer(src, dst, bits, use_buckets=True, bucket_type=bucket_type,
                                    bucket_size=bucket_size, **kw)
    return q, src, dst


@pytest.mark.parametrize('bits', range(1, 9))
@pytest.mark.parametrize('bucket_type', ['channel', 'split'])
def test_bucket_quantile_init_and_quantize_bit_exact(bucket_type, bits):
    cases = [c for c in SHAPES if c[1] == bucket_type]
    for shape, _, bsize in cases:
        ws = _weights([shape], 100 + bits)
        if shape == (1, 1, 30, 6):
            ws[0][:, :, :, 2] = 0.25                                  # a constant bucket: alpha = 1e-10
        q, src, dst = _quantizer(ws, bits, bucket_type, bsize, keep_index=True)
        q.quantile_init()
        q.forward()
        torch.cuda.synchronize()
        qx, c_ref, idx_ref, _, _ = B.nonuniform_quantize_buckets(ws[0], bits, bucket_type, bsize)
        cb = q.codebooks()[0].cpu().numpy()
        assert np.array_equal(cb[:1 << bits], c_ref), (shape, bsize)                  # exact order statistics
        assert not cb[1 << bits:].any()                                               # rows past 2^bits stay 0
        assert np.array_equal(dst[0].cpu().numpy(), qx), (shape, bsize)
        n = ws[0].size
        assert np.array_equal(q.idx[:n].cpu().numpy(), idx_ref.astype(np.uint8)), (shape, bsize)


@pytest.mark.parametrize('bucket_type', ['channel', 'split'])
def test_argmin_ties_take_the_first_centroid(bucket_type):
    """Duplicate centroids and points equidistant from two centroids: the first index wins (tf.argmin)."""
    shape, bsize = ((3, 3, 8, 7), 100) if bucket_type == 'split' else ((3, 3, 8, 7), 0)
    ws = _weights([shape], 7)
    ws[0].reshape(-1)[::5] = 0.0
    q, src, dst = _quantizer(ws, 3, bucket_type, bsize, keep_index=True)
    q.quantile_init()
    cb = q.codebooks()[0]
    c = cb[:8].cpu().numpy()
    c[1] = c[0]                                   # duplicates: index 1 and 3 can never win
    c[3] = c[2]
    c[4] = np.float32(0.25)                       # x_n = 0.5 lies as far from c4 as from c5
    c[5] = np.float32(0.75)
    cb[:8].copy_(torch.from_numpy(c))
    q.forward()
    torch.cuda.synchronize()
    qx, _, idx_ref, _, _ = B.nonuniform_quantize_buckets(ws[0], 3, bucket_type, bsize, clusters=c)
    assert np.array_equal(dst[0].cpu().numpy(), qx)
    got = q.idx[:ws[0].size].cpu().numpy()
    assert np.array_equal(got, idx_ref.astype(np.uint8))
    assert not np.isin(got, [1, 3]).any()


@pytest.mark.parametrize('bits', [1, 4, 8])
@pytest.mark.parametrize('bucket_type', ['channel', 'split'])
def test_bucket_cluster_grad_matches_autograd_and_is_deterministic(bucket_type, bits):
    shapes = [s for s, t, _ in SHAPES if t == bucket_type][:3] + [(3, 3, 64, 64)]
    bsize = 100 if bucket_type == 'split' else 0
    ws = _weights(shapes, 9)
    base = torch.zeros(sum((1 << bits) * ops.uq_bucket_layout(s, True, bucket_type, bsize)[0] + 4 for s in shapes),
                       device='cuda')
    views, off = [], 0
    for s in shapes:
        nb = ops.uq_bucket_layout(s, True, bucket_type, bsize)[0]
        views.append(base[off:off + (1 << bits) * nb].view(1 << bits, nb))
        off += ((1 << bits) * nb + 3) // 4 * 4
    q, src, dst = _quantizer(ws, bits, bucket_type, bsize, keep_index=True, cluster_views=views, cluster_base=base)
    q.quantile_init()
    q.forward()
    rng = np.random.default_rng(3)
    gs = [rng.standard_normal(s).astype(F32) for s in shapes]
    gdev = [torch.from_numpy(g).cuda() for g in gs]
    gbase = torch.zeros_like(base)
    q.cluster_grad(gdev, gbase)
    first = gbase.clone()
    gbase.zero_()
    q.cluster_grad(gdev, gbase)
    torch.cuda.synchronize()
    assert torch.equal(first, gbase)                                      # fixed-order reduction: same bits
    for i, (s, w, g) in enumerate(zip(shapes, ws, gs)):
        c = torch.from_numpy(views[i].cpu().numpy()).requires_grad_(True)
        out = B.codebook_quant_buckets(torch.from_numpy(w), c, bits, bucket_type, bsize)
        ref, = torch.autograd.grad(out, [c], torch.from_numpy(g))
        ref = ref.numpy()
        dev = gbase[views[i].data_ptr() // 4 - base.data_ptr() // 4:][:ref.size].view(ref.shape).cpu().numpy()
        assert np.abs(dev - ref).max() <= 1e-4 * max(np.abs(ref).max(), 1e-12), s
        _, _, idx, alpha, _ = B.nonuniform_quantize_buckets(w, bits, bucket_type, bsize, clusters=views[i].cpu().numpy())
        np.testing.assert_allclose(dev, B.bucket_nuq_grads(g, idx, 1 << bits, alpha), rtol=0,
                                   atol=1e-5 * max(np.abs(ref).max(), 1e-12))


def resnet50_kernel_shapes():
    """HWIO kernels of ResNet-50 (utils/external/resnet_model.py), creation order."""
    shapes = [(7, 7, 3, 64)]
    cin = 64
    for filters, blocks in zip([64, 128, 256, 512], [3, 4, 6, 3]):
        for b in range(blocks):
            if b == 0:
                shapes.append((1, 1, cin, filters * 4))
            shapes += [(1, 1, cin, filters), (3, 3, filters, filters), (1, 1, filters, filters * 4)]
            cin = filters * 4
    shapes.append((2048, 1001))
    return shapes


@pytest.mark.parametrize('bucket_type', ['channel', 'split'])
def test_resnet50_tensor_list_4bit(bucket_type):
    shapes = resnet50_kernel_shapes()[1:-1]          # the 52 quantized kernels (first conv and dense left out)
    assert len(shapes) == 52 and sum(int(np.prod(s)) for s in shapes) > 23e6
    torch.manual_seed(0)
    src = [torch.randn(s, device='cuda') * (2.0 / np.prod(s[:-1])) ** 0.5 for s in shapes]
    dst = [torch.empty_like(w) for w in src]
    bsize = 256 if bucket_type == 'split' else 0
    q = ops.CodebookWeightQuantizer(src, dst, 4, keep_index=True, use_buckets=True, bucket_type=bucket_type,
                                    bucket_size=bsize)
    q.quantile_init()
    q.forward()
    torch.cuda.synchronize()
    cbs = q.codebooks()
    for i in range(0, 52, 3):                                          # every third kernel through the numpy oracle
        w = src[i].cpu().numpy()
        qx, c_ref, idx_ref, _, _ = B.nonuniform_quantize_buckets(w, 4, bucket_type, bsize)
        assert np.array_equal(cbs[i][:16].cpu().numpy(), c_ref), i
        assert np.array_equal(dst[i].cpu().numpy(), qx), i
        assert np.array_equal(q.idx[q.idx_offsets[i]:q.idx_offsets[i] + w.size].cpu().numpy(), idx_ref.astype(np.uint8))


# ------------------------------------------------------------------------------------------------------------ learner
def make(**flags):
    FLAGS.reset()
    from pocketflow_b200.nets import resnet_at_cifar10 as R
    from pocketflow_b200.learners.learner_utils import create_learner
    import pocketflow_b200.learners.nonuniform_quantization.learner  # noqa: F401
    FLAGS.resnet_size, FLAGS.batch_size, FLAGS.learner = 8, 16, 'non-uniform'
    for k, v in dict(dict(nuql_use_buckets=True, summ_step=10 ** 9, save_step=10 ** 9), **flags).items():
        setattr(FLAGS, k, v)
    return create_learner(None, R.ModelHelper())


@pytest.mark.parametrize('mode,bucket_type', [('weights', 'channel'), ('cluster', 'channel'), ('both', 'channel'),
                                              ('weights', 'split'), ('both', 'split')])
def test_bucketed_learner_step_matches_oracle(monkeypatch, mode, bucket_type):
    from oracle.step_oracle import StepOracle
    monkeypatch.setenv('PF_CONV_PATH', 'fp32')
    bsize = 100
    lrn = make(nuql_weight_bits=4, enbl_dst=True, nuql_opt_mode=mode, nuql_bucket_type=bucket_type,
               nuql_bucket_size=bsize)
    ex = lrn.sess_train
    assert ex.wq.use_buckets
    state, tstate = ex.store.state_dict(), ex.teacher.store.state_dict()
    cnames = [op.vars['clusters'].name for op in ex.wq_ops]
    assert all(n.startswith('model/') and n.endswith('/nonuniform_bucket_quantize/clusters:0') for n in cnames)
    trainable = [v.name for v in lrn.trainable_vars]
    assert set(cnames) <= set(trainable)
    frozen = {'weights': cnames, 'cluster': [n for n in trainable if n not in cnames], 'both': []}[mode]
    for op, cn in zip(ex.wq_ops, cnames):
        w = state[op.vars['kernel'].name]
        nb = ops.uq_bucket_layout(w.shape, True, bucket_type, bsize)[0]
        assert state[cn].shape == (16, nb)
        _, c_ref, _, _, _ = B.nonuniform_quantize_buckets(w, 4, bucket_type, bsize)
        assert np.array_equal(state[cn], c_ref), cn                      # quantile init after the build
    teacher = StepOracle(ex.teacher.ops, ex.teacher.logits_t, lrn.images)
    orc = B.BucketStepOracle(ex.ops, ex.logits_t, lrn.images, lrn.labels, ex.loss, ex.weight_quant, ex.act_quant,
                             teacher)
    images, labels = lrn.iterator_train.next_batch()
    ex.buf[lrn.images].copy_(images)
    ex.buf[lrn.labels].copy_(labels)
    ex.run_step(lrn.lrn_rate(0))
    got = ex.fetch_losses()
    for op, cn in zip(ex.wq_ops, cnames):
        v = op.vars['kernel']
        q_ref, _, _, _, _ = B.nonuniform_quantize_buckets(state[v.name], 4, bucket_type, bsize, state[cn])
        assert np.array_equal(ex.store.view(v, ex.QW).cpu().numpy(), q_ref), v.name
    ref, new_state, grads = orc.step(state, images.numpy(), labels.numpy(), dict(kind='adam', slots={}),
                                     lrn.lrn_rate(0), teacher_state=tstate, frozen=frozen)
    for k in ('ce', 'l2', 'dst_loss', 'loss'):
        assert rel(got[k], ref[k]) <= 1e-5, (k, got[k], ref[k])
    assert any(v.name in cnames for v in ex.loss.l2)                        # the codebooks are in the l2 term
    after = ex.store.state_dict()
    for n in frozen:
        assert np.array_equal(after[n], state[n]), n
    if mode != 'weights':
        for op, cn in zip(ex.wq_ops, cnames):
            g_dev = ex.store.view(op.vars['clusters'], ex.G).cpu().numpy()
            assert np.abs(g_dev - grads[cn]).max() <= 1e-4 * max(np.abs(grads[cn]).max(), 1e-12), cn
    lr = lrn.lrn_rate(0)
    wd_of = {v.name: c for v, c in ex.loss.l2.items()}
    for n in [n for n in trainable if n not in frozen and 'batch_normalization' not in n]:
        d_dev = after[n] - state[n]
        if n in cnames:
            # Adam's first step is ~lr * sign(g + wd * c): a centroid whose total gradient lies within the gradient
            # tolerance above of 0 steps either way, so the codebook update is checked against TF's Adam applied to the
            # device's own (checked) gradient; the stored values round to fp32, hence one ulp of slack
            g_dev = ex.store.view(lrn.graph_train.variables[n], ex.G).cpu().numpy()
            w_exp, _, _ = O.adam_step(state[n], np.zeros_like(state[n]), np.zeros_like(state[n]), g_dev, lr,
                                      F32(0.9), F32(0.999), wd=wd_of.get(n, 0.0))
            assert (np.abs(after[n] - w_exp) <= 2e-2 * lr + np.spacing(np.abs(state[n]))).all(), n
            continue
        d_ref = new_state[n] - state[n]
        assert np.abs(d_dev - d_ref).max() <= 2e-2 * lr + 1e-12, n


def test_bucketed_checkpoint_roundtrip_and_bundle_names(tmp_path, capsys):
    from pocketflow_b200.utils import tf_bundle
    lrn = make(nuql_weight_bits=3, nuql_bucket_type='channel', nuql_opt_mode='both', enbl_dst=False,
               nuql_save_quant_model_path=str(tmp_path / 'nuql' / 'model.ckpt'), ckpt_format='tf')
    ex = lrn.sess_train
    for _ in range(2):
        lrn.train_step()
    lrn._NonUniformQuantLearner__save_model()                      # what train() does every save_step
    loss = lrn.evaluate(nb_iters=1)                                 # restores that checkpoint first
    assert np.isfinite(loss)
    out = capsys.readouterr().out
    nb_tot = sum(ops.uq_bucket_layout(op.vars['kernel'].shape, True, 'channel', 0)[0] for op in ex.wq_ops)
    nw = sum(lrn.statistics['num_weights'])
    assert ('bucket storage: %d bit' % (64 * nb_tot)) in out and ('weight storage: %d bit' % (3 * nw)) in out
    from pocketflow_b200.learners.abstract_learner import latest_checkpoint, load_checkpoint
    fn = latest_checkpoint(str(tmp_path / 'nuql'))
    tensors = tf_bundle.load(fn)
    saved = ex.store.state_dict()
    for op in ex.wq_ops:
        name = op.vars['clusters'].name.replace(':0', '')
        nb = op.vars['kernel'].shape[-1]
        assert name.endswith('/nonuniform_bucket_quantize/clusters') and tensors[name].shape == (8, nb)
        assert np.array_equal(tensors[name], saved[op.vars['clusters'].name])
    lrn2 = make(nuql_weight_bits=3, nuql_bucket_type='channel', nuql_opt_mode='both', enbl_dst=False)
    lrn2.sess_train.store.load_state_dict(load_checkpoint(fn), strict=False)
    got = lrn2.sess_train.store.state_dict()
    for op in ex.wq_ops:
        n = op.vars['clusters'].name
        assert np.array_equal(got[n], saved[n]), n


def test_rl_set_bits_reinitialises_every_bucket():
    lrn = make(nuql_weight_bits=4, nuql_bucket_type='split', nuql_bucket_size=64, enbl_dst=False)
    ex = lrn.sess_train
    nw = len(ex.wq_ops)
    w_bits = [1 + i % 4 for i in range(nw)]
    lrn.rl_set_bits(w_bits, [32] * len(ex.aq_ops))
    state = ex.store.state_dict()
    for op, b in zip(ex.wq_ops, w_bits):
        _, c_ref, _, _, _ = B.nonuniform_quantize_buckets(state[op.vars['kernel'].name], b, 'split', 64)
        c = state[op.vars['clusters'].name]
        assert np.array_equal(c[:1 << b], c_ref) and not c[1 << b:].any(), op.name
    ex.wq.forward()
    for op, b in zip(ex.wq_ops, w_bits):
        v = op.vars['kernel']
        q_ref, _, _, _, _ = B.nonuniform_quantize_buckets(state[v.name], b, 'split', 64, state[op.vars['clusters'].name])
        assert np.array_equal(ex.store.view(v, ex.QW).cpu().numpy(), q_ref), v.name


def test_mobilenet_channel_buckets_depthwise_is_one_bucket():
    import importlib
    import pocketflow_b200.datasets.ilsvrc12_dataset as D
    importlib.reload(D)
    from pocketflow_b200.nets import mobilenet_at_ilsvrc12 as M
    importlib.reload(M)
    from pocketflow_b200.learners.learner_utils import create_learner
    import pocketflow_b200.learners.nonuniform_quantization.learner  # noqa: F401
    FLAGS.reset()
    FLAGS.batch_size, FLAGS.learner, FLAGS.nb_classes = 2, 'non-uniform', 1001
    FLAGS.nuql_use_buckets, FLAGS.nuql_bucket_type, FLAGS.nuql_weight_bits = True, 'channel', 4
    FLAGS.summ_step = FLAGS.save_step = 10 ** 9
    lrn = create_learner(None, M.ModelHelper())
    ex = lrn.sess_train
    dw = [i for i, op in enumerate(ex.wq_ops) if op.type == 'DepthwiseConv2dNative']
    assert dw and all(ex.wq.nb[i] == 1 for i in dw)
    assert ex.wq.clusters is not None                                  # depthwise ops have no variable: private table
    ex.wq.forward()
    state = ex.store.state_dict()
    cbs = ex.wq.codebooks()
    for i, op in enumerate(ex.wq_ops):
        v = op.vars['kernel']
        qx, c_ref, _, _, _ = B.nonuniform_quantize_buckets(state[v.name], 4, 'channel', 0)
        assert np.array_equal(cbs[i][:16].cpu().numpy(), c_ref), v.name
        assert np.array_equal(ex.store.view(v, ex.QW).cpu().numpy(), qx), v.name
    lrn.train_step()
    assert np.isfinite(ex.fetch_losses()['loss'])
