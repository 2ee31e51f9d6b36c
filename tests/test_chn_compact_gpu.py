"""Compact (channel-pruned) inference graphs on the GPU: pf_gather_channels, the BN apply with a fused gather, the
compact convolutions teacher-forced against the full-width masked ones, end-to-end logits, the exported checkpoint's
round trip, and a compact model made from a `chn-pruned-gpu` learner's own checkpoint."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pocketflow_b200 import compact as C
from pocketflow_b200 import ops
from pocketflow_b200.engine import Executor
from pocketflow_b200.flags import FLAGS

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)


def _planes(n):
    return ops.Planes(n, DEV)


def _idx(kept, cout):
    return torch.tensor(list(kept) + [-1] * (cout - len(kept)), dtype=torch.int32, device=DEV)


def _ref_gather(x, idx):
    i = idx.long()
    return torch.where(i >= 0, x[..., i.clamp_min(0)], torch.zeros((), device=x.device))


def _split(x):
    p = _planes(x.numel())
    ops.split_bf16(x.contiguous(), p)
    return p


CASES = [(24, [1, 2, 3, 5, 20, 23], 8), (64, list(range(16, 48)), 32), (64, [0, 1, 2, 3, 8, 9, 10, 11, 60], 16),
         (260, list(range(0, 260, 3)), 96), (64, [], 16), (260, list(range(4, 260)), 256)]


@pytest.mark.parametrize('poison', [False, True])
@pytest.mark.parametrize('c,kept,cout', CASES)
def test_gather_channels_is_exact(c, kept, cout, poison, monkeypatch):
    if poison:
        monkeypatch.setenv('PF_POISON', '1')          # output planes start as NaN: every element must be written
    g = torch.Generator().manual_seed(c + cout)
    x = torch.randn(2, 4, 5, c, generator=g).to(DEV)
    idx = _idx(kept, cout)
    ref = _ref_gather(x, idx)
    y = torch.full((2, 4, 5, cout), float('nan'), device=DEV)
    yp = _planes(ref.numel())
    ops.gather_channels(x, idx, y, yp)
    torch.cuda.synchronize()
    assert torch.equal(y, ref)
    assert torch.equal(y[..., len(kept):], torch.zeros_like(y[..., len(kept):]))
    rp = _split(ref)
    assert torch.equal(yp.hi.view(torch.int16), rp.hi.view(torch.int16))
    assert torch.equal(yp.lo.view(torch.int16), rp.lo.view(torch.int16))
    # planes in: planes out copy the bits, fp32 out is hi + lo
    xp = _split(x)
    zp = _planes(ref.numel())
    z = torch.empty_like(y)
    m = x.numel() // c
    ops.gather_channels(None, idx, z, zp, x_planes=(xp, m, c))
    torch.cuda.synchronize()
    assert torch.equal(zp.hi.view(torch.int16), rp.hi.view(torch.int16))
    xs = (xp.hi.float() + xp.lo.float()).view(x.shape)
    assert torch.equal(z, _ref_gather(xs, idx))


@pytest.mark.parametrize('act', [0, 1, 2])
@pytest.mark.parametrize('c,kept,cout', CASES[:4])
def test_bn_apply_eval_gather_equals_bn_apply_then_gather(c, kept, cout, act):
    g = torch.Generator().manual_seed(act * 7 + c)
    x = (3 * torch.randn(4, 6, 6, c, generator=g)).to(DEV)
    mm, mv = torch.randn(c, generator=g).to(DEV), (torch.rand(c, generator=g) + 0.1).to(DEV)
    ga, be = torch.randn(c, generator=g).to(DEV), torch.randn(c, generator=g).to(DEV)
    m = x.numel() // c
    full = torch.empty_like(x)
    ops.bn_apply_eval(x, m, c, mm, mv, 1e-3, ga, be, act, full)
    idx = _idx(kept, cout)
    ref = _ref_gather(full, idx)
    y = torch.full(ref.shape, float('nan'), device=DEV)
    yp = _planes(ref.numel())
    ops.bn_apply_eval_gather(x, m, c, mm, mv, 1e-3, ga, be, act, idx, y, yp)
    torch.cuda.synchronize()
    assert torch.equal(y, ref)
    rp = _split(ref)
    assert torch.equal(yp.hi.view(torch.int16), rp.hi.view(torch.int16))
    assert torch.equal(yp.lo.view(torch.int16), rp.lo.view(torch.int16))


# ------------------------------------------------------------------ whole networks
def _net(name, batch):
    import importlib
    FLAGS.reset()
    mod = {'mobilenet_v1': 'mobilenet_at_ilsvrc12', 'mobilenet_v2': 'mobilenet_at_ilsvrc12', 'resnet50': 'resnet_at_ilsvrc12',
           'resnet20': 'resnet_at_cifar10', 'lenet': 'lenet_at_cifar10'}
    if name == 'mobilenet_v2':
        FLAGS.mobilenet_version = 2
    if name == 'resnet50':
        FLAGS.resnet_size = 50
    if name == 'resnet20':
        FLAGS.resnet_size = 20
    mh = importlib.import_module('pocketflow_b200.nets.' + mod[name]).ModelHelper()
    return C.build_eval_graph(mh, batch)


def _masked_state(g, lg, ratio, seed):
    rng = np.random.default_rng(seed)
    st = {}
    for op in C.reachable_ops(g, lg):
        for role, v in op.vars.items():
            a = v.initializer(rng, v.shape)
            if role == 'moving_variance':
                a = rng.uniform(0.5, 1.5, v.shape).astype(np.float32)
            elif role in ('moving_mean', 'beta'):
                a = (0.1 * rng.standard_normal(v.shape)).astype(np.float32)
            st[v.name] = a
    return C.fake_prune(g, lg, st, ratio, seed)


def _torch_conv64(x, k, op):
    (kh, kw), (sh, sw), (pt, pl) = op.attrs['ksize'], op.attrs['strides'], op.attrs['pad']
    n, h, w, c = x.shape
    p, q = op.output.shape[1:3]
    pb, pr = (p - 1) * sh + kh - h - pt, (q - 1) * sw + kw - w - pl
    xx = F.pad(x.permute(0, 3, 1, 2).double(), (pl, max(pr, 0), pt, max(pb, 0)))
    y = F.conv2d(xx, k.permute(3, 2, 0, 1).double(), stride=(sh, sw))
    return y[:, :, :p, :q].permute(0, 2, 3, 1)


@pytest.mark.parametrize('path', ['tc', 'fp32'])
@pytest.mark.parametrize('name,res_batch', [('mobilenet_v1', 2), ('mobilenet_v1', 100), ('resnet50', 2),
                                            ('resnet50', 100), ('mobilenet_v2', 2), ('mobilenet_v2', 64), ('lenet', 2),
                                            ('lenet', 100)])
def test_compact_convs_teacher_forced_against_the_masked_full_width_conv(name, res_batch, path):
    g, im, lg = _net(name, res_batch)
    st = _masked_state(g, lg, 0.5, 3)
    cm = C.CompactModel.from_masked(g, im, lg, st, DEV, conv_path=path)
    # a separate executor without the conv + residual epilogue, so every conv output is its own buffer
    ex = Executor(cm.graph, cm.images, cm.logits, DEV, train=False, conv_path=path, fuse_add=False)
    ex.store.load_state_dict(cm.state, strict=True)
    full = Executor(g, im, lg, DEV, train=False, conv_path=path)
    full.store.load_state_dict(st, strict=True)
    if path == 'tc':
        tc_full = {op.name for op in full.ops if op in full.tc or op in full.im2col}
        assert tc_full <= {op.name for op in ex.ops if op in ex.tc or op in ex.im2col}
    ex.buf[cm.images].copy_(torch.randn(im.shape, generator=torch.Generator().manual_seed(1)).to(DEV))
    ex.forward(training=False)
    torch.cuda.synchronize()
    fops = {op.name: op for op in C.reachable_ops(g, lg)}
    bar = 2e-5 if path == 'tc' else 1e-6
    checked = 0
    for op in ex.ops:
        if op.type != 'Conv2D':
            continue
        fop = fops[op.name]
        lin = C._input_layouts(fop, cm.rec)[0]
        lout = cm.rec['tensors'][fop.output.name]
        xp = ex.planes_of(op.inputs[0])
        xin = (xp.hi.float() + xp.lo.float()).view(op.inputs[0].shape) if xp is not None else ex.T(op.inputs[0])
        xfull = torch.zeros(fop.inputs[0].shape, dtype=torch.float64, device=DEV)
        rows = [j for j, c in enumerate(lin) if c >= 0]
        xfull[..., [lin[j] for j in rows]] = xin[..., rows].double()
        if path == 'fp32':
            # the full-width masked conv itself (exact-fp32 kernel) on the scattered input
            y = torch.empty(fop.output.shape, device=DEV)
            bias = full.store.view(fop.vars['bias']) if 'bias' in fop.vars else None
            ops.conv2d_fwd(full.desc[fop], xfull.float().contiguous(), full.kernel_of(fop), bias, fop in full.fused_act, y)
            ref = y.double()
        else:
            # split-bf16 operands: against the float64 conv of the same masked kernel
            k = torch.from_numpy(st[fop.vars['kernel'].name]).to(DEV)
            ref = _torch_conv64(xfull, k, fop)
            if 'bias' in fop.vars:
                ref = ref + torch.from_numpy(st[fop.vars['bias'].name]).to(DEV).double()
            if op in ex.fused_act:
                ref = ref.clamp_min(0.0)
        cols = [j for j, c in enumerate(lout) if c >= 0]
        got = ex.buf[op.output][..., cols].double()
        ref = ref[..., [lout[j] for j in cols]]
        scale = float(ref.abs().max())
        assert float((got - ref).abs().max()) <= bar * max(scale, 1e-30), (op.name, path)
        assert not torch.any(ex.buf[op.output][..., [j for j, c in enumerate(lout) if c < 0]])
        checked += 1
    assert checked == sum(1 for op in fops.values() if op.type == 'Conv2D')


@pytest.mark.parametrize('name', ['mobilenet_v1', 'resnet50', 'mobilenet_v2', 'lenet'])
def test_compact_logits_match_the_masked_full_width_model_and_round_trip(name, tmp_path):
    g, im, lg = _net(name, 16)
    st = _masked_state(g, lg, 0.5, 5)
    cm = C.CompactModel.from_masked(g, im, lg, st, DEV)
    full = Executor(g, im, lg, DEV, train=False)
    full.store.load_state_dict(st, strict=True)
    x = torch.randn(im.shape, generator=torch.Generator().manual_seed(2)).to(DEV)
    full.buf[im].copy_(x)
    ref = full.forward(training=False).clone()
    got = cm.forward(x).clone()
    torch.cuda.synchronize()
    assert float((got - ref).abs().max()) <= 1e-4 * float(ref.abs().max())
    top2 = ref.topk(2, dim=1).values
    clear = (top2[:, 0] - top2[:, 1]) > 2e-4 * float(ref.abs().max())
    assert torch.equal(got.argmax(1)[clear], ref.argmax(1)[clear])
    for fmt in ('npz', 'tf'):
        path = str(tmp_path / fmt / 'model')
        cm.export(path, fmt)
        cm2 = C.CompactModel.load(g, im, lg, path, DEV)
        again = cm2.forward(x).clone()
        torch.cuda.synchronize()
        assert torch.equal(again, got)


def test_compact_model_of_a_chn_pruned_gpu_learner_checkpoint(tmp_path):
    from pocketflow_b200.learners.abstract_learner import latest_checkpoint, load_checkpoint, save_checkpoint
    from pocketflow_b200.learners.channel_pruning_gpu.learner import ChannelPrunedGpuLearner
    from pocketflow_b200.nets import resnet_at_cifar10 as R
    FLAGS.reset()
    FLAGS.resnet_size, FLAGS.batch_size = 20, 32
    FLAGS.cpg_save_path = str(tmp_path / 'cpg' / 'model.ckpt')
    FLAGS.save_path = str(tmp_path / 'none' / 'model.ckpt')
    lrn = ChannelPrunedGpuLearner(None, R.ModelHelper())
    lrn.init_from_full()
    lrn.choose_channels(nb_iters_layer=3)
    ex = lrn.sess_train
    save_checkpoint(FLAGS.cpg_save_path, ex.store.state_dict(), 0)
    ckpt = load_checkpoint(latest_checkpoint(os.path.dirname(FLAGS.cpg_save_path)))
    g, im, lg = C.build_eval_graph(R.ModelHelper(), FLAGS.batch_size)
    cm = C.CompactModel.from_masked(g, im, lg, ckpt, DEV)
    # each conv's input count is what survives in the learner's channel mask of that kernel
    for (name, cin, kept), v in zip(cm.conv_report(), lrn.maskable_vars):
        assert name.split('/', 1)[1] == v.name.split('/', 1)[1].rsplit('/', 1)[0] + '/Conv2D'
        mask = ex.store.view(v, ex.MASK)
        assert kept == int(torch.count_nonzero(mask.reshape(-1, cin, mask.shape[-1]).abs().sum(dim=(0, 2))).item())
    # the eval losses of the learner's own evaluation pass and of the compact model agree on the same batches
    for _ in range(3):
        lrn.feed(ex, lrn.iterator_train)
        ex.forward_eval_loss()
        ref_loss = float(ex.fetch_losses()['ce'])
        labels = ex.buf[lrn.labels]
        logits = cm.forward(ex.buf[lrn.images])
        ce = float(-(labels * torch.log_softmax(logits.double(), dim=1)).sum(1).mean())
        assert abs(ce - ref_loss) <= 1e-4 * abs(ref_loss), (ce, ref_loss)
