"""The u8 x u8 inference path (pocketflow_b200/int8.py, pf_conv2d_u8_fwd, pf_bn_eval_levels_u8) on the GPU:
the kernel on every ResNet-50 and MobileNet-v1 pointwise and 3x3 shape at batch 128 (exact integer sums, the affine
epilogue against float64, the fused BN + ReLU + residual), the level producer against a float64 restatement, and whole
integer models against the float64 oracle forward of the fake-quantized model."""
import importlib
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from support import QUIET, free, make  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _release():
    """the learners, executors and integer models of a test hold GBs of device memory in reference cycles (an executor
    and its lowerings point at each other): collect them before the next test allocates"""
    yield
    from pocketflow_b200.flags import FLAGS
    FLAGS.reset()
    free()

BATCH = 128


def _dev():
    return torch.device('cuda', 0)


# distinct (H, W, Cin, Cout, filter, stride, (pad top, pad left), P, Q) of the u8 convolutions of ResNet-50 and
# MobileNet-v1 (int8.select on their inference graphs): every pointwise and 3x3 shape the integer models run
SHAPES = [
    (7, 7, 512, 512, 3, 1, (1, 1), 7, 7),
    (7, 7, 512, 1024, 1, 1, (0, 0), 7, 7),
    (7, 7, 512, 2048, 1, 1, (0, 0), 7, 7),
    (7, 7, 1024, 1024, 1, 1, (0, 0), 7, 7),
    (7, 7, 2048, 512, 1, 1, (0, 0), 7, 7),
    (14, 14, 256, 256, 3, 1, (1, 1), 14, 14),
    (14, 14, 256, 512, 1, 1, (0, 0), 14, 14),
    (14, 14, 256, 1024, 1, 1, (0, 0), 14, 14),
    (14, 14, 512, 512, 1, 1, (0, 0), 14, 14),
    (14, 14, 512, 512, 3, 2, (1, 1), 7, 7),
    (14, 14, 1024, 256, 1, 1, (0, 0), 14, 14),
    (14, 14, 1024, 512, 1, 1, (0, 0), 14, 14),
    (14, 14, 1024, 2048, 1, 2, (0, 0), 7, 7),
    (28, 28, 128, 128, 3, 1, (1, 1), 28, 28),
    (28, 28, 128, 256, 1, 1, (0, 0), 28, 28),
    (28, 28, 128, 512, 1, 1, (0, 0), 28, 28),
    (28, 28, 256, 256, 1, 1, (0, 0), 28, 28),
    (28, 28, 256, 256, 3, 2, (1, 1), 14, 14),
    (28, 28, 512, 128, 1, 1, (0, 0), 28, 28),
    (28, 28, 512, 256, 1, 1, (0, 0), 28, 28),
    (28, 28, 512, 1024, 1, 2, (0, 0), 14, 14),
    (56, 56, 64, 64, 1, 1, (0, 0), 56, 56),
    (56, 56, 64, 64, 3, 1, (1, 1), 56, 56),
    (56, 56, 64, 128, 1, 1, (0, 0), 56, 56),
    (56, 56, 64, 256, 1, 1, (0, 0), 56, 56),
    (56, 56, 128, 128, 1, 1, (0, 0), 56, 56),
    (56, 56, 128, 128, 3, 2, (1, 1), 28, 28),
    (56, 56, 256, 64, 1, 1, (0, 0), 56, 56),
    (56, 56, 256, 128, 1, 1, (0, 0), 56, 56),
    (56, 56, 256, 512, 1, 2, (0, 0), 28, 28),
]


def _conv64(x, w, k, s, pad, p, q):
    """float64 NHWC conv, zero padding (pt, pl), output cropped to p x q"""
    import torch.nn.functional as F
    pt, pl = pad
    xt = x.permute(0, 3, 1, 2)
    pb = max((p - 1) * s + k - x.shape[1] - pt, 0)
    pr = max((q - 1) * s + k - x.shape[2] - pl, 0)
    y = F.conv2d(F.pad(xt, (pl, pr, pt, pb)), w.permute(3, 2, 0, 1), stride=s)
    return y[:, :, :p, :q].permute(0, 2, 3, 1)


def _operands(shape, qa_hi, qw_hi, seed):
    h, w, c, k, ks, s, pad, p, q = shape
    g = torch.Generator(device='cuda').manual_seed(seed)
    qa = torch.randint(0, qa_hi + 1, (BATCH, h, w, c), generator=g, device='cuda', dtype=torch.int32).to(torch.uint8)
    qw = torch.randint(0, qw_hi + 1, (ks, ks, c, k), generator=g, device='cuda', dtype=torch.int32).to(torch.uint8)
    return qa, qw


def _run(shape, qa, qw, scale, alpha, beta, bits, residual=None, bn_out=None, relu=False):
    from pocketflow_b200 import ops
    h, w, c, k, ks, s, pad, p, q = shape
    d = ops.conv_desc(BATCH, h, w, c, k, ks, ks, p, q, s, s, pad[0], pad[1])
    hdr = torch.tensor([np.float32(scale).view(np.int32), 1], dtype=torch.int32, device='cuda')
    nseg = (c + 127) // 128
    csum = qa.view(-1, nseg, min(c, 128)).to(torch.float32).sum(-1).contiguous()
    wl = qw.reshape(-1, k).t().contiguous()
    y = torch.empty(BATCH, p, q, k, device='cuda')
    ops.conv2d_u8_fwd(d, qa, hdr, csum, wl, alpha, beta, bits, y, None, relu, residual, bn_out)
    return y


@pytest.mark.parametrize('shape', SHAPES, ids=lambda s: '%dx%d_%d-%d_k%ds%d' % (s[0], s[1], s[2], s[3], s[4], s[5]))
def test_u8_conv_exact_sums(shape):
    """scale 1, one bit (k_w = 1), alpha 1, beta 0: the output is the integer sum itself, kept below 2^24 by making one
    operand binary — so every byte value of the other operand is checked exactly, in both roles"""
    k = shape[3]
    one, zero = torch.ones(k, device='cuda'), torch.zeros(k, device='cuda')
    for i, (ah, wh) in enumerate(((255, 1), (1, 255))):
        qa, qw = _operands(shape, ah, wh, 11 + i)
        y = _run(shape, qa, qw, 1.0, one, zero, 1)
        ref = _conv64(qa.double(), qw.double(), shape[4], shape[5], shape[6], shape[7], shape[8])
        assert float(ref.abs().max()) < 2 ** 24
        assert torch.equal(y.double(), ref), (shape, (ah, wh), float((y.double() - ref).abs().max()))


def _affine_refs(shape, qa, qw, scale, alpha, beta, bits):
    """(float64 restatement of the kernel's formula with its fp32 column constants, float64 conv of the fake-quantized
    fp32 operands, magnitude bound |e1 S| + |e2 J|)"""
    kq = np.float32(2 ** bits - 1)
    rk = np.float32(1) / kq
    al, be = alpha.double().cpu().numpy().astype(np.float32), beta.double().cpu().numpy().astype(np.float32)
    e1 = torch.from_numpy(((al * rk).astype(np.float32) * np.float32(scale)).astype(np.float64)).cuda()
    e2 = torch.from_numpy((be * np.float32(scale)).astype(np.float64)).cuda()
    ks, s, pad, p, q = shape[4:]
    S = _conv64(qa.double(), qw.double(), ks, s, pad, p, q)
    J = _conv64(qa.double(), torch.ones_like(qw[..., :1], dtype=torch.float64), ks, s, pad, p, q)
    formula = e1 * S + e2 * J
    bound = (e1 * S).abs() + (e2 * J).abs()
    qa_v = (qa.float() * np.float32(scale)).double()          # fp32 values of the fake-quantized operands
    qw_v = ((alpha * (qw.float().reshape(-1, shape[3]) / float(kq))) + beta).reshape(qw.shape).double()
    fq = _conv64(qa_v, qw_v, ks, s, pad, p, q)
    return formula, fq, bound


@pytest.mark.parametrize('shape', SHAPES, ids=lambda s: '%dx%d_%d-%d_k%ds%d' % (s[0], s[1], s[2], s[3], s[4], s[5]))
def test_u8_conv_affine(shape):
    """full-range W8A8 levels, per-channel scales: the epilogue against float64"""
    k = shape[3]
    qa, qw = _operands(shape, 255, 255, 5)
    g = torch.Generator(device='cuda').manual_seed(7)
    alpha = (torch.rand(k, generator=g, device='cuda') * 0.2 + 0.01).contiguous()
    beta = (-alpha * torch.rand(k, generator=g, device='cuda')).contiguous()
    scale = np.float32(3.7) / np.float32(255)
    y = _run(shape, qa, qw, scale, alpha, beta, 8).double()
    formula, fq, bound = _affine_refs(shape, qa, qw, scale, alpha, beta, 8)
    assert bool(((y - formula).abs() <= 2.0 ** -22 * bound).all()), float(((y - formula).abs() / bound).max())
    err = float((y - fq).abs().max() / fq.abs().max())
    assert err <= 1e-6, err


@pytest.mark.parametrize('shape', SHAPES[::3], ids=lambda s: '%dx%d_%d-%d_k%ds%d' % (s[0], s[1], s[2], s[3], s[4], s[5]))
def test_u8_conv_bn_relu_residual(shape):
    """the folded inference batch norm + ReLU after the residual add, against float64 of pf_bn_apply_eval's chain"""
    from pocketflow_b200 import ops
    k = shape[3]
    qa, qw = _operands(shape, 255, 255, 9)
    g = torch.Generator(device='cuda').manual_seed(3)
    alpha = torch.rand(1, generator=g, device='cuda') * 0.1 + 0.01
    beta = -alpha * 0.1
    scale = np.float32(2.0) / np.float32(255)
    res = torch.randn(BATCH, shape[7], shape[8], k, generator=g, device='cuda')
    mean, var = torch.randn(k, generator=g, device='cuda'), torch.rand(k, generator=g, device='cuda') + 0.5
    gamma, bbeta = torch.randn(k, generator=g, device='cuda'), torch.randn(k, generator=g, device='cuda')
    post = torch.empty(BATCH, shape[7], shape[8], k, device='cuda')
    bn_out = ops.TcBnOut(mean, var, 1e-3, gamma, bbeta, 1, post)
    y = _run(shape, qa, qw, scale, alpha.contiguous(), beta.contiguous(), 8, residual=res, bn_out=bn_out)
    _, fq, _ = _affine_refs(shape, qa, qw, scale, alpha, beta, 8)
    ref = fq + res.double()
    assert float((y.double() - ref).abs().max() / ref.abs().max()) <= 1e-6
    # the BN of the kernel's own fp32 sum, in float64: only the BN's roundings separate the two
    z = ((y.double() - mean.double()) / torch.sqrt(var.double() + 1e-3)) * gamma.double() + bbeta.double()
    z = torch.clamp_min(z, 0)
    assert float((post.double() - z).abs().max() / z.abs().max()) <= 1e-6


@pytest.mark.parametrize('c,act', [(64, 1), (256, 2), (1024, 1)])
def test_u8_levels_producer(c, act):
    """levels, range, header and channel sums of pf_bn_eval_levels_u8 against a float64 restatement"""
    from pocketflow_b200 import ops
    m = BATCH * 14 * 14
    g = torch.Generator(device='cuda').manual_seed(c)
    x = torch.randn(m, c, generator=g, device='cuda') * 2
    mean, var = torch.randn(c, generator=g, device='cuda') * 0.1, torch.rand(c, generator=g, device='cuda') + 0.5
    gamma, beta = torch.rand(c, generator=g, device='cuda') + 0.5, torch.randn(c, generator=g, device='cuda') * 0.1
    rng = torch.zeros(2, dtype=torch.int32, device='cuda')
    levels = torch.empty(m * c, dtype=torch.uint8, device='cuda')
    hdr = torch.zeros(2, dtype=torch.int32, device='cuda')
    nseg = (c + 127) // 128
    csum = torch.empty(m * nseg, device='cuda')
    ops.bn_eval_levels_u8(x, m, c, mean, var, 1e-3, gamma, beta, act, 8, rng, levels, hdr, csum)
    # the fake-quant path's fp32 values: pf_bn_apply_eval writes y and the range, act_quant the quantized tensor
    y = torch.empty_like(x)
    rng2 = torch.tensor([-1, 0], dtype=torch.int32, device='cuda')
    ops.bn_apply_eval(x, m, c, mean, var, 1e-3, gamma, beta, act, y, rng2)
    assert torch.equal(rng, rng2)
    mx = float(y.max())
    assert float(y.min()) == 0.0
    alpha = np.float32(np.float32(mx) - np.float32(0)) + np.float32(1e-10)
    # float64 restatement of the level: rint(fp32((y / alpha)) * 255), the division and the product rounded to fp32
    xn = (y.double() / float(alpha)).float()
    lv = torch.round((xn.double() * 255).float().double())
    assert torch.equal(levels.view(m, c).double(), lv)
    hs = hdr.cpu().numpy()
    assert hs[1] == 1 and hs[0:1].view(np.float32)[0] == np.float32(alpha / np.float32(255))
    assert torch.equal(csum.view(m, nseg).double(), lv.view(m, nseg, -1).sum(-1))


def _model(net, batch, flags):
    from pocketflow_b200 import compact, int8
    from pocketflow_b200.flags import FLAGS
    mod = importlib.import_module('pocketflow_b200.nets.' + net)
    import pocketflow_b200.learners.uniform_quantization.learner  # noqa: F401
    FLAGS.reset()
    FLAGS.uql_weight_bits, FLAGS.uql_activation_bits = 8, 8
    for k, v in flags.items():
        setattr(FLAGS, k, v)
    mh = mod.ModelHelper()
    g, images, logits = compact.build_eval_graph(mh, batch)
    return g, images, logits, int8.config_from_flags()


def _learner_state(net, flags):
    """a --learner uniform checkpoint state: the learner's own store after two training steps"""
    reload = 'cifar10_dataset' if 'cifar' in net else 'ilsvrc12_dataset'
    lrn = make(net, 'uniform', 16, reload=reload, **dict(QUIET, uql_weight_bits=8, uql_activation_bits=8, **flags))
    for _ in range(2):
        lrn.train_step()
    return lrn.sess_train.store.state_dict()


CASES = [
    ('resnet_at_cifar10', 128, dict(resnet_size=20, uql_use_buckets=True, uql_bucket_type='channel')),
    ('resnet_at_cifar10', 128, dict(resnet_size=20, uql_use_buckets=True, uql_bucket_type='channel', enbl_dst=True)),
    ('resnet_at_ilsvrc12', 32, dict(resnet_size=50, uql_use_buckets=True, uql_bucket_type='channel')),
    ('mobilenet_at_ilsvrc12', 32, dict()),
]


@pytest.mark.parametrize('net,batch,flags', CASES, ids=['rn20', 'rn20_dst', 'rn50', 'mbv1'])
def test_int_model_against_oracle(net, batch, flags, tmp_path):
    from oracle.step_oracle import StepOracle
    from pocketflow_b200 import compact, int8
    state = _learner_state(net, flags)
    g, images, logits, cfg = _model(net, batch, flags)
    dev = _dev()
    im = int8.IntModel.from_checkpoint(g, images, logits, state, cfg, dev)
    assert any(why is None for _, why in im.sel)
    full = compact.map_state(g, compact.reachable_ops(g, logits), state)
    fq = int8.fake_quant_executor(g, images, logits, full, cfg, dev)
    x = torch.randn(images.shape, generator=torch.Generator().manual_seed(1)).to(dev)
    li = im.forward(x).clone()
    fq.buf[fq.images].copy_(x)
    lf = fq.forward(training=False).clone()
    assert bool(torch.isfinite(li).all())
    wq, aq = int8._specs(g, cfg)
    orc = StepOracle(compact.reachable_ops(g, logits), logits, images, weight_quant=wq, act_quant=aq)
    params = {k: torch.from_numpy(v).double().to(dev) for k, v in full.items()}
    ref = orc.forward(params, x.double(), training=False)[logits.name].double()
    scale = float(ref.abs().max())
    e_int = float((li.double() - ref).abs().max()) / scale
    e_fq = float((lf.double() - ref).abs().max()) / scale
    agree = float((li.argmax(1) == lf.argmax(1)).float().mean())
    print('%s: int %.3e fake-quant %.3e (of max|ref|), top-1 agreement %.4f' % (net, e_int, e_fq, agree))
    # Against the float64 oracle both fp32 forwards are dominated by quantizer levels that flip where a value lies
    # within rounding of a level boundary (a flip in an early layer moves every later layer), not by the convolutions'
    # arithmetic, which the kernel tests above hold to float64 layer by layer; measured on the H100: int / fake-quant
    # 4.2e-3 / 4.5e-3 (ResNet-20), 4.9e-3 / 4.8e-3 (with distillation), 4.0e-3 / 3.9e-3 (ResNet-50), 9.0e-4 / 7.5e-4
    # (MobileNet-v1).  The bar: the same distance within that spread.
    assert e_int <= 1.3 * e_fq, (e_int, e_fq)
    assert agree >= 0.99
    # round trip: export, load, the same logits
    fn = im.export(str(tmp_path / 'int8'))
    assert os.path.exists(fn)
    im2 = int8.IntModel.load(g, images, logits, str(tmp_path / 'int8'), dev)
    assert torch.equal(im2.forward(x), li)
