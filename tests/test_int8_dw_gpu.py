"""The u8 depthwise convolution of the integer inference model (pf_dwconv_u8_fwd, int8.select with
cfg['int8_depthwise']) on the GPU: every MobileNet-v1 depthwise shape at batch 256 (exact window sums S and J, the
affine epilogue against float64, NaN for a header that is not one plane of levels), the other filter shapes the kernel
takes, and a whole MobileNet-v1 integer model with u8 depthwise layers against the float64 oracle."""
import importlib
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from support import QUIET, dw_fwd_ref, free, make  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _release():
    """executors and integer models hold device memory in reference cycles: collect them before the next test"""
    yield
    from pocketflow_b200.flags import FLAGS
    FLAGS.reset()
    free()


BATCH = 256

# (H, W, C, stride) of MobileNet-v1's depthwise layers (3 x 3, SAME: pad 1 at stride 1, 0 top / left at stride 2 on
# an even input); 14 x 14 x 512 at stride 1 is five layers
SHAPES = [(112, 112, 32, 1), (112, 112, 64, 2), (56, 56, 128, 1), (56, 56, 128, 2), (28, 28, 256, 1),
          (28, 28, 256, 2), (14, 14, 512, 1), (14, 14, 512, 2), (7, 7, 1024, 1)]


def _sid(s):
    return '%dx%d_c%d_s%d' % s


def _desc(n, h, w, c, r, s, st, pt, pl):
    """depthwise descriptor with the SAME output size ceil(h / stride) x ceil(w / stride)"""
    from pocketflow_b200 import ops
    return ops.conv_desc(n, h, w, c, c, r, s, -(-h // st), -(-w // st), st, st, pt, pl)


def _mbv1_desc(shape):
    h, w, c, st = shape
    return _desc(BATCH, h, w, c, 3, 3, st, 1 if st == 1 else 0, 1 if st == 1 else 0)


def _hdr(scale, nplanes=1):
    return torch.tensor([np.float32(scale).view(np.int32), nplanes], dtype=torch.int32, device='cuda')


def _run(d, qa, qw, scale, alpha, beta, bits, nplanes=1):
    """qa uint8 [N, H, W, C], qw uint8 [R, S, C]"""
    from pocketflow_b200 import ops
    y = torch.empty(d.n, d.p, d.q, d.c, device='cuda')
    ops.dwconv_u8_fwd(d, qa, _hdr(scale, nplanes), qw.reshape(-1, d.c).contiguous(), alpha, beta, bits, y)
    return y


def _levels(d, hi, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    if hi == 'max':
        return (torch.full((d.n, d.h, d.w, d.c), 255, dtype=torch.uint8, device='cuda'),
                torch.full((d.r, d.s, d.c), 255, dtype=torch.uint8, device='cuda'))
    qa = torch.randint(0, hi + 1, (d.n, d.h, d.w, d.c), generator=g, device='cuda', dtype=torch.int32).to(torch.uint8)
    qw = torch.randint(0, hi + 1, (d.r, d.s, d.c), generator=g, device='cuda', dtype=torch.int32).to(torch.uint8)
    return qa, qw


def _sums(d, qa, qw):
    """float64 S = sum q_a q_w and J = sum q_a over each window (exact: integers far below 2^53)"""
    x = qa.double()
    return dw_fwd_ref(x, qw.double(), d), dw_fwd_ref(x, torch.ones(d.r, d.s, d.c, dtype=torch.float64, device='cuda'), d)


def _exact(d, hi, seed):
    """unit scales (k_w = 1, scale 1): (alpha, beta) = (1, 0) writes S, (0, 1) writes J, both exactly"""
    one, zero = torch.ones(1, device='cuda'), torch.zeros(1, device='cuda')
    qa, qw = _levels(d, hi, seed)
    S, J = _sums(d, qa, qw)
    assert float(S.max()) < 2 ** 20 and float(J.max()) < 2 ** 12
    ys = _run(d, qa, qw, 1.0, one, zero, 1)
    assert torch.equal(ys.double(), S), float((ys.double() - S).abs().max())
    del ys
    yj = _run(d, qa, qw, 1.0, zero, one, 1)
    assert torch.equal(yj.double(), J), float((yj.double() - J).abs().max())


@pytest.mark.parametrize('hi', [3, 31, 255, 'max'], ids=['2bit', '5bit', '8bit', 'all255'])
@pytest.mark.parametrize('shape', SHAPES, ids=_sid)
def test_u8_dw_exact_sums(shape, hi):
    _exact(_mbv1_desc(shape), hi, 17 + shape[2])


# filters and strides that take the one-pixel-per-item kernel: other filter sizes, unequal strides, and a 3 x 3
# layer with a single output row
OTHER = [(8, 20, 20, 48, 1, 9, 1, 0, 4), (8, 20, 20, 32, 5, 1, 2, 2, 0), (8, 9, 9, 16, 2, 2, 2, 0, 0),
         (8, 2, 2, 64, 3, 3, 2, 0, 0), (8, 17, 17, 32, 1, 1, 1, 0, 0)]


@pytest.mark.parametrize('geom', OTHER, ids=lambda g: '%dx%d_c%d_f%dx%d_s%d' % (g[1], g[2], g[3], g[4], g[5], g[6]))
def test_u8_dw_other_filters_exact(geom):
    from pocketflow_b200 import ops
    d = _desc(*geom)
    assert ops.dwconv_u8_supported(d)
    for hi, seed in ((255, 3), ('max', 0)):
        _exact(d, hi, seed)


def _affine_ref(d, qa, qw, scale, alpha, beta, bits):
    """(float64 of the kernel's formula with its fp32 constants e1 = (alpha / k_w) scale and e2 = beta scale, bound
    |e1 S| + |e2 J|)"""
    rk = np.float32(1) / np.float32(2 ** bits - 1)
    al, be = alpha.cpu().numpy(), beta.cpu().numpy()
    e1 = torch.from_numpy(((al * rk).astype(np.float32) * np.float32(scale)).astype(np.float64)).cuda()
    e2 = torch.from_numpy((be * np.float32(scale)).astype(np.float64)).cuda()
    S, J = _sums(d, qa, qw)
    return e1 * S + e2 * J, (e1 * S).abs() + (e2 * J).abs()


@pytest.mark.parametrize('per_channel', [False, True], ids=['per_layer', 'per_channel'])
@pytest.mark.parametrize('shape', SHAPES, ids=_sid)
def test_u8_dw_affine(shape, per_channel):
    """W8A8 levels with real scales.  fma(S, e1, J e2) rounds twice (J e2, then the sum), so it is within
    2^-23 (|e1 S| + |e2 J|) of float64; the bar is twice that, 2^-22, a few fp32 ulps."""
    d = _mbv1_desc(shape)
    qa, qw = _levels(d, 255, 5)
    g = torch.Generator(device='cuda').manual_seed(7)
    nb = d.c if per_channel else 1
    alpha = (torch.rand(nb, generator=g, device='cuda') * 0.2 + 0.01).contiguous()
    beta = (-alpha * torch.rand(nb, generator=g, device='cuda')).contiguous()
    scale = np.float32(3.7) / np.float32(255)
    y = _run(d, qa, qw, scale, alpha, beta, 8).double()
    ref, bound = _affine_ref(d, qa, qw, scale, alpha, beta, 8)
    ok = (y - ref).abs() <= 2.0 ** -22 * bound
    assert bool(ok.all()), float(((y - ref).abs() / bound.clamp_min(1e-300)).max())


@pytest.mark.parametrize('shape', [SHAPES[0], SHAPES[7]], ids=_sid)
def test_u8_dw_header_not_levels_is_nan(shape):
    """a header with nplanes != 1 (the activation's range did not start at 0) makes every output NaN"""
    d = _mbv1_desc(shape)
    qa, qw = _levels(d, 255, 1)
    one, zero = torch.ones(1, device='cuda'), torch.zeros(1, device='cuda')
    y = _run(d, qa, qw, 1.0, one, zero, 8, nplanes=0)
    assert bool(torch.isnan(y).all())


# ---------------------------------------------------------------------------------------------- whole model
def _model(batch, flags):
    from pocketflow_b200 import compact, int8
    from pocketflow_b200.flags import FLAGS
    mod = importlib.import_module('pocketflow_b200.nets.mobilenet_at_ilsvrc12')
    import pocketflow_b200.learners.uniform_quantization.learner  # noqa: F401
    FLAGS.reset()
    FLAGS.uql_weight_bits, FLAGS.uql_activation_bits = 8, 8
    for k, v in flags.items():
        setattr(FLAGS, k, v)
    g, images, logits = compact.build_eval_graph(mod.ModelHelper(), batch)
    return g, images, logits, dict(int8.config_from_flags(), int8_depthwise=True)


def _learner_state(flags):
    """a --learner uniform checkpoint state: the learner's own store after two training steps"""
    lrn = make('mobilenet_at_ilsvrc12', 'uniform', 16, reload='ilsvrc12_dataset',
               **dict(QUIET, uql_weight_bits=8, uql_activation_bits=8, **flags))
    for _ in range(2):
        lrn.train_step()
    return lrn.sess_train.store.state_dict()


@pytest.mark.parametrize('flags', [dict(), dict(uql_use_buckets=True, uql_bucket_type='channel')],
                         ids=['per_layer', 'channel_buckets'])
def test_int_model_planned_dw_against_oracle(flags, tmp_path):
    """the executor's plan lowers all 13 depthwise layers to pf_dwconv_u8_fwd; distance to the float64 oracle, top-1
    agreement with fake-quant and a bit-identical export / load"""
    from oracle.step_oracle import StepOracle
    from pocketflow_b200 import compact, int8
    from pocketflow_b200.engine import _U8DwConv
    state = _learner_state(flags)
    g, images, logits, cfg = _model(32, flags)
    dev = torch.device('cuda', 0)
    im = int8.IntModel.from_checkpoint(g, images, logits, state, cfg, dev)
    dws = [op for op in im.ex.ops if op.type == 'DepthwiseConv2dNative']
    assert len(dws) == 13 and all(isinstance(im.ex.depthwise[op], _U8DwConv) for op in dws)
    for op in dws:                       # the producers feeding only u8 layers no longer write the fp32 tensor
        assert im.ex.depthwise[op].bn.others is False, op.name
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
    print('mbv1 int8_depthwise %s: int %.3e fake-quant %.3e (of max|ref|), top-1 agreement %.4f'
          % (flags, e_int, e_fq, agree))
    # the measure of test_int8_gpu.py's whole-model test: quantizer level flips set both distances
    assert e_int <= 1.3 * e_fq, (e_int, e_fq)
    assert agree == 1.0
    fn = im.export(str(tmp_path / 'int8'))
    assert os.path.exists(fn)
    with open(str(tmp_path / 'int8') + '.int8.json') as f:
        rec = json.load(f)
    assert rec['version'] == int8.SIDECAR_VERSION == 2 and rec['config']['int8_depthwise'] is True
    im2 = int8.IntModel.load(g, images, logits, str(tmp_path / 'int8'), dev)
    assert {op.name for op, lo in im2.ex.depthwise.items() if isinstance(lo, _U8DwConv)} == {op.name for op in dws}
    assert torch.equal(im2.forward(x), li)
