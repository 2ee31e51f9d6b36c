"""The inference batch norm folded into the forward epilogue of the tensor-core convs (pf_conv2d_tc_fwd*_bn,
Executor._plan_bn_fold) gives the same bits as the conv followed by ops.bn_apply_eval:

* kernel level: the conv output y, the post-BN planes and the post-BN fp32 tensor, in the forward variants that can
  carry the fold (TMA feed at BN 64 / 128, cp.async feed at 16 / 32 channels; residual none, in registers and through
  the ring; ReLU / ReLU6 / none; ragged last tiles; several tiles per CTA);
* executor level (PF_POISON=1, so a buffer the fold forgot to write shows up as NaN): the ResNet-50 teacher at batch
  128 and the ResNet-20 teacher at batch 256 give bitwise the logits and every operand-plane buffer of the unfused plan,
  with one bn_apply_eval launch fewer per folded BN."""
import numpy as np
import pytest
import torch

from pocketflow_b200 import ops
from pocketflow_b200.flags import FLAGS

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')


@pytest.fixture(autouse=True)
def _flags_back_to_defaults():
    """the workloads' flag settings do not leak into the tests that run after these"""
    yield
    FLAGS.reset()


def bits(t):
    return t.contiguous().view(-1).view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


def same(a, b):
    return torch.equal(bits(a), bits(b))


# id, (n, h, w, c, k, r, s, stride, pad), x as planes, residual, bias + relu, PF_TC_* knobs,
# (feed, bn, ring) of the plan the fused call must run
CASES = [
    ('tma-bn128-3x3', (2, 11, 13, 64, 256, 3, 3, 1, 1), True, False, False, {}, (1, 128, 0)),
    ('tma-bn128-ragged-cols', (2, 11, 13, 64, 192, 3, 3, 1, 1), True, False, True, {}, (1, 128, 0)),
    ('tma-bn64', (2, 11, 13, 64, 64, 3, 3, 1, 1), True, False, False, {}, (1, 64, 0)),
    ('tma-bn64-res-ring2', (2, 9, 9, 64, 128, 1, 1, 1, 0), True, True, False, {'PF_TC_BN': 64}, (1, 64, 2)),
    ('tma-bn64-res-regs', (2, 9, 9, 64, 128, 1, 1, 1, 0), True, True, False, {'PF_TC_BN': 64, 'PF_TC_RING': 0},
     (1, 64, 0)),
    ('tma-bn128-res-regs', (2, 9, 9, 64, 256, 1, 1, 1, 0), True, True, False, {}, (1, 128, 0)),
    ('tma-many-tiles-res', (40, 28, 28, 64, 256, 1, 1, 1, 0), True, True, False, {}, (1, 128, 0)),
    ('tma-many-tiles-s2', (160, 28, 28, 128, 128, 3, 3, 2, 1), True, False, True, {}, (1, 128, 0)),
    ('cp-c16', (2, 9, 9, 16, 16, 3, 3, 1, 1), True, False, False, {}, (0, 16, 0)),
    ('cp-c16-res', (2, 9, 9, 16, 16, 3, 3, 1, 1), True, True, False, {}, (0, 16, 0)),
    ('cp-c32-res-fp32x', (2, 9, 9, 32, 32, 3, 3, 1, 1), False, True, True, {}, (0, 32, 0)),
    ('cp-c32-k64-s2', (4, 16, 16, 32, 64, 3, 3, 2, 1), True, False, False, {}, (0, 64, 0)),
    ('cp-many-tiles-res', (128, 32, 32, 16, 16, 3, 3, 1, 1), True, True, False, {}, (0, 16, 0)),
    ('cp-many-tiles-fp32x', (256, 16, 16, 32, 32, 3, 3, 1, 1), False, True, False, {}, (0, 32, 0)),
]
KNOBS = ('PF_TC_BN', 'PF_TC_RING')


@pytest.mark.parametrize('act', [0, 1, 2])
@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_fused_conv_bn_is_bitwise_the_unfused_pair(case, act, monkeypatch):
    name, (n, h, w, c, k, r, s, st, pad), planes_x, with_res, bias_relu, knobs, want = case
    for kname in KNOBS:
        monkeypatch.delenv(kname, raising=False)
    for kname, v in knobs.items():
        monkeypatch.setenv(kname, str(v))
    g = torch.Generator().manual_seed(sum(map(ord, name)) + act)
    p, q = (h + 2 * pad - r) // st + 1, (w + 2 * pad - s) // st + 1
    d = ops.conv_desc(n, h, w, c, k, r, s, p, q, st, st, pad, pad)
    x = torch.randn(n, h, w, c, generator=g).to(DEV)
    xp = ops.Planes(x.numel(), DEV)
    ops.split_bf16(x, xp)
    tw = ops.TcWeights(d, DEV, need_dgrad=False)
    tw.prepare((torch.randn(r, s, c, k, generator=g) / np.sqrt(r * s * c)).to(DEV))
    bias = torch.randn(k, generator=g).to(DEV) if bias_relu else None
    res = torch.randn(n, p, q, k, generator=g).to(DEV) if with_res else None
    mean, var = torch.randn(k, generator=g).to(DEV), (torch.rand(k, generator=g) * 2 + 0.05).to(DEV)
    gamma, beta = torch.randn(k, generator=g).to(DEV), torch.randn(k, generator=g).to(DEV)
    eps, m = 1e-3, n * p * q

    def conv(y, bn_out=None):
        if planes_x:
            ops.conv2d_tc_fwd_planes(d, xp, tw, bias, bias_relu, y, res, bn_out)
        else:
            ops.conv2d_tc_fwd(d, x, tw, bias, bias_relu, y, res, bn_out)

    nan = lambda: torch.full((n, p, q, k), float('nan'), device=DEV)
    y_ref, z_ref, pl_ref = nan(), nan(), ops.Planes(m * k, DEV)
    conv(y_ref)
    ops.bn_apply_eval(y_ref, m, k, mean, var, eps, gamma, beta, act, z_ref, None, pl_ref)
    for with_f32, with_planes in ((True, True), (False, True), (True, False)):
        y, z, pl = nan(), nan(), ops.Planes(m * k, DEV)
        pl.hi.fill_(float('nan'))
        pl.lo.fill_(float('nan'))
        conv(y, ops.TcBnOut(mean, var, eps, gamma, beta, act, z if with_f32 else None, pl if with_planes else None))
        plan = ops.conv2d_tc_last_plan()
        assert (plan['feed'], plan['bn'], plan['ring']) == want, plan
        torch.cuda.synchronize()
        assert same(y, y_ref), 'conv output differs'
        if with_f32:
            assert same(z, z_ref), 'post-BN fp32 differs'
        else:
            assert torch.isnan(z).all(), 'post-BN fp32 written without being asked for'
        if with_planes:
            assert same(pl.hi, pl_ref.hi) and same(pl.lo, pl_ref.lo), 'post-BN planes differ'


def test_fold_arguments_are_checked():
    d = ops.conv_desc(1, 4, 4, 64, 64, 1, 1, 4, 4, 1, 1, 0, 0)
    xp = ops.Planes(16 * 64, DEV)
    tw = ops.TcWeights(d, DEV, need_dgrad=False)
    y = torch.zeros(16 * 64, device=DEV)
    v = torch.ones(64, device=DEV)
    with pytest.raises(ValueError):          # neither output
        ops.conv2d_tc_fwd_planes(d, xp, tw, None, False, y, None, ops.TcBnOut(v, v, 1e-3, v, v, 0))
    with pytest.raises(ValueError):          # act out of range
        ops.conv2d_tc_fwd_planes(d, xp, tw, None, False, y, None, ops.TcBnOut(v, v, 1e-3, v, v, 3, y))


# ---------------------------------------------------------------------------------------------------- executor level
def teacher_graph(workload):
    import bench
    from pocketflow_b200 import graph as G
    mod = bench.setup_flags(workload)
    mh = mod.ModelHelper()
    g = G.Graph()
    with g.as_default():
        with G.variable_scope('data'):
            im, _ = mh.build_dataset_train().get_next()
        with G.variable_scope('distilled_model'):
            out = mh.forward_eval(im)
    return g, im, out


def run_eval(workload, fold, monkeypatch):
    """(logits, {BN name: (fp32 output or None, planes or None)}, bn_apply_eval launches, fold count) of one forward
    of a fresh eval executor (parameters from the store's seed, images from a fixed seed)"""
    from pocketflow_b200 import engine
    monkeypatch.setenv('PF_POISON', '1')
    if not fold:
        monkeypatch.setattr(engine.Executor, '_plan_bn_fold', lambda self: {})
    g, im, out = teacher_graph(workload)
    ex = engine.Executor(g, im, out, DEV, train=False)
    ex.buf[im].copy_(torch.randn(im.shape, generator=torch.Generator().manual_seed(7)).to(DEV))
    calls = []
    orig = ops.bn_apply_eval
    monkeypatch.setattr(ops, 'bn_apply_eval', lambda *a, **kw: (calls.append(1), orig(*a, **kw))[1])
    logits = ex.forward().clone()
    monkeypatch.setattr(ops, 'bn_apply_eval', orig)
    torch.cuda.synchronize()
    outs = {}
    for op in ex.ops:
        if op.type == 'FusedBatchNorm':
            f32, pl = ex.outputs_of(op)
            outs[op.name] = (f32.clone() if f32 is not None else None,
                             (pl.hi.clone(), pl.lo.clone()) if pl is not None else None)
    nfold = len(ex.bn_fold)
    del ex
    torch.cuda.empty_cache()
    return logits, outs, len(calls), nfold


@pytest.mark.parametrize('workload,n_fold', [('resnet50_uq8_dst_b128', 48), ('resnet20_uq8_dst_b256', None)])
def test_folded_eval_plan_is_bitwise_the_unfused_one(workload, n_fold, monkeypatch):
    with monkeypatch.context() as mp:
        lf, of, cf, nf = run_eval(workload, True, mp)
    with monkeypatch.context() as mp:
        lu, ou, cu, nu = run_eval(workload, False, mp)
    assert nu == 0 and nf > 0 and (n_fold is None or nf == n_fold)
    assert cu - cf == nf, (cu, cf, nf)
    assert torch.isfinite(lf).all() and same(lf, lu), 'logits differ'
    assert of.keys() == ou.keys()
    for name in of:
        (f1, p1), (f2, p2) = of[name], ou[name]
        assert (f1 is None) == (f2 is None) and (p1 is None) == (p2 is None), name
        if f1 is not None:
            assert not torch.isnan(f1).any() and same(f1, f2), name
        if p1 is not None:
            assert same(p1[0], p2[0]) and same(p1[1], p2[1]), name
