"""GPU parity of the layer kernels (conv fwd/dgrad/wgrad, batch-norm, pooling, add, softmax) against
a float64 PyTorch-CPU reference of the same op (these are floating-point kernels: tolerance 1e-5
relative to the tensor's scale — the north star's fp32 bar — written at each assert)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pocketflow_b200 import ops

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def close(got, ref, tol=1e-5):
    got = got.detach().cpu().double()
    ref = ref.detach().cpu().double()
    scale = ref.abs().max().item() + 1e-30
    err = (got - ref).abs().max().item()
    assert err <= tol * scale, 'max err %.3e vs scale %.3e' % (err, scale)


CONV_CASES = [
    # n, h, w, c, k, r, s, stride, pad_t/l, pad_b/r
    (4, 16, 16, 16, 32, 3, 3, 1, 1, 1),
    (2, 17, 15, 8, 12, 3, 3, 2, 1, 1),
    (3, 32, 32, 3, 16, 3, 3, 1, 1, 1),        # Cin=3: scalar path
    (2, 24, 24, 3, 64, 7, 7, 2, 3, 3),        # ResNet-50 stem shape family
    (2, 8, 8, 64, 256, 1, 1, 1, 0, 0),
    (2, 9, 9, 32, 64, 1, 1, 2, 0, 0),         # strided 1x1 projection
    (5, 14, 14, 32, 64, 5, 5, 1, 0, 0),       # LeNet VALID 5x5
    (2, 8, 8, 20, 10, 3, 3, 1, 1, 1),         # Cout=10: scalar path
    (2, 12, 12, 16, 16, 3, 3, 2, 0, 1),       # TF 'SAME' stride 2 on even size: pad (0,1)
]


@pytest.mark.parametrize('case', CONV_CASES)
def test_conv2d_fwd_dgrad_wgrad(case):
    n, h, w, c, k, r, s, st, p0, p1 = case
    g = torch.Generator().manual_seed(sum(case))
    x = torch.randn(n, h, w, c, generator=g)
    wt = torch.randn(r, s, c, k, generator=g) * (2.0 / (r * s * c)) ** 0.5
    bias = torch.randn(k, generator=g)
    p = (h + p0 + p1 - r) // st + 1
    q = (w + p0 + p1 - s) // st + 1
    # float64 reference
    xd = x.double().permute(0, 3, 1, 2).requires_grad_(True)
    wd = wt.double().permute(3, 2, 0, 1).requires_grad_(True)
    yd = F.conv2d(F.pad(xd, (p0, p1, p0, p1)), wd, stride=st)
    dy = torch.randn(n, p, q, k, generator=g)
    yd.backward(dy.double().permute(0, 3, 1, 2))
    y_ref = yd.permute(0, 2, 3, 1)
    dx_ref = xd.grad.permute(0, 2, 3, 1)
    dw_ref = wd.grad.permute(2, 3, 1, 0)
    d = ops.conv_desc(n, h, w, c, k, r, s, p, q, st, st, p0, p0)
    X, W, DY = x.to(DEV), wt.to(DEV).contiguous(), dy.to(DEV)
    Y = torch.empty(n, p, q, k, device=DEV)
    ops.conv2d_fwd(d, X, W, None, False, Y)
    close(Y, y_ref)
    ops.conv2d_fwd(d, X, W, bias.to(DEV), True, Y)
    close(Y, torch.relu(y_ref + bias.double()))
    DX = torch.full((n, h, w, c), 7.0, device=DEV)
    wt_ws = torch.empty(wt.numel(), device=DEV)
    ops.conv2d_dgrad(d, DY, W, wt_ws, False, DX)
    close(DX, dx_ref)
    ops.conv2d_dgrad(d, DY, W, wt_ws, True, DX)
    close(DX, 2 * dx_ref)
    ws = torch.empty(max(ops.conv2d_wgrad_workspace_floats(d), 4), device=DEV)
    DW = torch.empty_like(W)
    ops.conv2d_wgrad(d, X, DY, ws, DW)
    close(DW, dw_ref)


def test_dense_as_conv():
    g = torch.Generator().manual_seed(3)
    x, w, b = torch.randn(37, 64, generator=g), torch.randn(64, 10, generator=g), torch.randn(10, generator=g)
    d = ops.conv_desc(37, 1, 1, 64, 10, 1, 1, 1, 1, 1, 1, 0, 0)
    Y = torch.empty(37, 10, device=DEV)
    ops.conv2d_fwd(d, x.to(DEV), w.to(DEV), b.to(DEV), False, Y)
    close(Y, x.double() @ w.double() + b.double())
    dy = torch.randn(37, 10, generator=g)
    DW, ws = torch.empty(64, 10, device=DEV), torch.empty(max(ops.conv2d_wgrad_workspace_floats(d), 4), device=DEV)
    ops.conv2d_wgrad(d, x.to(DEV), dy.to(DEV), ws, DW)
    close(DW, x.double().t() @ dy.double())
    DX, wt = torch.empty(37, 64, device=DEV), torch.empty(640, device=DEV)
    ops.conv2d_dgrad(d, dy.to(DEV), w.to(DEV), wt, False, DX)
    close(DX, dy.double() @ w.double().t())


@pytest.mark.parametrize('shape', [(8, 16, 16, 16), (3, 7, 5, 64), (256, 1, 1, 256), (2, 9, 9, 2048)])
@pytest.mark.parametrize('act', [0, 1, 2])
def test_batch_norm_train_fwd_bwd(shape, act):
    g = torch.Generator().manual_seed(shape[0] + act)
    x = torch.randn(shape, generator=g) * 2 + 3.0
    c = shape[-1]
    m = x.numel() // c
    gamma, beta = torch.rand(c, generator=g) + 0.5, torch.randn(c, generator=g) * (2.0 if act == 2 else 0.3)
    dy = torch.randn(shape, generator=g)
    eps, mom = 1e-5, 0.997
    xd = x.double().requires_grad_(True)
    gd, bd = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    red = (0, 1, 2)
    mean, var = xd.mean(red), xd.var(red, unbiased=False)
    z = (xd - mean) * torch.rsqrt(var + eps) * gd + bd
    yd = z if act == 0 else (torch.relu(z) if act == 1 else torch.clamp(z, 0, 6))
    yd.backward(dy.double())
    X, DY = x.to(DEV), dy.to(DEV)
    mean_t, var_t, rstd_t = (torch.empty(c, device=DEV) for _ in range(3))
    mm, mv = torch.zeros(c, device=DEV), torch.ones(c, device=DEV)
    ws = torch.empty(3 * c * ops.BN_MAX_SPLITS, device=DEV)
    ops.bn_train_stats(X, m, c, eps, mom, mean_t, var_t, rstd_t, mm, mv, ws)
    close(mean_t, mean, 1e-6)
    close(var_t, var, 1e-5)
    close(mm, mean * (1 - mom), 1e-5)
    close(mv, mom + var * m / (m - 1) * (1 - mom), 1e-5)
    Y = torch.empty_like(X)
    slot = torch.zeros(2, dtype=torch.int32, device=DEV)
    ops.minmax_reset(slot)
    ops.bn_apply(X, m, c, mean_t, rstd_t, gamma.to(DEV), beta.to(DEV), act, Y, slot)
    close(Y, yd, 2e-5)
    mnmx = ops.decode_ordered(slot.cpu().numpy().view(np.uint32))
    assert mnmx[0] == Y.min().item() and mnmx[1] == Y.max().item()
    DX, DG, DB = torch.empty_like(X), torch.empty(c, device=DEV), torch.empty(c, device=DEV)
    ops.bn_bwd(DY, X, m, c, mean_t, rstd_t, gamma.to(DEV), beta.to(DEV), act, DG, DB, DX, False, ws)
    # float64 backward on the kernel's own fp32 statistics, with the activation mask taken from the fp32 op chain
    # the kernel evaluates: a pre-activation within rounding distance of 0 or 6 cannot flip the mask
    G, B = gamma.to(DEV), beta.to(DEV)
    z = ((X - mean_t) * rstd_t) * G + B
    mask = (z > 0) & (z < 6) if act == 2 else (z > 0 if act == 1 else torch.ones_like(z, dtype=torch.bool))
    xh = ((X.double() - mean_t.double()) * rstd_t.double()).view(m, c)
    dz = DY.double().view(m, c) * mask.view(m, c)
    db_ref, dg_ref = dz.sum(0), (dz * xh).sum(0)
    dx_ref = G.double() * rstd_t.double() * (dz - db_ref / m - xh * dg_ref / m)
    close(DG, dg_ref)
    close(DB, db_ref)
    close(DX.view(m, c), dx_ref)


def test_batch_norm_eval():
    g = torch.Generator().manual_seed(5)
    x = torch.randn(4, 6, 6, 32, generator=g)
    mm, mv = torch.randn(32, generator=g), torch.rand(32, generator=g) + 0.5
    ga, be = torch.rand(32, generator=g) + 0.5, torch.randn(32, generator=g)
    rstd = torch.empty(32, device=DEV)
    ops.bn_eval_prepare(mv.to(DEV), 32, 1e-5, rstd)
    Y = torch.empty(4, 6, 6, 32, device=DEV)
    ops.bn_apply(x.to(DEV), 4 * 36, 32, mm.to(DEV), rstd, ga.to(DEV), be.to(DEV), 1, Y)
    ref = torch.relu((x.double() - mm.double()) * torch.rsqrt(mv.double() + 1e-5) * ga.double() + be.double())
    close(Y, ref)
    Y2 = torch.empty_like(Y)                                            # one-launch inference BN: identical bits
    ops.bn_apply_eval(x.to(DEV), 4 * 36, 32, mm.to(DEV), mv.to(DEV), 1e-5, ga.to(DEV), be.to(DEV), 1, Y2)
    assert torch.equal(Y, Y2)


@pytest.mark.parametrize('cfg', [(2, 12, 12, 16, 3, 2, 0), (2, 11, 11, 8, 3, 2, 1), (3, 28, 28, 32, 2, 2, 0)])
def test_maxpool(cfg):
    n, h, w, c, k, s, pt = cfg
    g = torch.Generator().manual_seed(sum(cfg))
    x = torch.randn(n, h, w, c, generator=g)
    total = max((-(-h // s) - 1) * s + k - h, 0) if pt else 0
    pb = total - pt if pt else 0
    p = (h + pt + pb - k) // s + 1
    xd = x.double().permute(0, 3, 1, 2).requires_grad_(True)
    yd = F.max_pool2d(F.pad(xd, (pt, pb, pt, pb), value=float('-inf')), k, s)
    dy = torch.randn(n, p, p, c, generator=g)
    yd.backward(dy.double().permute(0, 3, 1, 2))
    d = ops.conv_desc(n, h, w, c, c, k, k, p, p, s, s, pt, pt)
    Y = torch.empty(n, p, p, c, device=DEV)
    AM = torch.empty(n, p, p, c, dtype=torch.uint8, device=DEV)
    ops.maxpool_fwd(d, x.to(DEV), Y, AM)
    close(Y, yd.permute(0, 2, 3, 1), 0.0)
    DX = torch.empty(n, h, w, c, device=DEV)
    ops.maxpool_bwd(d, dy.to(DEV), AM, DX)
    close(DX, xd.grad.permute(0, 2, 3, 1), 1e-6)


def test_avgpool_add_relu_colsum_softmax():
    g = torch.Generator().manual_seed(11)
    x = torch.randn(5, 7, 7, 64, generator=g)
    Y = torch.empty(5, 64, device=DEV)
    ops.global_avgpool_fwd(x.to(DEV), 5, 49, 64, Y)
    close(Y, x.double().mean((1, 2)))
    dy = torch.randn(5, 64, generator=g)
    DX = torch.empty(5, 7, 7, 64, device=DEV)
    ops.global_avgpool_bwd(dy.to(DEV), 5, 49, 64, DX)
    close(DX, (dy.double() / 49)[:, None, None, :].expand(5, 7, 7, 64))
    a, b = torch.randn(1003, generator=g), torch.randn(1003, generator=g)
    out = torch.empty(1003, device=DEV)
    ops.add(a.to(DEV), b.to(DEV), out)
    assert torch.equal(out.cpu(), a + b)
    ops.add(a.to(DEV), None, out, accumulate=True)
    close(out, (a + b + a).double(), 1e-6)
    y = torch.relu(torch.randn(300, generator=g))
    dz = torch.empty(300, device=DEV)
    ops.relu_bwd(a[:300].to(DEV).contiguous(), y.to(DEV), dz)
    assert torch.equal(dz.cpu(), a[:300] * (y > 0))
    mat = torch.randn(777, 10, generator=g)
    cs = torch.empty(10, device=DEV)
    ops.colsum(mat.to(DEV), 777, 10, cs)
    close(cs, mat.double().sum(0))
    lg = torch.randn(33, 10, generator=g)
    P = torch.empty(33, 10, device=DEV)
    ops.softmax_fwd(lg.to(DEV), P)
    pd = torch.softmax(lg.double().requires_grad_(True), -1)
    close(P, pd)
    lgd = lg.double().requires_grad_(True)
    pd = torch.softmax(lgd, -1)
    dp = torch.randn(33, 10, generator=g)
    pd.backward(dp.double())
    DXs = torch.empty(33, 10, device=DEV)
    ops.softmax_bwd(dp.to(DEV), P, DXs)
    close(DXs, lgd.grad)


@pytest.mark.parametrize('cfg', [(2, 12, 12, 32, 3, 1, 1, 1), (3, 15, 15, 16, 3, 2, 0, 1), (2, 14, 14, 64, 3, 2, 0, 1),
                                 (1, 7, 7, 1024, 3, 1, 1, 1), (2, 10, 10, 64, 3, 1, 1, 1), (2, 9, 9, 32, 3, 1, 0, 0),
                                 (3, 6, 6, 16, 3, 1, 1, 1), (2, 3, 3, 8, 3, 1, 1, 1), (2, 12, 12, 32, 3, 2, 1, 1), (2, 13, 13, 8, 3, 2, 1, 1),
                                 (2, 16, 16, 16, 3, 2, 0, 1)])
def test_depthwise_conv_fwd_dgrad_wgrad(cfg):
    n, h, w, c, k, st, p0, p1 = cfg
    g = torch.Generator().manual_seed(sum(cfg))
    x = torch.randn(n, h, w, c, generator=g)
    wt = torch.randn(k, k, c, 1, generator=g) * 0.3
    p = (h + p0 + p1 - k) // st + 1
    xd = x.double().permute(0, 3, 1, 2).requires_grad_(True)
    wd = wt.double().permute(2, 3, 0, 1).requires_grad_(True)          # [C,1,kh,kw]
    yd = F.conv2d(F.pad(xd, (p0, p1, p0, p1)), wd, stride=st, groups=c)
    dy = torch.randn(n, p, p, c, generator=g)
    yd.backward(dy.double().permute(0, 3, 1, 2))
    d = ops.conv_desc(n, h, w, c, c, k, k, p, p, st, st, p0, p0)
    X, W, DY = x.to(DEV), wt.to(DEV).contiguous(), dy.to(DEV)
    Y = torch.empty(n, p, p, c, device=DEV)
    ops.dwconv_fwd(d, X, W, Y)
    close(Y, yd.permute(0, 2, 3, 1))
    DX = torch.full((n, h, w, c), 2.0, device=DEV)
    ops.dwconv_dgrad(d, DY, W, False, DX)
    close(DX, xd.grad.permute(0, 2, 3, 1))
    ops.dwconv_dgrad(d, DY, W, True, DX)
    close(DX, 2 * xd.grad.permute(0, 2, 3, 1))
    ws = torch.empty(max(ops.dwconv_wgrad_workspace_floats(d), 4), device=DEV)
    DW = torch.empty_like(W)
    ops.dwconv_wgrad(d, X, DY, ws, DW)
    close(DW, wd.grad.permute(2, 3, 0, 1))


def _split_ref(t):
    hi = t.to(torch.bfloat16)
    return hi, (t - hi.float()).to(torch.bfloat16)


@pytest.mark.parametrize('act', [0, 1, 2])
def test_bn_and_act_quant_plane_outputs(act):
    """BN-apply / BN-backward / activation quantizer writing split-bf16 operand planes: the planes are exactly
    split(fp32 result), with or without the fp32 output."""
    g = torch.Generator().manual_seed(11 + act)
    m, c = 4 * 9 * 9, 64
    x = (torch.randn(m, c, generator=g) * 2 + 0.5).to(DEV)
    dy = torch.randn(m, c, generator=g).to(DEV)
    gamma, beta = (torch.rand(c, generator=g) + 0.5).to(DEV), (torch.randn(c, generator=g) * 0.3).to(DEV)
    mean, var, rstd = [torch.empty(c, device=DEV) for _ in range(3)]
    ws = torch.empty(3 * c * ops.BN_MAX_SPLITS, device=DEV)
    ops.bn_train_stats(x, m, c, 1e-5, 0.9, mean, var, rstd, None, None, ws)
    y = torch.empty_like(x)
    slot = torch.zeros(2, dtype=torch.int32, device=DEV)
    ops.minmax_reset(slot.view(1, 2))
    ops.bn_apply(x, m, c, mean, rstd, gamma, beta, act, y, slot)
    pl = ops.Planes(x.numel(), torch.device(DEV))
    y2 = torch.empty_like(x)
    ops.bn_apply(x, m, c, mean, rstd, gamma, beta, act, y2, None, pl)
    h, l = _split_ref(y.view(-1))
    assert torch.equal(y, y2) and torch.equal(pl.hi, h) and torch.equal(pl.lo, l)
    pl2 = ops.Planes(x.numel(), torch.device(DEV))
    ops.bn_apply(x, m, c, mean, rstd, gamma, beta, act, None, None, pl2)            # planes only
    assert torch.equal(pl2.hi, h) and torch.equal(pl2.lo, l)
    # activation quantizer: fp32 + planes, planes only
    q = torch.empty_like(y)
    ops.act_quant(y, q, slot, 8)
    q2 = torch.empty_like(y)
    ops.act_quant(y, q2, slot, 8, pl)
    h, l = _split_ref(q.view(-1))
    assert torch.equal(q, q2) and torch.equal(pl.hi, h) and torch.equal(pl.lo, l)
    ops.act_quant(y, None, slot, 8, pl2)
    assert torch.equal(pl2.hi, h) and torch.equal(pl2.lo, l)
    # BN backward
    dga, dbe, dga2, dbe2 = [torch.empty(c, device=DEV) for _ in range(4)]
    dx = torch.empty_like(x)
    ops.bn_bwd(dy, x, m, c, mean, rstd, gamma, beta, act, dga, dbe, dx, False, ws)
    ops.bn_bwd(dy, x, m, c, mean, rstd, gamma, beta, act, dga2, dbe2, None, False, ws, pl)
    h, l = _split_ref(dx.view(-1))
    assert torch.equal(dga, dga2) and torch.equal(dbe, dbe2) and torch.equal(pl.hi, h) and torch.equal(pl.lo, l)


@pytest.mark.parametrize('act', [0, 1, 2])
def test_bn_stats_range_and_fused_quant(act):
    """Range of act(bn(x)) from the per-channel extremes of x == min/max pass over y (bit-exact), and the fused
    BN + fake-quant pass == bn_apply followed by act_quant (bit-exact), incl. negative gammas."""
    g = torch.Generator().manual_seed(23 + act)
    m, c = 6 * 11 * 11, 96
    x = (torch.randn(m, c, generator=g) * 3 - 0.7).to(DEV)
    gamma, beta = (torch.randn(c, generator=g)).to(DEV), (torch.randn(c, generator=g) * 0.5 + 0.2).to(DEV)
    mean, var, rstd, mean2, var2, rstd2 = [torch.empty(c, device=DEV) for _ in range(6)]
    ws = torch.empty(5 * c * ops.BN_MAX_SPLITS, device=DEV)
    slots = torch.zeros(2, 2, dtype=torch.int32, device=DEV)
    ops.minmax_reset(slots)
    ops.bn_train_stats(x, m, c, 1e-5, 0.9, mean, var, rstd, None, None, ws)
    y = torch.empty_like(x)
    ops.bn_apply(x, m, c, mean, rstd, gamma, beta, act, y, slots[0])
    ops.bn_train_stats_range(x, m, c, 1e-5, 0.9, mean2, var2, rstd2, None, None, gamma, beta, act, slots[1], ws)
    assert torch.equal(mean, mean2) and torch.equal(var, var2) and torch.equal(rstd, rstd2)
    assert torch.equal(slots[0], slots[1]), (ops.decode_ordered(slots[0].cpu().numpy()), ops.decode_ordered(slots[1].cpu().numpy()))
    q = torch.empty_like(y)
    ops.act_quant(y, q, slots[0], 8)
    q2 = torch.empty_like(y)
    pl = ops.Planes(x.numel(), torch.device(DEV))
    ops.bn_apply_quant(x, m, c, mean, rstd, gamma, beta, act, slots[1], 8, q2, pl)
    h, l = _split_ref(q.view(-1))
    assert torch.equal(q, q2) and torch.equal(pl.hi, h) and torch.equal(pl.lo, l)


def test_im2col_planes_matches_fp32_im2col():
    g = torch.Generator().manual_seed(3)
    n, h, w, c, k, r, st, p0 = 3, 23, 23, 3, 64, 7, 2, 2
    p = (h + 2 * p0 + 1 - r) // st + 1
    x = torch.randn(n, h, w, c, generator=g).to(DEV)
    d = ops.conv_desc(n, h, w, c, k, r, r, p, p, st, st, p0, p0)
    kpad = (r * r * c + 15) // 16 * 16
    cols = torch.empty(n * p * p, kpad, device=DEV)
    ops.im2col(d, x, kpad, cols)
    pl = ops.Planes(cols.numel(), torch.device(DEV))
    ops.im2col_planes(d, x, kpad, pl)
    hh, ll = _split_ref(cols.view(-1))
    assert torch.equal(pl.hi, hh) and torch.equal(pl.lo, ll)
