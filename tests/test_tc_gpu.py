"""wgmma path: (1) the hardware probe pins the shared-memory / instruction descriptor conventions of
pf_tc_common.cuh; (2) pf_conv2d_tc_fwd / pf_conv2d_tc_dgrad against a float64 reference and against the
exact-fp32 CUDA-core kernels.  Tolerance: 2e-5 of the output scale (split-bf16: operands carry 16
mantissa bits, the dropped lo*lo term is 2^-18 relative) — two orders tighter than TF32 would be."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pocketflow_b200 import lib as _lib
from pocketflow_b200 import ops

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def probe(mode, N, K, la, sa, lb, sb, ka, kb):
    L = _lib.load()
    torch.manual_seed(N + K + mode)
    if mode == 0:
        A, B = torch.randn(128, K, device=DEV).bfloat16(), torch.randn(N, K, device=DEV).bfloat16()
        ref = A.float() @ B.float().t()
    else:
        A, B = torch.randn(K, 128, device=DEV).bfloat16(), torch.randn(K, N, device=DEV).bfloat16()
        ref = A.float().t() @ B.float()
    D = torch.zeros(128, N, device=DEV)
    st = L.pf_tc_probe(A.data_ptr(), B.data_ptr(), D.data_ptr(), N, K, mode, la, sa, lb, sb, ka, kb, None)
    torch.cuda.synchronize()
    assert st == 0
    return (D - ref).abs().max().item() / ref.abs().max().item()


@pytest.mark.parametrize('N,K', [(128, 64), (128, 256), (64, 128), (256, 128), (32, 64)])
def test_probe_k_major_sw128(N, K):
    # K-major, SWIZZLE_128B: SBO = 1024 B (8 rows x 128 B), K=16 step = 32 B, LBO unused
    assert probe(0, N, K, 16, 1024, 16, 1024, 32, 32) < 1e-5


@pytest.mark.parametrize('N,K', [(128, 64), (128, 256), (64, 128), (256, 128)])
def test_probe_mn_major_sw128(N, K):
    # MN-major: LBO = stride between 64-element MN blocks, SBO = stride between 8-k groups, K=16 step = 2*SBO
    mbA, mbB = 2, N // 64
    assert probe(1, N, K, 1024, mbA * 1024, 1024, mbB * 1024, 2 * mbA * 1024, 2 * mbB * 1024) < 1e-5


CASES = [
    # n, h, w, c, k, r, s, stride, pad0, pad1
    (4, 16, 16, 16, 32, 3, 3, 1, 1, 1),
    (2, 17, 15, 16, 48, 3, 3, 2, 1, 1),
    (2, 8, 8, 64, 256, 1, 1, 1, 0, 0),
    (2, 9, 9, 32, 64, 1, 1, 2, 0, 0),
    (3, 14, 14, 64, 64, 3, 3, 1, 1, 1),
    (2, 12, 12, 128, 128, 3, 3, 2, 0, 1),
    (2, 7, 7, 512, 2048, 1, 1, 1, 0, 0),
    (1, 7, 7, 512, 512, 3, 3, 1, 1, 1),
    (5, 10, 10, 32, 64, 5, 5, 1, 0, 0),
    (2, 32, 32, 16, 16, 3, 3, 1, 1, 1),
    # persistent kernel: several tiles per CTA, B-stationary 1x1 layers, 128-wide tiles, ragged channel tiles
    (8, 56, 56, 64, 256, 1, 1, 1, 0, 0),
    (8, 56, 56, 256, 64, 1, 1, 1, 0, 0),
    (2, 14, 14, 64, 192, 3, 3, 1, 1, 1),
    (6, 28, 28, 128, 512, 1, 1, 1, 0, 0),
    # strided dgrad by pixel-parity classes (Cout % 64 == 0): 'SAME' pads 0/1 and 1/1, odd sizes, 1x1 stride 2
    (16, 28, 28, 128, 128, 3, 3, 2, 0, 1),
    (4, 15, 15, 64, 128, 3, 3, 2, 1, 1),
    (2, 14, 14, 256, 512, 1, 1, 2, 0, 0),
    (3, 13, 16, 32, 64, 3, 3, 2, 1, 1),
]


@pytest.mark.parametrize('case', CASES)
def test_conv_tc_fwd_dgrad(case):
    n, h, w, c, k, r, s, st, p0, p1 = case
    g = torch.Generator().manual_seed(sum(case))
    x = torch.randn(n, h, w, c, generator=g)
    wt = torch.randn(r, s, c, k, generator=g) * (2.0 / (r * s * c)) ** 0.5
    bias = torch.randn(k, generator=g)
    p = (h + p0 + p1 - r) // st + 1
    q = (w + p0 + p1 - s) // st + 1
    xd = x.double().permute(0, 3, 1, 2).requires_grad_(True)
    wd = wt.double().permute(3, 2, 0, 1)
    yd = F.conv2d(F.pad(xd, (p0, p1, p0, p1)), wd, stride=st)
    dy = torch.randn(n, p, q, k, generator=g)
    yd.backward(dy.double().permute(0, 3, 1, 2))
    y_ref, dx_ref = yd.permute(0, 2, 3, 1).detach(), xd.grad.permute(0, 2, 3, 1)
    d = ops.conv_desc(n, h, w, c, k, r, s, p, q, st, st, p0, p0)
    assert ops.conv2d_tc_supported(d)
    X, W, DY = x.to(DEV), wt.to(DEV).contiguous(), dy.to(DEV)
    tw = ops.TcWeights(d, torch.device(DEV))
    tw.prepare(W)
    Y = torch.empty(n, p, q, k, device=DEV)
    ops.conv2d_tc_fwd(d, X, tw, None, False, Y)
    err = (Y.cpu().double() - y_ref).abs().max().item() / y_ref.abs().max().item()
    assert err <= 2e-5, 'fwd err %.3e' % err
    ops.conv2d_tc_fwd(d, X, tw, bias.to(DEV), True, Y)
    ref2 = torch.relu(y_ref + bias.double())
    assert (Y.cpu().double() - ref2).abs().max().item() <= 2e-5 * ref2.abs().max().item()
    res = torch.randn(n, p, q, k, generator=g)
    ops.conv2d_tc_fwd(d, X, tw, None, False, Y, res.to(DEV))           # fused residual add
    ref3 = y_ref + res.double()
    assert (Y.cpu().double() - ref3).abs().max().item() <= 2e-5 * ref3.abs().max().item()
    DX = torch.full((n, h, w, c), 3.0, device=DEV)
    ops.conv2d_tc_dgrad(d, DY, tw, False, DX)
    err = (DX.cpu().double() - dx_ref).abs().max().item() / dx_ref.abs().max().item()
    assert err <= 2e-5, 'dgrad err %.3e' % err
    ops.conv2d_tc_dgrad(d, DY, tw, True, DX)
    assert (DX.cpu().double() - 2 * dx_ref).abs().max().item() <= 4e-5 * dx_ref.abs().max().item()
    # pre-split operand planes: identical bits to convert-on-the-fly.  The planes call runs the TMA-fed kernel where
    # the gathered channel count is a multiple of 64 and the cp.async planes kernel otherwise; both add the same products
    # in the same order (tests/test_tc_variants_gpu.py checks the feeds against each other at every tile width)
    xp, dyp = ops.Planes(X.numel(), torch.device(DEV)), ops.Planes(DY.numel(), torch.device(DEV))
    ops.split_bf16(X, xp)
    ops.split_bf16(DY, dyp)
    Y2 = torch.empty_like(Y)
    ops.conv2d_tc_fwd(d, X, tw, bias.to(DEV), True, Y, res.to(DEV))
    ops.conv2d_tc_fwd_planes(d, xp, tw, bias.to(DEV), True, Y2, res.to(DEV))
    assert torch.equal(Y, Y2)
    DX2 = torch.full((n, h, w, c), 3.0, device=DEV)
    ops.conv2d_tc_dgrad(d, DY, tw, False, DX)
    ops.conv2d_tc_dgrad_planes(d, dyp, tw, False, DX2)
    assert torch.equal(DX, DX2)
    ops.conv2d_tc_dgrad_planes(d, dyp, tw, True, DX2)
    assert (DX2.cpu().double() - 2 * dx_ref).abs().max().item() <= 4e-5 * dx_ref.abs().max().item()
    # against the exact-fp32 kernel: same answer to split-bf16 accuracy
    Y32 = torch.empty_like(Y)
    ops.conv2d_fwd(d, X, W, None, False, Y32)
    ops.conv2d_tc_fwd(d, X, tw, None, False, Y)
    assert (Y - Y32).abs().max().item() <= 2e-5 * Y32.abs().max().item()


WG_CASES = [c for c in CASES if c[4] % 64 == 0] + [(8, 28, 28, 64, 128, 3, 3, 1, 1, 1), (16, 8, 8, 256, 64, 1, 1, 1, 0, 0),
                                                   (3, 9, 9, 16, 192, 3, 3, 1, 1, 1)]


@pytest.mark.parametrize('case', WG_CASES)
def test_conv_tc_wgrad(case):
    n, h, w, c, k, r, s, st, p0, p1 = case
    g = torch.Generator().manual_seed(sum(case) + 1)
    x = torch.randn(n, h, w, c, generator=g)
    p = (h + p0 + p1 - r) // st + 1
    q = (w + p0 + p1 - s) // st + 1
    dy = torch.randn(n, p, q, k, generator=g)
    xd = x.double().permute(0, 3, 1, 2)
    wd = torch.zeros(k, c, r, s, dtype=torch.float64, requires_grad=True)
    yd = F.conv2d(F.pad(xd, (p0, p1, p0, p1)), wd, stride=st)
    yd.backward(dy.double().permute(0, 3, 1, 2))
    dw_ref = wd.grad.permute(2, 3, 1, 0)
    d = ops.conv_desc(n, h, w, c, k, r, s, p, q, st, st, p0, p0)
    assert ops.conv2d_tc_wgrad_supported(d)
    ws = torch.empty(max(ops.conv2d_tc_wgrad_workspace_floats(d), 4), device=DEV)
    DW = torch.full((r, s, c, k), 5.0, device=DEV)
    ops.conv2d_tc_wgrad(d, x.to(DEV), dy.to(DEV), ws, DW)
    err = (DW.cpu().double() - dw_ref).abs().max().item() / dw_ref.abs().max().item()
    assert err <= 2e-5, 'wgrad err %.3e' % err


def test_conv_tc_rejects_unsupported_shapes():
    d = ops.conv_desc(2, 8, 8, 3, 16, 3, 3, 6, 6, 1, 1, 0, 0)
    assert not ops.conv2d_tc_supported(d)
    x, y = torch.zeros(2, 8, 8, 3, device=DEV), torch.zeros(2, 6, 6, 16, device=DEV)
    dummy = torch.zeros(1024, dtype=torch.bfloat16, device=DEV)

    class T:
        f_hi = f_lo = dummy
    with pytest.raises(ValueError):
        ops.conv2d_tc_fwd(d, x, T, None, False, y)


def test_split_bf16_planes():
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(4096 * 8, generator=g) * torch.logspace(-20, 20, 4096 * 8)).to(DEV)
    pl = ops.Planes(x.numel(), torch.device(DEV))
    ops.split_bf16(x, pl)
    hi, lo = pl.hi, pl.lo
    h_ref = x.to(torch.bfloat16)
    l_ref = (x - h_ref.float()).to(torch.bfloat16)
    assert torch.equal(hi, h_ref) and torch.equal(lo, l_ref)
    rec = hi.double() + lo.double()
    assert ((rec - x.double()).abs() <= x.double().abs() * 2.0 ** -16).all()


def test_multi_tensor_weight_prep_and_deferred_reduce():
    """One launch preparing several kernels == the per-kernel preparation (bit-equal); deferred multi-tensor split-K
    reduction == the immediate one."""
    dev = torch.device(DEV)
    g = torch.Generator().manual_seed(9)
    shapes = [(3, 3, 64, 64), (1, 1, 256, 64), (1, 1, 48, 160), (3, 3, 16, 32), (1, 1, 512, 2048)]
    items, singles, ws_ = [], [], []
    for (r, s, c, k) in shapes:
        w = (torch.randn(r, s, c, k, generator=g) * 0.1).to(dev).contiguous()
        d = ops.conv_desc(2, 8, 8, c, k, r, s, 8, 8, 1, 1, r // 2, s // 2)
        a, b = ops.TcWeights(d, dev), ops.TcWeights(d, dev)
        b.prepare(w)
        items.append((a, w))
        singles.append(b)
        ws_.append(w)
    ops.TcWeightsBatch(items, dev).prepare()
    for (a, _), b in zip(items, singles):
        assert torch.equal(a.f_hi, b.f_hi) and torch.equal(a.f_lo, b.f_lo)
        assert torch.equal(a.d_hi, b.d_hi) and torch.equal(a.d_lo, b.d_lo)
    # deferred reduction
    red, refs = [], []
    for n, splits in [(4096, 3), (36864, 7), (64 * 160, 1)]:
        part = torch.randn(splits * n, generator=g).to(dev)
        out = torch.empty(n, device=dev)
        red.append((part, out, splits))
        acc = torch.zeros(n, device=dev)
        for z in range(splits):
            acc = acc + part[z * n:(z + 1) * n]
        refs.append(acc)
    ops.TcWgradReduceBatch(red, dev).reduce()
    for (_, out, _), ref in zip(red, refs):
        assert torch.equal(out, ref)


@pytest.mark.parametrize('cfg', [(2, 23, 23, 3, 64, 7, 3, 3), (2, 24, 24, 3, 64, 7, 2, 3), (3, 17, 17, 3, 64, 3, 0, 1),
                                 (1, 32, 32, 4, 128, 5, 2, 2)])
def test_space_to_depth_stem(cfg):
    """Stride-2 first layer as space-to-depth + stride-1 tensor-core conv: forward and weight gradient vs float64."""
    n, h, w, c, k, r, p0, p1 = cfg
    dev = torch.device(DEV)
    g = torch.Generator().manual_seed(sum(cfg))
    x = torch.randn(n, h, w, c, generator=g)
    wt = torch.randn(r, r, c, k, generator=g) * (2.0 / (r * r * c)) ** 0.5
    p = (h + p0 + p1 - r) // 2 + 1
    xd = x.double().permute(0, 3, 1, 2)
    wd = wt.double().permute(3, 2, 0, 1).requires_grad_(True)
    yd = F.conv2d(F.pad(xd, (p0, p1, p0, p1)), wd, stride=2)
    dy = torch.randn(n, p, p, k, generator=g)
    yd.backward(dy.double().permute(0, 3, 1, 2))
    r2, s2, fwd_map, bwd_map = ops.s2d_weight_maps(r, r, c, 16)
    d2 = ops.conv_desc(n, p + r2 - 1, p + s2 - 1, 16, k, r2, s2, p, p, 1, 1, 0, 0)
    X, W, DY = x.to(dev), wt.to(dev).contiguous(), dy.to(dev)
    cols = ops.Planes(n * (p + r2 - 1) * (p + s2 - 1) * 16, dev)
    ops.s2d_planes(X, p0, p0, p + r2 - 1, p + s2 - 1, 16, cols)
    wpad = torch.zeros(r2 * s2 * 16 * k, device=dev)
    ops.gather_rows(W, torch.from_numpy(fwd_map).to(dev), wpad, k)
    tw = ops.TcWeights(d2, dev, need_dgrad=False)
    tw.prepare(wpad)
    Y = torch.empty(n, p, p, k, device=dev)
    ops.conv2d_tc_fwd_planes(d2, cols, tw, None, False, Y)
    y_ref = yd.permute(0, 2, 3, 1).detach()
    assert (Y.cpu().double() - y_ref).abs().max().item() <= 2e-5 * y_ref.abs().max().item()
    gp = ops.Planes(DY.numel(), dev)
    ops.split_bf16(DY, gp)
    ws = torch.empty(max(ops.conv2d_tc_wgrad_planes_workspace_floats(d2), 4), device=dev)
    dwpad = torch.empty(r2 * s2 * 16 * k, device=dev)
    ops.conv2d_tc_wgrad_planes(d2, cols, gp, ws, dwpad)
    DW = torch.empty_like(W)
    ops.gather_rows(dwpad, torch.from_numpy(bwd_map).to(dev), DW, k)
    dw_ref = wd.grad.permute(2, 3, 1, 0)
    assert (DW.cpu().double() - dw_ref).abs().max().item() <= 2e-5 * dw_ref.abs().max().item()


@pytest.mark.parametrize('cfg', [(4, 14, 14, 32, 32), (2, 8, 12, 32, 32), (3, 10, 10, 16, 16), (2, 6, 6, 48, 16)])
def test_small_cout_wgrad_by_pixel_pairing(cfg):
    """Weight gradient of a 1x1 conv with fewer than 64 output channels on the tensor cores (engine: the im2col'ed
    3 -> 32 stem of MobileNet-v1): g = 64 / Cout pixels share one GEMM row, the (g Cin) x (g Cout) result's diagonal
    blocks are folded (pf_fold_diag_blocks).  Against float64: 2e-5 of the largest entry, like every split-bf16 conv."""
    n, p, q, cin, cout = cfg
    g = 64 // cout
    if (cin * g) % 64 or (p * q) % g:
        pytest.skip('pairing does not apply')
    gen = torch.Generator().manual_seed(sum(cfg))
    cols = torch.randn(n * p * q, cin, generator=gen)
    dy = torch.randn(n * p * q, cout, generator=gen)
    ref = cols.double().t() @ dy.double()
    dev = torch.device(DEV)
    cp, dp = ops.Planes(cols.numel(), dev), ops.Planes(dy.numel(), dev)
    ops.split_bf16(cols.to(DEV), cp)
    ops.split_bf16(dy.to(DEV), dp)
    d_pair = ops.conv_desc(n, 1, p * q // g, cin * g, cout * g, 1, 1, 1, p * q // g, 1, 1, 0, 0)
    assert ops.conv2d_tc_wgrad_supported(d_pair)
    ws = torch.empty(max(ops.conv2d_tc_wgrad_planes_workspace_floats(d_pair), 4), device=DEV)
    dw_pair = torch.empty(cin * g * cout * g, device=DEV)
    ops.conv2d_tc_wgrad_planes(d_pair, cp, dp, ws, dw_pair)
    dw = torch.full((cin, cout), 7.0, device=DEV)
    ops.fold_diag_blocks(dw_pair, g, cin, cout, dw)
    err = (dw.cpu().double() - ref).abs().max().item()
    assert err <= 2e-5 * ref.abs().max().item(), (err, ref.abs().max().item())
