"""The integer inference model's kernels at the edges the batch-128 kernel tests do not reach, on every layer shape the
four integer models run (support.INT8_LAYERS): pf_conv2d_u8_fwd (TMA- and cp.async-fed), pf_dwconv_u8_fwd and the
level producer pf_bn_eval_levels_u8.

- Batches 1 and 3 on every shape, and 129 on large 7 x 7 and 14 x 14 ones: the last m-tile is partial (at 7 x 7 and
  batch 1 there are 49 rows, fewer than one tile).  The output is a view into a NaN-filled buffer followed by a
  sentinel: every output element must be written and the sentinel left alone, with the plain affine epilogue and with
  bias, ReLU, residual and the folded batch norm.
- Exact S and J on the MobileNet-v2 shapes the TMA-fed kernel runs (Cin 192, 384 and 960: a partial last 128-channel
  segment, an odd segment count, a partial last n-tile), ResNet-20's 8 x 8 64 -> 64 and the MobileNet-v2 depthwise
  shapes (C / 16 not a power of two).
- The affine epilogue below 8 bits: 1 / (2^b - 1) for b in {2, 4, 5, 7} and header scales alpha_a / k_a.
- The producer below 8 bits, at tails of m, with ReLU and ReLU6 and with the range given or found, and on a batch
  whose BN + ReLU output is all zeros."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from support import INT8_LAYERS, bn_chain, conv64, dw_fwd_ref, enc, free, rsqrt_rn  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _release():
    yield
    free()


def _distinct(kind):
    out = []
    for layers in INT8_LAYERS.values():
        for s in layers:
            if s[0] == kind and s[1:13] not in out:
                out.append(s[1:13])
    return out


# (H, W, Cin, Cout, R, S, stride, pad top, pad left, P, Q, kernel)
CONV = _distinct('conv')
DW = _distinct('dw')
MBV2 = INT8_LAYERS['mobilenet_v2_depthwise_narrow']
# exact sums: the MobileNet-v2 shapes of the TMA-fed kernel and ResNet-20's 8 x 8 64 -> 64, which it also runs
EXACT_CONV = [s[1:13] for s in MBV2 if s[0] == 'conv' and s[-2] == 'tma'] + \
    [s[1:13] for s in INT8_LAYERS['resnet20_narrow'] if s[-2] == 'tma']
EXACT_DW = [s[1:13] for s in MBV2 if s[0] == 'dw']
# a short last m-tile on large 7 x 7 and 14 x 14 shapes, both kernels: 129 * 49 = 49 tiles of 128 + 49 rows,
# 129 * 196 = 197 tiles + 68 rows
TAIL129 = [s for s in CONV if s[:4] in ((7, 7, 512, 2048), (7, 7, 960, 320), (7, 7, 960, 160), (14, 14, 1024, 256),
                                          (14, 14, 576, 96), (14, 14, 192, 64))]
# below 8 bits: (weight bits b, activation levels k_a = 2^b - 1)
BITS = [(2, 3), (4, 15), (5, 31), (7, 127)]
SENTINEL = 0x7fa5a5a5          # a NaN payload no fp32 arithmetic produces (it returns the canonical NaN)


def _sid(s):
    return '%dx%d_%d-%d_k%dx%d_s%d_%s' % (s[0], s[1], s[2], s[3], s[4], s[5], s[6], s[11])


def _dwid(s):
    return '%dx%d_c%d_s%d' % (s[0], s[1], s[2], s[6])


def _desc(s, n):
    from pocketflow_b200 import ops
    h, w, c, k, r, ss, st, pt, pl, p, q, _ = s
    return ops.conv_desc(n, h, w, c, k, r, ss, p, q, st, st, pt, pl)


def _guarded(shape, tail):
    """(a NaN-filled fp32 view of `shape`, the buffer it starts) with `tail` sentinel words after the view"""
    n = int(np.prod(shape))
    buf = torch.full((n + tail,), float('nan'), device='cuda')
    buf.view(torch.int32)[n:] = SENTINEL
    return buf[:n].view(shape), buf


def _assert_guarded(y, buf, what):
    """every element of the view written (finite), every sentinel word unchanged"""
    n = y.numel()
    bad = ~torch.isfinite(y)
    assert not bool(bad.any()), '%s: %d of %d outputs unwritten or non-finite, first at %s' % (
        what, int(bad.sum()), n, tuple(int(i) for i in bad.nonzero()[0]))
    assert bool((buf.view(torch.int32)[n:] == SENTINEL).all()), '%s: written past the end of the output' % what


def _levels(shape, hi, seed, wshape):
    g = torch.Generator(device='cuda').manual_seed(seed)
    whi = hi[1] if isinstance(hi, tuple) else hi
    ahi = hi[0] if isinstance(hi, tuple) else hi
    if hi == 'max':
        return (torch.full(shape, 255, dtype=torch.uint8, device='cuda'),
                torch.full(wshape, 255, dtype=torch.uint8, device='cuda'))
    qa = torch.randint(0, ahi + 1, shape, generator=g, device='cuda', dtype=torch.int32).to(torch.uint8)
    qw = torch.randint(0, whi + 1, wshape, generator=g, device='cuda', dtype=torch.int32).to(torch.uint8)
    return qa, qw


def _csum(qa, c):
    """the producer's channel sums: one per pixel and 128-channel segment, the last one partial"""
    pix = qa.reshape(-1, c).to(torch.float32)
    return torch.stack([pix[:, 128 * i:128 * (i + 1)].sum(1) for i in range(-(-c // 128))], 1).contiguous()


def _hdr(scale, nplanes=1):
    return torch.tensor([np.float32(scale).view(np.int32), nplanes], dtype=torch.int32, device='cuda')


def _conv(s, d, qa, qw, scale, alpha, beta, bits, bias=None, relu=False, residual=None, bn=None):
    """pf_conv2d_u8_fwd into a guarded output (and guarded folded-BN output with `bn` = (mean, var, gamma, beta));
    checks the kernel the inventory names ran and that every output was written.  Returns (y, post)."""
    from pocketflow_b200 import ops
    assert ops.conv2d_u8_supported(d) == (s[11] == 'tma')
    shape = (d.n, d.p, d.q, d.k)
    tail = 128 * d.k + 64                  # a whole m-tile of rows past the end
    y, ybuf = _guarded(shape, tail)
    bn_out, post = None, None
    if bn is not None:
        post, pbuf = _guarded(shape, tail)
        bn_out = ops.TcBnOut(bn[0], bn[1], 1e-3, bn[2], bn[3], 1, post)
    ops.conv2d_u8_fwd(d, qa, _hdr(scale), _csum(qa, d.c), qw.reshape(-1, d.k).t().contiguous(), alpha, beta, bits, y,
                      bias, relu, residual, bn_out)
    if s[11] == 'cp.async':
        plan = ops.conv2d_tc_last_plan()
        assert plan['feed'] == 0 and plan['pass'] == 0 and plan['aff'] == 2, plan
    _assert_guarded(y, ybuf, 'y')
    if bn is not None:
        _assert_guarded(post, pbuf, 'folded BN output')
    return y.double(), post


def _dw(d, qa, qw, scale, alpha, beta, bits):
    from pocketflow_b200 import ops
    y, buf = _guarded((d.n, d.p, d.q, d.c), 16 * d.c + 64)
    ops.dwconv_u8_fwd(d, qa, _hdr(scale), qw.reshape(-1, d.c).contiguous(), alpha, beta, bits, y)
    _assert_guarded(y, buf, 'y')
    return y.double()


def _sums(d, qa, qw, dw=False):
    """float64 S = sum q_a q_w and J = sum q_a over each window (exact: integers far below 2^53)"""
    x = qa.double()
    if dw:
        return dw_fwd_ref(x, qw.double(), d), dw_fwd_ref(x, torch.ones(d.r, d.s, d.c, dtype=torch.float64,
                                                                        device='cuda'), d)
    return conv64(x, qw.double(), d), conv64(x, torch.ones(d.r, d.s, d.c, 1, dtype=torch.float64, device='cuda'), d)


def _formula(d, qa, qw, scale, alpha, beta, bits, dw=False):
    """(float64 of the kernels' formula e1 S + e2 J with their fp32 constants e1 = (alpha * fp32(1 / (2^bits - 1))) *
    scale and e2 = beta * scale, magnitude bound |e1 S| + |e2 J|)"""
    rk = np.float32(1) / np.float32(2 ** bits - 1)
    al, be = alpha.cpu().numpy(), beta.cpu().numpy()
    e1 = torch.from_numpy(((al * rk).astype(np.float32) * np.float32(scale)).astype(np.float64)).cuda()
    e2 = torch.from_numpy((be * np.float32(scale)).astype(np.float64)).cuda()
    S, J = _sums(d, qa, qw, dw)
    return e1 * S + e2 * J, (e1 * S).abs() + (e2 * J).abs()


def _consts(nb, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    alpha = (torch.rand(nb, generator=g, device='cuda') * 0.2 + 0.01).contiguous()
    beta = (-alpha * torch.rand(nb, generator=g, device='cuda')).contiguous()
    return alpha, beta, g


def _within(y, ref, mag, what):
    """The bar of the existing u8 tests: |y - ref| <= 2^-22 |magnitude|.  S and J are exact integers; the epilogue
    rounds S to fp32, forms J e2 and one fma (three roundings of 2^-24 each of a term no larger than the magnitude),
    plus bias and residual adds: a few fp32 ulps, inside 2^-22 = 4 ulps."""
    err = (y - ref).abs()
    ok = err <= 2.0 ** -22 * mag
    assert bool(ok.all()), '%s: worst %.3g of the bound' % (what, float((err / (2.0 ** -22 * mag).clamp_min(1e-300)).max()))


# ---------------------------------------------------------------------------------------------- partial tiles
def _conv_tail(s, n):
    d = _desc(s, n)
    qa, qw = _levels((d.n, d.h, d.w, d.c), 255, 5 + n, (d.r, d.s, d.c, d.k))
    alpha, beta, g = _consts(d.k, 7)
    scale = np.float32(3.7) / np.float32(255)
    f, bound = _formula(d, qa, qw, scale, alpha, beta, 8)
    y, _ = _conv(s, d, qa, qw, scale, alpha, beta, 8)
    _within(y, f, bound, 'affine')
    # bias, ReLU and the residual (relu(formula + bias) + residual), then the folded inference BN + ReLU of that sum
    bias = torch.randn(d.k, generator=g, device='cuda')
    res = torch.randn(d.n, d.p, d.q, d.k, generator=g, device='cuda')
    mean, var = torch.randn(d.k, generator=g, device='cuda'), torch.rand(d.k, generator=g, device='cuda') + 0.5
    gamma, bbeta = torch.randn(d.k, generator=g, device='cuda'), torch.randn(d.k, generator=g, device='cuda')
    y, post = _conv(s, d, qa, qw, scale, alpha, beta, 8, bias=bias, relu=True, residual=res,
                    bn=(mean, var, gamma, bbeta))
    b64 = bias.double()
    _within(y, torch.clamp_min(f + b64, 0) + res.double(), bound + b64.abs() + res.double().abs(), 'residual')
    # the BN of the kernel's own fp32 sum in float64: only the BN's fp32 roundings (a handful) separate the two, the
    # bar of the existing folded-BN tests
    z = torch.clamp_min(((y - mean.double()) / torch.sqrt(var.double() + 1e-3)) * gamma.double() + bbeta.double(), 0)
    assert float((post.double() - z).abs().max() / z.abs().max().clamp_min(1e-30)) <= 1e-6


@pytest.mark.parametrize('batch', [1, 3])
@pytest.mark.parametrize('shape', CONV, ids=_sid)
def test_u8_conv_small_batches(shape, batch):
    _conv_tail(shape, batch)


@pytest.mark.parametrize('shape', TAIL129, ids=_sid)
def test_u8_conv_short_last_tile(shape):
    _conv_tail(shape, 129)


@pytest.mark.parametrize('batch', [1, 3])
@pytest.mark.parametrize('shape', DW, ids=_dwid)
def test_u8_dw_small_batches(shape, batch):
    d = _desc(shape, batch)
    qa, qw = _levels((d.n, d.h, d.w, d.c), 255, 5 + batch, (d.r, d.s, d.c))
    alpha, beta, _ = _consts(d.c, 7)
    scale = np.float32(3.7) / np.float32(255)
    y = _dw(d, qa, qw, scale, alpha, beta, 8)
    f, bound = _formula(d, qa, qw, scale, alpha, beta, 8, dw=True)
    _within(y, f, bound, 'depthwise')


# ---------------------------------------------------------------------------------------------- exact sums
@pytest.mark.parametrize('hi', [3, 31, 255, 'max'], ids=['2bit', '5bit', '8bit', 'all255'])
@pytest.mark.parametrize('shape', EXACT_CONV, ids=_sid)
def test_u8_conv_exact_sums_any_segments(shape, hi):
    """unit scales (k_w = 1, scale 1): (alpha, beta) = (1, 0) writes fp32(S) — the exact s32 sum rounded once on its
    way out of the accumulator — and (0, 1) writes J, exact (below 2^24).  csum per 128-channel segment, the last one
    partial at Cin 192 and 960."""
    d = _desc(shape, 3)
    one, zero = torch.ones(1, device='cuda'), torch.zeros(1, device='cuda')
    qa, qw = _levels((d.n, d.h, d.w, d.c), hi, 17 + d.c + d.k, (d.r, d.s, d.c, d.k))
    S, J = _sums(d, qa, qw)
    assert float(S.max()) < 2 ** 31 and float(J.max()) < 2 ** 24
    ys, _ = _conv(shape, d, qa, qw, 1.0, one, zero, 1)
    assert torch.equal(ys, S.float().double()), float((ys - S).abs().max())
    yj, _ = _conv(shape, d, qa, qw, 1.0, zero, one, 1)
    assert torch.equal(yj, J.expand_as(yj)), float((yj - J).abs().max())


@pytest.mark.parametrize('hi', [3, 31, 255, 'max'], ids=['2bit', '5bit', '8bit', 'all255'])
@pytest.mark.parametrize('shape', EXACT_DW, ids=_dwid)
def test_u8_dw_exact_sums_any_c(shape, hi):
    """the row-blocked depthwise kernel at C / 16 in {2, 6, 9, 12, 24, 36, 60}: S and J exact (below 2^24)"""
    d = _desc(shape, 3)
    one, zero = torch.ones(1, device='cuda'), torch.zeros(1, device='cuda')
    qa, qw = _levels((d.n, d.h, d.w, d.c), hi, 17 + d.c, (d.r, d.s, d.c))
    S, J = _sums(d, qa, qw, dw=True)
    assert float(S.max()) < 2 ** 24
    assert torch.equal(_dw(d, qa, qw, 1.0, one, zero, 1), S)
    assert torch.equal(_dw(d, qa, qw, 1.0, zero, one, 1), J)


# ---------------------------------------------------------------------------------------------- below 8 bits
AFFINE_CONV = EXACT_CONV + [s for s in CONV if s[11] == 'cp.async' and s[:4] in ((32, 32, 16, 16), (7, 7, 960, 160))]
AFFINE_DW = [s for s in DW if s[:3] in ((56, 56, 144), (7, 7, 960))]


@pytest.mark.parametrize('per_channel', [False, True], ids=['per_layer', 'per_channel'])
@pytest.mark.parametrize('bits', BITS, ids=lambda b: 'w%d_ka%d' % b)
@pytest.mark.parametrize('shape', AFFINE_CONV, ids=_sid)
def test_u8_conv_affine_below_8_bits(shape, bits, per_channel):
    """levels q_a <= k_a and q_w <= 2^b - 1, header scale alpha_a / k_a: the kernel's 1 / (2^b - 1) and the header
    against float64 of the formula with the same fp32 constants"""
    wb, ka = bits
    d = _desc(shape, 3)
    qa, qw = _levels((d.n, d.h, d.w, d.c), (ka, 2 ** wb - 1), 3 + wb, (d.r, d.s, d.c, d.k))
    alpha, beta, _ = _consts(d.k if per_channel else 1, wb)
    scale = np.float32(2.9) / np.float32(ka)
    y, _ = _conv(shape, d, qa, qw, scale, alpha, beta, wb)
    f, bound = _formula(d, qa, qw, scale, alpha, beta, wb)
    _within(y, f, bound, 'affine')


@pytest.mark.parametrize('per_channel', [False, True], ids=['per_layer', 'per_channel'])
@pytest.mark.parametrize('bits', BITS, ids=lambda b: 'w%d_ka%d' % b)
@pytest.mark.parametrize('shape', AFFINE_DW, ids=_dwid)
def test_u8_dw_affine_below_8_bits(shape, bits, per_channel):
    wb, ka = bits
    d = _desc(shape, 3)
    qa, qw = _levels((d.n, d.h, d.w, d.c), (ka, 2 ** wb - 1), 3 + wb, (d.r, d.s, d.c))
    alpha, beta, _ = _consts(d.c if per_channel else 1, wb)
    scale = np.float32(2.9) / np.float32(ka)
    y = _dw(d, qa, qw, scale, alpha, beta, wb)
    f, bound = _formula(d, qa, qw, scale, alpha, beta, wb, dw=True)
    _within(y, f, bound, 'depthwise affine')


# ---------------------------------------------------------------------------------------------- level producer
def _bn_inputs(m, c, seed, beta_shift=0.0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    x = torch.randn(m, c, generator=g, device='cuda') * 3
    mean, var = torch.randn(c, generator=g, device='cuda') * 0.1, torch.rand(c, generator=g, device='cuda') + 0.5
    gamma = torch.rand(c, generator=g, device='cuda') + 0.5
    beta = torch.randn(c, generator=g, device='cuda') * 0.1 + beta_shift
    return x, mean, var, gamma, beta


def _produce(x, m, c, mean, var, gamma, beta, act, bits, rng, have_range):
    """pf_bn_eval_levels_u8 into buffers that hold no levels: levels 0xff, header {NaN, 0}, channel sums NaN"""
    from pocketflow_b200 import ops
    nseg = -(-c // 128)
    levels = torch.full((m * c,), 0xff, dtype=torch.uint8, device='cuda')
    hdr = torch.tensor([0x7fc00000, 0], dtype=torch.int32, device='cuda')
    csum = torch.full((m * nseg,), float('nan'), device='cuda')
    ops.bn_eval_levels_u8(x, m, c, mean, var, 1e-3, gamma, beta, act, bits, rng, levels, hdr, csum,
                          have_range=have_range)
    return levels.view(m, c), hdr.cpu().numpy(), csum.view(m, nseg)


def _levels_ref(y, mn, mx, bits):
    """float64 restatement of the producer's levels of fp32 y with the range (mn, mx): alpha = fp32(mx - mn) + 1e-10,
    rint(fp32(fp32((y - mn) / alpha) * k)) with k = 2^bits - 1 (each quotient and product rounded to fp32: the double
    result of one fp32 operation rounds to the correctly rounded fp32 one)"""
    k = 2 ** bits - 1
    alpha = np.float32(np.float32(mx) - np.float32(mn)) + np.float32(1e-10)
    xn = ((y - mn).double() / float(alpha)).float()
    return torch.round((xn.double() * k).float().double()), alpha, k


@pytest.mark.parametrize('act', [1, 2], ids=['relu', 'relu6'])
@pytest.mark.parametrize('c', [64, 96, 192, 960, 1024])
@pytest.mark.parametrize('m', [1 * 7 * 7, 3 * 7 * 7, 3 * 14 * 14 + 1])
def test_u8_levels_producer_bits(m, c, act):
    """levels bit for bit against the float64 restatement on act(bn(x)) in fp32 (support.bn_chain, rstd correctly
    rounded), every level <= k, header {alpha / k, 1} and the per-segment channel sums exact, at activation bits 2 .. 8,
    with the range found by the producer or given to it"""
    x, mean, var, gamma, beta = _bn_inputs(m, c, m + c + act)
    rstd = rsqrt_rn(var + torch.tensor(np.float32(1e-3), device='cuda'))
    y = bn_chain(x, mean, rstd, gamma, beta, act)
    mn, mx = float(y.min()), float(y.max())
    assert mn == 0.0 and (act == 1 or mx == 6.0)
    nseg = -(-c // 128)
    for bits in (2, 4, 5, 7, 8):
        lv, alpha, k = _levels_ref(y, mn, mx, bits)
        want_csum = torch.stack([lv[:, 128 * i:128 * (i + 1)].sum(1) for i in range(nseg)], 1)
        for have_range in (False, True):
            rng = torch.from_numpy(enc([mn, mx]).view(np.int32)).cuda() if have_range else \
                torch.zeros(2, dtype=torch.int32, device='cuda')
            levels, hs, csum = _produce(x, m, c, mean, var, gamma, beta, act, bits, rng, have_range)
            what = (bits, have_range)
            assert np.array_equal(rng.cpu().numpy().view(np.uint32), enc([mn, mx])), what
            assert int(levels.max()) <= k, what
            assert torch.equal(levels.double(), lv), (what, int((levels.double() != lv).sum()))
            assert hs[1] == 1 and hs[0:1].view(np.float32)[0] == np.float32(alpha / np.float32(k)), (what, hs)
            assert torch.equal(csum.double(), want_csum), what


@pytest.mark.parametrize('shape', [s for s in CONV if s[:4] in ((7, 7, 960, 320), (7, 7, 960, 160))] +
                         [s for s in DW if s[:3] == (7, 7, 960)], ids=lambda s: _sid(s) if s[4] == 1 else _dwid(s))
def test_u8_all_zero_activations(shape):
    """a batch whose BN + ReLU output is all zeros (range [0, 0], alpha = 1e-10): every level 0, the header finite,
    and a layer fed by it writes exactly its bias (conv, e1 * 0 + e2 * 0 + bias) or 0 (depthwise)"""
    from pocketflow_b200 import ops
    d = _desc(shape, 3)
    m, c = d.n * d.h * d.w, d.c
    x, mean, var, gamma, beta = _bn_inputs(m, c, 1, beta_shift=-1000.0)
    levels, hdr, csum = _produce(x, m, c, mean, var, gamma, beta, 1, 8, torch.zeros(2, dtype=torch.int32,
                                                                                       device='cuda'), False)
    assert int(levels.max()) == 0 and float(csum.abs().max()) == 0.0
    scale = hdr[0:1].view(np.float32)[0]
    assert hdr[1] == 1 and np.isfinite(scale) and scale == np.float32(np.float32(1e-10) / np.float32(255))
    qa = levels.view(d.n, d.h, d.w, d.c)
    alpha, beta_w, g = _consts(d.k, 2)
    hdr_t = torch.from_numpy(hdr).cuda()
    if d.r == 1:
        qw = torch.randint(0, 256, (d.r, d.s, d.c, d.k), generator=g, device='cuda', dtype=torch.int32).to(torch.uint8)
        bias = torch.randn(d.k, generator=g, device='cuda')
        y = torch.empty(d.n, d.p, d.q, d.k, device='cuda')
        ops.conv2d_u8_fwd(d, qa, hdr_t, csum.reshape(-1).contiguous(), qw.reshape(-1, d.k).t().contiguous(), alpha,
                          beta_w, 8, y, bias)
        assert torch.equal(y, bias.expand_as(y))
    else:
        qw = torch.randint(0, 256, (d.r, d.s, d.c), generator=g, device='cuda', dtype=torch.int32).to(torch.uint8)
        y = torch.empty(d.n, d.p, d.q, d.c, device='cuda')
        ops.dwconv_u8_fwd(d, qa, hdr_t, qw.reshape(-1, d.c).contiguous(), alpha, beta_w, 8, y)
        assert bool((y == 0).all())
