"""The helpers of test_exact_reductions_gpu on the CPU: the per-tap DGEMM references against torch's float64 convolution
on small integer cases, the weight-plane writers against the readers of test_tc_bench_layers_gpu, and the operand
generator's bound and every-pixel-contributes construction."""
import types

import pytest
import torch
import torch.nn.functional as F

from pocketflow_b200 import ops
from support import (EXACT_BOUND, conv_dgrad_ref, conv_fwd_ref, conv_wgrad_ref, dgrad_weight, dw_dgrad_ref, dw_fwd_ref,
                     dw_wgrad_ref, every_pixel_contributes, fwd_weight, int_values, reduction_operands, split_terms,
                     wgrad_density, write_dgrad_weight, write_fwd_weight)


def same_pads(size, r, st):
    """TF 'SAME': (output size, pad before, pad after)"""
    p = -(-size // st)
    tot = max((p - 1) * st + r - size, 0)
    return p, tot // 2, tot - tot // 2


# (n, h, w, c, k, r, s, stride, padding)
CASES = [
    (2, 9, 9, 3, 4, 3, 3, 2, 'SAME'),        # stride 2, SAME on an odd size: pads 1 / 1
    (2, 8, 8, 3, 4, 3, 3, 2, 'SAME'),        # even size: pads 0 / 1, the bottom row no window reaches
    (2, 7, 6, 2, 3, 3, 3, 1, 'SAME'),
    (2, 10, 9, 2, 3, 5, 5, 1, 'VALID'),
    (1, 16, 16, 3, 4, 7, 7, 2, 'SAME'),      # the 7x7 stem
    (2, 9, 8, 4, 5, 1, 1, 2, 'VALID'),       # 1x1 stride 2: rows and columns no window reaches
    (3, 6, 6, 4, 4, 2, 2, 2, 'SAME'),
]


def desc_of(case):
    n, h, w, c, k, r, s, st, pad = case
    if pad == 'SAME':
        (p, pt, pb), (q, pl, pr) = same_pads(h, r, st), same_pads(w, s, st)
    else:
        p, q, pt, pb, pl, pr = (h - r) // st + 1, (w - s) // st + 1, 0, 0, 0, 0
    return (n, h, w, c, k, r, s, p, q, st, st, pt, pl), (pl, pr, pt, pb)


def torch_conv(x, w, case, groups=1):
    d, pads = desc_of(case)
    st = case[7]
    return F.conv2d(F.pad(x.permute(0, 3, 1, 2), pads), w, stride=st, groups=groups).permute(0, 2, 3, 1)


def ints(shape, g):
    return torch.randint(-3, 4, shape, generator=g).double()


@pytest.mark.parametrize('case', CASES, ids=lambda c: 'x'.join(map(str, c[:9])))
def test_per_tap_references_equal_conv2d(case):
    n, h, w, c, k, r, s, st, pad = case
    d, _ = desc_of(case)
    p, q = d[7], d[8]
    g = torch.Generator().manual_seed(sum(case[:8]))
    x, wt, dy = ints((n, h, w, c), g), ints((r, s, c, k), g), ints((n, p, q, k), g)
    y = torch_conv(x, wt.permute(3, 2, 0, 1), case)
    assert y.shape == (n, p, q, k)
    assert torch.equal(conv_fwd_ref(x, wt, d), y)
    xg = x.clone().requires_grad_(True)
    wg = wt.clone().requires_grad_(True)
    torch_conv(xg, wg.permute(3, 2, 0, 1), case).backward(dy)
    assert torch.equal(conv_dgrad_ref(dy, wt, d), xg.grad)
    dw, parts = conv_wgrad_ref(x, dy, d, [0, 5, 5, n * p * q - 1, n * p * q])
    assert torch.equal(dw, wg.grad)
    assert parts.shape[0] == 4 and torch.equal(parts[1], torch.zeros_like(parts[1]))
    assert torch.equal(parts.sum(0), dw)
    # a pixel range is the wgrad of those pixels alone
    keep = torch.zeros(n * p * q, dtype=torch.float64)
    keep[5:n * p * q - 1] = 1.0
    assert torch.equal(parts[2], conv_wgrad_ref(x, dy * keep.view(n, p, q, 1), d)[0])


@pytest.mark.parametrize('case', [c for c in CASES if c[5] > 1], ids=lambda c: 'x'.join(map(str, c[:9])))
def test_depthwise_references_equal_conv2d(case):
    n, h, w, c, k, r, s, st, pad = case
    d, _ = desc_of(case)
    p, q = d[7], d[8]
    g = torch.Generator().manual_seed(sum(case[:8]) + 1)
    x, wt, dy = ints((n, h, w, c), g), ints((r, s, c), g), ints((n, p, q, c), g)
    xg, wg = x.clone().requires_grad_(True), wt.clone().requires_grad_(True)
    y = torch_conv(xg, wg.permute(2, 0, 1).unsqueeze(1), case, groups=c)
    assert torch.equal(dw_fwd_ref(x, wt, d), y.detach())
    y.backward(dy)
    assert torch.equal(dw_dgrad_ref(dy, wt, d), xg.grad)
    assert torch.equal(dw_wgrad_ref(x, dy, d), wg.grad)


def test_split_terms_drop_lo_lo():
    f = lambda a, b: a * b                                     # noqa: E731
    a, b = [torch.tensor(3.0), torch.tensor(2.0)], [torch.tensor(5.0), torch.tensor(7.0)]
    assert split_terms(f, a, b).item() == 3 * 5 + 3 * 7 + 2 * 5
    assert split_terms(f, a[:1], b).item() == 3 * (5 + 7)
    assert split_terms(f, a, b[:1]).item() == 3 * 5 + 2 * 5


@pytest.mark.parametrize('r,s,c,k', [(3, 3, 16, 64), (1, 1, 64, 16), (7, 7, 16, 16), (3, 3, 48, 80)])
def test_plane_writers_round_trip_through_the_readers(r, s, c, k):
    d = ops.conv_desc(2, 8, 8, c, k, r, s, 8, 8, 1, 1, r // 2, s // 2)
    g = torch.Generator().manual_seed(r * c + k)
    hi, lo = ints((r, s, c, k), g), ints((r, s, c, k), g)
    kpad_f, kpad_d = -(-r * s * c // 64) * 64, -(-r * s * k // 64) * 64
    tw = types.SimpleNamespace(f_hi=torch.zeros(k * kpad_f, dtype=torch.bfloat16),
                               f_lo=torch.zeros(k * kpad_f, dtype=torch.bfloat16),
                               d_hi=torch.zeros(c * kpad_d, dtype=torch.bfloat16),
                               d_lo=torch.zeros(c * kpad_d, dtype=torch.bfloat16))
    write_fwd_weight(tw.f_hi, tw.f_lo, hi, lo)
    write_dgrad_weight(tw.d_hi, tw.d_lo, hi, lo)
    assert torch.equal(fwd_weight(tw.f_hi, tw.f_lo, d), hi + lo)
    assert torch.equal(fwd_weight(tw.f_hi, None, d), hi)
    assert torch.equal(dgrad_weight(tw, d), hi + lo)
    # the Kpad columns stay zero
    assert not tw.f_hi.view(k, kpad_f)[:, r * s * c:].float().any()
    assert not tw.d_lo.view(c, kpad_d)[:, r * s * k:].float().any()


@pytest.mark.parametrize('npix,planes', [(3_211_264, 2), (401_408, 2), (6272, 1), (50, 2)])
def test_density_keeps_the_bound(npix, planes):
    nterms = 3 if planes == 2 else 1
    p = wgrad_density(npix, nterms)
    assert 0 < p <= 0.5
    # the expected sum of |terms| of an entry, and the carrier entries (x dense, dy at density p, plus the forced
    # entries) stay well below the exact bound
    assert npix * nterms * p * p <= float(1 << 22) * 1.0001
    assert npix * (nterms * p + 1) < EXACT_BOUND


@pytest.mark.parametrize('xshape,yshape,planes,signed', [((2, 9, 9, 16), (2, 5, 5, 64), 2, True),
                                                         ((3, 7, 7, 32), (3, 7, 7, 16), 1, True),
                                                         ((2, 8, 8, 16), (2, 4, 4, 64), 1, False)])
def test_operands_keep_the_bound_and_every_pixel_contributes(xshape, yshape, planes, signed):
    g = torch.Generator().manual_seed(5)
    n, p, q, k = yshape
    xs, ys = reduction_operands(xshape, yshape, planes, 2, 0.3, g, x_signed=signed)
    assert len(xs) == planes and len(ys) == 2
    assert every_pixel_contributes(xs, ys)
    for v in xs + ys:
        assert set(v.unique().tolist()) <= ({-1.0, 0.0, 1.0} if signed or v is not xs[0] else {0.0, 1.0})
    # with a 1x1 window every pixel's terms land in entry (0, pixel % k): drop any one pixel and that entry changes
    d = (n, p, q, xshape[3], k, 1, 1, p, q, 1, 1, 0, 0)
    xv = [v[:, :p, :q].double() for v in xs]
    yv = [v.double() for v in ys]
    f = lambda a, b: conv_wgrad_ref(a, b, d)[0]                # noqa: E731
    full = split_terms(f, xv, yv)
    mag = split_terms(f, [v.abs() for v in xv], [v.abs() for v in yv])
    assert mag.max().item() < EXACT_BOUND
    for pix in (0, n * p * q // 2, n * p * q - 1):
        keep = torch.ones(n * p * q, dtype=torch.float64)
        keep[pix] = 0.0
        dropped = split_terms(f, xv, [v * keep.view(n, p, q, 1) for v in yv])
        assert not torch.equal(dropped, full), pix
    # a broken construction is seen
    xs[0][0, 0, 0, 0] = 0.0
    assert not every_pixel_contributes(xs, ys)
    bad = int_values((4, 4), 1.0, g)
    assert set(bad.abs().unique().tolist()) == {1.0}
