"""The ping-pong schedule of the TMA-fed fwd / unit-stride dgrad convolution (conv_tma_kernel).

Two consumer warpgroups take a CTA's tiles alternately and hand a mainloop turn and an epilogue turn to each other, so
the cases here are chosen by how many tiles each CTA gets: a grid of one tile (the second warpgroup has no work),
SMs + 1 tiles (one CTA gets two, the others one) and 3 x SMs + 5 (CTAs get three or four: odd and even counts), each
with one k-stage per tile and with k-loops longer than the stage ring (the handoff has to keep the ring's parity).
Every output starts as NaN (accumulate targets as a known tensor), and
  * split x split must give the same bits as the cp.async kernel at the same BN (same products, same order);
  * levels and single-plane operands must match a float64 convolution to DESIGN.md §6's bars, and the residual ring
    must give the same bits as the register-prefetched residual (PF_TC_RING=0)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pocketflow_b200 import ops
from support import rel_err, sms

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
HW = 8                            # 8 x 8 images: 64 GEMM rows per image


def tile_count(which):
    return {'one': 1, 'sms+1': sms() + 1, '3sms+5': 3 * sms() + 5}[which]


@pytest.fixture(autouse=True)
def _knobs(monkeypatch):
    for name in ('PF_TC_BN', 'PF_TC_RING'):
        monkeypatch.delenv(name, raising=False)
    yield
    ops.conv2d_tc_set_feed(-1)


def batch_for(m_tiles):
    """images of HW x HW such that the GEMM rows fill m_tiles tiles of 128, the last one half full"""
    return 2 * m_tiles - 1


def desc(n, c, k, r):
    return ops.conv_desc(n, HW, HW, c, k, r, r, HW, HW, 1, 1, r // 2, r // 2)


def conv_ref(x, w, r):
    """float64 NHWC x HWIO -> NHWC, stride 1, 'same' padding"""
    return F.conv2d(x.permute(0, 3, 1, 2), w.permute(3, 2, 0, 1), padding=r // 2).permute(0, 2, 3, 1)


def dgrad_ref(dy, w, r, shape):
    x = torch.zeros(shape, dtype=torch.float64, device=DEV, requires_grad=True)
    conv_ref(x, w, r).backward(dy)
    return x.grad


def split_planes(t):
    pl = ops.Planes(t.numel(), DEV)
    ops.split_bf16(t, pl)
    return pl, (pl.hi.double() + pl.lo.double()).view(t.shape)


def split_weights(c, k, r, g):
    wt = (torch.randn(r, r, c, k, generator=g) * (2.0 / (r * r * c)) ** 0.5).to(DEV).contiguous()
    tw = ops.TcWeights(desc(1, c, k, r), DEV)
    tw.prepare(wt)
    kp = tw.f_hi.numel() // k
    val = (tw.f_hi.double() + tw.f_lo.double()).view(k, kp)[:, :r * r * c].reshape(k, r, r, c).permute(1, 2, 3, 0)
    return tw, val.contiguous()


def check_plan(feed, pass_, tiles, bn=None, ring=None):
    plan = ops.conv2d_tc_last_plan()
    assert plan['feed'] == feed and plan['pass'] == pass_ and plan['tiles'] == tiles, plan
    assert plan['grid'] == min(tiles, sms()), plan
    if bn is not None:
        assert plan['bn'] == bn, plan
    if ring is not None:
        assert plan['ring'] == ring, plan
    return plan


# ------------------------------------------------------------------------------------------ fwd, split x split
# (id, tiles, c, k, r, knobs, epilogue, expected bn, expected ring); n-tiles = k / bn
FWD_SPLIT = [
    ('one-nk1', 'one', 64, 128, 1, {}, 'none', 128, 0),
    ('one-long-k', 'one', 128, 64, 5, {}, 'all', 64, 0),
    ('sms+1-nk1-residual', 'sms+1', 64, 128, 1, {}, 'residual', 128, 0),
    ('sms+1-long-k', 'sms+1', 128, 128, 5, {}, 'bias_relu', 128, 0),
    ('3sms+5-3x3', '3sms+5', 64, 128, 3, {}, 'all', 128, 0),
    ('3sms+5-nk1-ring2', '3sms+5', 64, 64, 1, {}, 'residual', 64, 2),
]


@pytest.mark.parametrize('spec', FWD_SPLIT, ids=[c[0] for c in FWD_SPLIT])
def test_fwd_split_matches_cp_async(spec, monkeypatch):
    cid, which, c, k, r, knobs, epi, bn, ring = spec
    for name, v in knobs.items():
        monkeypatch.setenv(name, str(v))
    tiles = tile_count(which)
    n_tiles = -(-k // bn)
    assert tiles % n_tiles == 0
    n = batch_for(tiles // n_tiles)
    g = torch.Generator().manual_seed(tiles + c + k + r)
    d = desc(n, c, k, r)
    xp, xv = split_planes((torch.randn(n, HW, HW, c, generator=g) * 1.3 + 0.2).to(DEV))
    tw, wv = split_weights(c, k, r, g)
    bias = torch.randn(k, generator=g).to(DEV) if epi in ('bias_relu', 'all') else None
    relu = epi in ('bias_relu', 'all')
    res = torch.randn(n, HW, HW, k, generator=g).to(DEV) if epi in ('residual', 'all') else None
    ref = conv_ref(xv, wv, r)
    if bias is not None:
        ref = ref + bias.double()
    if relu:
        ref = torch.relu(ref)
    if res is not None:
        ref = ref + res.double()
    outs = []
    for feed in (1, 0):
        ops.conv2d_tc_set_feed(feed)
        y = torch.full((n, HW, HW, k), float('nan'), device=DEV)
        ops.conv2d_tc_fwd_planes(d, xp, tw, bias, relu, y, res)
        torch.cuda.synchronize()
        check_plan(feed, 0, tiles, bn, ring if feed else None)
        outs.append(y)
    assert rel_err(outs[0], ref) <= 2e-5, cid
    assert torch.equal(outs[0], outs[1]), '%s: TMA and cp.async differ by %.3e' % (
        cid, (outs[0] - outs[1]).nan_to_num(1e30).abs().max().item())


# ------------------------------------------------------------------------------------------ fwd, levels
def hdr(scale, nplanes):
    return torch.from_numpy(np.array([(scale, nplanes)], dtype=ops.ACT_HDR).view(np.uint8)).to(DEV)


def act_levels(shape, g, scale):
    """one bf16 plane of integer activation levels (zeros included) and its per-pixel channel sums"""
    n, h, w, c = shape
    nseg = (c + 127) // 128
    j = torch.randint(0, 256, shape, generator=g).float() * (torch.rand(shape, generator=g) > 0.3)
    pl = ops.Planes(j.numel(), DEV)
    pl.hi.copy_(j.reshape(-1).to(torch.bfloat16))
    pl.lo.fill_(float('nan'))
    csum = j.to(DEV).double().reshape(-1, nseg, c // nseg).sum(2).float().contiguous()
    return pl, csum, nseg, j.double().to(DEV) * scale


def weight_levels(c, k, r, g, bits=8):
    kq, centre = (1 << bits) - 1, float(1 << (bits - 1))
    lv = torch.randint(0, kq + 1, (r, r, c, k), generator=g).float()
    alpha = torch.rand(k, generator=g) * 0.5 + 0.05
    beta = -alpha * (0.3 + 0.4 * torch.rand(k, generator=g))
    rk = float(np.float32(1.0) / np.float32(kq))
    val = ((alpha.double() * rk) * lv.double() + beta.double()).to(DEV)
    p0 = (lv - centre).permute(3, 0, 1, 2).reshape(k, r * r * c).to(torch.bfloat16).contiguous().to(DEV)
    pad = (-k) % 4
    return p0, torch.cat([alpha, torch.zeros(pad)]).to(DEV), torch.cat([beta, torch.zeros(pad)]).to(DEV), val


# (id, tiles: m-tiles x n-tiles, c, k, r, epilogue, expected bn, expected ring); k / bn > 1 with n-tiles that do not
# divide the grid: a CTA's tiles change columns, so the per-column table of the levels' epilogue is rebuilt
FWD_LVL = [
    ('one', (1, 1), 128, 64, 3, 'all', 64, 2),
    ('odd-tiles-per-cta-5-ntiles', (53, 5), 128, 640, 1, 'all', 128, 0),
    ('long-k-ring2', (67, 2), 128, 128, 5, 'residual', 64, 2),
]


@pytest.mark.parametrize('spec', FWD_LVL, ids=[c[0] for c in FWD_LVL])
def test_fwd_levels_against_float64(spec, monkeypatch):
    cid, (m_tiles, n_tiles), c, k, r, epi, bn, ring = spec
    monkeypatch.setenv('PF_TC_BN', str(bn))
    ops.conv2d_tc_set_feed(1)
    n = batch_for(m_tiles)
    g = torch.Generator().manual_seed(m_tiles + c + k)
    d = desc(n, c, k, r)
    s_a = 0.0173
    pl, csum, nseg, xv = act_levels((n, HW, HW, c), g, s_a)
    p0, alpha, beta, wv = weight_levels(c, k, r, g)
    bias = torch.randn(k, generator=g).to(DEV) if epi == 'all' else None
    res = torch.randn(n, HW, HW, k, generator=g).to(DEV)
    ref = conv_ref(xv, wv, r)
    if bias is not None:
        ref = torch.relu(ref + bias.double())
    ref = ref + res.double()
    act = ops.tc_act(pl, hdr(s_a, 1), csum, nseg)
    wt = ops.tc_wt(p0, None, alpha, beta, True, 8)
    y = torch.full((n, HW, HW, k), float('nan'), device=DEV)
    ops.conv2d_tc_fwd_ex(d, act, wt, bias, bias is not None, y, res)
    torch.cuda.synchronize()
    check_plan(1, 0, m_tiles * n_tiles, bn, ring)
    err = rel_err(y, ref)
    assert err <= 1e-5, '%s: err %.3e' % (cid, err)


# ------------------------------------------------------------------------------------------ fwd, residual ring depth 4
@pytest.mark.parametrize('which', ['one', '3sms+5'])
def test_fwd_ring4_matches_register_residual(which, monkeypatch):
    """single-plane levels x a single bf16 weight plane leaves room for a depth-4 ring; the ring and the
    register-prefetched residual must give the same bits"""
    tiles = tile_count(which)
    n, c, k, r = batch_for(tiles), 64, 64, 1
    g = torch.Generator().manual_seed(tiles)
    d = desc(n, c, k, r)
    pl, _, _, xv = act_levels((n, HW, HW, c), g, 1.0)
    tw, _ = split_weights(c, k, r, g)
    wv = tw.f_hi.double().view(k, -1)[:, :c].reshape(k, 1, 1, c).permute(1, 2, 3, 0)
    bias = torch.randn(k, generator=g).to(DEV)
    res = torch.randn(n, HW, HW, k, generator=g).to(DEV)
    ref = torch.relu(conv_ref(xv, wv, r) + bias.double()) + res.double()
    ops.conv2d_tc_set_feed(1)
    outs = []
    for ring_knob, ring in ((1, 4), (0, 0)):
        monkeypatch.setenv('PF_TC_RING', str(ring_knob))
        y = torch.full((n, HW, HW, k), float('nan'), device=DEV)
        ops.conv2d_tc_fwd_ex(d, ops.tc_act(pl, single=True), ops.tc_wt(tw.f_hi), bias, True, y, res)
        torch.cuda.synchronize()
        check_plan(1, 0, tiles, 64, ring)
        outs.append(y)
    assert rel_err(outs[0], ref) <= 1e-5
    assert torch.equal(outs[0], outs[1])


# ------------------------------------------------------------------------------------------ dgrad
# (id, tiles, c, k, r, accumulate, knobs, expected bn, expected ring); dgrad rows are the input pixels, columns c
DGRAD = [
    ('one-nk1', 'one', 128, 64, 1, False, {}, 128, 0),
    ('one-acc-ring2', 'one', 64, 64, 1, True, {}, 64, 2),
    ('sms+1-acc', 'sms+1', 128, 128, 1, True, {}, 128, 0),
    ('sms+1-long-k', 'sms+1', 64, 128, 5, False, {}, 64, 0),
    ('3sms+5-3x3-acc', '3sms+5', 64, 64, 3, True, {}, 64, 0),
    ('3sms+5-acc-ring2', '3sms+5', 64, 64, 1, True, {}, 64, 2),
]


@pytest.mark.parametrize('spec', DGRAD, ids=[c[0] for c in DGRAD])
def test_dgrad_matches_cp_async(spec, monkeypatch):
    cid, which, c, k, r, accumulate, knobs, bn, ring = spec
    for name, v in knobs.items():
        monkeypatch.setenv(name, str(v))
    tiles = tile_count(which)
    n_tiles = -(-c // bn)
    assert tiles % n_tiles == 0
    n = batch_for(tiles // n_tiles)
    g = torch.Generator().manual_seed(tiles + c + k + r + 1)
    d = desc(n, c, k, r)
    tw, wv = split_weights(c, k, r, g)
    dyp, dyv = split_planes(torch.randn(n, HW, HW, k, generator=g).to(DEV))
    prior = torch.randn(n, HW, HW, c, generator=g).to(DEV)
    ref = dgrad_ref(dyv, wv, r, (n, HW, HW, c)) + (prior.double() if accumulate else 0.0)
    outs = []
    for feed in (1, 0):
        ops.conv2d_tc_set_feed(feed)
        dx = prior.clone() if accumulate else torch.full((n, HW, HW, c), float('nan'), device=DEV)
        ops.conv2d_tc_dgrad_planes(d, dyp, tw, accumulate, dx)
        torch.cuda.synchronize()
        check_plan(feed, 1, tiles, bn, ring if feed else None)
        outs.append(dx)
    assert rel_err(outs[0], ref) <= 2e-5, cid
    assert torch.equal(outs[0], outs[1]), '%s: TMA and cp.async differ by %.3e' % (
        cid, (outs[0] - outs[1]).nan_to_num(1e30).abs().max().item())
