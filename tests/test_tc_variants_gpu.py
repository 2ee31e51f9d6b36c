"""Kernel-variant sweep of the tensor-core convolutions against float64.

Which kernel a call runs (TMA or cp.async feed, tile width BN, epilogue with or without the residual ring and its
depth, B-stationary or streamed weights, strided dgrad by pixel-parity classes or not, wgrad tile width and split-K)
is decided on the host from the shape, the operand form and the PF_TC_* knobs.  Every case here forces one variant,
runs it on seeded operands, and checks two things:
  * the launch plan (pf_conv2d_tc_last_plan) is the variant the case names, so a knob the launcher rejects fails here
    instead of running the default twice;
  * the output matches a float64 convolution of the operands the kernel was given (the represented values: hi + lo of
    split planes, scale x level of activation levels, alpha / k * level + beta of weight levels) to DESIGN.md §6's
    bars: 2e-5 of max|ref| when an operand is split-bf16, 1e-5 for levels x levels.
Outputs start as NaN, accumulate targets as a known tensor.  Split x split unit-stride fwd / dgrad must give the same
bits on both feeds at the same BN.  The last test asserts that every variant in REQUIRED was reached.

The knobs are read by getenv on every launch, so monkeypatch.setenv switches them in-process; the feed is switched with
ops.conv2d_tc_set_feed (PF_TC_FEED itself is read once per process)."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pocketflow_b200 import ops
from support import KEY_FIELDS, TC_REQUIRED, plan_key, rel_err, sms

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
S_A = 0.0173                      # value of one activation level

SEEN = {}                         # plan key -> first case id that produced it
RAN = set()
WORST = {}                        # (pass, operand form) -> worst error relative to max|ref|


def note(pass_, form, err):
    WORST[(pass_, form)] = max(WORST.get((pass_, form), 0.0), err)


@pytest.fixture(autouse=True)
def _feed_reset():
    yield
    ops.conv2d_tc_set_feed(-1)


def dims(case):
    n, h, w, c, k, r, s, st, p0, p1 = case
    return (h + p0 + p1 - r) // st + 1, (w + p0 + p1 - s) // st + 1


def auto_batch(case, pass_, bn):
    """n = 0 in a case: the smallest batch that gives >= 3 x SMs output tiles (fwd / dgrad rows are pixels)"""
    n, h, w, c, k, r, s, st, p0, p1 = case
    if n:
        return case
    p, q = dims(case)
    rows, ng = (p * q, k) if pass_ == 0 else (h * w, c)
    n_tiles = -(-ng // bn)
    n = max(1, math.ceil(3 * sms() * 128 / (n_tiles * rows)))
    return (n,) + tuple(case[1:])


def desc(case):
    n, h, w, c, k, r, s, st, p0, p1 = case
    p, q = dims(case)
    return ops.conv_desc(n, h, w, c, k, r, s, p, q, st, st, p0, p0)


def conv_ref(x, w, case):
    """float64 NHWC x HWIO -> NHWC on the GPU"""
    n, h, wd, c, k, r, s, st, p0, p1 = case
    return F.conv2d(F.pad(x.permute(0, 3, 1, 2), (p0, p1, p0, p1)), w.permute(3, 2, 0, 1), stride=st).permute(0, 2, 3, 1)


def dgrad_ref(dy, w, case):
    n, h, wd, c, k, r, s, st, p0, p1 = case
    x = torch.zeros(n, h, wd, c, dtype=torch.float64, device=DEV, requires_grad=True)
    conv_ref(x, w, case).backward(dy)
    return x.grad


def wgrad_ref(x, dy, case):
    n, h, wd, c, k, r, s, st, p0, p1 = case
    w = torch.zeros(r, s, c, k, dtype=torch.float64, device=DEV, requires_grad=True)
    conv_ref(x, w, case).backward(dy)
    return w.grad


# ------------------------------------------------------------------------------------------ operands
class Act:
    """activation operand in one of the forms of pf_tc_act, with the float64 value the kernels must see"""

    def __init__(self, form, shape, g):
        n, h, w, c = shape
        self.form, self.nseg = form, (c + 127) // 128
        self.pl = ops.Planes(n * h * w * c, DEV)
        self.hdr = self.csum = None
        if form in ('split', 'w8a32'):
            x = (torch.randn(shape, generator=g) * 1.3 + 0.2).to(DEV)
            ops.split_bf16(x, self.pl)
            self.fp32 = x
            self.val = (self.pl.hi.double() + self.pl.lo.double()).view(shape)
            if form == 'w8a32':       # W8A32: split planes under a header that says so (scale 1), real channel sums
                self.hdr = hdr(1.0, 2)
                self.csum = self._csum(self.pl.hi.float() + self.pl.lo.float(), shape)
        else:                          # integer levels of a quantized, post-ReLU activation (zeros included)
            j = torch.randint(0, 256, shape, generator=g).float() * (torch.rand(shape, generator=g) > 0.3)
            self.pl.hi.copy_(j.reshape(-1).to(torch.bfloat16))
            self.pl.lo.fill_(float('nan'))
            scale = S_A if form == 'lvl' else 1.0
            self.val = j.double().to(DEV) * scale
            self.csum = self._csum(j.to(DEV), shape)
            if form == 'lvl':
                self.hdr = hdr(S_A, 1)

    def _csum(self, v, shape):
        n, h, w, c = shape
        return v.double().reshape(-1, self.nseg, c // self.nseg).sum(2).float().contiguous()

    def tc(self):
        return ops.tc_act(self.pl, self.hdr, self.csum, self.nseg, single=self.form == 'single')


def hdr(scale, nplanes):
    return torch.from_numpy(np.array([(scale, nplanes)], dtype=ops.ACT_HDR).view(np.uint8)).to(DEV)


class Wt:
    """weight operand: split-bf16 planes (fwd and dgrad copies), a single bf16 plane, or integer levels"""

    def __init__(self, form, case, g, bits=8, per_channel=True, wrange='sym'):
        n, h, w, c, k, r, s, st, p0, p1 = case
        self.form, self.d = form, desc(case)
        rsc = r * s * c
        if form == 'levels':
            kq, centre = (1 << bits) - 1, float(1 << (bits - 1))
            lv = torch.randint(0, kq + 1, (r, s, c, k), generator=g).float()
            nb = k if per_channel else 1
            alpha = torch.rand(nb, generator=g) * 0.5 + 0.05
            if wrange == 'sym':
                beta = -alpha * (0.3 + 0.4 * torch.rand(nb, generator=g))
            elif wrange == 'pos':     # all weights >= 0
                beta = alpha * 0.2 * torch.rand(nb, generator=g)
            else:                     # range far from zero: the rank-1 term o_c * J dominates the sum
                beta = alpha * (20.0 + 10.0 * torch.rand(nb, generator=g))
            rk = float(np.float32(1.0) / np.float32(kq))
            self.val = ((alpha.double() * rk) * lv.double() + beta.double()).to(DEV)
            self.p0 = (lv - centre).permute(3, 0, 1, 2).reshape(k, rsc).to(torch.bfloat16).contiguous().to(DEV)
            pad = (-nb) % 4
            self.alpha = torch.cat([alpha, torch.zeros(pad)]).to(DEV)
            self.beta = torch.cat([beta, torch.zeros(pad)]).to(DEV)
            self.per_channel, self.bits = per_channel, bits
            return
        wt = (torch.randn(r, s, c, k, generator=g) * (2.0 / rsc) ** 0.5).to(DEV).contiguous()
        self.tw = ops.TcWeights(self.d, DEV)
        self.tw.prepare(wt)
        kp = self.tw.f_hi.numel() // k
        hi = self.tw.f_hi.double().view(k, kp)[:, :rsc]
        lo = self.tw.f_lo.double().view(k, kp)[:, :rsc] if form == 'split' else 0.0
        self.val = (hi + lo).reshape(k, r, s, c).permute(1, 2, 3, 0).contiguous()
        if form == 'split':
            kd = self.tw.d_hi.numel() // c
            dv = (self.tw.d_hi.double() + self.tw.d_lo.double()).view(c, kd)[:, :r * s * k].reshape(c, r, s, k)
            assert torch.equal(dv.permute(1, 2, 0, 3), self.val), 'dgrad copy differs from the fwd copy'

    def tc(self):
        if self.form == 'levels':
            return ops.tc_wt(self.p0, None, self.alpha, self.beta, self.per_channel, self.bits)
        return ops.tc_wt(self.tw.f_hi, self.tw.f_lo if self.form == 'split' else None)


def set_knobs(monkeypatch, knobs):
    for name in ('PF_TC_BN', 'PF_TC_RING', 'PF_TC_STATIONARY', 'PF_TC_CLASSES', 'PF_TC_WGRAD_BN', 'PF_TC_WGRAD_WAVES'):
        monkeypatch.delenv(name, raising=False)
    for name, v in knobs.items():
        monkeypatch.setenv(name, str(v))


def check_plan(cid, expect, big=None, ng=None):
    plan = ops.conv2d_tc_last_plan()
    for f, v in expect.items():
        assert plan[f] == v, '%s: plan %s = %s, the case needs %s (plan %s)' % (cid, f, plan[f], v, plan)
    if big:
        assert plan['tiles'] >= 3 * sms() and ng > plan['bn'], (cid, plan)
    SEEN.setdefault(plan_key(plan), cid)
    return plan


def key(feed, pass_, bn, aff=0, ring=0, stat=0, classes=0, fp32=0):
    return dict(feed=feed, **{'pass': pass_}, classes=classes, bn=bn, aff=aff, ring=ring, b_stationary=stat, a_fp32=fp32)


# ------------------------------------------------------------------------------------------ forward
# (id, case, act form, weight form, feed, knobs, epilogue, expected plan); n = 0: batch sized for >= 3 x SMs tiles
FWD = []
for _bn in (16, 32, 64, 128):
    _k = 2 * _bn + 16 if _bn > 16 else 48                        # ragged last n-tile where BN > 16
    # TMA, split x split, streamed weights over several n-tiles; bit-identical to the cp.async kernel at the same BN
    FWD.append(('tma-split-bn%d' % _bn, (2, 11, 13, 64, _k, 3, 3, 1, 1, 1), 'split', 'split', 1, {'PF_TC_BN': _bn},
                ('bias_relu', 'residual')[_bn % 3 == 1], key(1, 0, _bn)))
    # levels x levels with a residual: BN 64 keeps a depth-2 ring beside three stages, BN 128 has no room for one
    FWD.append(('tma-lvl-bn%d' % _bn, (2, 9, 7, 128, _k, 3, 3, 1, 1, 1), 'lvl', 'levels', 1, {'PF_TC_BN': _bn}, 'all',
                key(1, 0, _bn, aff=2, ring=2 if _bn == 64 else 0)))
    FWD.append(('tma-lvlsplit-bn%d' % _bn, (2, 12, 12, 64, _k, 3, 3, 2, 0, 1), 'lvl', 'split', 1, {'PF_TC_BN': _bn},
                'all', key(1, 0, _bn, aff=1)))
    FWD.append(('tma-w8a32-bn%d' % _bn, (3, 10, 10, 64, _k, 1, 1, 1, 0, 0), 'w8a32', 'levels', 1, {'PF_TC_BN': _bn},
                'bias_relu', key(1, 0, _bn, aff=2)))
    # cp.async: weights stationary (one n-tile, short k) and streamed (forced off), convert-on-the-fly and planes
    FWD.append(('cp-stat-bn%d' % _bn, (2, 9, 9, 48, _bn, 1, 1, 1, 0, 0), 'split', 'split', 0, {'PF_TC_BN': _bn}, 'all',
                key(0, 0, _bn, stat=1)))
    FWD.append(('cp-stream-bn%d' % _bn, (2, 9, 9, 48, _bn, 3, 3, 1, 1, 1), 'split', 'split', 0,
                {'PF_TC_BN': _bn, 'PF_TC_STATIONARY': 0}, 'residual', key(0, 0, _bn)))
FWD += [
    # residual ring: depth 2 (two planes, one k-stage), off by knob, depth 2 with levels, depth 4 with single planes
    ('tma-ring2-split', (2, 9, 9, 64, 128, 1, 1, 1, 0, 0), 'split', 'split', 1, {'PF_TC_BN': 64}, 'residual',
     key(1, 0, 64, ring=2)),
    ('tma-ring-off', (2, 9, 9, 64, 128, 1, 1, 1, 0, 0), 'split', 'split', 1, {'PF_TC_BN': 64, 'PF_TC_RING': 0}, 'residual',
     key(1, 0, 64)),
    ('tma-ring2-lvl', (2, 9, 7, 64, 64, 3, 3, 1, 1, 1), 'lvl', 'levels', 1, {}, 'all', key(1, 0, 64, aff=2, ring=2)),
    ('tma-ring4-single-lvl', (2, 9, 9, 64, 64, 1, 1, 1, 0, 0), 'single', 'levels', 1, {}, 'all',
     key(1, 0, 64, aff=2, ring=4)),
    ('tma-ring4-single', (2, 9, 9, 64, 64, 1, 1, 1, 0, 0), 'single', 'bf16', 1, {}, 'residual', key(1, 0, 64, ring=4)),
    ('tma-ring2-single-nk2', (2, 9, 9, 128, 64, 1, 1, 1, 0, 0), 'single', 'bf16', 1, {}, 'residual', key(1, 0, 64, ring=2)),
    # nk == 1; a k-loop of 50 stages that wraps the stage ring many times
    ('tma-nk1', (3, 7, 7, 64, 256, 1, 1, 1, 0, 0), 'split', 'split', 1, {}, 'none', key(1, 0, 128)),
    ('tma-long-k', (2, 9, 9, 128, 64, 5, 5, 1, 2, 2), 'lvl', 'levels', 1, {}, 'all', key(1, 0, 64, aff=2, ring=2)),
    ('cp-long-k', (2, 9, 9, 48, 128, 5, 5, 1, 2, 2), 'split', 'split', 0, {}, 'bias_relu', key(0, 0, 128)),
    # >= 3 x SMs tiles and several n-tiles: every CTA walks several tiles with changing n0
    ('tma-big-split', (0, 28, 28, 64, 256, 1, 1, 1, 0, 0), 'split', 'split', 1, {}, 'residual', key(1, 0, 128)),
    ('tma-big-lvl', (0, 14, 14, 512, 2048, 1, 1, 1, 0, 0), 'lvl', 'levels', 1, {}, 'all', key(1, 0, 128, aff=2)),
    ('tma-big-lvl-bn16', (0, 14, 14, 64, 64, 3, 3, 1, 1, 1), 'lvl', 'levels', 1, {'PF_TC_BN': 16}, 'residual',
     key(1, 0, 16, aff=2)),
    ('tma-big-lvlsplit', (0, 14, 14, 256, 512, 3, 3, 1, 1, 1), 'lvl', 'split', 1, {}, 'bias_relu', key(1, 0, 128, aff=1)),
    ('cp-big', (0, 28, 28, 48, 256, 1, 1, 1, 0, 0), 'split', 'split', 0, {}, 'all', key(0, 0, 128)),
]
FWD_IDS = [c[0] for c in FWD]


def run_fwd(d, act, wt, use_planes_api, bias, relu, res, y):
    y.fill_(float('nan'))
    if use_planes_api:
        ops.conv2d_tc_fwd_planes(d, act.pl, wt.tw, bias, relu, y, res)
    else:
        ops.conv2d_tc_fwd_ex(d, act.tc(), wt.tc(), bias, relu, y, res)
    torch.cuda.synchronize()
    return ops.conv2d_tc_last_plan()


@pytest.mark.parametrize('spec', FWD, ids=FWD_IDS)
def test_fwd_variant(spec, monkeypatch):
    cid, case, aform, wform, feed, knobs, epi, expect = spec
    set_knobs(monkeypatch, knobs)
    ops.conv2d_tc_set_feed(feed)
    case = auto_batch(case, 0, expect['bn'])
    n, h, w, c, k, r, s, st, p0, p1 = case
    p, q = dims(case)
    g = torch.Generator().manual_seed(sum(case) + len(cid))
    d = desc(case)
    act = Act(aform, (n, h, w, c), g)
    wt = Wt(wform, case, g, wrange='pos' if 'w8a32' in cid else 'sym')
    bias = torch.randn(k, generator=g).to(DEV) if epi in ('bias_relu', 'all') else None
    relu = epi in ('bias_relu', 'all')
    res = torch.randn(n, p, q, k, generator=g).to(DEV) if epi in ('residual', 'all') else None
    ref = conv_ref(act.val, wt.val, case)
    if bias is not None:
        ref = ref + bias.double()
    if relu:
        ref = torch.relu(ref)
    if res is not None:
        ref = ref + res.double()
    y = torch.empty(n, p, q, k, device=DEV)
    planes_api = aform == 'split' and wform == 'split'
    run_fwd(d, act, wt, planes_api, bias, relu, res, y)
    check_plan(cid, expect, big=case is not spec[1], ng=k)
    bar = 1e-5 if aform in ('lvl', 'single') and wform in ('levels', 'bf16') else 2e-5
    err = rel_err(y, ref)
    note('fwd', '%s x %s' % (aform, wform), err)
    assert err <= bar, '%s: err %.3e' % (cid, err)
    if planes_api and feed == 0:
        # the same kernel converting fp32 on the fly: the split is the same, so are the bits
        y2 = torch.full_like(y, float('nan'))
        ops.conv2d_tc_fwd(d, act.fp32, wt.tw, bias, relu, y2, res)
        torch.cuda.synchronize()
        check_plan(cid, dict(expect, a_fp32=1))
        assert torch.equal(y, y2), cid
    if planes_api and feed == 1 and c % 64 == 0:
        # split x split: the TMA and cp.async kernels add the same products in the same order
        ops.conv2d_tc_set_feed(0)
        y2 = torch.empty_like(y)
        plan = run_fwd(d, act, wt, True, bias, relu, res, y2)
        assert plan['feed'] == 0 and plan['bn'] == expect['bn'], plan
        SEEN.setdefault(plan_key(plan), cid + '/cp')
        assert torch.equal(y, y2), '%s: TMA and cp.async differ by %.3e' % (cid, (y - y2).abs().max().item())
    RAN.add(cid)


# ------------------------------------------------------------------------------------------ dgrad
DGRAD = []
for _bn in (16, 32, 64, 128):
    _c = 2 * _bn + 16 if _bn > 16 else 48
    DGRAD.append(('tma-bn%d' % _bn, (2, 9, 11, _c, 64, 3, 3, 1, 1, 1), 1, {'PF_TC_BN': _bn}, False, key(1, 1, _bn)))
    DGRAD.append(('cp-stat-bn%d' % _bn, (2, 9, 9, _bn, 48, 1, 1, 1, 0, 0), 0, {'PF_TC_BN': _bn}, True, key(0, 1, _bn, stat=1)))
    DGRAD.append(('cp-stream-bn%d' % _bn, (2, 9, 9, _c, 48, 3, 3, 1, 1, 1), 0, {'PF_TC_BN': _bn}, False, key(0, 1, _bn)))
    DGRAD.append(('classes-bn%d' % _bn, (2, 15, 15, _c, 64, 3, 3, 2, 1, 1), 1, {'PF_TC_BN': _bn}, True,
                  key(0, 1, _bn, classes=1)))
    DGRAD.append(('no-classes-bn%d' % _bn, (2, 14, 14, _c, 64, 3, 3, 2, 0, 1), 1, {'PF_TC_BN': _bn, 'PF_TC_CLASSES': 0},
                  False, key(0, 1, _bn)))
DGRAD += [
    ('tma-ring2-acc', (2, 9, 9, 128, 64, 1, 1, 1, 0, 0), 1, {'PF_TC_BN': 64}, True, key(1, 1, 64, ring=2)),
    ('tma-acc-nk1-bn128', (2, 9, 9, 128, 64, 1, 1, 1, 0, 0), 1, {}, True, key(1, 1, 128)),
    ('classes-1x1-s2', (2, 14, 14, 256, 512, 1, 1, 2, 0, 0), 1, {}, True, key(0, 1, 128, classes=1)),
    ('tma-long-k', (2, 9, 9, 64, 128, 5, 5, 1, 2, 2), 1, {}, False, key(1, 1, 64)),
    ('tma-big', (0, 28, 28, 256, 64, 1, 1, 1, 0, 0), 1, {}, True, key(1, 1, 128)),
    ('cp-big', (0, 28, 28, 256, 48, 3, 3, 1, 1, 1), 1, {}, False, key(0, 1, 128)),
    ('classes-big', (0, 28, 28, 256, 128, 3, 3, 2, 0, 1), 1, {}, True, key(0, 1, 128, classes=1)),
]


@pytest.mark.parametrize('spec', DGRAD, ids=[c[0] for c in DGRAD])
def test_dgrad_variant(spec, monkeypatch):
    cid, case, feed, knobs, accumulate, expect = spec
    set_knobs(monkeypatch, knobs)
    ops.conv2d_tc_set_feed(feed)
    case = auto_batch(case, 1, expect['bn'])
    n, h, w, c, k, r, s, st, p0, p1 = case
    p, q = dims(case)
    g = torch.Generator().manual_seed(sum(case) + len(cid) + 7)
    d = desc(case)
    wt = Wt('split', case, g)
    dy = torch.randn(n, p, q, k, generator=g).to(DEV)
    dyp = ops.Planes(dy.numel(), DEV)
    ops.split_bf16(dy, dyp)
    dyv = (dyp.hi.double() + dyp.lo.double()).view(n, p, q, k)
    prior = torch.randn(n, h, w, c, generator=g).to(DEV)
    ref = dgrad_ref(dyv, wt.val, case) + (prior.double() if accumulate else 0.0)

    def run(fn, operand):
        dx = prior.clone() if accumulate else torch.full((n, h, w, c), float('nan'), device=DEV)
        fn(d, operand, wt.tw, accumulate, dx)
        torch.cuda.synchronize()
        return dx

    dx = run(ops.conv2d_tc_dgrad_planes, dyp)
    check_plan(cid, expect, big=case is not spec[1], ng=c)
    err = rel_err(dx, ref)
    note('dgrad', 'split x split', err)
    assert err <= 2e-5, '%s: err %.3e' % (cid, err)
    if expect['feed'] == 0 and not expect['classes'] and st == 1:
        dx2 = run(ops.conv2d_tc_dgrad, dy)                         # fp32 dy converted by the producers
        check_plan(cid, dict(expect, a_fp32=1))
        assert torch.equal(dx, dx2), cid
    if expect['feed'] == 1:
        ops.conv2d_tc_set_feed(0)
        dx2 = run(ops.conv2d_tc_dgrad_planes, dyp)
        plan = ops.conv2d_tc_last_plan()
        assert plan['feed'] == 0 and plan['bn'] == expect['bn'], plan
        SEEN.setdefault(plan_key(plan), cid + '/cp')
        assert torch.equal(dx, dx2), '%s: TMA and cp.async differ by %.3e' % (cid, (dx - dx2).abs().max().item())
    RAN.add(cid)


# ------------------------------------------------------------------------------------------ wgrad
# (id, case, x form, feed, knobs, deferred, expected plan, split-K: 1 / 'ragged')
WGRAD = []
for _bn in (64, 128):
    for _form, _aff in (('split', 0), ('lvl', 1), ('w8a32', 1)):
        WGRAD.append(('tma-%s-bn%d-s1' % (_form, _bn), (1, 12, 12, 64, 256, 3, 3, 1, 1, 1), _form, 1,
                      {'PF_TC_WGRAD_BN': _bn}, False, key(1, 2, _bn, aff=_aff), 1))
        WGRAD.append(('tma-%s-bn%d-ragged' % (_form, _bn), (3, 23, 23, 128, 192, 3, 3, 1, 1, 1), _form, 1,
                      {'PF_TC_WGRAD_BN': _bn}, False, key(1, 2, _bn, aff=_aff), 'ragged'))
        WGRAD.append(('tma-%s-bn%d-deferred' % (_form, _bn), (6, 23, 23, 128, 192, 3, 3, 2, 0, 1), _form, 1,
                      {'PF_TC_WGRAD_BN': _bn, 'PF_TC_WGRAD_WAVES': 2}, True, key(1, 2, _bn, aff=_aff), 'ragged'))
    WGRAD.append(('cp-bn%d-s1' % _bn, (1, 12, 12, 48, 256, 3, 3, 1, 1, 1), 'split', 0, {'PF_TC_WGRAD_BN': _bn}, False,
                  key(0, 2, _bn), 1))
    WGRAD.append(('cp-bn%d-ragged' % _bn, (3, 23, 23, 48, 192, 3, 3, 1, 1, 1), 'split', 0,
                  {'PF_TC_WGRAD_BN': _bn, 'PF_TC_WGRAD_WAVES': 3}, False, key(0, 2, _bn), 'ragged'))
    WGRAD.append(('cp-bn%d-deferred' % _bn, (6, 23, 23, 64, 192, 3, 3, 2, 0, 1), 'split', 0, {'PF_TC_WGRAD_BN': _bn},
                  True, key(0, 2, _bn), 'ragged'))
WGRAD += [
    # 4 waves: 14 splits of 36 tiles (one wave would give 3)
    ('tma-big-lvl', (15, 28, 28, 256, 256, 3, 3, 1, 1, 1), 'lvl', 1, {'PF_TC_WGRAD_WAVES': 4}, True, key(1, 2, 128, aff=1),
     'ragged'),
]


@pytest.mark.parametrize('spec', WGRAD, ids=[c[0] for c in WGRAD])
def test_wgrad_variant(spec, monkeypatch):
    cid, case, xform, feed, knobs, deferred, expect, split_kind = spec
    set_knobs(monkeypatch, knobs)
    ops.conv2d_tc_set_feed(feed)
    n, h, w, c, k, r, s, st, p0, p1 = case
    p, q = dims(case)
    g = torch.Generator().manual_seed(sum(case) + len(cid) + 11)
    d = desc(case)
    act = Act(xform, (n, h, w, c), g)
    dy = torch.randn(n, p, q, k, generator=g).to(DEV)
    dyp = ops.Planes(dy.numel(), DEV)
    ops.split_bf16(dy, dyp)
    dyv = (dyp.hi.double() + dyp.lo.double()).view(n, p, q, k)
    ref = wgrad_ref(act.val, dyv, case)
    splits = ops.conv2d_tc_wgrad_splits(d)
    nel = r * s * c * k
    ws = torch.full((max(ops.conv2d_tc_wgrad_planes_workspace_floats(d), 4),), float('nan'), device=DEV)
    dw = None if deferred else torch.full((r, s, c, k), float('nan'), device=DEV)
    if xform == 'split':
        ops.conv2d_tc_wgrad_planes(d, act.pl, dyp, ws, dw)
    else:
        ops.conv2d_tc_wgrad_ex(d, act.tc(), ops.tc_act(dyp), ws, dw)
    plan = check_plan(cid, dict(expect, splits=splits))
    npix = n * p * q
    if split_kind == 1:
        assert plan['splits'] == 1, plan
    else:
        assert plan['splits'] > 1 and npix % plan['pps'] != 0, ('the last split must be ragged', plan)
    if 'big' in cid:
        assert plan['tiles'] >= 3 * sms() and k > plan['bn'], plan
    if deferred:
        dw = torch.full((r, s, c, k), float('nan'), device=DEV)
        ops.TcWgradReduceBatch([(ws[:splits * nel], dw.view(-1), splits)], DEV).reduce()
    torch.cuda.synchronize()
    err = rel_err(dw, ref)
    note('wgrad', '%s x split' % xform, err)
    assert err <= 2e-5, '%s: err %.3e' % (cid, err)
    RAN.add(cid)


# ------------------------------------------------------------------------------------------ dgrad_ex
def test_dgrad_ex_refuses_weight_levels_and_matches_planes_form():
    case = (2, 9, 11, 64, 128, 3, 3, 1, 1, 1)
    n, h, w, c, k, r, s, st, p0, p1 = case
    p, q = dims(case)
    d = desc(case)
    g = torch.Generator().manual_seed(3)
    wt = Wt('split', case, g)
    dy = torch.randn(n, p, q, k, generator=g).to(DEV)
    dyp = ops.Planes(dy.numel(), DEV)
    ops.split_bf16(dy, dyp)
    dx = torch.full((n, h, w, c), float('nan'), device=DEV)
    alpha, beta = torch.ones(k, device=DEV), torch.zeros(k, device=DEV)
    with pytest.raises(ValueError, match='weight levels'):
        ops.conv2d_tc_dgrad_ex(d, ops.tc_act(dyp), ops.tc_wt(wt.tw.d_hi, None, alpha, beta, True, 8), False, dx)
    ref = dgrad_ref((dyp.hi.double() + dyp.lo.double()).view(n, p, q, k), wt.val, case)
    for feed in (1, 0):
        ops.conv2d_tc_set_feed(feed)
        dx.fill_(float('nan'))
        ops.conv2d_tc_dgrad_ex(d, ops.tc_act(dyp), ops.tc_wt(wt.tw.d_hi, wt.tw.d_lo), False, dx)
        assert ops.conv2d_tc_last_plan()['feed'] == feed
        dx2 = torch.full_like(dx, float('nan'))
        ops.conv2d_tc_dgrad_planes(d, dyp, wt.tw, False, dx2)
        torch.cuda.synchronize()
        assert torch.equal(dx, dx2)
        assert rel_err(dx, ref) <= 2e-5


# ------------------------------------------------------------------------------------------ coverage
def test_every_variant_was_reached():
    """Runs last: the union of the plans above covers REQUIRED (skipped when only part of the module ran)."""
    cases = {c[0] for c in FWD} | {c[0] for c in DGRAD} | {c[0] for c in WGRAD}
    if not cases <= RAN:
        pytest.skip('only part of the sweep ran')
    print('variant combinations reached (%d): ' % len(SEEN) + ', '.join(
        '%s=%s' % (dict(zip(KEY_FIELDS, k)), v) for k, v in sorted(SEEN.items())))
    print('worst error / max|ref|: ' + ', '.join('%s %s %.2e' % (p, f, e) for (p, f), e in sorted(WORST.items())))
    missing = TC_REQUIRED - set(SEEN)
    assert not missing, 'variants never reached: %s' % sorted(missing)
