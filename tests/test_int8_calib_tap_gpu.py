"""Calibrated integer models layer by layer against float64, with static ranges that clamp: every integer model of
support.INT8_MODELS at batch 3 and 8/8 bits, from a --learner uniform checkpoint, with each activation's range set to
[0, 0.7 * its range on the evaluated batch], so that every quantized activation has values above hi.

Each _U8Bn, _U8Conv and _U8DwConv of the calibrated plan is wrapped so that its operands are cloned just before its
kernels run and its outputs just after:
- every level producer against its captured fp32 input (support.bn_chain with a correctly rounded rstd), clamped to the
  static range and quantized with it: levels, header and channel sums bit for bit, and its range slot unchanged;
  every call of the first forward and of the four forwards of the whole-model comparison is checked;
- every integer layer against float64 of its formula on the captured levels and its own weight levels, within 2^-22 of
  its magnitude, with bias, ReLU, residual and the folded batch norm the plan wired to it.
Then the whole model: the calibrated integer and fake-quant logits against the float64 oracle with the same static ranges
(StaticRangeOracle: the oracle's forward with every quantized activation clamped and quantized with lo / hi instead of
its batch's min / max), under the bar the per-batch models meet (tests/test_int8_tap_gpu.py)."""
import collections
import gc
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from support import (INT8_MODELS, QUIET, bn_chain, conv64, dw_fwd_ref, free, int8_graph, make, planes_value,  # noqa: E402
                     rsqrt_rn)

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
BATCH = 3
IMAGES = 12
SHRINK = np.float32(0.7)


@pytest.fixture(autouse=True)
def _release():
    yield
    from pocketflow_b200.flags import FLAGS
    FLAGS.reset()
    gc.collect()
    free()


def _state(key):
    net, flags, _ = INT8_MODELS[key]
    reload = 'cifar10_dataset' if 'cifar' in net else 'ilsvrc12_dataset'
    lrn = make(net, 'uniform', 16, reload=reload, **dict(QUIET, uql_weight_bits=8, uql_activation_bits=8, **flags))
    for _ in range(2):
        lrn.train_step()
    state = lrn.sess_train.store.state_dict()
    del lrn
    free()
    return state


class _StaticQuant(dict):
    """the `force` table of StaticRangeOracle: a quantized activation's output is replaced by its static-range
    fake-quant, computed in float64 from the value the oracle has just recorded in `local`"""

    def __init__(self, static, local):
        super().__init__()
        self.static, self.local = static, local

    def __contains__(self, name):
        return name in self.static

    def __getitem__(self, name):
        (lo, hi), bits = self.static[name]
        y = torch.clamp(self.local[name], float(lo), float(hi))
        alpha, k = float(hi) - float(lo) + 1e-10, float(2 ** bits - 1)
        return alpha * (torch.round((y - float(lo)) / alpha * k) / k) + float(lo)


def static_range_oracle(ops, logits, images, wq, aq, ranges):
    """StaticRangeOracle over `ops`: the float64 oracle (mbv2_oracle.DropoutStepOracle, inference) with no per-batch
    activation quantizer and every activation of `aq` clamped to ranges[name] and quantized with it"""
    from oracle.mbv2_oracle import DropoutStepOracle

    class StaticRangeOracle(DropoutStepOracle):
        def forward(self, params, x):
            local = {}
            static = {op.output.name: (ranges[op.name], b) for op, b in zip(aq['ops'], aq['bits'])}
            return super().forward(params, x, training=False, force=_StaticQuant(static, local), local_out=local)

    return StaticRangeOracle(ops, logits, images, weight_quant=wq)


class Tap:
    """wraps forward() of every integer lowering of `ex`: the operands cloned just before its kernels run, the outputs
    just after"""

    def __init__(self, ex):
        from pocketflow_b200.engine import _U8Bn, _U8Conv, _U8DwConv
        self.ex, self.calls, self.bn, self.layers = ex, collections.Counter(), [], []
        for table, cls, cap in ((ex.batch_norm, _U8Bn, self._bn), (ex.conv, _U8Conv, self._layer),
                                (ex.depthwise, _U8DwConv, self._layer)):
            for lo in table.values():
                if isinstance(lo, cls):
                    lo.forward = (lambda lo, run, cap: lambda *a: cap(lo, run, *a))(lo, lo.forward, cap)

    def _bn(self, lo, run, training):
        x, slot = self.ex.T(lo.op.inputs[0]).clone(), lo.base.slot.clone()
        run(training)
        self.calls[lo.op.name] += 1
        self.bn.append(dict(lo=lo, x=x, levels=lo.levels.clone(), hdr=lo.hdr.clone(), csum=lo.csum.clone(),
                            slot_before=slot, slot=lo.base.slot.clone()))

    def _layer(self, lo, run):
        ex, op = self.ex, lo.op
        rec = dict(lo=lo, levels=lo.bn.levels.clone(), hdr=lo.bn.hdr.clone(), csum=lo.bn.csum.clone())
        if op.type == 'Conv2D':
            bias, relu, y = lo._epilogue()
            rec.update(bias=None if bias is None else bias.clone(), relu=relu,
                       res=ex.T(lo.res).clone() if lo.res is not None else None)
        run()
        self.calls[op.name] += 1
        rec['y'] = ex.buf[op.output].clone()
        if op.type == 'Conv2D' and lo.bn_out is not None:
            fb = ex.batch_norm[ex.bn_fold[op]]
            rec['folded'] = fb
            rec['post'] = fb.y_out.clone() if fb.y_out is not None else None
            rec['post_planes'] = planes_value(fb.pl, tuple(op.output.shape)) if fb.pl is not None else None
        self.layers.append(rec)


def _check_producer(ex, r):
    """levels, header and channel sums of one static-range _U8Bn call bit for bit; returns the elements clamped"""
    lo = r['lo']
    base = lo.base
    m, c, mm, mv, eps, gamma, beta = base.moving
    bits = ex.act_quant['bits'][base.aq]
    name = lo.op.name
    assert torch.equal(r['slot'], r['slot_before']), name          # read only
    rlo, rhi = ex.act_quant['ranges'][base.aq]
    assert rlo == 0, name
    y = bn_chain(r['x'].view(m, c), mm, rsqrt_rn(mv + torch.tensor(np.float32(eps), device=mv.device)), gamma, beta,
                 base.act)
    clamped = int((y > float(rhi)).sum())
    yc = torch.clamp(y, 0.0, float(rhi))
    k = 2 ** bits - 1
    alpha = np.float32(rhi) + np.float32(1e-10)
    lv = torch.round(((yc.double() / float(alpha)).float().double() * k).float().double())
    levels = r['levels'].view(m, c).double()
    assert float(levels.max()) <= k, name
    assert torch.equal(levels, lv), (name, int((levels != lv).sum()))
    hs = r['hdr'].cpu().numpy()
    assert hs[1] == 1 and hs[0:1].view(np.float32)[0] == np.float32(alpha / np.float32(k)), (name, hs)
    nseg = -(-c // 128)
    want = torch.stack([lv[:, 128 * i:128 * (i + 1)].sum(1) for i in range(nseg)], 1)
    assert torch.equal(r['csum'].view(m, nseg).double(), want), name
    return clamped


def _check_layer(r):
    """one integer layer against float64 of its formula on its captured operands; returns the error in units of the
    bar 2^-22 |magnitude|"""
    lo = r['lo']
    d, op = lo.d, lo.op
    dw = op.type == 'DepthwiseConv2dNative'
    hs = r['hdr'].cpu().numpy()
    assert hs[1] == 1, op.name
    scale = hs[0:1].view(np.float32)[0]
    qa = r['levels'].view(d.n, d.h, d.w, d.c).double()
    rk = np.float32(1) / np.float32(2 ** lo.bits - 1)
    al, be = lo.alpha.cpu().numpy(), lo.beta.cpu().numpy()
    e1 = torch.from_numpy(((al * rk).astype(np.float32) * scale).astype(np.float64)).cuda()
    e2 = torch.from_numpy((be * scale).astype(np.float64)).cuda()
    if dw:
        w = lo.wl.view(d.r, d.s, d.c).double()
        S, J = dw_fwd_ref(qa, w, d), dw_fwd_ref(qa, torch.ones_like(w), d)
    else:
        w = lo.wl.view(d.k, d.r, d.s, d.c).permute(1, 2, 3, 0).double()
        S, J = conv64(qa, w, d), conv64(qa, torch.ones_like(w[..., :1]), d)
    ref, mag = e1 * S + e2 * J, (e1 * S).abs() + (e2 * J).abs()
    if not dw:
        if r['bias'] is not None:
            ref, mag = ref + r['bias'].double(), mag + r['bias'].double().abs()
        if r['relu']:
            ref = torch.clamp_min(ref, 0)
        if r['res'] is not None:
            res = r['res'].double().view(ref.shape)
            ref, mag = ref + res, mag + res.abs()
    y = r['y'].double().view(ref.shape)
    assert bool(torch.isfinite(y).all()), op.name
    ratio = float(((y - ref).abs() / (2.0 ** -22 * mag).clamp_min(1e-300)).max())
    assert ratio <= 1.0, (op.name, ratio)
    if 'folded' in r:
        fb = r['folded']
        _, _, mm, mv, eps, gamma, beta = fb.moving
        z = ((y - mm.double()) / torch.sqrt(mv.double() + float(np.float32(eps)))) * gamma.double() + beta.double()
        z = torch.clamp(z, 0, 6 if fb.act == 2 else None) if fb.act else z
        scale_z = float(z.abs().max()) or 1.0
        if r['post'] is not None:
            assert float((r['post'].double().view(z.shape) - z).abs().max()) <= 1e-6 * scale_z, op.name
        if r['post_planes'] is not None:
            assert float((r['post_planes'].view(z.shape) - z).abs().max()) <= 2.0 ** -16 * scale_z, op.name
    return ratio


@pytest.mark.parametrize('key', sorted(INT8_MODELS))
def test_calibrated_model_teacher_forced(key):
    from pocketflow_b200 import compact, int8
    from pocketflow_b200.engine import _U8Bn
    state = _state(key)
    g, images, logits, cfg = int8_graph(key, BATCH)
    full = compact.map_state(g, compact.reachable_ops(g, logits), state)
    x = torch.randn(images.shape, generator=torch.Generator().manual_seed(7)).to(DEV)
    # static ranges that clamp: 0.7 of each activation's range on this batch
    r = int8.IntModel.from_checkpoint(g, images, logits, state, cfg, DEV).calibrate([x])
    ranges = {n: (lo, np.float32(hi * SHRINK)) for n, (lo, hi) in r.items()}
    im = int8.IntModel.from_checkpoint(g, images, logits, state, cfg, DEV, act_ranges=ranges)
    fq = int8.fake_quant_executor(g, images, logits, full, cfg, DEV, act_ranges=ranges)
    tap = Tap(im.ex)
    li0 = im.forward(x).clone()
    assert bool(torch.isfinite(li0).all())
    ints = sorted(n for n, why in im.sel if why is None)
    producers = sorted(op.name for op, lo in im.ex.batch_norm.items() if isinstance(lo, _U8Bn))
    assert sorted(t['lo'].op.name for t in tap.layers) == ints
    assert sorted(t['lo'].op.name for t in tap.bn) == producers
    assert set(tap.calls.values()) == {1}, tap.calls
    # the whole model against float64 with the same static ranges, over IMAGES images BATCH at a time
    wq, aq = int8._specs(g, cfg)
    orc = static_range_oracle(compact.reachable_ops(g, logits), logits, images, wq, aq, ranges)
    params = {k: torch.from_numpy(v).double().to(DEV) for k, v in full.items()}
    xs = torch.randn((IMAGES,) + tuple(images.shape[1:]), generator=torch.Generator().manual_seed(1)).to(DEV)
    li, lf, ref = [], [], []
    for i in range(0, IMAGES, BATCH):
        xb = xs[i:i + BATCH]
        li.append(im.forward(xb).clone())
        fq.buf[fq.images].copy_(xb)
        lf.append(fq.forward(training=False).clone())
        ref.append(orc.forward(params, xb.double())[logits.name].double())
    li, lf, ref = torch.cat(li), torch.cat(lf), torch.cat(ref)
    # every producer and integer layer call of the five forwards
    clamped = [_check_producer(im.ex, t) for t in tap.bn]
    # the first producer's input on the calibration batch is the one its range was measured on, so it clamps; deeper
    # ones see activations that upstream clamping has already shrunk, and most of them still clamp
    assert clamped[0] > 0 and sum(n > 0 for n in clamped) >= len(clamped) // 2, clamped
    worst = max(_check_layer(t) for t in tap.layers)
    s = float(ref.abs().max())
    e_int, e_fq = float((li.double() - ref).abs().max()) / s, float((lf.double() - ref).abs().max()) / s
    agree = float((li.argmax(1) == lf.argmax(1)).float().mean())
    agree_ref = float((lf.argmax(1) == ref.argmax(1)).float().mean())
    print('%s calibrated (hi x %.1f): %d integer layers, %d producers (%d of them clamping) checked; worst epilogue '
          'error %.3f of its bound; int %.3e fake-quant %.3e (of max|ref|, %d images), top-1 int / fq %.4f, fq / ref %.4f'
          % (key, SHRINK, len(tap.layers), len(tap.bn), sum(n > 0 for n in clamped), worst, e_int, e_fq, IMAGES, agree,
             agree_ref))
    # the bar the per-batch models meet against the per-batch oracle: quantizer level flips set both distances
    assert e_int <= 1.3 * e_fq, (e_int, e_fq)
    assert agree >= 0.99 and agree_ref >= 0.99
