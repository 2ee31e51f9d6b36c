"""The integer inference model layer by layer, teacher-forced: every integer layer of the four integer models
(support.INT8_MODELS) checked in float64 on the operands it was handed in a real forward, at batch 1 and 3, at 8/8 and
4/4 weight / activation bits and at 4/8 on ResNet-20.

Each _U8Bn, _U8Conv and _U8DwConv lowering of the executor's plan is wrapped so that its operands are cloned just
before its kernels run and its outputs just after, whatever buffers the plan shares:
- every level producer against float64 of its captured fp32 input (support.bn_chain with a correctly rounded rstd, the
  range of this batch): levels, header and channel sums bit for bit;
- every integer layer against float64 of the formula on its captured levels and its own weight levels, with bias,
  ReLU, residual and the folded batch norm the plan wired to it.
The forward runs with PF_POISON=1 and every producer's header and channel sums set to NaN beforehand, so finite logits
mean every element an integer layer read was written in this forward.  One loose whole-model comparison against the
fake-quant executor and the float64 oracle stays, and at 4/4 the export / load round trip."""
import collections
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from support import (INT8_MODELS, QUIET, bn_chain, conv64, dw_fwd_ref, enc, free, int8_graph, make, planes_value,  # noqa: E402
                     rsqrt_rn)

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _release():
    yield
    from pocketflow_b200.flags import FLAGS
    FLAGS.reset()
    free()


# (model, batch, weight bits, activation bits)
CONFIGS = [(key, batch, wb, ab) for key in INT8_MODELS for wb, ab in ((8, 8), (4, 4)) for batch in (1, 3)] + \
    [('resnet20_narrow', batch, 4, 8) for batch in (1, 3)]

_STATES, _RSTD = {}, {}
IMAGES = 12              # images of the loose whole-model comparison, at every batch


def _state(key, wb, ab):
    """a --learner uniform checkpoint state at these widths: the learner's own store after two training steps (shared
    by the batches of one model and width)"""
    if (key, wb, ab) not in _STATES:
        net, flags, _ = INT8_MODELS[key]
        reload = 'cifar10_dataset' if 'cifar' in net else 'ilsvrc12_dataset'
        lrn = make(net, 'uniform', 16, reload=reload, **dict(QUIET, uql_weight_bits=wb, uql_activation_bits=ab, **flags))
        for _ in range(2):
            lrn.train_step()
        _STATES[(key, wb, ab)] = lrn.sess_train.store.state_dict()
        del lrn
        free()
    return _STATES[(key, wb, ab)]


class Tap:
    """wraps forward() of every integer lowering of `ex`: per call, the operands cloned just before its kernels run and
    the outputs just after"""

    def __init__(self, ex):
        from pocketflow_b200.engine import _U8Bn, _U8Conv, _U8DwConv
        self.ex, self.calls, self.bn, self.layers = ex, collections.Counter(), [], []
        for table, cls, cap in ((ex.batch_norm, _U8Bn, self._bn), (ex.conv, _U8Conv, self._layer),
                                (ex.depthwise, _U8DwConv, self._layer)):
            for lo in table.values():
                if isinstance(lo, cls):
                    lo.forward = (lambda lo, run, cap: lambda *a: cap(lo, run, *a))(lo, lo.forward, cap)

    def _bn(self, lo, run, training):
        x = self.ex.T(lo.op.inputs[0]).clone()
        run(training)
        self.calls[lo.op.name] += 1
        self.bn.append(dict(lo=lo, x=x, levels=lo.levels.clone(), hdr=lo.hdr.clone(), csum=lo.csum.clone(),
                            slot=lo.base.slot.clone()))

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


def _rstd(key, op, mv, eps):
    """correctly rounded fp32 1 / sqrt(fp32(var + eps)), what the producer forms (per model and weights: cached)"""
    k = (key, op.name, float(mv.double().sum()))
    if k not in _RSTD:
        _RSTD[k] = rsqrt_rn(mv + torch.tensor(np.float32(eps), device=mv.device))
    return _RSTD[k]


def _levels_ref(y, mn, mx, bits):
    """float64 restatement of the producer's levels (as tests/test_int8_edges_gpu.py states it): alpha =
    fp32(mx - mn) + 1e-10, rint(fp32(fp32((y - mn) / alpha) * k)), k = 2^bits - 1"""
    k = 2 ** bits - 1
    alpha = np.float32(np.float32(mx) - np.float32(mn)) + np.float32(1e-10)
    xn = ((y - mn).double() / float(alpha)).float()
    return torch.round((xn.double() * k).float().double()), alpha, k


def _check_producer(key, ex, r):
    """levels, header, channel sums and range slot of one _U8Bn call, bit for bit"""
    lo = r['lo']
    base = lo.base
    m, c, mm, mv, eps, gamma, beta = base.moving
    bits = ex.act_quant['bits'][base.aq]
    y = bn_chain(r['x'].view(m, c), mm, _rstd(key, lo.op, mv, eps), gamma, beta, base.act)
    mn, mx = float(y.min()), float(y.max())
    name = lo.op.name
    assert np.array_equal(r['slot'].cpu().numpy().view(np.uint32), enc([mn, mx])), name
    lv, alpha, k = _levels_ref(y, mn, mx, bits)
    levels = r['levels'].view(m, c).double()
    assert float(levels.max()) <= k, name
    assert torch.equal(levels, lv), (name, int((levels != lv).sum()))
    hs = r['hdr'].cpu().numpy()
    if mn == 0.0:
        assert hs[1] == 1 and hs[0:1].view(np.float32)[0] == np.float32(alpha / np.float32(k)), (name, hs)
    else:
        assert hs[1] == 0 and hs[0:1].view(np.float32)[0] == np.float32(1), (name, hs)
    nseg = -(-c // 128)
    want = torch.stack([lv[:, 128 * i:128 * (i + 1)].sum(1) for i in range(nseg)], 1)
    assert torch.equal(r['csum'].view(m, nseg).double(), want), name


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
    kq = d.c if dw else d.k
    rk = np.float32(1) / np.float32(2 ** lo.bits - 1)          # the kernels' fp32 1 / (2^b - 1)
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
    assert ref.shape[-1] == kq
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
    # the bar of the kernel tests: S and J exact, then a few fp32 roundings of terms no larger than the magnitude
    ratio = float(((y - ref).abs() / (2.0 ** -22 * mag).clamp_min(1e-300)).max())
    assert ratio <= 1.0, (op.name, ratio)
    if 'folded' in r:
        # the folded inference BN + act of the kernel's own fp32 sum, in float64: a handful of fp32 roundings
        fb = r['folded']
        _, _, mm, mv, eps, gamma, beta = fb.moving
        z = ((y - mm.double()) / torch.sqrt(mv.double() + float(np.float32(eps)))) * gamma.double() + beta.double()
        z = torch.clamp(z, 0, 6 if fb.act == 2 else None) if fb.act else z
        scale_z = float(z.abs().max()) or 1.0
        if r['post'] is not None:
            assert float((r['post'].double().view(z.shape) - z).abs().max()) <= 1e-6 * scale_z, op.name
        if r['post_planes'] is not None:
            # hi + lo of the split-bf16 planes holds fp32 to 2^-17 of each value (two 8-bit significands, each
            # rounded to nearest); with the 1e-6 of the fp32 chain, 2^-16 of the largest value
            assert float((r['post_planes'].view(z.shape) - z).abs().max()) <= 2.0 ** -16 * scale_z, op.name
    return ratio


def _int_names(im):
    return sorted(name for name, why in im.sel if why is None)


@pytest.mark.parametrize('key,batch,wb,ab', CONFIGS, ids=['%s_b%d_w%da%d' % c for c in CONFIGS])
def test_int_model_teacher_forced(key, batch, wb, ab, monkeypatch, tmp_path):
    from oracle.mbv2_oracle import DropoutStepOracle      # StepOracle, with MobileNet-v2's inference-mode Dropout
    from pocketflow_b200 import compact, int8
    from pocketflow_b200.engine import _U8Bn
    state = _state(key, wb, ab)
    g, images, logits, cfg = int8_graph(key, batch, wb, ab)
    assert (cfg['weight_bits'], cfg['activation_bits']) == (wb, ab)
    dev = torch.device('cuda', 0)
    full = compact.map_state(g, compact.reachable_ops(g, logits), state)
    fq = int8.fake_quant_executor(g, images, logits, full, cfg, dev)
    # PF_POISON=1: every activation and scratch buffer of the integer model's plan starts as NaN
    monkeypatch.setenv('PF_POISON', '1')
    im = int8.IntModel.from_checkpoint(g, images, logits, state, cfg, dev)
    monkeypatch.delenv('PF_POISON')
    tap = Tap(im.ex)
    producers = sorted(op.name for op, lo in im.ex.batch_norm.items() if isinstance(lo, _U8Bn))
    for lo in im.ex.batch_norm.values():
        if isinstance(lo, _U8Bn):                        # no levels in them until this forward writes them
            lo.csum.fill_(float('nan'))
            lo.hdr.copy_(torch.tensor([0x7fc00000, 0], dtype=torch.int32))
    x = torch.randn(images.shape, generator=torch.Generator().manual_seed(batch)).to(dev)
    l0 = im.forward(x).clone()
    assert bool(torch.isfinite(l0).all())
    # the tap saw every layer select() marked as integer and every level producer, each exactly once
    ints = _int_names(im)
    assert sorted(r['lo'].op.name for r in tap.layers) == ints
    assert sorted(r['lo'].op.name for r in tap.bn) == producers
    assert {r['lo'].bn.op.name for r in tap.layers} == set(producers)
    assert set(tap.calls.values()) == {1}, tap.calls
    for r in tap.bn:
        _check_producer(key, im.ex, r)
    worst = max(_check_layer(r) for r in tap.layers)
    n_layers, n_producers = len(tap.layers), len(tap.bn)
    # the loose whole-model comparison of test_int8_gpu.py: quantizer level flips set both distances to the oracle.
    # That bar was set on the max over a batch of 32 .. 128 images; the max over one image's logits is a single draw of
    # where a level flips (measured on an H100 80GB HBM3 at 700 W, batch 1, one image: int / fake-quant 1.3 - 1.5 on
    # three of the nine configurations, 0.4 - 1.2 on the others).  So the distances here are maxima over the same IMAGES images at every batch, run
    # through the model `batch` at a time.
    wq, aq = int8._specs(g, cfg)
    orc = DropoutStepOracle(compact.reachable_ops(g, logits), logits, images, weight_quant=wq, act_quant=aq)
    params = {k: torch.from_numpy(v).double().to(dev) for k, v in full.items()}
    xs = torch.randn((IMAGES,) + tuple(images.shape[1:]), generator=torch.Generator().manual_seed(1)).to(dev)
    li, lf, ref = [], [], []
    for i in range(0, IMAGES, batch):
        xb = xs[i:i + batch]
        li.append(im.forward(xb).clone())
        fq.buf[fq.images].copy_(xb)
        lf.append(fq.forward(training=False).clone())
        ref.append(orc.forward(params, xb.double(), training=False)[logits.name].double())
    li, lf, ref = torch.cat(li), torch.cat(lf), torch.cat(ref)
    assert bool(torch.isfinite(li).all())
    s = float(ref.abs().max())
    e_int, e_fq = float((li.double() - ref).abs().max()) / s, float((lf.double() - ref).abs().max()) / s
    agree = float((li.argmax(1) == lf.argmax(1)).float().mean())
    print('%s batch %d W%dA%d: %d integer layers, %d producers checked; worst epilogue error %.3f of its bound; '
          'int %.3e fake-quant %.3e (of max|ref|, %d images), top-1 agreement %.4f'
          % (key, batch, wb, ab, n_layers, n_producers, worst, e_int, e_fq, IMAGES, agree))
    assert e_int <= 1.3 * e_fq, (e_int, e_fq)
    # top-1 agreement, the bar test_int8_gpu.py set on 8-bit activations.  At 4-bit activations one level is 1/15 of a
    # layer's range, and after two training steps ResNet-50's two largest logits can lie closer than a flip of one
    # such level moves them (measured on an H100 at 700 W, batch 3: 11 of 12 images agree), so there it is reported only.
    if ab == 8:
        assert agree >= 0.99
    if (wb, ab) == (4, 4):
        im.export(str(tmp_path / 'int8'))
        im2 = int8.IntModel.load(g, images, logits, str(tmp_path / 'int8'), dev)
        assert (im2.cfg['weight_bits'], im2.cfg['activation_bits']) == (4, 4)
        assert _int_names(im2) == ints
        assert torch.equal(im2.forward(x), l0)
