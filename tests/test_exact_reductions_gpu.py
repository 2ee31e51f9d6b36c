"""The long reductions of the benchmarked steps, checked exactly on integer-valued operands.

The bench-layer tests (test_tc_bench_layers_gpu, test_nn_bench_layers_gpu) hold a weight gradient to a fraction of its
largest sum of |terms|.  Such a bar tolerates about bar x Npix pixels' worth of terms lost or counted twice: at 3.2 M
pixels, some 60.  Here the answer is exact instead.  Every partial sum of integers below EXACT_BOUND is an integer an
fp32 accumulator holds exactly, whatever the order of the additions and however split-K partitions the pixels, so the
kernel must equal a float64 reference bit for bit, and one missing or duplicated pixel fails.

For each run (the benchmark workloads of test_nn_bench_layers_gpu.RUNS and the compact fine-tune steps of ResNet-50 and
MobileNet-v1) one eager step records, for the first call of each distinct (entry point, geometry, operand form,
epilogue, deferred or not), the descriptor, the form and the launch plan (pf_conv2d_tc_last_plan, or the depthwise
variant).  The learner is freed, and every key is replayed through the same `ops` call on fresh integer operands of the
same form; the replay must run the recorded plan.  The references are float64 DGEMMs, one per filter tap over strided,
shifted slices (exact on integers, unlike Winograd / FFT convolutions), chunked over the batch.  Split operand planes
count as hi.hi + hi.lo + lo.hi: the kernels drop lo.lo (pf_conv_tc.cu).  A deferred weight gradient is checked split
by split against the reference over that split's pixel range, then through TcWgradReduceBatch.reduce.

What is compared, and why not more:
  * conv2d_tc_{fwd,dgrad,wgrad} in the fp32, `_planes` and `_ex` forms, with bias, ReLU, residual and accumulate; of a
    forward with a folded inference batch norm (bn_out) only y, the batch norm's output is not integer.  Weight levels
    (`_ex`) use alpha = 2^bits - 1, so one level step is fp32(alpha * fp32(1 / alpha)) = 1, and beta = 1 - 2^(bits-1),
    so the epilogue's window-sum term J * (centre + beta) is J: every step of its op chain stays integer;
  * conv2d_{fwd,dgrad,wgrad} (CUDA-core, at the recorded operands' offsets from 16-byte alignment),
    dwconv_{fwd,dgrad,wgrad}, fold_diag_blocks, colsum, l2_loss at scale 2, the codebook gradient with every scale 1,
    TcWgradReduceBatch.reduce;
  * BN-backward dbeta and dgamma at mean 0, rstd 1, gamma 1, beta 0, where every fp32 step of
    ((x - mean) * rstd) * gamma + beta gives x: both are integer sums over the rows (dx divides by m and is not).
Every call of a wrapped entry point must have a replayed key, or one in SKIPPED with its reason; every other public
entry point the step calls must be checked by test_nn_bench_layers_gpu or be in NOT_REPLAYED with its reason."""
import gc
import time
import types
import zlib

import numpy as np
import pytest
import torch

from pocketflow_b200 import ops
from support import (CLASSES, EXACT_BOUND, EXEMPT, QUIET, RUNS, NnRecorder, after_step, conv_dgrad_ref, conv_fwd_ref,
                     conv_wgrad_ref, dw_dgrad_ref, dw_fwd_ref, dw_wgrad_ref, every_pixel_contributes, geom, int_values,
                     make, plan_key, prune_interior, reduction_operands, run_workload, split_terms, wgrad_density,
                     write_dgrad_weight, write_fwd_weight)

DEV = torch.device('cuda:0')

TC_NAMES = ('conv2d_tc_fwd', 'conv2d_tc_fwd_planes', 'conv2d_tc_fwd_ex', 'conv2d_tc_dgrad', 'conv2d_tc_dgrad_planes',
            'conv2d_tc_dgrad_ex', 'conv2d_tc_wgrad', 'conv2d_tc_wgrad_planes', 'conv2d_tc_wgrad_ex')
NAMES = TC_NAMES + ('conv2d_fwd', 'conv2d_dgrad', 'conv2d_wgrad', 'dwconv_fwd', 'dwconv_dgrad', 'dwconv_wgrad',
                    'fold_diag_blocks', 'colsum', 'l2_loss', 'bn_bwd')
METHODS = (('CodebookWeightQuantizer', 'cluster_grad'), ('TcWgradReduceBatch', 'reduce'))
# keys of these entry points are recorded and not replayed, and why
SKIPPED = {'conv2d_tc_dgrad_ex': 'the engine does not call it (the dgrad operands are split planes)'}
# the entry points test_nn_bench_layers_gpu checks against float64 or bit for bit, and its host-side helpers
CHECKED_ELSEWHERE = ({n[3:] for n in dir(NnRecorder) if n.startswith('_c_')} |
                     {n[3:].replace('_', '.', 1) for n in dir(NnRecorder) if n.startswith('_m_')} | set(EXEMPT))
# entry points the steps call that are not replayed here, and why; any other one the step calls fails the test
NOT_REPLAYED = {
    'bn_train_stats': 'mean and variance divide by the row count: not integer (1e-6 / 1e-5 bars elsewhere)',
    'bn_train_stats_range': 'mean and variance divide by the row count: not integer (1e-6 / 1e-5 bars elsewhere)',
    'global_avgpool_fwd': 'divides by the pixel count: not integer',
    'softmax_ce': 'a reduction over one row of logits through exponentials',
    'softmax_fwd': 'a reduction over one row of logits through exponentials',
    'softmax_bwd': 'a reduction over one row of logits',
    'bn_apply_quant_levels': 'its channel sums run over at most 128 channels of one pixel, bit-exact elsewhere',
    'UniformWeightQuantizer.minmax': 'a min / max: exact in any order, bit-exact elsewhere',
    'act_minmax': 'a min / max: exact in any order, bit-exact elsewhere',
    'select_desc': 'an order statistic, bit-exact elsewhere',
    'gather_channels': 'a channel gather, no reduction (bit-exact in test_compact_train_gpu)',
    'scatter_channels': 'a channel scatter, no reduction (bit-exact in test_compact_train_gpu)',
    'bn_apply_gather': 'BN apply + channel gather, no reduction (bit-exact in test_compact_train_gpu)',
    'bn_apply_eval_gather': 'BN apply + channel gather, no reduction (bit-exact in test_compact_train_gpu)',
    'scatter_table': 'host-side table',
}
# the bar each weight gradient is held to by the bench-layer tests, relative to the largest sum of |terms|
FLOAT_BAR = {'conv2d_tc_wgrad': 2e-5, 'conv2d_tc_wgrad_planes': 2e-5, 'conv2d_tc_wgrad_ex': 2e-5,
             'conv2d_wgrad': 1e-5, 'dwconv_wgrad': 1e-5}


def dv(t):
    return t.double()


# ------------------------------------------------------------------------------------------------ recorder
class ExactRecorder:
    """wraps NAMES and METHODS of `ops`; keeps, for the first call of each key, what a replay needs (never a tensor)"""

    def __init__(self, monkeypatch):
        self.orig = {name: getattr(ops, name) for name in NAMES + ('tc_act', 'tc_wt', 'conv2d_tc_last_plan',
                                                                   'dwconv_last_variant')}
        self.orig.update({'%s.%s' % cm: getattr(getattr(ops, cm[0]), cm[1]) for cm in METHODS})
        self.first, self.calls, self.label, self.secs, self.peak = {}, {}, None, 0.0, 0.0
        orig_act, orig_wt = ops.tc_act, ops.tc_wt

        def tc_act(planes, hdr=None, csum=None, nseg=0, single=False):
            a = orig_act(planes, hdr, csum, nseg, single)
            a._src = (planes, hdr, csum, int(nseg), single)
            return a

        def tc_wt(p0, p1=None, alpha=None, beta=None, per_channel=False, bits=0):
            w = orig_wt(p0, p1, alpha, beta, per_channel, bits)
            w._src = (p0, p1, alpha, beta, bool(per_channel), int(bits))
            return w

        monkeypatch.setattr(ops, 'tc_act', tc_act)
        monkeypatch.setattr(ops, 'tc_wt', tc_wt)
        for name in NAMES:
            monkeypatch.setattr(ops, name, self._wrap(name, getattr(ops, name)))
        for cname, mname in METHODS:
            cls = getattr(ops, cname)
            monkeypatch.setattr(cls, mname, self._wrap('%s.%s' % (cname, mname), getattr(cls, mname)))
        # every other public callable of ops only notes that the step called it (finish() freezes the set)
        self.called, self.step_called = set(), None
        for name in dir(ops):
            obj = getattr(ops, name)
            if name in NAMES or name.startswith('_') or isinstance(obj, type) or not callable(obj) or \
                    getattr(obj, '__module__', None) != ops.__name__:
                continue
            monkeypatch.setattr(ops, name, self._note(name, obj))
        for cname in CLASSES:
            cls = getattr(ops, cname)
            for mname, fn in list(vars(cls).items()):
                if not mname.startswith('_') and callable(fn) and (cname, mname) not in METHODS:
                    monkeypatch.setattr(cls, mname, self._note('%s.%s' % (cname, mname), fn))

    def _note(self, name, fn):
        def call(*args, **kw):
            self.called.add(name)
            return fn(*args, **kw)
        return call

    def _wrap(self, name, fn):
        def call(*args, **kw):
            meta = getattr(self, '_m_' + name.split('.')[-1])(name, *args, **kw)
            key = (name,) + meta['key']
            first = key not in self.first
            out = fn(*args, **kw)
            self.calls[key] = self.calls.get(key, 0) + 1
            if first:
                if name in TC_NAMES:
                    meta['plan'] = self.orig['conv2d_tc_last_plan']()
                elif name.startswith('dwconv_'):
                    meta['variant'] = self.orig['dwconv_last_variant']()
                self.first[key] = meta
            return out
        return call

    # ---- what identifies a call, and what its replay needs
    @staticmethod
    def _act(a):
        planes, hdr, csum, nseg, single = a._src
        nplanes = int(hdr.cpu().numpy().view(ops.ACT_HDR)[0]['nplanes']) if hdr is not None else 0
        form = 'single' if single else ('hdr%d' % nplanes if hdr is not None else 'split')
        return dict(form=form, numel=planes.numel, csum=csum is not None, nseg=nseg)

    @staticmethod
    def _wt(w):
        p0, p1, alpha, beta, per_channel, bits = w._src
        return dict(levels=alpha is not None, numel=p0.numel(), two=p1 is not None, per_channel=per_channel,
                    bits=bits, nalpha=alpha.numel() if alpha is not None else 0)

    def _m_fwd(self, name, d, x, w, bias, relu, y, residual=None, bn_out=None):
        torch.cuda.synchronize()              # an operand header may come from a producer on another stream
        m = dict(g=geom(d), y=y.numel(), bias=bias is not None, relu=bool(relu), res=residual is not None,
                 bn=None)
        if name == 'conv2d_tc_fwd_ex':
            m['act'], m['wt'] = self._act(x), self._wt(w)
            form = m['act']['form'] + (' x levels' if m['wt']['levels'] else ' x split')
        else:
            m['x'], m['wf'] = (x.numel() if name == 'conv2d_tc_fwd' else x.numel), w.f_hi.numel()
            form = ('fp32' if name == 'conv2d_tc_fwd' else 'split') + ' x split'
        if bn_out is not None:
            m['bn'] = dict(eps=float(bn_out.eps), act=int(bn_out.act), y=bn_out._keep[4] is not None,
                           planes=bn_out._keep[5].numel if bn_out._keep[5] is not None else 0)
        m['key'] = (m['g'], form, m['bias'], m['relu'], m['res'], bn_out is not None)
        return m

    _m_conv2d_tc_fwd = _m_conv2d_tc_fwd_planes = _m_conv2d_tc_fwd_ex = _m_fwd

    def _m_dgrad(self, name, d, dy, w, acc, dx):
        m = dict(g=geom(d), acc=bool(acc), dx=dx.numel())
        if name == 'conv2d_tc_dgrad_ex':
            m['key'] = (m['g'], 'ex', m['acc'])
            return m
        m['dy'] = dy.numel() if name == 'conv2d_tc_dgrad' else dy.numel
        m['wd'] = w.d_hi.numel()
        m['key'] = (m['g'], 'fp32 x split' if name == 'conv2d_tc_dgrad' else 'split x split', m['acc'])
        return m

    _m_conv2d_tc_dgrad = _m_conv2d_tc_dgrad_planes = _m_conv2d_tc_dgrad_ex = _m_dgrad

    def _m_wgrad(self, name, d, x, dy, ws, dw):
        torch.cuda.synchronize()
        m = dict(g=geom(d), ws=ws.numel(), dw=dw.numel() if dw is not None else 0)
        if name == 'conv2d_tc_wgrad_ex':
            m['act'], m['dy_act'] = self._act(x), self._act(dy)
            form = m['act']['form'] + ' x ' + m['dy_act']['form']
        elif name == 'conv2d_tc_wgrad':
            m['x'], m['dy'] = x.numel(), dy.numel()
            form = 'fp32 x fp32'
        else:
            m['x'], m['dy'] = x.numel, dy.numel
            form = 'split x split'
        m['key'] = (m['g'], form, dw is None)
        return m

    _m_conv2d_tc_wgrad = _m_conv2d_tc_wgrad_planes = _m_conv2d_tc_wgrad_ex = _m_wgrad

    @staticmethod
    def _mis(*ts):
        """byte offset of each operand from 16-byte alignment: the CUDA-core kernels pick their vectorised or scalar
        form from it (pf_conv.cu: aligned16), so a replay reproduces it"""
        return tuple(t.data_ptr() % 16 if t is not None else 0 for t in ts)

    def _m_conv2d_fwd(self, name, d, x, w, bias, relu, y):
        return dict(g=geom(d), x=x.numel(), y=y.numel(), bias=bias is not None, relu=bool(relu),
                    mis=self._mis(x, w, y), key=(geom(d), bias is not None, bool(relu), self._mis(x, w, y)))

    def _m_conv2d_dgrad(self, name, d, dy, w, wt_ws, acc, dx):
        mis = self._mis(dy, wt_ws, dx)
        return dict(g=geom(d), dy=dy.numel(), dx=dx.numel(), wt_ws=wt_ws.numel() if wt_ws is not None else 0,
                    acc=bool(acc), mis=mis, key=(geom(d), bool(acc), mis))

    def _m_conv2d_wgrad(self, name, d, x, dy, ws, dw):
        mis = self._mis(x, dy, dw, ws)
        return dict(g=geom(d), x=x.numel(), dy=dy.numel(), ws=ws.numel() if ws is not None else 0, dw=dw.numel(),
                    mis=mis, key=(geom(d), mis))

    def _m_bn_bwd(self, name, dy, x, m, c, mean, rstd, gamma, beta, act, dgamma, dbeta, dx, acc, ws, planes=None):
        return dict(m=int(m), c=int(c), act=int(act), acc=bool(acc), dx=dx.numel() if dx is not None else 0,
                    planes=planes.numel if planes is not None else 0, ws=ws.numel(),
                    key=(int(m), int(c), int(act), bool(acc), dx is not None, planes is not None))

    def _m_dwconv_fwd(self, name, d, x, w, y):
        return dict(g=geom(d), x=x.numel(), y=y.numel(), key=(geom(d),))

    def _m_dwconv_dgrad(self, name, d, dy, w, acc, dx):
        return dict(g=geom(d), dy=dy.numel(), dx=dx.numel(), acc=bool(acc), key=(geom(d), bool(acc)))

    def _m_dwconv_wgrad(self, name, d, x, dy, ws, dw):
        return dict(g=geom(d), x=x.numel(), dy=dy.numel(), ws=ws.numel() if ws is not None else 0, dw=dw.numel(),
                    key=(geom(d),))

    def _m_fold_diag_blocks(self, name, src, g, m, n, dst):
        return dict(src=src.numel(), dst=dst.numel(), gmn=(int(g), int(m), int(n)), key=(int(g), int(m), int(n)))

    def _m_colsum(self, name, a, m, c, out):
        return dict(a=a.numel(), out=out.numel(), mc=(int(m), int(c)), key=(int(m), int(c)))

    def _m_l2_loss(self, name, v, scale, out, partial_ws, accumulate=False):
        return dict(v=v.numel(), out=out.numel(), ws=partial_ws.numel(), acc=bool(accumulate),
                    key=(v.numel(), bool(accumulate)))

    def _m_cluster_grad(self, name, q, grads, grad_base):
        assert not q.use_buckets, 'bucketed codebooks are not benchmarked'
        shapes = tuple(tuple(s.shape) for s in q.srcs)
        return dict(shapes=shapes, bits=tuple(q.uq.bits), grads=tuple(g.numel() for g in grads),
                    base=grad_base.numel(), key=(shapes, tuple(q.uq.bits)))

    def _m_reduce(self, name, rb):
        items = tuple((int(part.numel()), int(out.numel()), int(splits)) for part, out, splits in rb.keep)
        return dict(items=items, key=(items,))

    def finish(self, label, secs, peak_gb):
        self.label, self.secs, self.peak = label, secs, peak_gb
        self.step_called = set(self.called) | {k[0] for k in self.calls}


# ------------------------------------------------------------------------------------------------ replay
def _planes(numel, vals):
    """ops.Planes of `numel` elements holding vals[0] (hi) and vals[1] (lo) in their first elements; the rest zero"""
    pl = ops.Planes(numel, DEV)
    pl.buf.zero_()
    for dst, v in zip((pl.hi, pl.lo), vals):
        dst[:v.numel()] = v.reshape(-1).to(torch.bfloat16)
    return pl


def _fp32(numel, v, mis=0):
    """fp32 buffer of numel elements starting `mis` bytes past a 16-byte boundary, holding v in its first elements"""
    t = torch.zeros(numel + 4, device=DEV)[mis // 4:mis // 4 + numel]
    if v is not None:
        t[:v.numel()] = v.reshape(-1)
    return t


def _nan(numel, mis=0):
    return torch.full((max(numel, 1) + 4,), float('nan'), device=DEV)[mis // 4:mis // 4 + max(numel, 1)]


def _hdr(scale, nplanes):
    return torch.from_numpy(np.array([(scale, nplanes)], dtype=ops.ACT_HDR).view(np.uint8)).to(DEV)


class Replay:
    """replays the keys of one ExactRecorder with fresh integer operands; see the module docstring"""

    def __init__(self, rec, seed):
        self.rec, self.f = rec, rec.orig
        self.g = torch.Generator(device=DEV).manual_seed(seed)
        self.fails, self.replayed, self.skipped, self.notes, self.tolerated = [], set(), {}, [], []

    def run(self):
        for key, meta in self.rec.first.items():
            name = key[0]
            if name in SKIPPED:
                self.skipped[key] = SKIPPED[name]
                continue
            getattr(self, '_r_' + name.split('.')[-1])(name, key, meta)
            self.replayed.add(key)
            torch.cuda.synchronize()
            gc.collect()
            torch.cuda.empty_cache()
        return self

    # ---- helpers
    def _exact(self, key, got, ref, what=''):
        got = got.double()
        if not torch.equal(got, ref):
            bad = int((got != ref).sum())
            self.fails.append((key, what, '%d of %d entries differ, worst by %g' % (
                bad, ref.numel(), (got - ref).abs().max().item())))

    def _bound(self, key, mag, what=''):
        m = mag.abs().max().item() if mag.numel() else 0.0
        assert m < EXACT_BOUND, ('operands too large for an exact reference', key, what, m)

    def _plan(self, key, meta):
        got = self.f['conv2d_tc_last_plan']()
        want = meta['plan']
        diff = {f: (want[f], got[f]) for f in want if f != 'seq' and want[f] != got[f]}
        if diff:
            self.fails.append((key, 'plan %s' % (plan_key(want),), diff))
        return got

    def _variant(self, key, meta):
        got = self.f['dwconv_last_variant']()
        if got != meta['variant']:
            self.fails.append((key, 'depthwise variant', (meta['variant'], got)))

    def _act_operand(self, a, shape, density, signed=True, carrier=None):
        """(pf_tc_act, planes of the value it represents) of form a (ExactRecorder._act): split (hi, lo), single (hi),
        hdr1 (levels in hi, scale 1), hdr2 (split planes under a header with scale 1).  Levels are non-negative."""
        form = a['form']
        levels = form in ('hdr1', 'single')
        if carrier is not None:
            vals = carrier
        else:
            vals = [int_values(shape, density, self.g, signed and not levels) for _ in range(1 if levels else 2)]
        if form == 'hdr1' or form == 'single':
            vals = [v.abs() for v in vals[:1]]
        pl = _planes(a['numel'], vals)
        if form == 'hdr1':
            pl.lo.fill_(float('nan'))                  # one plane under the header: the lo plane is never read
        hdr = _hdr(1.0, int(form[3])) if form.startswith('hdr') else None
        csum = None
        if a['csum']:
            n, h, w, c = shape
            tot = sum(vals)
            csum = tot.reshape(-1, a['nseg'], c // a['nseg']).sum(2).contiguous()
        act = self.f['tc_act'](pl, hdr, csum, a['nseg'], form == 'single')
        act._keep = (pl, hdr, csum)
        return act, [dv(v) for v in vals]

    def _tolerated(self, key, name, npix):
        self.tolerated.append((key, FLOAT_BAR[name] * npix))

    # ---- tensor-core convolutions
    def _r_conv2d_tc_fwd(self, name, key, meta):
        n, h, w, c, k, r, s, p, q = meta['g'][:9]
        g = self.g
        xshape, wshape = (n, h, w, c), (r, s, c, k)
        if name == 'conv2d_tc_fwd_ex':
            act, xv = self._act_operand(meta['act'], xshape, 0.5)
            wm = meta['wt']
            if wm['levels']:
                bits = wm['bits']
                kq, centre = (1 << bits) - 1, float(1 << (bits - 1))
                p0 = int_values(wshape, 0.5, g)                               # stored level - centre
                pk = torch.zeros(wm['numel'], dtype=torch.bfloat16, device=DEV)
                write_fwd_weight(pk, None, p0, None)
                alpha = torch.full((max(wm['nalpha'], 4),), float(kq), device=DEV)
                beta = torch.full((max(wm['nalpha'], 4),), 1.0 - centre, device=DEV)
                wt = self.f['tc_wt'](pk, None, alpha, beta, wm['per_channel'], bits)
                wt._keep = (pk, alpha, beta)
                wv = [dv(p0 + 1.0)]                   # alpha / k * (p0 + centre) + beta with alpha / k = 1
            else:
                wv32 = [int_values(wshape, 0.5, g) for _ in range(2 if wm['two'] else 1)]
                hi = torch.zeros(wm['numel'], dtype=torch.bfloat16, device=DEV)
                lo = torch.zeros(wm['numel'], dtype=torch.bfloat16, device=DEV) if wm['two'] else None
                write_fwd_weight(hi, lo, wv32[0], wv32[1] if wm['two'] else None)
                wt = self.f['tc_wt'](hi, lo)
                wt._keep = (hi, lo)
                wv = [dv(v) for v in wv32]
            xop = act
        else:
            xv32 = [int_values(xshape, 0.5, g)] + ([int_values(xshape, 0.5, g)] if name.endswith('_planes') else [])
            xop = _fp32(meta['x'], xv32[0]) if name == 'conv2d_tc_fwd' else _planes(meta['x'], xv32)
            xv = [dv(v) for v in xv32]
            wv32 = [int_values(wshape, 0.5, g), int_values(wshape, 0.5, g)]
            wt = types.SimpleNamespace(f_hi=torch.zeros(meta['wf'], dtype=torch.bfloat16, device=DEV),
                                       f_lo=torch.zeros(meta['wf'], dtype=torch.bfloat16, device=DEV))
            write_fwd_weight(wt.f_hi, wt.f_lo, *wv32)
            wv = [dv(v) for v in wv32]
        bias = int_values((k,), 0.5, g) if meta['bias'] else None
        res = int_values((n, p, q, k), 0.5, g) if meta['res'] else None
        y = _nan(meta['y'])
        d = ops.conv_desc(*meta['g'])
        args = (d, xop, wt, bias, meta['relu'], y, _fp32(meta['y'], res) if res is not None else None)
        if meta['bn'] is not None:
            b = meta['bn']
            bn_y = _nan(meta['y']) if b['y'] else None
            bn_pl = ops.Planes(b['planes'], DEV) if b['planes'] else None
            bn = ops.TcBnOut(torch.zeros(k, device=DEV), torch.ones(k, device=DEV), b['eps'], torch.ones(k, device=DEV),
                             torch.zeros(k, device=DEV), b['act'], bn_y, bn_pl)
            self.f[name](*args, bn)
        else:
            self.f[name](*args)
        self._plan(key, meta)
        ref = split_terms(lambda a, b: conv_fwd_ref(a, b, meta['g']), xv, wv)
        mag = split_terms(lambda a, b: conv_fwd_ref(a, b, meta['g']), [v.abs() for v in xv], [v.abs() for v in wv])
        if bias is not None:
            ref, mag = ref + dv(bias), mag + dv(bias).abs()
        if meta['relu']:
            ref = torch.relu(ref)
        if res is not None:
            ref, mag = ref + dv(res), mag + dv(res).abs()
        self._bound(key, mag)
        self._exact(key, y[:ref.numel()].view(ref.shape), ref, 'y')

    _r_conv2d_tc_fwd_planes = _r_conv2d_tc_fwd_ex = _r_conv2d_tc_fwd

    def _r_conv2d_tc_dgrad(self, name, key, meta):
        n, h, w, c, k, r, s, p, q = meta['g'][:9]
        g = self.g
        yshape, wshape = (n, p, q, k), (r, s, c, k)
        dv32 = [int_values(yshape, 0.5, g)] + ([int_values(yshape, 0.5, g)] if name.endswith('_planes') else [])
        dyop = _fp32(meta['dy'], dv32[0]) if name == 'conv2d_tc_dgrad' else _planes(meta['dy'], dv32)
        wv32 = [int_values(wshape, 0.5, g), int_values(wshape, 0.5, g)]
        wt = types.SimpleNamespace(d_hi=torch.zeros(meta['wd'], dtype=torch.bfloat16, device=DEV),
                                   d_lo=torch.zeros(meta['wd'], dtype=torch.bfloat16, device=DEV))
        write_dgrad_weight(wt.d_hi, wt.d_lo, *wv32)
        prior = int_values((n, h, w, c), 0.5, g) if meta['acc'] else None
        dx = _fp32(meta['dx'], prior) if prior is not None else _nan(meta['dx'])
        self.f[name](ops.conv_desc(*meta['g']), dyop, wt, meta['acc'], dx)
        self._plan(key, meta)
        yv, wv = [dv(v) for v in dv32], [dv(v) for v in wv32]
        ref = split_terms(lambda a, b: conv_dgrad_ref(a, b, meta['g']), yv, wv)
        mag = split_terms(lambda a, b: conv_dgrad_ref(a, b, meta['g']), [v.abs() for v in yv], [v.abs() for v in wv])
        if prior is not None:
            ref, mag = ref + dv(prior), mag + dv(prior).abs()
        self._bound(key, mag)
        self._exact(key, dx[:ref.numel()].view(ref.shape), ref, 'dx')

    _r_conv2d_tc_dgrad_planes = _r_conv2d_tc_dgrad

    def _r_conv2d_tc_wgrad(self, name, key, meta):
        n, h, w, c, k, r, s, p, q = meta['g'][:9]
        npix = n * p * q
        xshape, yshape = (n, h, w, c), (n, p, q, k)
        if name == 'conv2d_tc_wgrad_ex':
            xa, ya = meta['act'], meta['dy_act']
            nx = 1 if xa['form'] in ('hdr1', 'single') else 2
            xs, ys = reduction_operands(xshape, yshape, nx, 2, wgrad_density(npix, 3), self.g,
                                        x_signed=nx == 2)
            xop, xv = self._act_operand(xa, xshape, 0, carrier=xs)
            yop, yv = self._act_operand(ya, yshape, 0, carrier=ys)
        else:
            two = name == 'conv2d_tc_wgrad_planes'
            xs, ys = reduction_operands(xshape, yshape, 2 if two else 1, 2 if two else 1,
                                        wgrad_density(npix, 3 if two else 1), self.g)
            if two:
                xop, yop = _planes(meta['x'], xs), _planes(meta['dy'], ys)
            else:
                xop, yop = _fp32(meta['x'], xs[0]), _fp32(meta['dy'], ys[0])
            xv, yv = [dv(v) for v in xs], [dv(v) for v in ys]
        assert every_pixel_contributes(xs, ys), key
        del xs, ys
        ws = _nan(meta['ws'])
        dw = _nan(meta['dw']) if meta['dw'] else None
        self.f[name](ops.conv_desc(*meta['g']), xop, yop, ws, dw)
        plan = self._plan(key, meta)
        splits, pps = max(plan['splits'], 1), plan['pps']
        bounds = [min(npix, i * pps) for i in range(splits)] + [npix] if dw is None else None
        tot, parts = conv_wgrad_ref(xv[0], yv[0] + yv[1] if len(yv) > 1 else yv[0], meta['g'], bounds)
        if len(xv) > 1:
            t2, p2 = conv_wgrad_ref(xv[1], yv[0], meta['g'], bounds)
            tot, parts = tot + t2, (parts + p2 if parts is not None else None)
        mag = split_terms(lambda a, b: conv_wgrad_ref(a, b, meta['g'])[0], [v.abs() for v in xv],
                          [v.abs() for v in yv])
        self._bound(key, mag)
        self._tolerated(key, name, npix)
        nel = r * s * c * k
        if dw is None:
            got = ws[:splits * nel].view(splits, r, s, c, k)
            for i in range(splits):
                self._exact(key, got[i], parts[i], 'split %d of %d (pixels %d..%d)' % (i, splits, bounds[i],
                                                                                     bounds[i + 1]))
            self._exact(key, got.double().sum(0), tot, 'sum of the partials')
            # the deferred reduction of these partials
            out = _nan(nel)
            rb = ops.TcWgradReduceBatch([(ws, out, splits)], DEV)
            self.f['TcWgradReduceBatch.reduce'](rb)
            self._exact(key, out.view(tot.shape), tot, 'TcWgradReduceBatch.reduce')
        else:
            self._exact(key, dw[:nel].view(tot.shape), tot, 'dw')

    _r_conv2d_tc_wgrad_planes = _r_conv2d_tc_wgrad_ex = _r_conv2d_tc_wgrad

    # ---- CUDA-core convolutions
    def _r_conv2d_fwd(self, name, key, meta):
        n, h, w, c, k, r, s, p, q = meta['g'][:9]
        x, wt = int_values((n, h, w, c), 0.5, self.g), int_values((r, s, c, k), 0.5, self.g)
        bias = int_values((k,), 0.5, self.g) if meta['bias'] else None
        mx, mw, my = meta['mis']
        y = _nan(meta['y'], my)
        self.f[name](ops.conv_desc(*meta['g']), _fp32(meta['x'], x, mx), _fp32(wt.numel(), wt, mw), bias,
                     meta['relu'], y)
        ref, mag = conv_fwd_ref(dv(x), dv(wt), meta['g']), conv_fwd_ref(dv(x).abs(), dv(wt).abs(), meta['g'])
        if bias is not None:
            ref, mag = ref + dv(bias), mag + dv(bias).abs()
        if meta['relu']:
            ref = torch.relu(ref)
        self._bound(key, mag)
        self._exact(key, y[:ref.numel()].view(ref.shape), ref, 'y')

    def _r_conv2d_dgrad(self, name, key, meta):
        n, h, w, c, k, r, s, p, q = meta['g'][:9]
        dy, wt = int_values((n, p, q, k), 0.5, self.g), int_values((r, s, c, k), 0.5, self.g)
        prior = int_values((n, h, w, c), 0.5, self.g) if meta['acc'] else None
        mdy, mws, mdx = meta['mis']
        dx = _fp32(meta['dx'], prior, mdx) if prior is not None else _nan(meta['dx'], mdx)
        wt_ws = _nan(meta['wt_ws'], mws) if meta['wt_ws'] else None
        self.f[name](ops.conv_desc(*meta['g']), _fp32(meta['dy'], dy, mdy), wt.contiguous(), wt_ws, meta['acc'], dx)
        ref, mag = conv_dgrad_ref(dv(dy), dv(wt), meta['g']), conv_dgrad_ref(dv(dy).abs(), dv(wt).abs(), meta['g'])
        if prior is not None:
            ref, mag = ref + dv(prior), mag + dv(prior).abs()
        self._bound(key, mag)
        self._exact(key, dx[:ref.numel()].view(ref.shape), ref, 'dx')

    def _r_conv2d_wgrad(self, name, key, meta):
        n, h, w, c, k, r, s, p, q = meta['g'][:9]
        npix = n * p * q
        xs, ys = reduction_operands((n, h, w, c), (n, p, q, k), 1, 1, wgrad_density(npix, 1), self.g)
        assert every_pixel_contributes(xs, ys), key
        mx, mdy, mdw, mws = meta['mis']
        ws, dw = (_nan(meta['ws'], mws) if meta['ws'] else None), _nan(meta['dw'], mdw)
        self.f[name](ops.conv_desc(*meta['g']), _fp32(meta['x'], xs[0], mx), _fp32(meta['dy'], ys[0], mdy), ws, dw)
        ref = conv_wgrad_ref(dv(xs[0]), dv(ys[0]), meta['g'])[0]
        self._bound(key, conv_wgrad_ref(dv(xs[0]).abs(), dv(ys[0]).abs(), meta['g'])[0])
        self._tolerated(key, name, npix)
        self._exact(key, dw[:ref.numel()].view(ref.shape), ref, 'dw')

    # ---- depthwise
    def _r_dwconv_fwd(self, name, key, meta):
        n, h, w, c, k, r, s, p, q = meta['g'][:9]
        x, wt = int_values((n, h, w, c), 0.5, self.g), int_values((r, s, c), 0.5, self.g)
        y = _nan(meta['y'])
        self.f[name](ops.conv_desc(*meta['g']), _fp32(meta['x'], x), wt.contiguous(), y)
        self._variant(key, meta)
        ref = dw_fwd_ref(dv(x), dv(wt), meta['g'])
        self._exact(key, y[:ref.numel()].view(ref.shape), ref, 'y')

    def _r_dwconv_dgrad(self, name, key, meta):
        n, h, w, c, k, r, s, p, q = meta['g'][:9]
        dy, wt = int_values((n, p, q, c), 0.5, self.g), int_values((r, s, c), 0.5, self.g)
        prior = int_values((n, h, w, c), 0.5, self.g) if meta['acc'] else None
        dx = _fp32(meta['dx'], prior) if prior is not None else _nan(meta['dx'])
        self.f[name](ops.conv_desc(*meta['g']), _fp32(meta['dy'], dy), wt.contiguous(), meta['acc'], dx)
        self._variant(key, meta)
        ref = dw_dgrad_ref(dv(dy), dv(wt), meta['g']) + (dv(prior) if prior is not None else 0.0)
        self._exact(key, dx[:ref.numel()].view(ref.shape), ref, 'dx')

    def _r_dwconv_wgrad(self, name, key, meta):
        n, h, w, c, k, r, s, p, q = meta['g'][:9]
        npix = n * p * q
        # the depthwise form of reduction_operands: channel 0 of x and of dy non-zero everywhere
        xs, ys = reduction_operands((n, h, w, c), (n, p, q, c), 1, 1, wgrad_density(npix, 1), self.g)
        ys[0][..., 0] = torch.where(torch.rand(n, p, q, generator=self.g, device=DEV) < 0.5, -1.0, 1.0)
        assert bool((xs[0][..., 0] != 0).all()) and bool((ys[0][..., 0] != 0).all()), key
        ws, dw = (_nan(meta['ws']) if meta['ws'] else None), _nan(meta['dw'])
        self.f[name](ops.conv_desc(*meta['g']), _fp32(meta['x'], xs[0]), _fp32(meta['dy'], ys[0]), ws, dw)
        self._variant(key, meta)
        ref = dw_wgrad_ref(dv(xs[0]), dv(ys[0]), meta['g'])
        self._bound(key, dw_wgrad_ref(dv(xs[0]).abs(), dv(ys[0]).abs(), meta['g']))
        self._tolerated(key, name, npix)
        self._exact(key, dw[:ref.numel()].view(ref.shape), ref, 'dw')

    # ---- other reductions
    def _r_bn_bwd(self, name, key, meta):
        """dbeta and dgamma of the BN backward at mean 0, rstd 1, gamma 1, beta 0: every fp32 step of
        ((x - mean) * rstd) * gamma + beta gives x, the mask is x > 0 (and x < 6 for ReLU6, none without activation),
        dbeta = sum of dy * mask and dgamma = sum of dy * mask * x, integers.  dx divides by m and is not compared."""
        m, c, act = meta['m'], meta['c'], meta['act']
        x = int_values((m, c), 0.5, self.g) + int_values((m, c), 0.25, self.g, signed=False)   # -1 .. 2
        dy = int_values((m, c), 0.5, self.g)
        # every row has an entry with x = 1 and dy = +-1 (column row % c): its term survives every mask
        col = (torch.arange(m, device=DEV) % c).view(m, 1)
        x.scatter_(1, col, torch.ones(m, 1, device=DEV))
        dy.scatter_(1, col, torch.where(torch.rand(m, 1, generator=self.g, device=DEV) < 0.5, -1.0, 1.0))
        zero, one = torch.zeros(c, device=DEV), torch.ones(c, device=DEV)
        dgamma, dbeta = _nan(c), _nan(c)
        dx = _fp32(meta['dx'], None) if meta['dx'] else None
        planes = ops.Planes(meta['planes'], DEV) if meta['planes'] else None
        self.f[name](dy, x, m, c, zero, one, one, zero, act, dgamma, dbeta, dx, meta['acc'], _nan(meta['ws']), planes)
        mask = torch.ones_like(x, dtype=torch.bool) if act == 0 else x > 0
        if act == 2:
            mask &= x < 6
        dz = dv(dy) * mask
        self._bound(key, dz.abs().sum(0) * 2)
        self._exact(key, dbeta, dz.sum(0), 'dbeta')
        self._exact(key, dgamma, (dz * dv(x)).sum(0), 'dgamma')

    def _r_fold_diag_blocks(self, name, key, meta):
        gg, m, n = meta['gmn']
        src = int_values((gg * m, gg * n), 0.5, self.g)
        dst = _nan(meta['dst'])
        self.f[name](_fp32(meta['src'], src), gg, m, n, dst)
        a = dv(src)
        ref = sum(a[b * m:(b + 1) * m, b * n:(b + 1) * n] for b in range(gg))
        self._exact(key, dst[:m * n].view(m, n), ref, 'folded blocks')

    def _r_colsum(self, name, key, meta):
        m, c = meta['mc']
        a = int_values((m, c), wgrad_density(m, 1) ** 2, self.g)
        # every row has a +-1 in column row % c: dropping or repeating any row changes that column's sum
        a.scatter_(1, (torch.arange(m, device=DEV) % c).view(m, 1),
                   torch.where(torch.rand(m, 1, generator=self.g, device=DEV) < 0.5, -1.0, 1.0))
        assert bool((a != 0).any(1).all()), key
        out = _nan(meta['out'])
        self.f[name](_fp32(meta['a'], a), m, c, out)
        self._bound(key, dv(a).abs().sum(0))
        self._exact(key, out[:c], dv(a).sum(0), 'column sums')

    def _r_l2_loss(self, name, key, meta):
        # every element a term up to 2^23 elements; a longer vector cannot be all non-zero below the exact bound
        v = int_values((meta['v'],), min(1.0, float(1 << 23) / meta['v']), self.g)
        if meta['v'] <= 1 << 23:
            assert bool((v != 0).all()), key
        out = _nan(meta['out'])
        prior = 3.0
        if meta['acc']:
            out[0] = prior
        self.f[name](v, 2.0, out, _nan(meta['ws']), meta['acc'])
        ref = (dv(v) ** 2).sum() + (prior if meta['acc'] else 0.0)
        self._bound(key, ref.view(1))
        self._exact(key, out[:1], ref.view(1), 'l2 loss at scale 2')

    def _r_cluster_grad(self, name, key, meta):
        srcs = [torch.zeros(s, device=DEV) for s in meta['shapes']]
        dsts = [torch.zeros_like(s) for s in srcs]
        base = torch.zeros(256 * len(srcs), device=DEV)
        views = [base[256 * i:256 * (i + 1)] for i in range(len(srcs))]
        q = ops.CodebookWeightQuantizer(srcs, dsts, list(meta['bits']), keep_index=True, cluster_views=views,
                                        cluster_base=base)
        q.uq.scales.fill_(1.0)                        # alpha = 1 in every scale the gradient reads
        grads, refs = [], []
        for i, (s, b) in enumerate(zip(srcs, meta['bits'])):
            gi = int_values(tuple(s.shape), 1.0, self.g)       # every element adds +-1 to its centroid
            assert bool((gi != 0).all()), key
            idx = torch.randint(0, 1 << b, (s.numel(),), generator=self.g, device=DEV)
            q.idx[q.idx_offsets[i]:q.idx_offsets[i] + s.numel()] = idx.to(torch.uint8)
            grads.append(gi)
            refs.append(torch.zeros(1 << b, dtype=torch.float64, device=DEV).index_add_(0, idx, dv(gi).reshape(-1)))
            self._bound(key, torch.zeros(1 << b, dtype=torch.float64, device=DEV).index_add_(
                0, idx, dv(gi).abs().reshape(-1)))
        gbase = _nan(base.numel())                  # the layout of this quantizer's cluster_base
        self.f[name](q, grads, gbase)
        for i, ref in enumerate(refs):
            o = int(q.cluster_off[i].item())
            self._exact(key, gbase[o:o + ref.numel()], ref, 'codebook gradient of tensor %d' % i)

    def _r_reduce(self, name, key, meta):
        items, refs = [], []
        for npart, nout, splits in meta['items']:
            part = int_values((npart,), 0.5, self.g)
            out = _nan(nout)
            items.append((part, out, splits))
            refs.append(dv(part[:splits * nout]).view(splits, nout).sum(0))
        self.f[name](ops.TcWgradReduceBatch(items, DEV))
        for (_, out, _), ref in zip(items, refs):
            self._exact(key, out, ref, 'split-K reduction')

    # ---- report
    def finish(self, label, secs, peak_gb):
        per = {}
        for key in self.rec.first:
            per[key[0]] = per.get(key[0], 0) + 1
        ncalls = sum(self.rec.calls.values())
        print('%s: %d calls, %d keys (%d replayed against float64, %d skipped); step %.0f s, peak %.1f GB; '
              'replay %.0f s, peak %.1f GB' % (self.rec.label, ncalls, len(self.rec.first), len(self.replayed),
                                               len(self.skipped), self.rec.secs, self.rec.peak, secs, peak_gb))
        print('  keys per entry point: %s' % ', '.join('%s %d' % kv for kv in sorted(per.items())))
        for key, npix in self.tolerated:
            print('  %s %s: the float bar tolerates %.1f pixels of terms' % (key[0], key[1:], npix))
        for key, why in self.skipped.items():
            print('  skipped %s %s: %s' % (key[0], key[1:], why))
        for f in self.fails:
            print('  NOT EXACT: %s' % (f,))
        # every entry point the step called is replayed here, skipped with a reason, listed in NOT_REPLAYED with one,
        # or checked by test_nn_bench_layers_gpu; a new entry point in the step fails here until it is placed
        others = self.rec.step_called - {k[0] for k in self.replayed} - {k[0] for k in self.skipped}
        for name in sorted(others & set(NOT_REPLAYED)):
            print('  not replayed: %s: %s' % (name, NOT_REPLAYED[name]))
        unknown = others - set(NOT_REPLAYED) - CHECKED_ELSEWHERE - set(TC_NAMES)
        assert not unknown, ('entry points the step calls that are neither replayed nor placed', sorted(unknown))
        unreplayed = [k for k in self.rec.calls if k not in self.replayed and k not in self.skipped]
        assert not unreplayed, ('calls of the wrapped entry points with no replayed key', unreplayed)
        assert not self.fails, self.fails[:20]
        assert self.replayed


def replay_and_check(rec, seed):
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    rep = Replay(rec, seed).run()
    torch.cuda.synchronize()
    rep.finish(rec.label, time.time() - t0, torch.cuda.max_memory_allocated() / 2 ** 30)
    return rep


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.gpu
def test_wgmma_accumulates_integers_exactly():
    """the precondition: bf16 wgmma with fp32 accumulation adds integer products exactly while every partial sum stays
    below 2^24.  pf_tc_probe at K = 256 with rows of 255 x 255 (sums of 16,646,400) and random levels; then one TMA
    weight gradient of all-ones x and dy over 255 x 256 x 256 = 16,711,680 pixels, where every dw entry must be Npix."""
    from pocketflow_b200 import lib as _lib
    L = _lib.load()
    g = torch.Generator(device=DEV).manual_seed(7)
    K, N = 256, 128
    A = torch.randint(0, 256, (128, K), generator=g, device=DEV).float()
    B = torch.randint(0, 256, (N, K), generator=g, device=DEV).float()
    A[:8], B[:8] = 255.0, 255.0                         # entries at 256 * 255^2, 2^24 - 130816
    A[8:16] = -255.0                                    # and their negatives
    Ab, Bb = A.to(torch.bfloat16).contiguous(), B.to(torch.bfloat16).contiguous()
    D = torch.full((128, N), float('nan'), device=DEV)
    assert L.pf_tc_probe(Ab.data_ptr(), Bb.data_ptr(), D.data_ptr(), N, K, 0, 16, 1024, 16, 1024, 32, 32, None) == 0
    torch.cuda.synchronize()
    ref = A.double() @ B.double().t()
    assert ref.abs().max().item() < EXACT_BOUND and ref.abs().max().item() > EXACT_BOUND - (1 << 18)
    assert torch.equal(D.double(), ref)

    n, h, w, c, k = 255, 256, 256, 64, 64
    npix = n * h * w
    assert npix < EXACT_BOUND
    d = ops.conv_desc(n, h, w, c, k, 1, 1, h, w, 1, 1, 0, 0)
    xp, yp = ops.Planes(npix * c, DEV), ops.Planes(npix * k, DEV)
    for pl in (xp, yp):
        pl.hi.fill_(1.0)
        pl.lo.zero_()
    ws = torch.empty(ops.conv2d_tc_wgrad_planes_workspace_floats(d), device=DEV)
    dw = torch.full((c * k,), float('nan'), device=DEV)
    ops.conv2d_tc_wgrad_planes(d, xp, yp, ws, dw)
    plan = ops.conv2d_tc_last_plan()
    torch.cuda.synchronize()
    print('all-ones wgrad over %d pixels: plan %s' % (npix, plan))
    assert plan['feed'] == 1 and plan['pass'] == 2
    assert torch.equal(dw, torch.full_like(dw, float(npix)))


def recorder_into(holder):
    def make(monkeypatch, lrn):
        holder.append(ExactRecorder(monkeypatch))
        return holder[-1]
    return make


@pytest.mark.gpu
@pytest.mark.parametrize('workload,batch,flags', [
    pytest.param(w, b, f, id='%s-%d' % (w, b) + ''.join('-%s' % v for _, v in sorted((f or {}).items())))
    for w, b, f in RUNS])
def test_bench_step_reductions_are_exact(workload, batch, flags, monkeypatch):
    holder = []
    run_workload(workload, batch, monkeypatch, recorder_into(holder), flags=flags, after=after_step(workload))
    replay_and_check(holder[0], zlib.crc32(('%s %d' % (workload, batch)).encode()) & 0xffff)


@pytest.mark.gpu
@pytest.mark.parametrize('net,learner', [('resnet50', 'chn-pruned-gpu'), ('mobilenet', 'chn-pruned-rmt')])
def test_compact_step_reductions_are_exact(net, learner, monkeypatch):
    """the compact fine-tune step as test_compact_train_gpu builds it: half of every interior kernel's input channels
    pruned, at batch 128"""
    from pocketflow_b200 import compact as C
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    mod, nflags = {'resnet50': ('resnet_at_ilsvrc12', dict(resnet_size=50)), 'mobilenet': ('mobilenet_at_ilsvrc12', {})}[net]
    lrn = make(mod, learner, 128, **dict(QUIET, nb_classes=1001, **nflags))
    prune_interior(lrn, 0.5, 3)
    ex = lrn.sess_train
    images, labels = lrn.iterator_train.next_batch()
    ex.buf[lrn.images].copy_(images)
    ex.buf[lrn.labels].copy_(labels)
    ct = C.CompactTrainer(ex)
    rec = ExactRecorder(monkeypatch)
    ct.ex.run_step(0.05)
    torch.cuda.synchronize()
    assert np.isfinite(ct.ex.fetch_losses()['loss'])
    rec.finish('%s %s compact fine-tune at batch 128' % (net, learner), time.time() - t0,
               torch.cuda.max_memory_allocated() / 2 ** 30)
    del lrn, ex, ct
    gc.collect()
    torch.cuda.empty_cache()
    rep = replay_and_check(rec, 11 if net == 'resnet50' else 13)
    if net == 'resnet50':
        assert any(k[0] == 'conv2d_wgrad' for k in rep.replayed), 'no compact convolution ran the CUDA-core wgrad'
