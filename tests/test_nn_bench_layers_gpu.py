"""The layers between the tensor-core convolutions, in one training step of the benchmarked workloads at the
benchmarked batch, against float64 or bit for bit.

The harness is test_tc_bench_layers_gpu.run_workload: the learner is built at the batch bench.py measures, under
PF_POISON=1, and one eager step runs with entry points of `ops` wrapped.  Each call passes through unchanged; then
  * its output must be finite;
  * the first call of each (entry point, geometry, form, flags) is compared on exactly the operands it was given, with
    "prior" outputs (accumulate targets, moving statistics, range slots) cloned before the call:
      - batch-norm statistics: mean within 1e-6 of |mean| + std, var 1e-5 relative, rstd within one ulp of
        fp32(1 / sqrt(fl(var + eps))), moving statistics 1e-6 of float64 from the prior (the mean at the scale
        |prior| momentum + (|mean| + std)(1 - momentum), and bit-exact as the fp32 chain of the batch mean), the range
        slot bit-exact;
      - BN apply, fake-quant, planes, levels and range slots: bit-exact against the fp32 op chain
        ((x - mean) * rstd) * gamma + beta and the quantizer's op chain (test_nn_variants_gpu);
      - BN backward: mask from that fp32 chain, dgamma / dbeta within 1e-6 of the sum of |terms| per channel, dx 1e-5
        of max|ref| on the fed fp32 statistics, planes == split(fp32 dx);
      - depthwise fwd / dgrad 1e-5 of max|ref|; wgrad against max|ref|, the sum of |terms| and an fp32 reference;
      - max-pool: y and argmax (first maximum) bit-exact, dx 1e-6; the rest float64 at 1e-5 or bit-exact.
The weight-sparse and codebook workloads also run what their learners do besides the step (run_workload's `after`):
      - mask rebuild: masks, weights (as uint32: -0.0 counts), backups and thresholds bit-exact against
        oracle.ws_build_mask at the ratios passed in;
      - codebook forward: quantized weights (and kept indices, ties to the first centroid) bit-exact against
        oracle.nonuniform_quantize with the device codebook; quantile init: every codebook bit-exact against
        oracle.nuq_quantile_init of the normalised tensor, entries past 2^bits zero; order statistics (pf_select_desc)
        bit-exact against a sort; codebook gradient within 1e-6 of each centroid's sum of |terms| of float64
        oracle.nuq_grads, and the same bits on a second call.
      Each of them must cover every tensor its object holds.
Every public callable of `ops` is wrapped: the test fails when the step calls one that is neither a tensor-core entry
point (test_tc_bench_layers_gpu), nor checked here, nor in EXEMPT with its reason."""
import os
import sys
from fractions import Fraction

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import pf_oracle as O  # noqa: E402
from pocketflow_b200 import ops  # noqa: E402
from test_nn_variants_gpu import bn_chain, fq_chain, pool_dx_ref, pool_ref, split_planes  # noqa: E402
from test_tc_bench_layers_gpu import Recorder as TcRecorder, after_step, conv64, geom, run_workload  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')

# called by the step and not compared, and why: host-side helpers, and steps of an entry point checked as a whole
EXEMPT = {
    'conv_desc': 'host-side descriptor',
    'Planes': 'host-side buffer holder',
    'tc_act': 'host-side operand descriptor',
    'tc_wt': 'host-side operand descriptor',
    'conv2d_tc_wgrad_splits': 'host-side query',
    'conv2d_tc_last_plan': 'host-side query',
    'dwconv_last_variant': 'host-side query',
    'conv2d_tc_supported': 'host-side query',
    'conv2d_tc_wgrad_supported': 'host-side query',
    'conv2d_tc_tma_supported': 'host-side query',
    'conv2d_tc_set_feed': 'host-side switch',
    'conv2d_wgrad_workspace_floats': 'host-side query',
    'conv2d_tc_wgrad_workspace_floats': 'host-side query',
    'conv2d_tc_wgrad_planes_workspace_floats': 'host-side query',
    'dwconv_wgrad_workspace_floats': 'host-side query',
    'decode_ordered': 'host-side decoding',
    'flat_works': 'host-side work table',
    'percentile_rank_desc': 'host-side rank arithmetic',
    'ws_rank_desc': 'host-side rank arithmetic',
    'UniformWeightQuantizer.ranges': 'host-side copy of the range slots',
    'minmax_reset': 'fills the range slots with the empty range; every slot it resets is checked where it is consumed',
    'launch_count': 'host-side counter',
    'launch_count_reset': 'host-side counter',
    'UniformWeightQuantizer.reset_ranges': 'part of UniformWeightQuantizer.forward, whose output is checked',
    'UniformWeightQuantizer.minmax': 'part of UniformWeightQuantizer.forward and of the codebook forward and '
                                     'quantile init, whose outputs are checked',
    'UniformWeightQuantizer.quantize': 'part of UniformWeightQuantizer.forward, whose output is checked',
}
CLASSES = ('UniformWeightQuantizer', 'CodebookWeightQuantizer', 'MaskBuilder', 'TcWeights', 'TcWeightsBatch',
           'TcWgradReduceBatch')


def enc(v):
    """ordered-uint encoding of fp32 values (the range slots; inverse of ops.decode_ordered)"""
    u = np.asarray(v, np.float32).view(np.uint32)
    return np.where(u & 0x80000000, ~u, u | 0x80000000).astype(np.uint32)


def slot_after(prior, y):
    """the range slot [min, max] after folding y's range into `prior` (int32[2] as uint32)"""
    p = prior.cpu().numpy().view(np.uint32)
    lo, hi = enc([y.min().item(), y.max().item()])
    return np.array([min(p[0], lo), max(p[1], hi)], np.uint32)


def rsqrt_rn(v):
    """correctly rounded fp32 1 / sqrt(v) of a positive fp32 tensor (what __frsqrt_rn returns): the float64 estimate,
    then the neighbour whose rounding interval holds 1 / sqrt(v), decided exactly with rationals"""
    r = (1.0 / torch.sqrt(v.double())).float().cpu().numpy()
    vs = v.cpu().numpy()
    out = r.copy()
    up, dn = np.float32(np.inf), np.float32(0)
    for i, (ri, vi) in enumerate(zip(r.reshape(-1), vs.reshape(-1))):
        fv = Fraction(float(vi))
        for c in (ri, np.nextafter(ri, dn), np.nextafter(ri, up)):
            # t = 1 / sqrt(v) rounds to c iff mid(c-, c) <= t <= mid(c, c+), i.e. mid^2 * v <= 1 <= mid'^2 * v
            fc = Fraction(float(c))
            lo, hi = (Fraction(float(np.nextafter(c, dn))) + fc) / 2, (fc + Fraction(float(np.nextafter(c, up)))) / 2
            if lo * lo * fv <= 1 <= hi * hi * fv:
                out.reshape(-1)[i] = c
                break
        else:
            raise AssertionError('no correctly rounded rsqrt found for %r' % vi)
    return torch.from_numpy(out).to(v.device)


def relerr(got, ref, scale=None):
    assert torch.isfinite(got).all(), 'non-finite output'
    s = ref.abs().max() if scale is None else scale
    return ((got.double() - ref).abs().max() / s).item()


class NnRecorder:
    """wraps every public callable of `ops`; see the module docstring"""

    def __init__(self, monkeypatch, expect=None):
        """expect: {check tag: tensors it must cover, or None where the tag only has to appear}"""
        self.checked, self.worst, self.calls, self.called, self.fail = set(), {}, 0, set(), []
        self.wgrad_notes = []
        self.oracle_done, self.quant_seen = False, False
        self.expect, self.covered, self._codebooks = dict(expect or {}), {}, {}
        for name in dir(ops):
            obj = getattr(ops, name)
            if name.startswith('_') or isinstance(obj, type) or not callable(obj) or \
                    getattr(obj, '__module__', None) != ops.__name__:
                continue
            check = getattr(self, '_c_' + name, None)
            monkeypatch.setattr(ops, name, self._wrap(name, obj, check))
        for cname in CLASSES:
            cls = getattr(ops, cname)
            for mname, fn in list(vars(cls).items()):
                if not mname.startswith('_') and callable(fn):
                    check = getattr(self, '_m_%s_%s' % (cname, mname), None)
                    monkeypatch.setattr(cls, mname, self._wrap('%s.%s' % (cname, mname), fn, check))

    def _wrap(self, name, fn, check):
        def call(*args, **kw):
            self.called.add(name)
            if check is None:
                return fn(*args, **kw)
            self.calls += 1
            return check(fn, *args, **kw)
        return call

    def _first(self, key):
        if key in self.checked:
            return False
        self.checked.add(key)
        return True

    def _note(self, tag, err, bar):
        self.worst[tag] = max(self.worst.get(tag, 0.0), err)
        if not err <= bar:
            self.fail.append((tag, err, bar))

    def _exact(self, tag, ok, where=None):
        self.worst.setdefault(tag, 0.0)
        if not ok:
            self.fail.append((tag, 'not bit-exact', where))

    def _per_tensor(self, results):
        """results: {tag: [bit-exact per tensor]}; one entry per tag, naming the tensors that differ"""
        for tag, oks in results.items():
            bad = [i for i, ok in enumerate(oks) if not ok]
            self._exact(tag, not bad, 'tensors %s of %d' % (bad, len(oks)) if bad else None)

    # ---------------------------------------------------------------------------------------------- batch-norm
    def _stats(self, fn, name, x, m, c, eps, mom, mean, var, rstd, mm, mv, gamma=None, beta=None, act=0, slot=None,
               ws=None):
        key = (name, m, c, act, mm is not None)
        first = self._first(key)
        prior = (mm.clone(), mv.clone()) if (first and mm is not None) else None
        pslot = slot.clone() if (first and slot is not None) else None
        if name == 'bn_train_stats':
            fn(x, m, c, eps, mom, mean, var, rstd, mm, mv, ws)
        else:
            fn(x, m, c, eps, mom, mean, var, rstd, mm, mv, gamma, beta, act, slot, ws)
        torch.cuda.synchronize()
        assert torch.isfinite(mean).all() and torch.isfinite(var).all() and torch.isfinite(rstd).all(), key
        if not first:
            return
        xd = x.reshape(-1)[:m * c].view(m, c).double()
        m64, v64 = xd.mean(0), xd.var(0, unbiased=False)
        self._note('bn stats mean', ((mean.double() - m64).abs() / (m64.abs() + v64.sqrt()).clamp_min(1e-30)).max().item(),
                   1e-6)
        self._note('bn stats var', ((var.double() - v64).abs() / v64.clamp_min(1e-30)).max().item(), 1e-5)
        r64 = 1.0 / torch.sqrt((var + eps).double())
        r32 = r64.float()
        ulp = (torch.nextafter(r32, torch.full_like(r32, float('inf'))) - r32).double()
        self._exact('bn stats rstd (1 ulp)', bool(((rstd.double() - r64).abs() <= ulp).all()))
        if prior is not None:
            # moving mean: the fp32 op chain of the batch mean it was given (checked above), bit for bit; and against
            # float64 per channel at the mean's own scale carried through the update, |prior| mom + (|mean| + std) om
            # (a bar of max|moving mean| fails where every batch mean is small beside its std: ResNet-20 at batch 256)
            mo, om32 = np.float32(mom), np.float32(1) - np.float32(mom)
            self._exact('bn stats moving mean (fp32 chain)',
                        np.array_equal(mm.cpu().numpy(), prior[0].cpu().numpy() * mo + mean.cpu().numpy() * om32))
            om = 1.0 - float(mo)
            scale = prior[0].double().abs() * float(mo) + (m64.abs() + v64.sqrt()) * om
            e = max(((mm.double() - (prior[0].double() * float(mo) + m64 * om)).abs() / scale.clamp_min(1e-30)).max()
                    .item(), relerr(mv, prior[1].double() * float(mo) + xd.var(0, unbiased=True) * om))
            self._note('bn stats moving', e, 1e-6)
        if pslot is not None:
            y = bn_chain(x.reshape(-1)[:m * c].view(m, c), mean, rstd, gamma, beta, act)
            self._exact('bn stats range slot', np.array_equal(slot.cpu().numpy().view(np.uint32), slot_after(pslot, y)))

    def _c_bn_train_stats(self, fn, *a):
        self._stats(fn, 'bn_train_stats', *a[:10], ws=a[10])

    def _c_bn_train_stats_range(self, fn, *a):
        self._stats(fn, 'bn_train_stats_range', *a)

    def _apply_check(self, tag, y_ref, y, planes, slot, pslot):
        if y is not None:
            self._exact(tag + ' y', torch.equal(y.reshape(-1)[:y_ref.numel()], y_ref.reshape(-1)))
        if planes is not None:
            h, l = split_planes(y_ref)
            self._exact(tag + ' planes', torch.equal(planes.hi[:h.numel()], h) and torch.equal(planes.lo[:l.numel()], l))
        if pslot is not None:
            self._exact(tag + ' range slot', np.array_equal(slot.cpu().numpy().view(np.uint32), slot_after(pslot, y_ref)))

    def _c_bn_apply(self, fn, x, m, c, mean, rstd, gamma, beta, act, y, minmax=None, planes=None):
        key = ('bn_apply', m, c, act, y is not None, minmax is not None, planes is not None)
        first = self._first(key)
        pslot = minmax.clone() if (first and minmax is not None) else None
        fn(x, m, c, mean, rstd, gamma, beta, act, y, minmax, planes)
        self._finite(y, planes, m * c, key)
        if first:
            y_ref = bn_chain(x.reshape(-1)[:m * c].view(m, c), mean, rstd, gamma, beta, act)
            self._apply_check('bn_apply', y_ref, y, planes, minmax, pslot)

    def _c_bn_apply_eval(self, fn, x, m, c, mm, mv, eps, gamma, beta, act, y, minmax=None, planes=None):
        key = ('bn_apply_eval', m, c, act, y is not None, minmax is not None, planes is not None)
        first = self._first(key)
        pslot = minmax.clone() if (first and minmax is not None) else None
        fn(x, m, c, mm, mv, eps, gamma, beta, act, y, minmax, planes)
        self._finite(y, planes, m * c, key)
        if first:
            rstd = rsqrt_rn(mv + eps)
            y_ref = bn_chain(x.reshape(-1)[:m * c].view(m, c), mm, rstd, gamma, beta, act)
            self._apply_check('bn_apply_eval', y_ref, y, planes, minmax, pslot)

    def _c_bn_apply_quant(self, fn, x, m, c, mean, rstd, gamma, beta, act, rng, bits, y=None, planes=None):
        key = ('bn_apply_quant', m, c, act, bits, y is not None, planes is not None)
        fn(x, m, c, mean, rstd, gamma, beta, act, rng, bits, y, planes)
        self._finite(y, planes, m * c, key)
        if self._first(key):
            q_ref = self._fq(bn_chain(x.reshape(-1)[:m * c].view(m, c), mean, rstd, gamma, beta, act), rng, bits)[0]
            self._apply_check('bn_apply_quant', q_ref, y, planes, None, None)

    def _c_bn_apply_quant_levels(self, fn, x, m, c, mean, rstd, gamma, beta, act, rng, bits, y, planes, hdr, csum):
        key = ('bn_apply_quant_levels', m, c, act, bits, y is not None)
        fn(x, m, c, mean, rstd, gamma, beta, act, rng, bits, y, planes, hdr, csum)
        torch.cuda.synchronize()
        if not self._first(key):
            return
        yb = bn_chain(x.reshape(-1)[:m * c].view(m, c), mean, rstd, gamma, beta, act)
        q_ref, lv = self._fq(yb, rng, bits)
        hd = hdr.cpu().numpy().view(ops.ACT_HDR)[0]
        nseg = -(-c // 128)
        if y is not None:
            self._exact('bn_apply_quant_levels y', torch.equal(y.reshape(-1)[:m * c], q_ref.reshape(-1)))
        mn = ops.decode_ordered(rng.cpu().numpy().view(np.uint32))[0]
        if int(hd['nplanes']) == 1:
            self._exact('bn_apply_quant_levels header', mn == 0.0 and bits <= 8)
            self._exact('bn_apply_quant_levels levels', torch.equal(planes.hi[:m * c].float(), lv.reshape(-1)) and
                        bool(((lv >= 0) & (lv <= float(2 ** bits - 1))).all()))
            e = ((lv.double() * float(hd['scale']) - q_ref.double()).abs().max()).item()
            self._note('bn_apply_quant_levels scale x level - fq', e, 3e-7 * max(1.0, q_ref.abs().max().item()))
            cs = lv.double().view(m, nseg, min(c, 128)).sum(-1).reshape(-1)
            self._exact('bn_apply_quant_levels csum', torch.equal(csum[:m * nseg].double(), cs))
        else:
            self._exact('bn_apply_quant_levels header', float(hd['scale']) == 1.0 and int(hd['nplanes']) == 2)
            self._apply_check('bn_apply_quant_levels', q_ref, None, planes, None, None)
            qs = q_ref.double().view(m, nseg, min(c, 128))
            e = ((csum[:m * nseg].double() - qs.sum(-1).reshape(-1)).abs() /
                 qs.abs().sum(-1).reshape(-1).clamp_min(1e-30)).max().item()
            self._note('bn_apply_quant_levels csum / sum|terms|', e, 1e-6)

    def _c_act_quant(self, fn, x, y, minmax, bits, planes=None):
        key = ('act_quant', x.numel(), bits, y is not None, planes is not None)
        fn(x, y, minmax, bits, planes)
        self._finite(y, planes, x.numel(), key)
        if self._first(key):
            self._apply_check('act_quant', self._fq(x, minmax, bits)[0], y, planes, None, None)

    def _c_act_minmax(self, fn, x, minmax):
        key = ('act_minmax', x.numel())
        first = self._first(key)
        pslot = minmax.clone() if first else None
        fn(x, minmax)
        if first:
            torch.cuda.synchronize()
            self._apply_check('act_minmax', x, None, None, minmax, pslot)

    def _fq(self, y, rng, bits):
        """fake-quant reference of y with the range slot `rng`; the first tensor of up to 16 M elements whose range is
        exactly its own also goes through the numpy oracle (oracle/pf_oracle.uniform_quantize)"""
        self.quant_seen = True
        mn, mx = ops.decode_ordered(rng.cpu().numpy().view(np.uint32))[:2]
        q, lv = fq_chain(y, torch.tensor(mn, device=y.device), torch.tensor(mx, device=y.device), bits)
        if not self.oracle_done and y.numel() <= 1 << 24 and y.min().item() == mn and y.max().item() == mx:
            ref = O.uniform_quantize(y.cpu().numpy(), bits, mode='activation')
            self._exact('numpy oracle (one activation tensor)', np.array_equal(q.cpu().numpy(), ref))
            self.oracle_done = True
        return q, lv

    def _c_bn_bwd(self, fn, dy, x, m, c, mean, rstd, gamma, beta, act, dgamma, dbeta, dx, acc, ws, planes=None):
        key = ('bn_bwd', m, c, act, bool(acc), dx is not None, planes is not None)
        first = self._first(key)
        prior = dx.clone() if (first and acc) else None
        fn(dy, x, m, c, mean, rstd, gamma, beta, act, dgamma, dbeta, dx, acc, ws, planes)
        self._finite(dx, planes, m * c, key)
        if not first:
            return
        xv, dyv = x.reshape(-1)[:m * c].view(m, c), dy.reshape(-1)[:m * c].view(m, c)
        z = ((xv - mean) * rstd) * gamma + beta
        mask = torch.ones_like(z, dtype=torch.bool) if act == 0 else z > 0
        if act == 2:
            mask &= z < 6
        del z
        xh = (xv.double() - mean.double()) * rstd.double()
        dz = dyv.double() * mask
        del mask
        db, dg = dz.sum(0), (dz * xh).sum(0)
        self._note('bn_bwd dbeta / sum|terms|', ((dbeta.double() - db).abs() / dz.abs().sum(0).clamp_min(1e-30)).max().item(), 1e-6)
        self._note('bn_bwd dgamma / sum|terms|', ((dgamma.double() - dg).abs() / (dz * xh).abs().sum(0).clamp_min(1e-30)).max().item(), 1e-6)
        ref = gamma.double() * rstd.double() * (dz - db / m - xh * dg / m)
        del dz, xh
        if prior is not None:
            ref += prior.reshape(-1)[:m * c].view(m, c).double()
        if dx is None:          # planes only: the same launch into an fp32 target, then planes == split(fp32)
            dx = torch.empty(m * c, device=DEV)
            fn(dy, x, m, c, mean, rstd, gamma, beta, act, torch.empty_like(dgamma), torch.empty_like(dbeta), dx, False,
               ws, None)
        else:
            dx = dx.reshape(-1)[:m * c]
        self._note('bn_bwd dx', relerr(dx.view(m, c), ref), 1e-5)
        if planes is not None:
            h, l = split_planes(dx)
            self._exact('bn_bwd planes', torch.equal(planes.hi[:m * c], h) and torch.equal(planes.lo[:m * c], l))

    # ---------------------------------------------------------------------------------------------- depthwise
    @staticmethod
    def _dw64(x, w, d):
        n, h, wd, c, k, r, s, p, q, sh, sw, pt, pl = geom(d)
        pb, pr = (p - 1) * sh + r - h - pt, (q - 1) * sw + s - wd - pl
        return F.conv2d(F.pad(x.permute(0, 3, 1, 2), (pl, pr, pt, pb)), w.reshape(r, s, c, 1).permute(2, 3, 0, 1),
                        stride=(sh, sw), groups=c).permute(0, 2, 3, 1)

    def _c_dwconv_fwd(self, fn, d, x, w, y):
        key = ('dwconv_fwd', geom(d))
        fn(d, x, w, y)
        self._finite(y, None, y.numel(), key)
        if self._first(key):
            n, h, wd, c = geom(d)[:4]
            ref = self._dw64(x.reshape(-1)[:n * h * wd * c].view(n, h, wd, c).double(), w.double(), d)
            self._note('dwconv fwd', relerr(y.reshape(-1)[:ref.numel()].view(ref.shape), ref), 1e-5)

    def _c_dwconv_dgrad(self, fn, d, dy, w, acc, dx):
        key = ('dwconv_dgrad', geom(d), bool(acc))
        first = self._first(key)
        prior = dx.clone() if (first and acc) else None
        fn(d, dy, w, acc, dx)
        self._finite(dx, None, dx.numel(), key)
        if first:
            n, h, wd, c, k, r, s, p, q = geom(d)[:9]
            xg = torch.zeros(n, h, wd, c, dtype=torch.float64, device=DEV, requires_grad=True)
            self._dw64(xg, w.double(), d).backward(dy.reshape(-1)[:n * p * q * c].view(n, p, q, c).double())
            ref = xg.grad + (prior.reshape(-1)[:xg.numel()].view(xg.shape).double() if acc else 0.0)
            self._note('dwconv dgrad' + (' acc' if acc else ''), relerr(dx.reshape(-1)[:ref.numel()].view(ref.shape), ref),
                       1e-5)

    def _c_dwconv_wgrad(self, fn, d, x, dy, ws, dw):
        key = ('dwconv_wgrad', geom(d))
        fn(d, x, dy, ws, dw)
        self._finite(dw, None, dw.numel(), key)
        if not self._first(key):
            return
        n, h, wd, c, k, r, s, p, q = geom(d)[:9]
        xv = x.reshape(-1)[:n * h * wd * c].view(n, h, wd, c)
        dyv = dy.reshape(-1)[:n * p * q * c].view(n, p, q, c)
        out = []
        for dt, absolute in ((torch.float64, False), (torch.float64, True), (torch.float32, False)):
            wg = torch.zeros(r, s, c, dtype=dt, device=DEV, requires_grad=True)
            a, b = (xv.abs(), dyv.abs()) if absolute else (xv, dyv)
            tf32 = torch.backends.cudnn.allow_tf32
            torch.backends.cudnn.allow_tf32 = False           # the fp32 reference: exact fp32 products
            try:
                self._dw64(a.to(dt), wg, d).backward(b.to(dt))
            finally:
                torch.backends.cudnn.allow_tf32 = tf32
            out.append(wg.grad.double())
        ref, mag, ref32 = out
        got = dw.reshape(-1)[:ref.numel()].view(ref.shape)
        err, errm, err32 = relerr(got, ref), relerr(got, ref, mag.abs().max()), relerr(ref32, ref)
        self.wgrad_notes.append((geom(d), err, errm, err32))
        self.worst['dwconv wgrad / sum|terms|'] = max(self.worst.get('dwconv wgrad / sum|terms|', 0.0), errm)
        self._note('dwconv wgrad', err, 1e-5)

    # ---------------------------------------------------------------------------------------------- pooling
    def _c_maxpool_fwd(self, fn, d, x, y, argmax=None):
        key = ('maxpool_fwd', geom(d), argmax is not None)
        fn(d, x, y, argmax)
        self._finite(y, None, y.numel(), key)
        if self._first(key):
            n, h, wd, c, k, r, s, p, q, sh, sw, pt, pl = geom(d)
            assert r == s and sh == sw and pt == pl and h == wd
            pb = (p - 1) * sh + r - h - pt
            y_ref, am_ref = pool_ref(x.reshape(-1)[:n * h * wd * c].view(n, h, wd, c), r, sh, pt, pb, p, q)[:2]
            self._exact('maxpool y', torch.equal(y.reshape(-1)[:y_ref.numel()].view(y_ref.shape), y_ref))
            if argmax is not None:
                self._exact('maxpool argmax', torch.equal(argmax.reshape(-1)[:y_ref.numel()].view(y_ref.shape).long(),
                                                          am_ref.long()))

    def _c_maxpool_bwd(self, fn, d, dy, argmax, dx, acc=False):
        key = ('maxpool_bwd', geom(d), bool(acc))
        first = self._first(key)
        prior = dx.clone() if (first and acc) else None
        fn(d, dy, argmax, dx, acc)
        self._finite(dx, None, dx.numel(), key)
        if first:
            n, h, wd, c, k, r, s, p, q, sh, sw, pt, pl = geom(d)
            pb = (p - 1) * sh + r - h - pt
            am = argmax.reshape(-1)[:n * p * q * c].view(n, p, q, c).long()
            hp = h + pt + max(pb, 0)
            ref = pool_dx_ref(dy.reshape(-1)[:n * p * q * c].view(n, p, q, c), am, r, sh, pt, p, q, n, h, wd, c, hp, hp)
            if acc:
                ref = ref + prior.reshape(-1)[:ref.numel()].view(ref.shape).double()
            self._note('maxpool dx', relerr(dx.reshape(-1)[:ref.numel()].view(ref.shape), ref), 1e-6)

    def _c_global_avgpool_fwd(self, fn, x, n, hw, c, y):
        key = ('global_avgpool_fwd', n, hw, c)
        fn(x, n, hw, c, y)
        self._finite(y, None, n * c, key)
        if self._first(key):
            ref = x.reshape(-1)[:n * hw * c].view(n, hw, c).double().mean(1)
            self._note('global_avgpool fwd', relerr(y.reshape(-1)[:n * c].view(n, c), ref), 1e-5)

    def _c_global_avgpool_bwd(self, fn, dy, n, hw, c, dx, acc=False):
        key = ('global_avgpool_bwd', n, hw, c, bool(acc))
        first = self._first(key)
        prior = dx.clone() if (first and acc) else None
        fn(dy, n, hw, c, dx, acc)
        self._finite(dx, None, n * hw * c, key)
        if first:
            ref = (dy.reshape(-1)[:n * c].view(n, 1, c).double() / hw).expand(n, hw, c)
            if acc:
                ref = ref + prior.reshape(-1)[:n * hw * c].view(n, hw, c).double()
            self._note('global_avgpool bwd', relerr(dx.reshape(-1)[:n * hw * c].view(n, hw, c), ref), 1e-5)

    # ---------------------------------------------------------------------------------------------- the rest
    def _c_softmax_fwd(self, fn, x, y):
        fn(x, y)
        self._finite(y, None, y.numel(), 'softmax_fwd')
        if self._first(('softmax_fwd', tuple(x.shape))):
            self._note('softmax fwd', relerr(y, torch.softmax(x.double(), -1)), 1e-5)

    def _c_softmax_bwd(self, fn, dy, y, dx):
        fn(dy, y, dx)
        self._finite(dx, None, dx.numel(), 'softmax_bwd')
        if self._first(('softmax_bwd', tuple(y.shape))):
            yd, dyd = y.double(), dy.double()
            terms = dyd * yd
            ref = (dyd - terms.sum(-1, keepdim=True)) * yd
            mag = ((dyd.abs() + terms.abs().sum(-1, keepdim=True)) * yd.abs()).max()
            self._note('softmax bwd / sum|terms|', relerr(dx, ref, mag), 1e-5)

    def _c_add(self, fn, a, b, out, accumulate=False):
        key = ('add', a.numel(), b is not None, bool(accumulate))
        first = self._first(key)
        prior = out.clone() if (first and accumulate) else None
        fn(a, b, out, accumulate)
        self._finite(out, None, a.numel(), key)
        if first:
            ref = a if b is None else a + b.reshape(-1)[:a.numel()].view(a.shape)
            if accumulate:
                ref = ref + prior.reshape(-1)[:a.numel()].view(a.shape)
            self._exact('add', torch.equal(out.reshape(-1)[:a.numel()], ref.reshape(-1)))

    def _c_relu_bwd(self, fn, dy, y, dx, act=1, accumulate=False):
        key = ('relu_bwd', y.numel(), act, bool(accumulate))
        first = self._first(key)
        prior = dx.clone() if (first and accumulate) else None
        fn(dy, y, dx, act, accumulate)
        self._finite(dx, None, y.numel(), key)
        if first:
            mask = (y > 0) & ((y < 6) if act == 2 else torch.ones_like(y, dtype=torch.bool))
            ref = torch.where(mask, dy.reshape(-1)[:y.numel()].view(y.shape), torch.zeros_like(y))
            if accumulate:
                ref = prior.reshape(-1)[:y.numel()].view(y.shape) + ref
            self._exact('relu_bwd', torch.equal(dx.reshape(-1)[:y.numel()], ref.reshape(-1)))

    def _c_split_bf16(self, fn, src, planes):
        fn(src, planes)
        if self._first(('split_bf16', src.numel())):
            torch.cuda.synchronize()
            h, l = split_planes(src)
            self._exact('split_bf16', torch.equal(planes.hi[:h.numel()], h) and torch.equal(planes.lo[:l.numel()], l))

    def _c_mul(self, fn, a, b, out):
        fn(a, b, out)
        if self._first(('mul', a.numel())):
            torch.cuda.synchronize()
            self._exact('mul', torch.equal(out.reshape(-1)[:a.numel()], (a * b).reshape(-1)))

    def _c_colsum(self, fn, a, m, c, out):
        fn(a, m, c, out)
        self._finite(out, None, c, 'colsum')
        if self._first(('colsum', m, c)):
            av = a.reshape(-1)[:m * c].view(m, c).double()
            self._note('colsum / sum|terms|', relerr(out.reshape(-1)[:c], av.sum(0), av.abs().sum(0).max()), 1e-5)

    def _c_conv2d_fwd(self, fn, d, x, w, bias, relu, y):
        key = ('conv2d_fwd', geom(d), bias is not None, bool(relu))
        fn(d, x, w, bias, relu, y)
        self._finite(y, None, y.numel(), key)
        if self._first(key):
            n, h, wd, c, k, r, s, p, q = geom(d)[:9]
            ref = conv64(x.reshape(-1)[:n * h * wd * c].view(n, h, wd, c).double(), w.double().view(r, s, c, k), d)
            if bias is not None:
                ref = ref + bias.double()
            if relu:
                ref = torch.relu(ref)
            self._note('conv2d fp32 fwd', relerr(y.reshape(-1)[:ref.numel()].view(ref.shape), ref), 1e-5)

    def _c_conv2d_dgrad(self, fn, d, dy, w, wt_ws, acc, dx):
        key = ('conv2d_dgrad', geom(d), bool(acc))
        first = self._first(key)
        prior = dx.clone() if (first and acc) else None
        fn(d, dy, w, wt_ws, acc, dx)
        self._finite(dx, None, dx.numel(), key)
        if first:
            n, h, wd, c, k, r, s, p, q = geom(d)[:9]
            xg = torch.zeros(n, h, wd, c, dtype=torch.float64, device=DEV, requires_grad=True)
            conv64(xg, w.double().view(r, s, c, k), d).backward(dy.reshape(-1)[:n * p * q * k].view(n, p, q, k).double())
            ref = xg.grad + (prior.reshape(-1)[:xg.numel()].view(xg.shape).double() if acc else 0.0)
            self._note('conv2d fp32 dgrad', relerr(dx.reshape(-1)[:ref.numel()].view(ref.shape), ref), 1e-5)

    def _c_conv2d_wgrad(self, fn, d, x, dy, ws, dw):
        key = ('conv2d_wgrad', geom(d))
        fn(d, x, dy, ws, dw)
        self._finite(dw, None, dw.numel(), key)
        if self._first(key):
            n, h, wd, c, k, r, s, p, q = geom(d)[:9]
            xv, dyv = x.reshape(-1)[:n * h * wd * c].view(n, h, wd, c), dy.reshape(-1)[:n * p * q * k].view(n, p, q, k)
            refs = []
            for a, b in ((xv, dyv), (xv.abs(), dyv.abs())):
                wg = torch.zeros(r, s, c, k, dtype=torch.float64, device=DEV, requires_grad=True)
                conv64(a.double(), wg, d).backward(b.double())
                refs.append(wg.grad)
            got = dw.reshape(-1)[:refs[0].numel()].view(refs[0].shape)
            self._note('conv2d fp32 wgrad', relerr(got, refs[0]), 1e-5)
            self._note('conv2d fp32 wgrad / sum|terms|', relerr(got, refs[0], refs[1].abs().max()), 1e-5)

    # ---------------------------------------------------------------------------------------------- losses
    def _c_softmax_ce(self, fn, logits, labels, teacher=None, tempr=4.0, w_dst=4.0, dlogits=None, out=None,
                      row_ws=None):
        res = fn(logits, labels, teacher, tempr, w_dst, dlogits, out, row_ws)
        o, dl = res
        self._finite(dl, None, dl.numel(), 'softmax_ce')
        if self._first(('softmax_ce', tuple(logits.shape), teacher is not None)):
            n = logits.shape[0]
            s, lab = logits.double(), labels.double()
            ls = torch.log_softmax(s, -1)
            hard = -(lab * ls).sum(-1).mean()
            g = (torch.softmax(s, -1) - lab) / n
            got = o.cpu().double()
            self._note('softmax_ce hard loss', abs(got[0].item() - hard.item()) / abs(hard.item()), 1e-5)
            if teacher is not None:
                T = float(np.float32(tempr))
                soft = torch.softmax(teacher.double() / T, -1)
                dst = float(np.float32(w_dst)) * -(soft * torch.log_softmax(s / T, -1)).sum(-1).mean()
                self._note('softmax_ce distillation loss', abs(got[1].item() - dst.item()) / abs(dst.item()), 1e-5)
                g = g + float(np.float32(w_dst)) * (torch.softmax(s / T, -1) - soft) / (n * T)
            self._note('softmax_ce dlogits', relerr(dl, g), 1e-5)
            ln, sn = labels.cpu().numpy(), logits.cpu().numpy()
            self._exact('softmax_ce top-1', got[2].item() == float(O.accuracy(ln, sn)))
            top5 = np.mean([(np.sum(sn[i] > sn[i, np.argmax(ln[i])]) < 5) for i in range(n)])
            self._note('softmax_ce top-5', abs(got[3].item() - top5), 1e-6)
        return res

    def _c_l2_loss(self, fn, v, scale, out, partial_ws, accumulate=False):
        key = ('l2_loss', v.numel(), bool(accumulate))
        first = self._first(key)
        prior = out[:1].clone() if first else None
        fn(v, scale, out, partial_ws, accumulate)
        if first:
            vd = v.double()
            ref = float(np.float32(scale)) * (vd * vd).sum() / 2 + (prior.double()[0] if accumulate else 0.0)
            self._note('l2_loss', abs(out[0].item() - ref.item()) / abs(ref.item()), 1e-5)

    # ---------------------------------------------------------------------------------------------- optimizers
    def _c_momentum_step(self, fn, w, acc, g, mask, hp, momentum, wd=0.0, grad_scale=1.0):
        key = ('momentum_step', w.numel(), mask is not None)
        first = self._first(key)
        if first:
            torch.cuda.synchronize()
            w0, a0, g0 = w.cpu().numpy(), acc.cpu().numpy(), g.cpu().numpy()
            m0 = mask.cpu().numpy() if mask is not None else None
            lr = float(hp[0].item())
        fn(w, acc, g, mask, hp, momentum, wd, grad_scale)
        if first:
            rw, ra = O.momentum_step(w0, a0, g0, lr, momentum, mask=m0, wd=wd, grad_scale=grad_scale)
            self._exact('momentum_step', np.array_equal(w.cpu().numpy(), rw) and np.array_equal(acc.cpu().numpy(), ra))

    def _c_adam_step(self, fn, w, m, v, g, hp, beta1=0.9, beta2=0.999, eps=1e-8, wd=0.0, grad_scale=1.0):
        key = ('adam_step', w.numel())
        first = self._first(key)
        if first:
            torch.cuda.synchronize()
            w0, m0, v0, g0 = (t.cpu().numpy() for t in (w, m, v, g))
            lr, b1p, b2p = (np.float32(x) for x in hp[:3].cpu().numpy())
        fn(w, m, v, g, hp, beta1, beta2, eps, wd, grad_scale)
        if first:
            rw, rm, rv = O.adam_step(w0, m0, v0, g0, lr, b1p, b2p, beta1, beta2, eps, wd=wd, grad_scale=grad_scale)
            self._exact('adam_step', np.array_equal(w.cpu().numpy(), rw) and np.array_equal(m.cpu().numpy(), rm) and
                        np.array_equal(v.cpu().numpy(), rv))

    # ---------------------------------------------------------------------------------------------- weight quantizer
    @staticmethod
    def _buckets(q, i):
        """(use_buckets, bucket_type, bucket_size) of tensor i of a UniformWeightQuantizer, from its layout"""
        seg, shape = q.segs[i], tuple(q.srcs[i].shape)
        ncols, padded = int(seg['ncols']), int(seg['padded'])
        if ncols == 1 and padded == q.srcs[i].numel():
            return False, 'channel', 0
        if padded == q.srcs[i].numel() and ncols == shape[-1]:
            return True, 'channel', 0
        return True, 'split', padded // ncols

    def _m_UniformWeightQuantizer_forward(self, fn, q):
        fn(q)
        if not self._first(('UniformWeightQuantizer.forward', id(q))):
            return
        torch.cuda.synchronize()
        for i, (src, dst) in enumerate(zip(q.srcs, q.dsts)):
            ub, bt, bs = self._buckets(q, i)
            ref = O.uniform_quantize(src.cpu().numpy(), q.bits[i], 'weight', ub, bt, bs or 256)
            self._exact('weight quantizer (%s)' % (bt if ub else 'per layer'), np.array_equal(dst.cpu().numpy(), ref))

    def _m_UniformWeightQuantizer_ste_backward_(self, fn, q, grads, indices=None):
        idx = list(range(len(grads))) if indices is None else list(indices)
        key = ('UniformWeightQuantizer.ste_backward_', id(q), tuple(idx))
        first = self._first(key)
        if first:
            torch.cuda.synchronize()
            pre = {i: grads[i].cpu().numpy() for i in idx}
        fn(q, grads, indices)
        if not first:
            return
        torch.cuda.synchronize()
        alpha = q.scales[:q.n_buckets].cpu().numpy()
        for i in idx:
            seg = q.segs[i]
            b0, ncols = int(seg['bucket0']), int(seg['ncols'])
            g = pre[i].reshape(-1)
            a = alpha[b0 + np.arange(g.size) % ncols]
            ref = O.uq_ste_grad(g, a, q.bits[i]).reshape(pre[i].shape)
            self._exact('weight quantizer STE', np.array_equal(grads[i].cpu().numpy(), ref))

    # ---------------------------------------------------------------------------------------------- codebooks
    def _cover(self, tag, n, held):
        """one run of a per-tensor check: n tensors compared of the `held` its object holds"""
        self.covered.setdefault(tag, []).append((n, held))

    @staticmethod
    def _codebook(q, i):
        """the whole device codebook of tensor i: its store-resident `clusters` variable, or its private table row"""
        return q.cluster_views[i] if q.cluster_views is not None else q.clusters[i]

    def _quantile_ref(self, q, i):
        """oracle.nuq_quantile_init of tensor i's normalised weights from ONE sort: the elements at the oracle's
        percentile_index positions of the descending order (16 full sorts of a 2.36M tensor per kernel would dominate
        the run; the shortcut is cross-checked against the oracle itself in the quantile-init check)"""
        key = (id(q), i)
        if key not in self._codebooks:
            xn = O.uq_scale(q.srcs[i].cpu().numpy().reshape(-1), None)[0]
            k = 1 << q.uq.bits[i]
            desc = np.sort(xn)[::-1]
            self._codebooks[key] = desc[[O.percentile_index(xn.size, (j + 1) * 100 / (k + 1)) for j in range(k)]]
        return self._codebooks[key]

    def _c_select_desc(self, fn, tensors, queries):
        out = fn(tensors, queries)
        if self._first(('select_desc', tuple(t.numel() for t in tensors), tuple(queries))):
            got, desc, ok = out.cpu().numpy(), {}, True
            for qi, (ti, rank) in enumerate(queries):
                if ti not in desc:
                    desc[ti] = np.sort(tensors[ti].cpu().numpy().reshape(-1))[::-1]
                ok = ok and got[qi] == desc[ti][rank]
            self._exact('order statistics (select_desc)', ok)
        return out

    def _m_CodebookWeightQuantizer_quantile_values(self, fn, q):
        vals = fn(q)
        if self._first(('CodebookWeightQuantizer.quantile_values', id(q))):
            assert not q.use_buckets, 'bucketed codebooks are not benchmarked (test_nuq_buckets_gpu checks them)'
            oks = [np.array_equal(v.view(np.uint32), self._quantile_ref(q, i).view(np.uint32))
                   for i, v in enumerate(vals)]
            self._per_tensor({'codebook quantile values': oks})
            self._cover('codebook quantile values', len(oks), len(q.srcs))
        return vals

    def _m_CodebookWeightQuantizer_quantile_init(self, fn, q):
        fn(q)
        if not self._first(('CodebookWeightQuantizer.quantile_init', id(q))):
            return
        torch.cuda.synchronize()
        assert not q.use_buckets, 'bucketed codebooks are not benchmarked (test_nuq_buckets_gpu checks them)'
        res = {'codebook quantile init': [], 'codebook quantile init: entries past 2^bits zero': []}
        for i in range(len(q.srcs)):
            k = 1 << q.uq.bits[i]
            cb = self._codebook(q, i).cpu().numpy().view(np.uint32)
            res['codebook quantile init'].append(np.array_equal(cb[:k], self._quantile_ref(q, i).view(np.uint32)))
            res['codebook quantile init: entries past 2^bits zero'].append(not cb[k:].any())
        self._per_tensor(res)
        self._cover('codebook quantile init', len(res['codebook quantile init']), len(q.srcs))
        sizes = [s.numel() for s in q.srcs]
        for i in sorted({int(np.argmin(sizes)), int(np.argmax(sizes))}):
            xn = O.uq_scale(q.srcs[i].cpu().numpy(), None)[0]
            self._exact('codebook quantile init: one sort == oracle (smallest, largest tensor)',
                        np.array_equal(self._quantile_ref(q, i), O.nuq_quantile_init(xn, 1 << q.uq.bits[i])))
        self._codebooks = {key: v for key, v in self._codebooks.items() if key[0] != id(q)}

    def _m_CodebookWeightQuantizer_forward(self, fn, q):
        fn(q)
        if not self._first(('CodebookWeightQuantizer.forward', id(q))):
            return
        torch.cuda.synchronize()
        assert not q.use_buckets, 'bucketed codebooks are not benchmarked (test_nuq_buckets_gpu checks them)'
        res = {'codebook forward': []}
        for i, (src, dst) in enumerate(zip(q.srcs, q.dsts)):
            bits = q.uq.bits[i]
            ref, _, idx = O.nonuniform_quantize(src.cpu().numpy(), bits,
                                                clusters=self._codebook(q, i)[:1 << bits].cpu().numpy())
            res['codebook forward'].append(np.array_equal(dst.cpu().numpy().view(np.uint32), ref.view(np.uint32)))
            if q.idx is not None:           # ties go to the first centroid (tf.argmin)
                o = q.idx_offsets[i]
                res.setdefault('codebook forward kept index', []).append(
                    np.array_equal(q.idx[o:o + src.numel()].cpu().numpy(), idx.reshape(-1).astype(np.uint8)))
        self._per_tensor(res)
        self._cover('codebook forward', len(res['codebook forward']), len(q.srcs))

    def _m_CodebookWeightQuantizer_cluster_grad(self, fn, q, grads, grad_base):
        first = self._first(('CodebookWeightQuantizer.cluster_grad', id(q)))
        fn(q, grads, grad_base)
        if not first:
            return
        torch.cuda.synchronize()
        assert not q.use_buckets, 'bucketed codebooks are not benchmarked (test_nuq_buckets_gpu checks them)'
        outs = [grad_base[int(o):int(o) + (1 << b)].clone() for o, b in zip(q.cluster_off.cpu().numpy(), q.uq.bits)]
        scales = q.uq.scales.cpu().numpy()
        worst, n = 0.0, 0
        for i, g in enumerate(grads):
            k, gn = 1 << q.uq.bits[i], g.cpu().numpy().reshape(-1)
            idx = q.idx[q.idx_offsets[i]:q.idx_offsets[i] + gn.size].cpu().numpy().astype(np.int64)
            alpha = scales[int(q.uq.segs[i]['bucket0'])]
            ref = O.nuq_grads(gn, idx, k, alpha)[1].astype(np.float64)
            mag = np.bincount(idx, weights=np.abs((gn * alpha).astype(np.float32).astype(np.float64)), minlength=k)
            err = np.abs(outs[i].cpu().numpy().astype(np.float64) - ref) / np.maximum(mag, 1e-30)
            worst = max(worst, err.max())
            n += 1
        self._note('codebook gradient / sum|terms|', worst, 1e-6)
        self._cover('codebook gradient', n, len(q.srcs))
        fn(q, grads, grad_base)            # the reduction runs in a fixed order: a second call gives the same bits
        torch.cuda.synchronize()
        self._exact('codebook gradient run to run', all(
            torch.equal(grad_base[int(o):int(o) + t.numel()].view(torch.int32), t.view(torch.int32))
            for o, t in zip(q.cluster_off.cpu().numpy(), outs)))

    # ---------------------------------------------------------------------------------------------- masks
    def _m_MaskBuilder_build(self, fn, mb, prune_ratios):
        first = self._first(('MaskBuilder.build', id(mb), tuple(float(r) for r in prune_ratios)))
        if first:
            torch.cuda.synchronize()
            pre = [(w.cpu().numpy(), b.cpu().numpy(), m.cpu().numpy()) for w, b, m in zip(mb.ws, mb.bkups, mb.masks)]
        ranks = fn(mb, prune_ratios)
        if not first:
            return ranks
        torch.cuda.synchronize()
        u32 = lambda t: t.cpu().numpy().view(np.uint32)        # noqa: E731
        res = {'mask rebuild mask': [], 'mask rebuild weights': [], 'mask rebuild backups': [],
               'mask rebuild thresholds': []}
        thr = u32(mb.thr)
        for i, ((w0, b0, m0), r) in enumerate(zip(pre, prune_ratios)):
            rw, rb, rm, rt = O.ws_build_mask(w0, b0, m0, r)
            res['mask rebuild mask'].append(np.array_equal(u32(mb.masks[i]), rm.view(np.uint32)))
            res['mask rebuild weights'].append(np.array_equal(u32(mb.ws[i]), rw.view(np.uint32)))
            res['mask rebuild backups'].append(np.array_equal(u32(mb.bkups[i]), rb.view(np.uint32)))
            res['mask rebuild thresholds'].append(thr[i] == np.float32(rt).view(np.uint32))
        self._per_tensor(res)
        self._cover('mask rebuild', len(res['mask rebuild mask']), len(mb.ws))
        return ranks

    # ---------------------------------------------------------------------------------------------- tc operands
    def _check_tc_weights(self, tw, w, seg):
        """forward / dgrad copies of one kernel against the fp32 tensor they stand for (pf_conv2d_tc_prep_*)"""
        r, s_, c, k = tw.d.r, tw.d.s, tw.d.c, tw.d.k
        rsc = r * s_ * c
        wm = w.reshape(rsc, k)
        bits = int(seg['q_bits']) if seg is not None else 0
        fh = tw.f_hi.view(k, -1)
        if bits:
            w0, al, be, ra, ncols, _ = seg['levels']
            w0n = w0.reshape(rsc, k).cpu().numpy()
            a, b = al[:ncols].cpu().numpy(), be[:ncols].cpu().numpy()
            kq = O.uq_k(bits)
            lv = np.rint(((((w0n - b).astype(np.float32)) / a).astype(np.float32) * kq).astype(np.float32))
            want = torch.from_numpy((lv - float(1 << (bits - 1))).T.copy()).to(DEV)
            self._exact('tc weight levels', torch.equal(fh[:, :rsc].float(), want))
            # the quantized fp32 weight the levels stand for is what the step's fp32 kernel holds
            q = O.uq_inv_scale((lv / kq).astype(np.float32), a, b)
            self._exact('tc weight levels == quantized weight', np.array_equal(q, wm.cpu().numpy()))
        else:
            h, l = split_planes(wm.t().contiguous())
            self._exact('tc weight planes', torch.equal(fh[:, :rsc].reshape(-1), h) and
                        torch.equal(tw.f_lo.view(k, -1)[:, :rsc].reshape(-1), l))
            self._exact('tc weight Kpad zero', bool((tw.f_lo.view(k, -1)[:, rsc:] == 0).all()))
        self._exact('tc weight Kpad zero', bool((fh[:, rsc:] == 0).all()))
        if tw.d_hi is not None:
            # dgrad copy [c][(r, s), k]: split of the fp32 weight, transposed
            wd = w.reshape(r * s_, c, k).permute(1, 0, 2).reshape(c, r * s_ * k)
            h, l = split_planes(wd.contiguous())
            dh, dl = tw.d_hi.view(c, -1), tw.d_lo.view(c, -1)
            n = r * s_ * k
            self._exact('tc dgrad weight planes', torch.equal(dh[:, :n].reshape(-1), h) and
                        torch.equal(dl[:, :n].reshape(-1), l))
            self._exact('tc weight Kpad zero', bool((dh[:, n:] == 0).all() and (dl[:, n:] == 0).all()))

    def _m_TcWeightsBatch_prepare(self, fn, tb, levels=True):
        fn(tb, levels)
        if not self._first(('TcWeightsBatch.prepare', id(tb), bool(levels))):
            return
        torch.cuda.synchronize()
        segs = tb.segs if levels else tb.segs_plain
        for i, (tw, w) in enumerate(tb.keep):
            seg = {'q_bits': int(segs[i]['q_bits']), 'levels': tb.levels.get(i)}
            self._check_tc_weights(tw, w, seg)

    def _m_TcWeights_prepare(self, fn, tw, w):
        fn(tw, w)
        if self._first(('TcWeights.prepare', id(tw))):
            torch.cuda.synchronize()
            self._check_tc_weights(tw, w, None)

    def _m_TcWgradReduceBatch_reduce(self, fn, rb):
        fn(rb)
        if not self._first(('TcWgradReduceBatch.reduce', id(rb))):
            return
        torch.cuda.synchronize()
        worst = 0.0
        for part, out, splits in rb.keep:
            n = out.numel()
            p = part[:splits * n].view(splits, n).double()
            e = ((out.reshape(-1).double() - p.sum(0)).abs() / p.abs().sum(0).clamp_min(1e-30)).max().item()
            worst = max(worst, e)
        self._note('split-K reduction / sum|partials|', worst, 1e-6)

    # ---------------------------------------------------------------------------------------------- producers
    @staticmethod
    def _cols_ref(d, x, kpad, n0, n1):
        """im2col columns [(n1 - n0)*p*q, kpad] of images n0..n1 of NHWC x, (r, s, c) order, zero padding and zero
        columns past r*s*c"""
        n, h, wd, c, k, r, s, p, q, sh, sw, pt, pl = geom(d)
        x = x.reshape(-1)[n0 * h * wd * c:n1 * h * wd * c]
        n = n1 - n0
        pb, pr = (p - 1) * sh + r - h - pt, (q - 1) * sw + s - wd - pl      # negative: rows / columns no window reaches
        xp = F.pad(x.reshape(-1)[:n * h * wd * c].view(n, h, wd, c).permute(0, 3, 1, 2), (pl, pr, pt, pb))
        cols = F.unfold(xp, (r, s), stride=(sh, sw))
        cols = cols.view(n, c, r, s, p * q).permute(0, 4, 2, 3, 1).reshape(n * p * q, r * s * c)
        return F.pad(cols, (0, kpad - r * s * c))

    def _c_im2col(self, fn, d, x, kpad, cols):
        fn(d, x, kpad, cols)
        if self._first(('im2col', geom(d), kpad)):
            torch.cuda.synchronize()
            ok, n, pq = True, geom(d)[0], geom(d)[7] * geom(d)[8]
            for n0 in range(0, n, 8):                          # 8 images at a time: the stem's columns are GBs
                ref = self._cols_ref(d, x, kpad, n0, min(n, n0 + 8)).reshape(-1)
                ok = ok and torch.equal(cols.reshape(-1)[n0 * pq * kpad:n0 * pq * kpad + ref.numel()], ref)
            self._exact('im2col', ok)

    def _c_im2col_planes(self, fn, d, x, kpad, planes):
        fn(d, x, kpad, planes)
        if self._first(('im2col_planes', geom(d), kpad)):
            torch.cuda.synchronize()
            ok, n, pq = True, geom(d)[0], geom(d)[7] * geom(d)[8]
            for n0 in range(0, n, 8):
                h, l = split_planes(self._cols_ref(d, x, kpad, n0, min(n, n0 + 8)))
                o = n0 * pq * kpad
                ok = ok and torch.equal(planes.hi[o:o + h.numel()], h) and torch.equal(planes.lo[o:o + l.numel()], l)
            self._exact('im2col_planes', ok)

    def _c_s2d_planes(self, fn, x, pad_t, pad_l, hp, wp, cpad, planes):
        fn(x, pad_t, pad_l, hp, wp, cpad, planes)
        if not self._first(('s2d_planes', tuple(x.shape), pad_t, pad_l, hp, wp, cpad)):
            return
        torch.cuda.synchronize()
        n, h, w, c = x.shape
        xp = F.pad(x.permute(0, 3, 1, 2), (pad_l, max(2 * wp + 2 - w - pad_l, 0), pad_t, max(2 * hp + 2 - h - pad_t, 0)))
        ref = torch.zeros(n, hp, wp, cpad, device=DEV)
        for blk in range(4):
            u, v = blk >> 1, blk & 1
            ref[..., blk * c:(blk + 1) * c] = xp[:, :, u::2, v::2][:, :, :hp, :wp].permute(0, 2, 3, 1)
        h2, l2 = split_planes(ref)
        self._exact('s2d_planes', torch.equal(planes.hi[:h2.numel()], h2) and torch.equal(planes.lo[:l2.numel()], l2))

    def _c_gather_rows(self, fn, src, idx, dst, row_len):
        fn(src, idx, dst, row_len)
        if self._first(('gather_rows', src.numel(), idx.numel(), row_len)):
            torch.cuda.synchronize()
            rows = src.reshape(-1)[:src.numel() // row_len * row_len].view(-1, row_len)
            ix = idx.long()
            ref = torch.where((ix >= 0).view(-1, 1), rows[ix.clamp_min(0)], torch.zeros((), device=DEV))
            self._exact('gather_rows', torch.equal(dst.reshape(-1)[:ref.numel()], ref.reshape(-1)))

    def _c_fold_diag_blocks(self, fn, src, g, m, n, dst):
        fn(src, g, m, n, dst)
        if self._first(('fold_diag_blocks', g, m, n)):
            torch.cuda.synchronize()
            a = src.reshape(-1)[:g * m * g * n].view(g * m, g * n).double()
            blocks = torch.stack([a[b * m:(b + 1) * m, b * n:(b + 1) * n] for b in range(g)])
            e = ((dst.reshape(-1)[:m * n].view(m, n).double() - blocks.sum(0)).abs() /
                 blocks.abs().sum(0).clamp_min(1e-30)).max().item()
            self._note('fold_diag_blocks / sum|terms|', e, 1e-6)

    @staticmethod
    def _finite(t, planes, nel, key):
        torch.cuda.synchronize()
        if t is not None:
            assert torch.isfinite(t.reshape(-1)[:nel]).all(), ('non-finite output', key)
        if planes is not None:
            assert torch.isfinite(planes.hi[:nel]).all() and torch.isfinite(planes.lo[:nel]).all(), \
                ('non-finite planes', key)

    def finish(self, label, secs, peak_gb):
        print('%s: %d calls of the wrapped layers, %d checked; worst %s; %.0f s, peak %.1f GB' % (
            label, self.calls, len(self.checked), {k: '%.2e' % v for k, v in sorted(self.worst.items())}, secs, peak_gb))
        for g, e, em, e32 in self.wgrad_notes:
            print('  dwconv wgrad %s: %.2e of max|ref|, %.2e of max sum|terms|, fp32 reference %.2e' % (g, e, em, e32))
        for tag, runs in sorted(self.covered.items()):
            print('  %s: %s tensors' % (tag, ', '.join('%d of %d' % r for r in runs)))
        checked_here = {n[3:] for n in dir(self) if n.startswith('_c_')} | \
            {n[3:].replace('_', '.', 1) for n in dir(self) if n.startswith('_m_')}
        unknown = self.called - checked_here - set(TcRecorder.NAMES) - set(EXEMPT)
        for what, v in (('unchecked entry points', sorted(unknown)), ('failed checks', self.fail)):
            if v:
                print('  %s: %s' % (what, v))
        assert not unknown, 'the step calls entry points that are neither checked nor exempt: %s' % sorted(unknown)
        assert not self.fail, self.fail
        # every per-tensor check covered every tensor its object holds, and each check the plan calls for ran
        assert all(n == held for runs in self.covered.values() for n, held in runs), self.covered
        missing = {t: n for t, n in self.expect.items()
                   if (t not in self.worst if n is None else
                       not self.covered.get(t) or any(r[0] != n for r in self.covered[t]))}
        assert not missing, ('checks the plan calls for that did not run (over every tensor)', missing, self.covered)
        # one activation tensor per workload through the numpy oracle itself (when the workload quantizes activations)
        assert self.oracle_done or not self.quant_seen, 'no activation tensor went through the numpy oracle'
        assert len(self.checked) >= 10


def expected_checks(workload, lrn):
    """the checks the learner's plan calls for: {tag: tensors each run must cover, or None where the tag only has to
    appear} — the weight-sparse mask rebuild over every maskable variable, the codebook checks over every quantized
    kernel, and the producer of each first layer that computes its own operand (the stem's folded weight gradient
    included)"""
    import bench
    ex = lrn.sess_train
    want = {}
    if bench.WORKLOADS[workload][2] == 'weight-sparse':
        want['mask rebuild'] = len(ex.maskable)
    if isinstance(ex.wq, ops.CodebookWeightQuantizer):
        for tag in ('codebook forward', 'codebook quantile values', 'codebook quantile init'):
            want[tag] = len(ex.wq_ops)
        if ex.train_clusters:
            want['codebook gradient'] = len(ex.wq_ops)
    for e in (ex, ex.teacher):
        for im in (e.im2col.values() if e is not None else ()):
            if im['compute']:
                want['s2d_planes' if im['mode'] == 's2d' else ('im2col_planes' if im['planes'] else 'im2col')] = None
            if e.train and 'pair' in im:
                want['fold_diag_blocks / sum|terms|'] = None
    return want


# (workload, batch, flag overrides): the benchmarked workloads at their batch, and the codebook learner also in the
# 'both' optimisation mode, where the codebook gradient runs
RUNS = [('resnet50_uq8_dst_b128', 128, None), ('mobilenet_cpg50_b256', 256, None), ('lenet_uq8_b128', 128, None),
        ('resnet50_ws50_dst_b128', 128, None), ('resnet50_nuq4_dst_b128', 128, None),
        ('resnet50_nuq4_dst_b128', 128, {'nuql_opt_mode': 'both'}), ('resnet20_uq8_dst_b256', 256, None),
        ('resnet20_ws50_dst_b256', 256, None)]


@pytest.mark.parametrize('workload,batch,flags', [
    pytest.param(w, b, f, id='%s-%d' % (w, b) + ''.join('-%s' % v for _, v in sorted((f or {}).items())))
    for w, b, f in RUNS])
def test_bench_layers_besides_the_tc_convs(workload, batch, flags, monkeypatch):
    run_workload(workload, batch, monkeypatch, lambda mp, lrn: NnRecorder(mp, expected_checks(workload, lrn)),
                 flags=flags, after=after_step(workload))
