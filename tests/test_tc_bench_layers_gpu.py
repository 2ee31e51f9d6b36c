"""Every tensor-core convolution of one training step of the benchmarked workloads, at the benchmarked batch, against
float64.

bench.py measures its workloads at batch 128 (ResNet-50) and 256 (ResNet-20, MobileNet) (DESIGN.md §8); the other step
tests run ResNet-50 at batch 2, where no CTA of the persistent kernels ever sees a second tile.  Here the learner of a
workload is built at the benchmarked batch under PF_POISON=1 (activation and scratch buffers start as NaN) and one
eager step runs with the tensor-core entry points of `ops` wrapped: each call is passed through unchanged, then
  * its output must be finite, and its launch plan (pf_conv2d_tc_last_plan) is collected;
  * the first call of each (entry point, geometry, operand form, epilogue) is compared with a float64 convolution of
    exactly the operands it was fed — split planes as hi + lo, activation levels as scale x level, weight levels as
    alpha / k * level + beta — with its own epilogue (bias, ReLU, residual, accumulate) and, for a deferred weight
    gradient, the sum of its split-K partials.  Bars as DESIGN.md §6: 2e-5 of max|ref| with a split-bf16 operand,
    1e-5 for levels x levels.  Repeated geometries are checked once: the float64 references of every layer would
    dominate the run time.
Finally every plan the step used must be one the kernel-variant sweep (test_tc_variants_gpu.py) proves it reaches,
so the small-shape sweep covers what the benchmark runs."""
import gc
import os
import sys
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from pocketflow_b200 import ops  # noqa: E402
from test_tc_variants_gpu import KEY_FIELDS, REQUIRED, plan_key  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')


def geom(d):
    return tuple(int(getattr(d, f)) for f in ('n', 'h', 'w', 'c', 'k', 'r', 's', 'p', 'q', 'stride_h', 'stride_w',
                                               'pad_t', 'pad_l'))


def conv64(x, w, d):
    """float64 conv of NHWC x with HWIO w as pf_conv_desc d describes it (implicit bottom / right padding), by unfold +
    DGEMM; differentiable in x and w"""
    n, h, wd, c, k, r, s, p, q, sh, sw, pt, pl = geom(d)
    pb, pr = (p - 1) * sh + r - h - pt, (q - 1) * sw + s - wd - pl      # negative: rows / columns no window reaches
    xp = F.pad(x.permute(0, 3, 1, 2), (pl, pr, pt, pb))
    cols = F.unfold(xp, (r, s), stride=(sh, sw))                          # [n, c*r*s, p*q], channel-major
    wm = w.permute(3, 2, 0, 1).reshape(k, c * r * s)
    return (wm @ cols).view(n, k, p, q).permute(0, 2, 3, 1)


def split_value(x, shape):
    """value of an fp32 operand as the producers split it: hi + lo"""
    x = x.reshape(-1)[:int(np.prod(shape))]
    hi = x.to(torch.bfloat16)
    return (hi.double() + (x - hi.float()).to(torch.bfloat16).double()).view(shape)


def planes_value(pl, shape):
    nel = int(np.prod(shape))
    return (pl.hi[:nel].double() + pl.lo[:nel].double()).view(shape)


def act_value(act, shape):
    """(value, is integer levels) of a pf_tc_act made by ops.tc_act"""
    planes, hdr, single = act._src
    if hdr is not None:
        h = hdr.cpu().numpy().view(ops.ACT_HDR)[0]
        if int(h['nplanes']) == 1:
            return planes.hi[:int(np.prod(shape))].double().view(shape) * float(h['scale']), True
        return planes_value(planes, shape), False
    if single:
        return planes.hi[:int(np.prod(shape))].double().view(shape), True
    return planes_value(planes, shape), False


def fwd_weight(tw_hi, tw_lo, d):
    n, h, wd, c, k, r, s = geom(d)[:7]
    v = tw_hi.double() + (tw_lo.double() if tw_lo is not None else 0.0)
    return v.view(k, -1)[:, :r * s * c].reshape(k, r, s, c).permute(1, 2, 3, 0)


def wt_value(wt, d):
    """(value, is integer levels) of a pf_tc_wt made by ops.tc_wt"""
    p0, p1, alpha, beta, per_channel, bits = wt._src
    if alpha is None:
        return fwd_weight(p0, p1, d), False
    k = geom(d)[4]
    lv = fwd_weight(p0, None, d) + float(1 << (bits - 1))
    rk = float(np.float32(1.0) / np.float32((1 << bits) - 1))
    a, b = (alpha[:k], beta[:k]) if per_channel else (alpha[:1], beta[:1])
    return (a.double() * rk) * lv + b.double(), True


def dgrad_weight(tw, d):
    n, h, wd, c, k, r, s = geom(d)[:7]
    v = tw.d_hi.double() + tw.d_lo.double()
    return v.view(c, -1)[:, :r * s * k].reshape(c, r, s, k).permute(1, 2, 0, 3)


class Recorder:
    """wraps the tensor-core entry points of `ops`; see the module docstring"""

    NAMES = ('conv2d_tc_fwd', 'conv2d_tc_fwd_planes', 'conv2d_tc_fwd_ex', 'conv2d_tc_dgrad', 'conv2d_tc_dgrad_planes',
             'conv2d_tc_dgrad_ex', 'conv2d_tc_wgrad', 'conv2d_tc_wgrad_planes', 'conv2d_tc_wgrad_ex')

    def __init__(self, monkeypatch, min_calls, fwd_geoms=()):
        """fwd_geoms: geometries that must each make a forward call"""
        self.plans, self.checked, self.worst, self.calls, self.max_tiles = {}, set(), {}, 0, 0
        self.min_calls, self.fwd_geoms, self.fwd_seen = min_calls, set(fwd_geoms), set()
        self.over = []                 # checks above the DESIGN §6 bar: (key, error, error of an fp32 GEMM)
        orig_act, orig_wt = ops.tc_act, ops.tc_wt

        def tc_act(planes, hdr=None, csum=None, nseg=0, single=False):
            a = orig_act(planes, hdr, csum, nseg, single)
            a._src = (planes, hdr, single)
            return a

        def tc_wt(p0, p1=None, alpha=None, beta=None, per_channel=False, bits=0):
            w = orig_wt(p0, p1, alpha, beta, per_channel, bits)
            w._src = (p0, p1, alpha, beta, per_channel, bits)
            return w

        monkeypatch.setattr(ops, 'tc_act', tc_act)
        monkeypatch.setattr(ops, 'tc_wt', tc_wt)
        for name in self.NAMES:
            monkeypatch.setattr(ops, name, self._wrap(name, getattr(ops, name)))

    def _wrap(self, name, fn):
        def call(d, *args):
            pass_ = 0 if '_fwd' in name else (1 if '_dgrad' in name else 2)
            form = self._form(name, args)
            key = (name, geom(d), form) + self._epilogue(pass_, args)
            check = key not in self.checked
            prior = args[3].clone() if (check and pass_ == 1 and args[2]) else None
            fn(d, *args)
            plan = ops.conv2d_tc_last_plan()
            self.plans.setdefault(plan_key(plan), '%s %s' % (name, geom(d)))
            self.calls += 1
            if pass_ == 0:
                self.fwd_seen.add(geom(d))
            self.max_tiles = max(self.max_tiles, plan['tiles'])
            out = args[4] if pass_ == 0 else args[3]
            if out is not None:
                n, h, wd, c, k, r, s, p, q = geom(d)[:9]
                nel = (n * p * q * k, n * h * wd * c, r * s * c * k)[pass_]
                torch.cuda.synchronize()
                assert torch.isfinite(out.reshape(-1)[:nel]).all(), ('non-finite output', key)
            if check:
                self.checked.add(key)
                torch.cuda.synchronize()
                err, err32, levels = self._check(name, pass_, d, args, prior)
                tag = ('fwd', 'dgrad', 'wgrad')[pass_] + ' ' + form
                self.worst[tag] = max(self.worst.get(tag, 0.0), err)
                if err > (1e-5 if levels else 2e-5):
                    self.over.append((key, err, err32, self._magnitude_error(name, pass_, d, args, prior)))
        return call

    @staticmethod
    def _form(name, args):
        if name.endswith('_ex'):
            torch.cuda.synchronize()             # the header may come from a producer on another stream
            a = args[0]
            planes, hdr, single = a._src
            af = 'single' if single else ('hdr%d' % int(hdr.cpu().numpy().view(ops.ACT_HDR)[0]['nplanes'])
                                          if hdr is not None else 'split')
            if name == 'conv2d_tc_wgrad_ex':
                return af + ' x split'
            return af + (' x levels' if args[1]._src[2] is not None else ' x split')
        return ('fp32' if name in ('conv2d_tc_fwd', 'conv2d_tc_dgrad', 'conv2d_tc_wgrad') else 'split') + ' x split'

    @staticmethod
    def _epilogue(pass_, args):
        if pass_ == 0:       # (x, w, bias, relu, y, residual)
            return (args[2] is not None, bool(args[3]), len(args) > 5 and args[5] is not None)
        if pass_ == 1:       # (dy, w, accumulate, dx)
            return (bool(args[2]),)
        return (args[-1] is None,)   # wgrad: deferred split-K partials

    def _check(self, name, pass_, d, args, prior):
        """(error of the kernel, error of a plain fp32 GEMM of the same operands, levels x levels), both relative to
        max|float64 reference|; the fp32 error is only computed when the kernel misses the DESIGN §6 bar"""
        ref, got, levels = self._reference(name, pass_, d, args, prior)
        assert torch.isfinite(got).all()
        scale = ref.abs().max()
        err = ((got.double() - ref).abs().max() / scale).item()
        err32 = 0.0
        if err > (1e-5 if levels else 2e-5):
            # the same contraction accumulated in fp32 (exact fp32 products, no TF32): the accuracy a plain fp32
            # implementation reaches where the sum cancels (BN-backward gradients are zero-mean per channel)
            tf32 = torch.backends.cuda.matmul.allow_tf32
            torch.backends.cuda.matmul.allow_tf32 = False
            try:
                ref32 = self._reference(name, pass_, d, args, prior, torch.float32)[0]
            finally:
                torch.backends.cuda.matmul.allow_tf32 = tf32
            err32 = ((ref32.double() - ref).abs().max() / scale).item()
        return err, err32, levels

    def _magnitude_error(self, name, pass_, d, args, prior):
        """max |kernel - float64| relative to the largest sum of |terms| (|x|^T |dy| for wgrad): the error bound of a
        dot product that does not depend on how much the sum cancels"""
        ref, got = self._reference(name, pass_, d, args, prior)[:2]
        mag = self._reference(name, pass_, d, args, prior, absolute=True)[0]
        return ((got.double() - ref).abs().max() / mag.abs().max()).item()

    def _reference(self, name, pass_, d, args, prior, dt=torch.float64, absolute=False):
        """(reference in dtype dt, kernel output, levels x levels); absolute: wgrad of |x| and |dy|"""
        n, h, wd, c, k, r, s, p, q = geom(d)[:9]
        if pass_ == 0:
            x, w, bias, relu, y = args[:5]
            res = args[5] if len(args) > 5 else None
            if name == 'conv2d_tc_fwd_ex':
                xv, xl = act_value(x, (n, h, wd, c))
                wv, wl = wt_value(w, d)
            else:
                xv = (split_value if name == 'conv2d_tc_fwd' else planes_value)(x, (n, h, wd, c))
                xl = False
                wv, wl = fwd_weight(w.f_hi, w.f_lo, d), False
            ref = conv64(xv.to(dt), wv.to(dt), d)
            if bias is not None:
                ref = ref + bias.to(dt)
            if relu:
                ref = torch.relu(ref)
            if res is not None:
                ref = ref + res.reshape(-1)[:ref.numel()].to(dt).view(ref.shape)
            return ref, y.reshape(-1)[:ref.numel()].view(ref.shape), xl and wl
        if pass_ == 1:
            dy, w, acc, dx = args
            assert name != 'conv2d_tc_dgrad_ex', 'the engine does not call pf_conv2d_tc_dgrad_ex'
            dyv = (split_value if name == 'conv2d_tc_dgrad' else planes_value)(dy, (n, p, q, k))
            xg = torch.zeros(n, h, wd, c, dtype=dt, device=DEV, requires_grad=True)
            conv64(xg, dgrad_weight(w, d).to(dt), d).backward(dyv.to(dt))
            ref = xg.grad + (prior.reshape(-1)[:xg.numel()].to(dt).view(n, h, wd, c) if acc else 0.0)
            return ref, dx.reshape(-1)[:ref.numel()].view(ref.shape), False
        x, dy, ws, dw = args
        assert not absolute or pass_ == 2
        if name == 'conv2d_tc_wgrad_ex':
            xv, _ = act_value(x, (n, h, wd, c))
            dyv = planes_value(dy._src[0], (n, p, q, k))
        elif name == 'conv2d_tc_wgrad':
            xv, dyv = split_value(x, (n, h, wd, c)), split_value(dy, (n, p, q, k))
        else:
            xv, dyv = planes_value(x, (n, h, wd, c)), planes_value(dy, (n, p, q, k))
        if absolute:
            xv, dyv = xv.abs(), dyv.abs()
        wg = torch.zeros(r, s, c, k, dtype=dt, device=DEV, requires_grad=True)
        conv64(xv.to(dt), wg, d).backward(dyv.to(dt))
        ref = wg.grad
        if dw is None:
            splits = ops.conv2d_tc_wgrad_splits(d)
            got = ws[:splits * ref.numel()].view(splits, -1).double().sum(0).view(ref.shape)
        else:
            got = dw.reshape(-1)[:ref.numel()].view(ref.shape)
        return ref, got, False

    def finish(self, label, secs, peak_gb):
        print('%s: %d tensor-core calls, %d checked against float64; worst errors %s; %d distinct plans, '
              'at most %d tiles in one launch; %.0f s, peak %.1f GB' % (
                  label, self.calls, len(self.checked), {k: '%.2e' % v for k, v in sorted(self.worst.items())},
                  len(self.plans), self.max_tiles, secs, peak_gb))
        for k, first in sorted(self.plans.items()):
            print('  plan %s: first %s' % (' '.join('%s=%s' % f for f in zip(KEY_FIELDS, k)), first))
        for key, err, err32, errm in self.over:
            print('  above the bar: %s %s: %.2e of max|ref| (an fp32 GEMM of the same operands: %.2e); %.2e of max '
                  'sum of |terms|' % (key[0], key[1:], err, err32, errm))
        # DESIGN.md §6 bars hold for every forward and dgrad call.  The weight gradients reduce over every pixel of the
        # batch (6272 at ResNet-50's last stage, batch 128) of BN-backward gradients, which are zero-mean per channel:
        # the sum cancels, and the tensor-core accumulation then loses more than an fp32 GEMM does (DESIGN.md §4).
        # There the bar is 2e-5 of the largest sum of |terms|, which does not depend on the cancellation.
        bad = [(k, e, m) for k, e, _, m in self.over if not (k[0].startswith('conv2d_tc_wgrad') and m <= 2e-5)]
        assert not bad, bad
        assert self.calls >= self.min_calls and len(self.checked) >= 3
        assert not self.fwd_geoms - self.fwd_seen, ('planned tensor-core convolutions that made no forward call',
                                                    sorted(self.fwd_geoms - self.fwd_seen))
        assert self.max_tiles >= 3 * torch.cuda.get_device_properties(0).multi_processor_count
        outside = {k: v for k, v in self.plans.items() if k not in REQUIRED}
        assert not outside, 'plans the variant sweep does not reach: %s' % {
            str(dict(zip(KEY_FIELDS, k))): v for k, v in outside.items()}


def tc_recorder(monkeypatch, lrn):
    """a Recorder expecting what the executors planned: every convolution they put on the tensor cores, student and
    teacher, makes at least one forward call, at its own geometry (the first layer's lowered one)"""
    geoms = []
    for ex in (lrn.sess_train, lrn.sess_train.teacher):
        for op in (set(ex.tc) | set(ex.im2col) if ex is not None else ()):
            geoms.append(geom(ex.im2col[op]['d1'] if op in ex.im2col else ex.desc[op]))
    return Recorder(monkeypatch, len(geoms), set(geoms))


def ws_prune(lrn):
    """two mask rebuilds inside the pruning window (steps 6 and 8 of 20): the second finds the weights the first pruned
    at zero under a zero mask, so their backups must be kept"""
    lrn.nb_iters_train = 20
    for step in (6, 8):
        lrn.sess_train.step_count = step
        lrn.prune()


def after_step(workload):
    """what runs after the step besides it, by learner: the weight-sparse mask rebuild, and the codebook quantile init
    (which the learner first ran at construction, before any entry point was wrapped)"""
    import bench
    learner = bench.WORKLOADS[workload][2]
    if learner == 'weight-sparse':
        return ws_prune
    if learner == 'non-uniform':
        return lambda lrn: lrn.cluster_init()
    return None


def run_workload(workload, batch, monkeypatch, recorder, flags=None, after=None):
    """One eager step of a bench workload at `batch` under PF_POISON=1, with recorder(monkeypatch, learner) wrapping
    entry points of `ops` from just before the step; after(learner), if given, runs next with the recorder still
    installed; then recorder.finish(label, seconds, peak GB) prints and asserts.  flags: overrides of the workload's
    flags."""
    import bench
    monkeypatch.setenv('PF_POISON', '1')
    if flags:
        net, size, learner, over, descr = bench.WORKLOADS[workload]
        monkeypatch.setitem(bench.WORKLOADS, workload, (net, size, learner, dict(over, **flags), descr))
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    lrn = bench.build_learner(workload, 1, batch)
    ex = lrn.sess_train
    rec = recorder(monkeypatch, lrn)
    images, labels = lrn.iterator_train.next_batch()
    ex.buf[lrn.images].copy_(images)
    ex.buf[lrn.labels].copy_(labels)
    ex.run_step(lrn.lrn_rate(0))
    torch.cuda.synchronize()
    losses = ex.fetch_losses()
    assert np.isfinite(losses['loss']), losses
    if after is not None:
        after(lrn)
        torch.cuda.synchronize()
    label = '%s at batch %d' % (workload, batch) + ''.join(' %s=%s' % kv for kv in sorted((flags or {}).items()))
    try:
        rec.finish(label, time.time() - t0, torch.cuda.max_memory_allocated() / 2 ** 30)
    finally:
        del lrn, ex, rec
        gc.collect()
        torch.cuda.empty_cache()


def test_resnet50_uq8_bench_layers_at_batch_128(monkeypatch):
    run_workload('resnet50_uq8_dst_b128', 128, monkeypatch, tc_recorder)


def test_mobilenet_cpg50_bench_layers_at_batch_256(monkeypatch):
    run_workload('mobilenet_cpg50_b256', 256, monkeypatch, tc_recorder)


@pytest.mark.parametrize('workload,batch', [('resnet50_ws50_dst_b128', 128), ('resnet50_nuq4_dst_b128', 128),
                                            ('resnet20_uq8_dst_b256', 256), ('resnet20_ws50_dst_b256', 256)])
def test_bench_tc_convs(workload, batch, monkeypatch):
    run_workload(workload, batch, monkeypatch, tc_recorder, after=after_step(workload))
