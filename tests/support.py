"""What more than one test module uses: float64 references, the split-bf16 value model, error metrics, the learner
builder and the layer-by-layer parity harnesses (the backward tap, the tensor-core and CUDA-core entry-point
recorders, the per-tap exact-reduction references).  Not a test module: pytest collects nothing here."""
import gc
import importlib
import json
import os
import tempfile
import time
from fractions import Fraction

import numpy as np
import torch
import torch.nn.functional as F

from oracle import pf_oracle as O
from oracle.step_oracle import StepOracle
from pocketflow_b200 import compact as C
from pocketflow_b200 import ops
from pocketflow_b200.flags import FLAGS

DEV = torch.device('cuda:0')
F32 = np.float32


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def rel_err(got, ref):
    assert torch.isfinite(got).all(), 'non-finite output'
    return ((got.double() - ref).abs().max() / ref.abs().max()).item()


def max_rel(got, ref, slack=0.0):
    """max |got - ref| relative to max|ref|, after `slack` per element (the fp32 rounding of an accumulate)"""
    assert torch.isfinite(got).all(), 'non-finite gradient'
    return (((got - ref).abs() - slack).clamp_min(0.0).max() / ref.abs().max().clamp_min(1e-300)).item()


def free():
    gc.collect()
    torch.cuda.empty_cache()


def rel(a, b):
    return abs(float(a) - float(b)) / max(abs(float(b)), 1e-30)


def record(name, **kw):
    # outside the source tree, which may be read-only: $PF_PARITY_DIR, else the system temp directory
    out = os.environ.get('PF_PARITY_DIR') or tempfile.gettempdir()
    os.makedirs(out, exist_ok=True)
    p = os.path.join(out, 'parity_flips.json')
    d = json.load(open(p)) if os.path.exists(p) else {}
    d[name] = kw
    json.dump(d, open(p, 'w'), indent=1, sort_keys=True)


def split_value(x, shape=None):
    """hi + lo in float64 of the bf16 split the producers write of an fp32-valued x (hi = bf16(x), lo = bf16(x - hi));
    with `shape`, of x's first prod(shape) elements, viewed as `shape`"""
    if shape is not None:
        x = x.reshape(-1)[:int(np.prod(shape))]
    x = x.float()
    hi = x.to(torch.bfloat16)
    v = hi.double() + (x - hi.float()).to(torch.bfloat16).double()
    return v if shape is None else v.view(shape)


def planes_value(pl, shape):
    """hi + lo in float64 of ops.Planes pl, its first prod(shape) elements viewed as `shape`"""
    nel = int(np.prod(shape))
    return (pl.hi[:nel].double() + pl.lo[:nel].double()).view(shape)


def dbl(t, shape):
    return t.reshape(-1)[:int(np.prod(shape))].double().view(shape)


def split_planes(t):
    """the (hi, lo) bf16 planes, flat, of the split of fp32 t"""
    hi = t.reshape(-1).to(torch.bfloat16)
    return hi, (t.reshape(-1) - hi.float()).to(torch.bfloat16)


def bn_chain(x, mean, rstd, gamma, beta, act):
    """act(((x - mean) * rstd) * gamma + beta), each op rounded to fp32 on its own (eager torch)"""
    y = ((x - mean) * rstd) * gamma + beta
    if act >= 1:
        y = torch.clamp_min(y, 0.0)
    if act == 2:
        y = torch.clamp_max(y, 6.0)
    return y


def fq_chain(y, mn, mx, bits):
    """the activation fake-quant op chain of oracle/pf_oracle.uniform_quantize in fp32 torch, range (mn, mx) given"""
    alpha = (mx - mn) + torch.tensor(1e-10, dtype=torch.float32, device=y.device)
    k = torch.tensor(float(O.uq_k(bits)), dtype=torch.float32, device=y.device)
    lv = torch.round(((y - mn) / alpha) * k)
    return alpha * (lv / k) + mn, lv


def pool_ref(x, k, st, pt, pb, P, Q):
    """(y, first-max argmax code r * k + q, float64 dx of dy routed to it) with an unfold of the -inf padded input"""
    n, h, w, c = x.shape
    pr = (Q - 1) * st + k - w - pt
    xp = F.pad(x.permute(0, 3, 1, 2), (pt, pr, pt, pb), value=float('-inf'))
    cols = F.unfold(xp, k, stride=st).view(n, c, k * k, P * Q)
    y = cols.max(2).values
    idx = torch.arange(k * k, device=x.device).view(1, 1, -1, 1)
    at_max = cols == y.unsqueeze(2)
    am = torch.where(at_max, idx, k * k).min(2).values                          # first maximum, row-major
    ties = (at_max.sum(2) > 1).float().mean().item()
    return y.view(n, c, P, Q).permute(0, 2, 3, 1), am.view(n, c, P, Q).permute(0, 2, 3, 1), xp.shape, ties


def pool_dx_ref(dy, am, k, st, pt, P, Q, n, h, w, c, hp, wp):
    oh = torch.arange(P, device=dy.device).view(1, P, 1, 1)
    ow = torch.arange(Q, device=dy.device).view(1, 1, Q, 1)
    ih = oh * st + am // k
    iw = ow * st + am % k
    flat = ((torch.arange(n, device=dy.device).view(n, 1, 1, 1) * hp + ih) * wp + iw) * c + \
        torch.arange(c, device=dy.device).view(1, 1, 1, c)
    dxp = torch.zeros(n * hp * wp * c, dtype=torch.float64, device=dy.device)
    dxp.index_add_(0, flat.reshape(-1), dy.double().reshape(-1))
    return dxp.view(n, hp, wp, c)[:, pt:pt + h, pt:pt + w, :]


LEARNER_MODULE = {'uniform': 'uniform_quantization', 'non-uniform': 'nonuniform_quantization',
                  'full-prec': 'full_precision', 'weight-sparse': 'weight_sparsification',
                  'chn-pruned-gpu': 'channel_pruning_gpu', 'chn-pruned-rmt': 'channel_pruning_rmt'}
# what the tests build learners with beyond their own flags: no summaries or checkpoints inside a short run
QUIET = dict(summ_step=10 ** 9, save_step=10 ** 9)


def make(net_module, learner, batch, reload='ilsvrc12_dataset', **flags):
    """A learner as the command line would build it: FLAGS reset, the learner's module imported, the dataset module
    `reload` and the net module reloaded (each re-declares its defaults; reload=None: the net module imported as it
    is, with the defaults the last imported modules declared), `flags` set, then create_learner."""
    FLAGS.reset()
    importlib.import_module('pocketflow_b200.learners.%s.learner' % LEARNER_MODULE[learner])
    importlib.import_module('pocketflow_b200.learners.distillation_helper')
    if reload is not None:
        importlib.reload(importlib.import_module('pocketflow_b200.datasets.' + reload))
    mod = importlib.import_module('pocketflow_b200.nets.' + net_module)
    if reload is not None:
        mod = importlib.reload(mod)
    from pocketflow_b200.learners.learner_utils import create_learner
    FLAGS.learner, FLAGS.batch_size = learner, batch
    for k, v in flags.items():
        setattr(FLAGS, k, v)
    return create_learner(None, mod.ModelHelper())


# plan key: (feed, pass, classes, bn, aff, ring, b_stationary, a_fp32) — pass 0 fwd, 1 dgrad, 2 wgrad
KEY_FIELDS = ('feed', 'pass', 'classes', 'bn', 'aff', 'ring', 'b_stationary', 'a_fp32')


def plan_key(plan):
    return tuple(plan[f] for f in KEY_FIELDS)


def _required():
    req = set()
    for bn in (16, 32, 64, 128):
        for aff in (0, 1, 2):
            req.add((1, 0, 0, bn, aff, 0, 0, 0))               # TMA fwd: split / act levels / weight levels
        req.add((1, 1, 0, bn, 0, 0, 0, 0))                     # TMA unit-stride dgrad
        for stat in (0, 1):
            for fp32 in (0, 1):
                req.add((0, 0, 0, bn, 0, 0, stat, fp32))       # cp.async fwd: streamed / stationary weights
                req.add((0, 1, 0, bn, 0, 0, stat, fp32))       # cp.async dgrad (unit stride)
        req.add((0, 1, 1, bn, 0, 0, 0, 0))                     # strided dgrad by pixel-parity classes
        req.add((0, 1, 0, bn, 0, 0, 0, 0))                     # strided dgrad, classes off
    for aff in (0, 2):
        req.add((1, 0, 0, 64, aff, 2, 0, 0))                   # residual ring, depth 2
        req.add((1, 0, 0, 64, aff, 4, 0, 0))                   # residual ring, depth 4
    req.add((1, 1, 0, 64, 0, 2, 0, 0))                         # dgrad accumulate through the ring
    for bn in (64, 128):
        req.update({(1, 2, 0, bn, 0, 0, 0, 0), (1, 2, 0, bn, 1, 0, 0, 0), (0, 2, 0, bn, 0, 0, 0, 0)})
    return req


# Every variant the launchers can produce for the operand forms of test_tc_variants_gpu.py.  cp.async kernels never get a ring on sm_90:
# beside a 128 KB ring the shared memory holds fewer than two stages at BN >= 64 (pf_conv_tc.cu: launch_persist).
TC_REQUIRED = frozenset(_required())


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
    k = w.shape[-1]                                                       # w may have fewer output channels than d
    wm = w.permute(3, 2, 0, 1).reshape(k, c * r * s)
    return (wm @ cols).view(n, k, p, q).permute(0, 2, 3, 1)


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


class TcRecorder:
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
        outside = {k: v for k, v in self.plans.items() if k not in TC_REQUIRED}
        assert not outside, 'plans the variant sweep does not reach: %s' % {
            str(dict(zip(KEY_FIELDS, k))): v for k, v in outside.items()}


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


# (workload, batch, flag overrides): the benchmarked workloads at their batch, and the codebook learner also in the
# 'both' optimisation mode, where the codebook gradient runs
RUNS = [('resnet50_uq8_dst_b128', 128, None), ('mobilenet_cpg50_b256', 256, None), ('lenet_uq8_b128', 128, None),
        ('resnet50_ws50_dst_b128', 128, None), ('resnet50_nuq4_dst_b128', 128, None),
        ('resnet50_nuq4_dst_b128', 128, {'nuql_opt_mode': 'both'}), ('resnet20_uq8_dst_b256', 256, None),
        ('resnet20_ws50_dst_b256', 256, None)]


EXACT_BOUND = 1 << 24          # integers below this add exactly in fp32 in any order (pinned on wgmma below)


CHUNK_PIXELS = 1 << 20         # rows of one per-tap DGEMM in the references


def dims(d):
    """(n, h, w, c, k, r, s, p, q, sh, sw, pt, pl) of a descriptor or of such a tuple"""
    return d if isinstance(d, tuple) else geom(d)


def padded_hw(d):
    n, h, w, c, k, r, s, p, q, sh, sw, pt, pl = dims(d)
    return max((p - 1) * sh + r, pt + h), max((q - 1) * sw + s, pl + w)


def pad_input(x, d):
    """NHWC x inside a zero frame: top / left padding pt / pl, bottom / right as far as any window reaches"""
    n, h, w, c, k, r, s, p, q, sh, sw, pt, pl = dims(d)
    hp, wp = padded_hw(d)
    xp = torch.zeros(x.shape[0], hp, wp, x.shape[3], dtype=x.dtype, device=x.device)
    xp[:, pt:pt + h, pl:pl + w] = x
    return xp


def tap(xp, d, i, j):
    """[n, p, q, c] view of padded input xp that filter tap (i, j) reads at every output pixel"""
    n, h, w, c, k, r, s, p, q, sh, sw, pt, pl = dims(d)
    return xp[:, i:i + (p - 1) * sh + 1:sh, j:j + (q - 1) * sw + 1:sw]


def batch_chunks(d):
    n, p, q = dims(d)[0], dims(d)[7], dims(d)[8]
    step = max(1, CHUNK_PIXELS // max(p * q, 1))
    return [(n0, min(n, n0 + step)) for n0 in range(0, n, step)]


def conv_fwd_ref(x, w, d):
    """y[n, p, q, k] = sum over taps of x_tap @ w[i, j]  (x NHWC, w HWIO), in x's dtype"""
    n, h, wd, c, k, r, s, p, q = dims(d)[:9]
    y = torch.zeros(n, p, q, k, dtype=x.dtype, device=x.device)
    for n0, n1 in batch_chunks(d):
        xp = pad_input(x[n0:n1], d)
        for i in range(r):
            for j in range(s):
                y[n0:n1] += (tap(xp, d, i, j).reshape(-1, c) @ w[i, j]).view(n1 - n0, p, q, k)
    return y


def conv_dgrad_ref(dy, w, d):
    """dx of y = conv(x, w): every tap scatters dy @ w[i, j]^T into its strided slice of the padded input"""
    n, h, wd, c, k, r, s, p, q, sh, sw, pt, pl = dims(d)
    dx = torch.zeros(n, h, wd, c, dtype=dy.dtype, device=dy.device)
    for n0, n1 in batch_chunks(d):
        hp, wp = padded_hw(d)
        dxp = torch.zeros(n1 - n0, hp, wp, c, dtype=dy.dtype, device=dy.device)
        g = dy[n0:n1].reshape(-1, k)
        for i in range(r):
            for j in range(s):
                tap(dxp, d, i, j)[...] += (g @ w[i, j].t()).view(n1 - n0, p, q, c)
        dx[n0:n1] = dxp[:, pt:pt + h, pl:pl + wd]
    return dx


def conv_wgrad_ref(x, dy, d, bounds=None):
    """dw[i, j] = x_tap^T @ dy over the pixels (n, p, q) in row-major order; bounds = [0, b1, ..., Npix]: also the sum
    over each pixel range [b_s, b_s+1), as [ranges, r, s, c, k].  Returns (dw, per-range sums or None)."""
    n, h, wd, c, k, r, s, p, q = dims(d)[:9]
    dw = torch.zeros(r, s, c, k, dtype=x.dtype, device=x.device)
    parts = None if bounds is None else torch.zeros(len(bounds) - 1, r, s, c, k, dtype=x.dtype, device=x.device)
    for n0, n1 in batch_chunks(d):
        xp = pad_input(x[n0:n1], d)
        g = dy[n0:n1].reshape(-1, k)
        row0, row1 = n0 * p * q, n1 * p * q
        for i in range(r):
            for j in range(s):
                xt = tap(xp, d, i, j).reshape(-1, c)
                dw[i, j] += xt.t() @ g
                if bounds is None:
                    continue
                for sp in range(len(bounds) - 1):
                    a, b = max(bounds[sp], row0) - row0, min(bounds[sp + 1], row1) - row0
                    if a < b:
                        parts[sp, i, j] += xt[a:b].t() @ g[a:b]
    return dw, parts


def dw_fwd_ref(x, w, d):
    """depthwise: y[n, p, q, c] = sum over taps of x_tap * w[i, j]  (w [r, s, c])"""
    n, h, wd, c, k, r, s, p, q = dims(d)[:9]
    y = torch.zeros(n, p, q, c, dtype=x.dtype, device=x.device)
    for n0, n1 in batch_chunks(d):
        xp = pad_input(x[n0:n1], d)
        for i in range(r):
            for j in range(s):
                y[n0:n1] += tap(xp, d, i, j) * w[i, j]
    return y


def dw_dgrad_ref(dy, w, d):
    n, h, wd, c, k, r, s, p, q, sh, sw, pt, pl = dims(d)
    dx = torch.zeros(n, h, wd, c, dtype=dy.dtype, device=dy.device)
    for n0, n1 in batch_chunks(d):
        hp, wp = padded_hw(d)
        dxp = torch.zeros(n1 - n0, hp, wp, c, dtype=dy.dtype, device=dy.device)
        for i in range(r):
            for j in range(s):
                tap(dxp, d, i, j)[...] += dy[n0:n1] * w[i, j]
        dx[n0:n1] = dxp[:, pt:pt + h, pl:pl + wd]
    return dx


def dw_wgrad_ref(x, dy, d):
    n, h, wd, c, k, r, s, p, q = dims(d)[:9]
    dw = torch.zeros(r, s, c, dtype=x.dtype, device=x.device)
    for n0, n1 in batch_chunks(d):
        xp = pad_input(x[n0:n1], d)
        g = dy[n0:n1].reshape(-1, c)
        for i in range(r):
            for j in range(s):
                dw[i, j] += (tap(xp, d, i, j).reshape(-1, c) * g).sum(0)
    return dw


def split_terms(f, a, b):
    """f over operand planes a = [hi(, lo)], b = [hi(, lo)], without the lo.lo term the kernels drop:
    f(a_hi, b_hi (+ b_lo)) + f(a_lo, b_hi).  With absolute=True-style inputs this is the largest sum of |terms|."""
    bb = b[0] + b[1] if len(b) > 1 else b[0]
    out = f(a[0], bb)
    if len(a) > 1:
        out = out + f(a[1], b[0])
    return out


def int_values(shape, density, g, signed=True):
    """float32 tensor of 0 and (+-)1, each entry non-zero with probability `density`"""
    dev = g.device
    v = (torch.rand(shape, generator=g, device=dev) < density).float()
    if signed:
        v = v * torch.where(torch.rand(shape, generator=g, device=dev) < 0.5, -1.0, 1.0)
    return v


def wgrad_density(npix, nterms):
    """density of x and dy such that the expected sum of |terms| of a weight-gradient entry, npix * nterms * density^2,
    stays near 2^22 (at most 1/2)"""
    return min(0.5, (float(1 << 22) / (npix * nterms)) ** 0.5)


def reduction_operands(xshape, yshape, x_planes, y_planes, density, g, x_signed=True):
    """x [n, h, w, c] and dy [n, p, q, k] as lists of planes (one or two), integer valued, built so that every output
    pixel contributes a non-zero term to the weight gradient: channel 0 of x is +-1 in its hi plane and 0 in its lo
    plane everywhere, and every pixel of dy has one entry (at channel pixel % k) that is +-1 in hi and 0 in lo; so each
    pixel with an in-bounds tap puts x_hi * dy_hi != 0 into entry (tap, 0, pixel % k)."""
    xs = [int_values(xshape, density, g, x_signed) for _ in range(x_planes)]
    ys = [int_values(yshape, density, g) for _ in range(y_planes)]
    xs[0][..., 0] = torch.where(torch.rand(xshape[:3], generator=g, device=g.device) < 0.5, -1.0, 1.0) \
        if x_signed else 1.0
    for pl in xs[1:]:
        pl[..., 0] = 0.0
    n, p, q, k = yshape
    kf = (torch.arange(n * p * q, device=g.device) % k).view(n, p, q, 1)
    sign = torch.where(torch.rand(n, p, q, 1, generator=g, device=g.device) < 0.5, -1.0, 1.0)
    ys[0].scatter_(3, kf, sign)
    for pl in ys[1:]:
        pl.scatter_(3, kf, torch.zeros_like(sign))
    return xs, ys


def every_pixel_contributes(xs, ys):
    """the construction of reduction_operands holds: x channel 0 non-zero in hi and zero in lo at every position, and
    every pixel of dy has an entry non-zero in hi and zero in lo"""
    ok = bool((xs[0][..., 0] != 0).all()) and all(bool((pl[..., 0] == 0).all()) for pl in xs[1:])
    carrier = ys[0] != 0
    for pl in ys[1:]:
        carrier &= pl == 0
    return ok and bool(carrier.any(-1).all())


def write_fwd_weight(f_hi, f_lo, w_hi, w_lo):
    """inverse of fwd_weight: HWIO planes -> the K-major forward copy [k][Kpad] with columns
    in (r, s, c) order; the Kpad columns stay as they are (zero in a fresh TcWeights)"""
    r, s, c, k = w_hi.shape
    for dst, src in ((f_hi, w_hi), (f_lo, w_lo)):
        if dst is not None and src is not None:
            dst.view(k, -1)[:, :r * s * c] = src.permute(3, 0, 1, 2).reshape(k, r * s * c).to(dst.dtype)


def write_dgrad_weight(d_hi, d_lo, w_hi, w_lo):
    """inverse of dgrad_weight: HWIO planes -> the dgrad copy [c][Kpad_d], columns (r, s, k)"""
    r, s, c, k = w_hi.shape
    for dst, src in ((d_hi, w_hi), (d_lo, w_lo)):
        dst.view(c, -1)[:, :r * s * k] = src.permute(2, 0, 1, 3).reshape(c, r * s * k).to(dst.dtype)


def oracles(lrn):
    ex = lrn.sess_train
    teacher = StepOracle(ex.teacher.ops, ex.teacher.logits_t, lrn.images) if ex.teacher is not None else None
    return StepOracle(ex.ops, ex.logits_t, lrn.images, lrn.labels, ex.loss, ex.weight_quant, ex.act_quant, teacher)


def gpu_activation(ex, relu_op):
    """Value of a quantized activation as the consuming convolutions see it (fp32 copy, split planes or levels)."""
    bn = ex.fused_into.get(relu_op)
    pl = ex.xplanes.get(bn) if bn is not None else None
    if pl is None:
        return ex.T(relu_op.output).float().cpu().numpy()
    shape = relu_op.output.shape
    lv = ex.act_lv.get(bn)
    if lv is not None and ex._lv_on:
        hdr = lv['hdr'].cpu().numpy().view(ops.ACT_HDR)[0]
        if int(hdr['nplanes']) == 1:
            return (pl.hi.float() * float(hdr['scale'])).cpu().numpy().reshape(shape)
    return (pl.hi.float() + pl.lo.float()).cpu().numpy().reshape(shape)


def local_parity(ex, orc, state, img, training=True):
    """Teacher-forced comparison: (worst conv error relative to the output scale, # fused BN+act+quant elements on a
    different level, # such elements, worst non-flip difference in units of one level).  training=False: the device
    ran an inference-mode pass (moving statistics, no dropout), and so does the oracle.  A non-finite output (a buffer
    no kernel wrote, under PF_POISON) counts as an infinite error."""
    params = {k: torch.from_numpy(np.array(v, dtype=F32, copy=True)) for k, v in state.items()}
    force = {}
    for op in ex.ops:
        if op.type == 'GatherChannels':
            # a compact graph's channel gather, as the next conv reads it (fp32 or operand planes)
            y, pl = ex.outputs_of(op)
            if y is None:
                n = op.output.numel
                force[op.output.name] = (pl.hi[:n].float() + pl.lo[:n].float()).cpu().view(op.output.shape)
            else:
                force[op.output.name] = y.float().cpu().view(op.output.shape)
        elif any(c in ex.gather_fused for c in ex._consumers(op.output)):
            # a BN (+ activation) whose gather is fused into its apply (pf_bn_apply_gather) never writes its
            # full-width output: the oracle computes it, and the gather's output is compared instead
            continue
        elif op.type in ('Relu', 'Relu6'):
            force[op.output.name] = torch.from_numpy(np.ascontiguousarray(gpu_activation(ex, op)))
        elif op.type in ('Conv2D', 'MatMul', 'DepthwiseConv2dNative') and op not in ex.fused_add and op not in ex.fused_act:
            force[op.output.name] = ex.T(op.output).float().cpu()
        elif op.type in ('MaxPool', 'Add', 'Mean'):
            pl = ex.xplanes.get(op)                  # a linear bottleneck's Add that only its planes hold
            if pl is not None and not ex.bn_need_f32[op]:
                n = op.output.numel
                force[op.output.name] = (pl.hi[:n].float() + pl.lo[:n].float()).cpu().view(op.output.shape)
            else:
                force[op.output.name] = ex.T(op.output).float().cpu()
    local = {}
    with torch.no_grad():
        orc.forward(params, torch.from_numpy(img), training, force=force, local_out=local)
    worst_conv, worst_name, flips, total, worst_frac = 0.0, '', 0, 0, 0.0
    bits_of = dict(zip([o.name for o in ex.aq_ops], ex.act_quant['bits'])) if ex.aq_ops else {}
    for op in ex.ops:
        name = op.output.name
        if name not in force or name not in local:
            continue
        got, ref = force[name].numpy(), local[name].numpy()
        if not np.isfinite(got).all():
            worst_conv, worst_name = float('inf'), op.name + ' (non-finite)'
            continue
        if op.type in ('Relu', 'Relu6') and op.name in bits_of and int(bits_of[op.name]) <= 16:
            step = (float(ref.max()) - float(ref.min())) / float(2 ** int(bits_of[op.name]) - 1)
            if step > 0:
                dlev = np.abs(got - ref) / step
                f = dlev > 0.5
                flips += int(f.sum())
                total += ref.size
                if (~f).any():
                    worst_frac = max(worst_frac, float(dlev[~f].max()))
        else:
            e = float(np.abs(got - ref).max() / (np.abs(ref).max() + 1e-30))
            if e > worst_conv:
                worst_conv, worst_name = e, op.name
    return worst_conv, worst_name, flips, total, worst_frac


# bars of the backward tap (Parity)
BAR_DX = 2e-5          # of max|float64 reference|
BAR_W = 2e-5           # of the largest sum of |terms| of the reduction
BAR_CHAIN = 1e-6       # of the sum of |terms| per element
BAR_FWD = 4e-5         # of max|float64| of a forward output, layer-local (test_config_sweep_gpu.py explains it)
SPLIT = 2.0 ** -16     # |hi + lo - v| <= 2^-16 |v| for the bf16 split of an fp32 v (8 significant bits each)
# op types whose backward passes the gradient through unchanged (no launch)
THROUGH = ('Reshape', 'Identity', 'Dropout', 'Relu', 'Relu6')

# variables the tap does not compare, and why: {variable key in op.vars: reason}
VAR_EXEMPT = {
    'clusters': "codebooks in the non-uniform learner's 'weights' mode: frozen, so the step computes no gradient for "
                "them (cluster_grad runs only when they train); asserted: their gradient stays zero and the optimizer "
                "leaves them and their slots alone.  Trained codebooks are compared (Parity.codebook_terms)",
}


class Parity:
    """Taps one executor's backward pass; see the module docstring."""

    def __init__(self, ex, controls=False):
        self.ex, self.controls = ex, controls
        self.worst, self.checked_ops, self.var_ref, self.pending = {}, set(), {}, {}
        self.fails, self.ctrl, self._prev_gz = [], {}, {}
        self.only_of = {pl: ex.bn_gplanes_only[bn] for bn, pl in ex.bn_gplanes.items()}
        self.rec = None

    # ------------------------------------------------------------------------------------------ tap
    def install(self):
        ex = self
        e = self.ex
        grad_of, grad_target, lab = e.grad_of, e.grad_target, e.loss_and_backward

        def t_grad_of(t):
            g = grad_of(t)
            ex._boundary(t.op, g)
            return g

        def t_grad_target(t):
            buf, acc = grad_target(t)
            torch.cuda.synchronize()
            ex.rec['writes'].append((t, buf, acc, dbl(buf, t.shape) if acc else None))
            return buf, acc

        def t_loss_and_backward(*a, **k):
            ex.rec = dict(op=None, writes=[], dy=[])
            lab(*a, **k)
            torch.cuda.synchronize()
            ex._finish()
        e.grad_of, e.grad_target, e.loss_and_backward = t_grad_of, t_grad_target, t_loss_and_backward
        for lo in e.conv.values():
            self._wrap_conv(lo)

    def _wrap_conv(self, lo):
        wgrad, dgrad = lo.wgrad, lo.dgrad

        def used(gy):
            torch.cuda.synchronize()
            shape = lo.op.output.shape
            if getattr(lo, 'tc_wgrad', False):
                return planes_value(lo.dy, shape)
            return dbl(gy, shape)

        def t_wgrad(gy, ws, dw=None, dy_buf=None):
            wgrad(gy, ws, dw, dy_buf)
            self.rec['dy'].append(('wgrad', used(gy)))

        def t_dgrad(gy, gx, acc):
            dgrad(gy, gx, acc)
            self.rec['dy'].append(('dgrad', used(gy)))
        lo.wgrad, lo.dgrad = t_wgrad, t_dgrad

    def _boundary(self, op, g):
        torch.cuda.synchronize()
        self._finish()
        ex = self.ex
        shape = op.output.shape
        s = self.pending.pop(op.output, None)
        read = None
        if g is not None:
            pl = ex.conv_dy_planes.get(op)
            only = pl is not None and self.only_of[pl]
            read = (planes_value(pl, shape) if only else dbl(g, shape), only)
        self.rec = dict(op=op, writes=[], dy=[], read=read, sem=s)

    # ------------------------------------------------------------------------------------------ bookkeeping
    def note(self, tag, err, bar):
        self.worst[tag] = max(self.worst.get(tag, 0.0), err)
        if not err <= bar:
            self.fails.append((tag, self.rec['op'].name if self.rec['op'] is not None else 'loss', err, bar))

    def _contribute(self, t, c):
        s = self.pending.get(t)
        if s is None:
            self.pending[t] = [c.clone(), c.abs(), 1, c]
        else:
            s[0] += c
            s[1] += c.abs()
            s[2] += 1
            s[3] = c

    def _contribution(self, t, buf, acc, pre):
        """(what one grad_target write added to dL/dt, whether it is dy planes, the rounding allowed per element):
        post - pre of the buffer, which carries the fp32 rounding of the sum (half an ulp of post: 2^-24 |post|), or the dy
        planes that live in the buffer's memory"""
        op, shape = self.rec['op'], t.shape
        if op is not None and op.type == 'FusedBatchNorm' and self.ex.batch_norm[op].only:
            return planes_value(self.ex.bn_gplanes[op], shape), True, 0.0
        post = dbl(buf, shape)
        return ((post - pre), False, 2.0 ** -24 * post.abs()) if acc else (post, False, 0.0)

    def _finish(self):
        rec = self.rec
        if rec is None:
            return
        op, ex = rec['op'], self.ex
        writes = {}
        for t, buf, acc, pre in rec['writes']:
            assert t not in writes, ('two writes of one gradient by one op', op, t.name)
            writes[t] = self._contribution(t, buf, acc, pre)
        if op is None:                                            # the loss
            self._loss(writes)
        elif rec['read'] is not None and self._chain(rec):
            through = op.type in THROUGH and (ex._passthrough(op) or op in ex.fused_into)
            if through:
                self._contribute(op.inputs[0], rec['sem'][0].view(op.inputs[0].shape))
            else:
                getattr(self, '_op_' + op.type)(op, rec, writes)
                self.checked_ops.add(op)
                if op.type == 'Add':
                    for x in op.inputs:
                        if x not in writes:                       # the plan-time alias: the output's own buffer
                            self._contribute(x, rec['sem'][0])
        for t, (c, _, _) in writes.items():
            self._contribute(t, c)
        self.rec = None

    # ------------------------------------------------------------------------------------------ chain
    def _chain(self, rec):
        """the gradient the op read against the sum of its consumers' contributions; False: there were none"""
        op = rec['op']
        r, only = rec['read']
        s = rec['sem']
        if s is None:
            self.note('chain: a gradient no consumer wrote', float('inf'), BAR_CHAIN)
            return False
        tol = SPLIT * s[0].abs() if only else 0.0
        err = self._chain_err(r, s[0], s[1], tol)
        self.note('chain', err, BAR_CHAIN)
        if self.controls and 'dropped accumulate' not in self.ctrl and s[2] >= 2:
            self.ctrl['dropped accumulate'] = (self._chain_err(r, s[0] - s[3], s[1], tol) / BAR_CHAIN, op.name)
        return True

    @staticmethod
    def _chain_err(r, s, a, tol):
        ex_ = ((r - s).abs() - tol).clamp_min(0.0)
        return (ex_ / a.clamp_min(1e-300)).max().item()

    def gz_of(self, op, rec):
        """the upstream gradient of a conv / matmul times the mask of its fused ReLU (from the device's own output)"""
        r = rec['read'][0]
        if op in self.ex.fused_act:
            y = self.ex.buf[op.output].view(op.output.shape)
            r = r * (y > 0)
        return r

    # ------------------------------------------------------------------------------------------ local references
    def _loss(self, writes):
        ex, L = self.ex, self.ex.loss
        z_t = L.ce[1]
        (c, _, e), = [v for t, v in writes.items() if t is z_t]
        z = dbl(ex.T(z_t), z_t.shape).requires_grad_(True)
        lab = dbl(ex.T(ex.labels_t), z_t.shape)
        loss = (-(lab * torch.log_softmax(z, -1)).sum(-1)).mean()
        if L.dst is not None:
            assert L.dst[0] is z_t
            tl = dbl(ex.teacher.T(ex.teacher.logits_t), z_t.shape)
            w, T = L.dst[2], L.dst[3]
            loss = loss + w * (-(torch.softmax(tl / T, -1) * torch.log_softmax(z / T, -1)).sum(-1)).mean()
        g, = torch.autograd.grad(loss, [z])
        self.note('loss dlogits', max_rel(c, g, e), BAR_DX)
        self.checked_ops.add('loss')

    def _x_value(self, op):
        """the conv's input as its kernels read it: operand planes (hi + lo, or scale x level) or the fp32 buffer"""
        ex, lo, x = self.ex, self.ex.conv[op], op.inputs[0]
        xp = getattr(lo, 'xp', None)
        if xp is not None:
            if lo._levels():
                hdr = lo.x_lv['hdr'].cpu().numpy().view(ops.ACT_HDR)[0]
                if int(hdr['nplanes']) == 1:
                    return dbl(xp.hi, x.shape) * float(hdr['scale'])
            return planes_value(xp, x.shape)
        return dbl(ex.T(x), x.shape)

    def _wref(self, v, g, mag):
        self.var_ref[v] = (g.detach(), mag.detach())

    def _conv_ref(self, op, x, w, gz):
        """(dx, dW, |x|^T|gz|) of y = conv(x, w) (matmul) at upstream gz, float64 autograd"""
        xg, wg = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
        f = (lambda a, b: a @ b) if op.type == 'MatMul' else (lambda a, b: conv64(a, b, self.ex.desc[op]))
        dx, dw = torch.autograd.grad(f(xg, wg), [xg, wg], gz)
        wa = torch.zeros_like(w, requires_grad=True)
        mag, = torch.autograd.grad(f(x.abs(), wa), [wa], gz.abs())
        return dx, dw, mag

    def _op_Conv2D(self, op, rec, writes):
        ex = self.ex
        gz = self.gz_of(op, rec)
        lo = ex.conv[op]
        # what the kernels read is, bit for bit, what they were handed: the same planes, the split of the fp32 gradient
        # into planes, or the fp32 gradient itself
        want = gz if rec['read'][1] or not getattr(lo, 'tc_wgrad', False) else split_value(gz)
        for which, d in rec['dy']:
            self.note('conv dy read (%s)' % which, float(not torch.equal(d, want)), 0.0)
        kv = op.vars['kernel']
        w = dbl(ex.kernel_of(op), kv.shape)
        x = self._x_value(op) if op.inputs[0].op.type != 'Placeholder' else dbl(ex.T(op.inputs[0]), op.inputs[0].shape)
        # the reference takes that operand as it is (then only the kernels' own rounding is measured)
        dx, dw, mag = self._conv_ref(op, x, w, want)
        self._wref(kv, dw, mag)
        if 'bias' in op.vars:
            red = tuple(range(gz.dim() - 1))
            self._wref(op.vars['bias'], gz.sum(red), gz.abs().sum(red))
        if op.inputs[0].op.type == 'Placeholder':
            assert not writes
            return
        (c, _, e), = writes.values()
        self.note('conv dx', max_rel(c, dx, e), BAR_DX)
        if self.controls:
            self._conv_controls(op, x, w, gz, c, e)

    _op_MatMul = _op_Conv2D

    def _conv_controls(self, op, x, w, gz, c, e):
        ex = self.ex
        if 'unquantized kernel' not in self.ctrl and op in ex.qvars:
            w0 = dbl(ex.store.view(op.vars['kernel']), w.shape)
            self.ctrl['unquantized kernel'] = (max_rel(c, self._conv_ref(op, x, w0, gz)[0], e) / BAR_DX, op.name)
        key = (op.output.shape, tuple(w.shape))
        prev = self._prev_gz.get(key)
        if 'swapped gy' not in self.ctrl and prev is not None:
            self.ctrl['swapped gy'] = (max_rel(c, self._conv_ref(op, x, w, prev[1])[0], e) / BAR_DX,
                                       '%s with %s' % (op.name, prev[0]))
        if 'swapped gy' not in self.ctrl:
            self._prev_gz[key] = (op.name, gz)
        else:
            self._prev_gz.clear()

    def _op_DepthwiseConv2dNative(self, op, rec, writes):
        ex = self.ex
        gz = rec['read'][0]
        kv = op.vars['kernel']
        x = dbl(ex.T(op.inputs[0]), op.inputs[0].shape)
        w = dbl(ex.kernel_of(op), kv.shape)
        (sh, sw), (pt, pl), (kh, kw) = op.attrs['strides'], op.attrs['pad'], op.attrs['ksize']
        p, q, c_ = op.output.shape[1], op.output.shape[2], x.shape[-1]

        def f(a, b):
            pb = (p - 1) * sh + kh - a.shape[1] - pt
            pr = (q - 1) * sw + kw - a.shape[2] - pl
            y = F.conv2d(F.pad(a.permute(0, 3, 1, 2), (pl, pr, pt, pb)), b.permute(2, 3, 0, 1), stride=(sh, sw),
                         groups=c_)
            return y.permute(0, 2, 3, 1)
        xg, wg = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
        dx, dw = torch.autograd.grad(f(xg, wg), [xg, wg], gz)
        wa = torch.zeros_like(w, requires_grad=True)
        mag, = torch.autograd.grad(f(x.abs(), wa), [wa], gz.abs())
        self._wref(kv, dw, mag)
        if writes:
            (c, _, e), = writes.values()
            self.note('depthwise dx', max_rel(c, dx, e), BAR_DX)

    def _op_FusedBatchNorm(self, op, rec, writes):
        ex, st = self.ex, self.ex.store
        assert op.attrs['training'], 'a training step through an inference-mode BN'
        gy = rec['read'][0]
        x32 = ex.T(op.inputs[0]).view(op.inputs[0].shape)
        s = ex.bn[op]
        ga32, be32 = st.view(op.vars['gamma']), st.view(op.vars['beta'])
        act = ex.fused_act.get(op, 0)
        z = bn_chain(x32, s['mean'], s['rstd'], ga32, be32, 0)
        mask = torch.ones_like(z, dtype=torch.bool) if act == 0 else (z > 0)
        if act == 2:
            mask &= z < 6
        x, ga, be = x32.double().requires_grad_(True), ga32.double().requires_grad_(True), \
            be32.double().requires_grad_(True)
        red = tuple(range(x.dim() - 1))
        mean = x.mean(red)
        var = ((x - mean) ** 2).mean(red)
        xh = (x - mean) * torch.rsqrt(var + op.attrs['epsilon'])
        dz = gy * mask
        dx, dga, dbe = torch.autograd.grad(xh * ga + be, [x, ga, be], dz)
        xh = xh.detach()
        self._wref(op.vars['gamma'], dga, (dz * xh).abs().sum(red))
        self._wref(op.vars['beta'], dbe, dz.abs().sum(red))
        (c, planes, e), = writes.values()
        self.note('bn dx (dy planes)' if planes else 'bn dx', max_rel(c, dx, e), BAR_DX)

    def _op_MaxPool(self, op, rec, writes):
        x = op.inputs[0]
        n, h, w, c = x.shape
        _, p, q, _ = op.output.shape
        (kh, kw), (sh, sw), (pt, pl) = op.attrs['ksize'], op.attrs['strides'], op.attrs['pad']
        assert kh == kw and sh == sw and pt == pl
        hp, wp = max((p - 1) * sh + kh, pt + h), max((q - 1) * sw + kw, pl + w)
        am = self.ex.pool_argmax[op].long()
        ref = pool_dx_ref(rec['read'][0], am, kh, sh, pt, p, q, n, h, w, c, hp, wp)
        (cc, _, e), = writes.values()
        self.note('max-pool dx', max_rel(cc, ref, e), BAR_DX)

    def _op_Mean(self, op, rec, writes):
        n, h, w, c = op.inputs[0].shape
        ref = (rec['read'][0].reshape(n, 1, 1, c) / (h * w)).expand(n, h, w, c)
        (cc, _, e), = writes.values()
        self.note('mean dx', max_rel(cc, ref, e), BAR_DX)

    def _op_Add(self, op, rec, writes):
        for t, (c, _, e) in writes.items():
            self.note('add dx', max_rel(c, rec['read'][0].view(t.shape), e), BAR_DX)

    def _op_Softmax(self, op, rec, writes):
        x = dbl(self.ex.T(op.inputs[0]), op.inputs[0].shape).requires_grad_(True)
        ref, = torch.autograd.grad(torch.softmax(x, -1), [x], rec['read'][0])
        (c, _, e), = writes.values()
        self.note('softmax dx', max_rel(c, ref, e), BAR_DX)

    def _op_Dropout(self, op, rec, writes):
        m = self.ex.dropout[op].view(op.output.shape).double()
        ref = rec['read'][0] * m / float(F32(op.attrs['keep_prob']))
        (c, _, e), = writes.values()
        self.note('dropout dx', max_rel(c, ref, e), BAR_DX)

    # ------------------------------------------------------------------------------------------ after the step
    def codebook_terms(self):
        """Trained codebooks ('cluster' / 'both' mode): per quantized op (kernel's float64 gradient g, its sum of |terms|,
        the device's centroid index of every weight, alpha, codebook size 2^bits).  The quantizer's STE sends the
        gradient of the quantized kernel unchanged to the gathered centroid (utils.py:303-306), through the inverse
        scale: dL/dc_j = alpha * sum over {i: idx_i = j} of g_i."""
        ex, wq = self.ex, self.ex.wq
        assert not wq.use_buckets, 'bucketed codebook training has no float64 reference here'
        idx, rng, out = wq.idx.cpu().numpy(), wq.uq.ranges(), {}
        for i, op in enumerate(ex.wq_ops):
            kv = op.vars['kernel']
            g, mag = self.var_ref[kv]
            a = wq.idx_offsets[i]
            mn, mx = rng[i]
            alpha = float(F32(F32(mx[0]) - F32(mn[0])) + F32(1e-10))
            out[op] = (g, mag, torch.from_numpy(idx[a:a + kv.numel].astype(np.int64)).to(g.device), alpha,
                       1 << wq.uq.bits[i])
        return out

    @staticmethod
    def codebook_ref(shape, g, mag, idx, alpha, k):
        """(dL/dc, sum of |terms|) of one codebook variable of `shape` (entries >= k get no gradient)"""
        n = int(np.prod(shape))
        assert int(idx.max()) < k <= n
        ref = torch.zeros(n, dtype=torch.float64, device=g.device).index_add_(0, idx, g.reshape(-1)) * alpha
        m = torch.zeros(n, dtype=torch.float64, device=g.device).index_add_(0, idx, mag.reshape(-1)) * alpha
        return ref.view(shape), m.view(shape)

    def variables(self):
        """every trainable variable's gradient in G against its float64 reference; returns (compared, exempt)"""
        ex, st = self.ex, self.ex.store
        key_of = {v: k for op in ex.ops for k, v in op.vars.items()}
        done, exempt = 0, 0
        self.rec = dict(op=None)
        if ex.train_clusters:
            self.codebooks = self.codebook_terms()
            for op, t in self.codebooks.items():
                self._wref(op.vars['clusters'], *self.codebook_ref(op.vars['clusters'].shape, *t))
        for v in st.train_vars:
            g = st.view(v, ex.G).double()
            if v not in self.var_ref:
                assert key_of[v] in VAR_EXEMPT, ('variable gradient not compared', v.name)
                assert torch.count_nonzero(g) == 0, v.name
                exempt += 1
                continue
            ref, mag = self.var_ref.pop(v)
            assert torch.isfinite(g).all(), v.name
            err = ((g - ref).abs().max() / mag.max().clamp_min(1e-300)).item()
            self.worst['dW ' + key_of[v]] = max(self.worst.get('dW ' + key_of[v], 0.0), err)
            if not err <= BAR_W:
                self.fails.append(('dW', v.name, err, BAR_W))
            done += 1
        return done, exempt


def backward_ops(ex):
    """the ops of the executor that have a gradient and a backward of their own"""
    return [op for op in ex.ops if op.type != 'Placeholder' and not ex._passthrough(op) and op not in ex.fused_into]


def snapshot(ex):
    return dict(P=ex.store.P.clone(), O=ex.store.O.clone(), S1=ex.S1.clone(),
                S2=ex.S2.clone() if ex.S2 is not None else None, b1=ex.beta1_power, b2=ex.beta2_power)


def check_optimizer(ex, before, lr, frozen):
    """P, S1, S2 bit-exact per variable from the device's G; moving statistics within 1e-6 of float64"""
    st, o = ex.store, ex.optimizer
    wd_of = {v: float(c) for v, c in ex.loss.l2.items()}
    maskable = set(ex.maskable)
    G = ex.G.cpu().numpy()
    cur = {k: (t.cpu().numpy() if t is not None else None) for k, t in
           (('P', st.P), ('S1', ex.S1), ('S2', ex.S2))}
    old = {k: (before[k].cpu().numpy() if before[k] is not None else None) for k in ('P', 'S1', 'S2')}
    mask = ex.MASK.cpu().numpy() if ex.MASK is not None else None
    n = 0
    for v in st.train_vars:
        a, b = st.offset[v], st.offset[v] + v.numel
        sl = lambda d, k: d[k][a:b].reshape(v.shape)       # noqa: E731
        if v.name in frozen:
            for k in ('P', 'S1', 'S2'):
                if cur[k] is not None:
                    assert np.array_equal(sl(cur, k), sl(old, k)), (v.name, k)
            continue
        g = G[a:b].reshape(v.shape)
        wd = wd_of.get(v, 0.0)
        if o['kind'] == 'adam':
            w1, m1, v1 = O.adam_step(sl(old, 'P'), sl(old, 'S1'), sl(old, 'S2'), g, lr, F32(before['b1']),
                                     F32(before['b2']), o.get('beta1', 0.9), o.get('beta2', 0.999), o.get('eps', 1e-8),
                                     wd, ex.grad_scale)
            want = dict(P=w1, S1=m1, S2=v1)
        else:
            mk = mask[a:b].reshape(v.shape) if (v in maskable and mask is not None) else None
            w1, a1 = O.momentum_step(sl(old, 'P'), sl(old, 'S1'), g, lr, o.get('momentum', 0.9), mk, wd, ex.grad_scale)
            want = dict(P=w1, S1=a1)
        for k, ref in want.items():
            assert np.array_equal(sl(cur, k).view(np.uint32), np.asarray(ref, F32).view(np.uint32)), (v.name, k)
        n += 1
    # BN moving statistics from the device's own batch statistics
    worst = 0.0
    for op in ex.ops:
        if op.type != 'FusedBatchNorm' or not op.attrs['training'] or not ex.update_moving_stats:
            continue
        c = op.output.shape[-1]
        m = op.output.numel // c
        mom = float(F32(op.attrs['momentum']))
        s = ex.bn[op]
        mean, var = s['mean'].double(), s['var'].double()
        unbiased = var * m / max(m - 1, 1)
        for vk, stat, scale in (('moving_mean', mean, mean.abs() + var.sqrt()), ('moving_variance', unbiased, unbiased)):
            v = op.vars[vk]
            a = st.offset[v]
            prior = before['O'][a:a + c].double()
            ref = prior * mom + stat * (1.0 - mom)
            got = st.view(v).double()
            err = ((got - ref).abs() / (prior.abs() * mom + scale * (1.0 - mom)).clamp_min(1e-30)).max().item()
            worst = max(worst, err)
    assert worst <= 1e-6, worst
    return n, worst


def run_parity(name, lrn, frozen=(), controls=False):
    ex = lrn.sess_train
    assert ex._graph is None, 'the tap needs an eager step'
    t0 = time.time()
    images, labels = lrn.iterator_train.next_batch()
    ex.buf[lrn.images].copy_(images)
    ex.buf[lrn.labels].copy_(labels)
    before = snapshot(ex)
    lr = lrn.lrn_rate(ex.step_count)
    par = Parity(ex, controls)
    par.install()
    ex.run_step(lr)
    torch.cuda.synchronize()
    assert not par.pending or all(t.op.type == 'Placeholder' for t in par.pending), \
        ('gradients nobody read', [t.name for t in par.pending if t.op.type != 'Placeholder'])
    want_ops = backward_ops(ex)
    missing = [op.name for op in want_ops if op not in par.checked_ops]
    assert not missing, ('ops with a gradient that were not checked', missing)
    assert 'loss' in par.checked_ops
    nvar, nexempt = par.variables()
    want_vars = len(ex.store.train_vars)
    nopt, worst_mov = check_optimizer(ex, before, lr, set(frozen))
    secs = time.time() - t0
    worst = {k: float('%.3g' % v) for k, v in sorted(par.worst.items())}
    print('%s: %d backward ops + the loss checked (of %d), %d variable gradients compared (+ %d exempt, of %d), '
          '%d optimizer updates bit-exact, moving statistics %.2e; worst %s; %.0f s' % (
              name, len(par.checked_ops) - 1, len(want_ops), nvar, nexempt, want_vars, nopt, worst_mov, worst, secs))
    record('backward_' + name, ops=len(par.checked_ops) - 1, variables=nvar, exempt=nexempt, moving_stats=worst_mov,
           seconds=round(secs), **worst)
    assert not par.fails, par.fails[:20]
    assert nvar + nexempt == want_vars and nopt + len(frozen) == want_vars
    if controls:
        print('%s: negative controls (error / bar): %s' % (name, par.ctrl))
        assert set(par.ctrl) == {'unquantized kernel', 'swapped gy', 'dropped accumulate'}, par.ctrl
        for k, (ratio, where) in par.ctrl.items():
            assert ratio > 10.0, (k, ratio, where)
        record('backward_%s_controls' % name, **{k: r for k, (r, _) in par.ctrl.items()})
    return par


class CompactParity(Parity):
    """Parity's tap (every op's backward rebuilt alone in float64 from the device's own
    inputs and upstream gradient, the chain of contributions, coverage) with the backward of a channel gather:
    dx[..., c] = dy[..., j] where index[j] == c, zero elsewhere.  A scatter that writes a whole buffer must give those
    bits; one that accumulates, the fp32 sum; one that emits dy planes alone, their bf16 split."""

    def __init__(self, ex):
        super().__init__(ex)
        self.scatters = []                                   # (op, accumulate, dy planes, planes only)

    def _contribution(self, t, buf, acc, pre):
        op = self.rec['op']
        if op is not None and op.type == 'GatherChannels' and self.ex.bn_gplanes_only.get(op, False):
            return planes_value(self.ex.bn_gplanes[op], t.shape), True, 0.0
        return super()._contribution(t, buf, acc, pre)

    def _op_GatherChannels(self, op, rec, writes):
        idx = torch.from_numpy(np.asarray(op.attrs['index'], np.int64)).to(DEV)
        gy = rec['read'][0]
        ref = torch.zeros(op.inputs[0].shape, dtype=torch.float64, device=DEV)
        ref[..., idx[idx >= 0]] = gy[..., idx >= 0]
        (t, (c, planes, e)), = writes.items()
        acc = [a for tt, _, a, _ in rec['writes'] if tt is t][0]
        self.scatters.append((op, acc, op in self.ex.bn_gplanes, planes))
        if acc or planes:
            self.note('scatter dx (accumulate)' if acc else 'scatter dx (dy planes)', max_rel(c, ref, e), BAR_DX)
        else:
            self.note('scatter dx', float(not torch.equal(c, ref)), 0.0)


def tapped_step(cex, lr):
    """one eager step of `cex` under the tap: every backward op and the loss against float64, every variable's gradient,
    the optimizer update bit for bit from the device's gradient, the moving statistics.  Returns the tap."""
    before = snapshot(cex)
    par = CompactParity(cex)
    par.install()
    cex.run_step(lr)
    torch.cuda.synchronize()
    assert all(t.op.type == 'Placeholder' for t in par.pending), [t.name for t in par.pending]
    missing = [op.name for op in backward_ops(cex) if op not in par.checked_ops]
    assert not missing and 'loss' in par.checked_ops, missing
    nvar, nexempt = par.variables()
    nopt, _ = check_optimizer(cex, before, lr, set())
    print('compact step: %d backward ops, %d variable gradients, %d updates bit-exact; worst %s'
          % (len(par.checked_ops) - 1, nvar, nopt, {k: float('%.3g' % v) for k, v in sorted(par.worst.items())}))
    assert not par.fails, par.fails[:20]
    assert nexempt == 0 and nvar == nopt == len(cex.store.train_vars)
    del cex.grad_of, cex.grad_target, cex.loss_and_backward          # the tap lives on the instances: take it off
    for lo in cex.conv.values():
        del lo.wgrad, lo.dgrad
    return par


def prune_interior(lrn, ratio, seed):
    """zero int(cin * ratio) random input channels of every maskable kernel but the first and the last, and set the
    learner's masks from them (what the selection leaves behind)"""
    ex = lrn.sess_train
    lrn.init_from_full()
    rng = np.random.RandomState(seed)
    for v in lrn.maskable_vars[1:-1]:
        w = ex.store.view(v)
        cin = w.shape[2]
        w[:, :, torch.from_numpy(rng.permutation(cin)[:int(cin * ratio)]).to(DEV), :] = 0.0
    for v in lrn.maskable_vars:
        ops.cpg_channel_mask(ex.store.view(v), ex.store.view(v, ex.MASK))
    ex.reset_optimizer_state()


MASK32 = 0xffffffff


def philox4x32_10(ctr, key):
    """numpy restatement of Philox4x32-10 (Salmon et al., SC'11): ctr [..., 4] uint32, key (k0, k1)"""
    c = [ctr[..., i].astype(np.uint64) for i in range(4)]
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    m0, m1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
    for r in range(10):
        if r:
            k0, k1 = (k0 + np.uint64(0x9E3779B9)) & np.uint64(MASK32), (k1 + np.uint64(0xBB67AE85)) & np.uint64(MASK32)
        p0, p1 = m0 * c[0], m1 * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & np.uint64(MASK32)
        hi1, lo1 = p1 >> np.uint64(32), p1 & np.uint64(MASK32)
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
    return np.stack(c, -1).astype(np.uint32)


def ref_mask(n, keep, seed, rank, step, stream=0):
    """counter (element group [2 words], step [low word], stream), key (seed, rank)"""
    g = np.arange((n + 3) // 4, dtype=np.uint64)
    ctr = np.stack([g & np.uint64(MASK32), g >> np.uint64(32), np.full_like(g, step & MASK32),
                    np.full_like(g, stream)], -1).astype(np.uint32)
    w = philox4x32_10(ctr, (seed, rank)).reshape(-1)[:n]
    u = ((w & np.uint32(0x7fffff)) | np.uint32(0x3f800000)).view(np.float32) - np.float32(1.0)
    return np.floor(np.float32(keep) + u).astype(np.float32)


def mapped_mask(rows, layout, cfull, keep, seed, rank, step, stream=0):
    """pf_dropout_fwd_mapped in numpy: element (row, j) of the compact [rows, len(layout)] tensor takes the uniform of
    full-width element f = row * cfull + layout[j], word f & 3 of Philox block f >> 2; padding (layout[j] < 0) is 0"""
    lay = np.asarray(layout, np.int64)
    f = (np.arange(rows, dtype=np.uint64)[:, None] * np.uint64(cfull) + np.maximum(lay, 0).astype(np.uint64)[None, :])
    g = f >> np.uint64(2)
    ctr = np.stack([g & np.uint64(MASK32), g >> np.uint64(32), np.full_like(g, step & MASK32),
                    np.full_like(g, stream)], -1).astype(np.uint32)
    w = np.take_along_axis(philox4x32_10(ctr, (seed, rank)), (f & np.uint64(3)).astype(np.int64)[..., None], -1)[..., 0]
    u = ((w & np.uint32(0x7fffff)) | np.uint32(0x3f800000)).view(np.float32) - np.float32(1.0)
    m = np.floor(np.float32(keep) + u).astype(np.float32)
    m[:, lay < 0] = 0.0
    return m


def train_graph(net):
    import make_golden_chn_export as M
    mod, flags = M.NETS[net]
    FLAGS.reset()
    for k, v in flags.items():
        setattr(FLAGS, k, v)
    mh = importlib.import_module('pocketflow_b200.nets.' + mod).ModelHelper()
    return C.build_train_graph(mh, 2)


def seed_state(g, lg, rng):
    return {v.name: np.asarray(v.initializer(rng, v.shape), np.float32) + (0.5 if v.name.endswith('beta:0') else 0.0)
            for op in C.reachable_ops(g, lg) for v in op.vars.values()}


def kept_channels(w):
    return int((np.square(w).sum(axis=(0, 1, 3)) > 0).sum())


def check_selection(lrn, full_state):
    ex = lrn.sess_train
    assert len(lrn.selection_log) == lrn.nb_layers
    for rec, v in zip(lrn.selection_log, lrn.maskable_vars):
        w = ex.store.view(v).cpu().numpy()
        cin = w.shape[2]
        assert rec['nnz_target'] == int(cin * (1.0 - rec['ratio']))
        assert np.all(rec['err'] < 1e-6)
        # the search meets its target, or stops only once its bracket is below 1e-8 (:803): from 0.1 that takes more
        # than 20 halvings.  A ratio-0 layer (target = Cin) always meets it.
        if rec['ratio'] == 0.0:
            assert rec['nnz'] == cin, v.name
        if rec['nnz'] != rec['nnz_target']:
            assert len(rec['search']) > 20, (v.name, rec['search'])
        assert kept_channels(w) == rec['nnz'], v.name
        # the channels the search dropped are zero; the kept ones were refit
        assert np.all(w[:, :, rec['mask'] == 0, :] == 0)
    # layer 0: ratio 0, still sampled, searched and refit — every channel kept, the weights changed
    w0 = ex.store.view(lrn.maskable_vars[0]).cpu().numpy()
    full0 = full_state[lrn.conv_ops_full[0].vars['kernel'].name]
    assert lrn.prune_ratios[0] == 0.0 and lrn.selection_log[0]['nnz_target'] == w0.shape[2] == kept_channels(w0)
    assert not np.array_equal(w0, full0)


def grad_inputs(ex, op):
    """Tensors whose gradient buffer op's backward WRITES (mirrors Executor.loss_and_backward)."""
    if op.type in ('Placeholder', 'Reshape', 'Identity') or op in ex.fused_into:
        return []
    ins = op.inputs if op.type == 'Add' else op.inputs[:1]
    out = []
    for t in ins:
        if t.op.type == 'Placeholder':
            continue
        if op.type == 'Add' and ex.gkey(t) is ex.gkey(op.output):
            continue                                   # shared buffer: the Add's backward is a no-op for this input
        out.append(t)
    return out


def expected_contributions(ex, t, memo):
    """The set of WRITER ops whose contributions make up dL/dt."""
    if t in memo:
        return memo[t]
    s = set()
    for c in ex._consumers(t):
        if c.type in ('Reshape', 'Identity') or c in ex.fused_into:
            s |= expected_contributions(ex, c.output, memo)              # pass-through: same gradient
        elif c.type == 'Add' and ex.gkey(t) is ex.gkey(c.output):
            s |= expected_contributions(ex, c.output, memo)              # identity: shares the Add output's gradient
        else:
            s.add(c)
    if t is ex.loss.ce[1] or (t in ex.alias and False):
        s.add('loss')
    memo[t] = s
    return s


# ---------------------------------------------------------------------------------------------- integer models
# The four integer inference models (int8.IntModel): network module, its flags, the int8 options.  The weight buckets
# are per channel on the ResNets and per layer on the MobileNets, so both forms of the weight scales run.
INT8_MODELS = {
    'resnet20_narrow': ('resnet_at_cifar10', dict(resnet_size=20, uql_use_buckets=True, uql_bucket_type='channel'),
                        dict(int8_narrow=True)),
    'resnet50': ('resnet_at_ilsvrc12', dict(resnet_size=50, uql_use_buckets=True, uql_bucket_type='channel'), {}),
    'mobilenet_v1_depthwise': ('mobilenet_at_ilsvrc12', {}, dict(int8_depthwise=True)),
    'mobilenet_v2_depthwise_narrow': ('mobilenet_at_ilsvrc12', dict(mobilenet_version=2, nb_classes=1001),
                                      dict(int8_depthwise=True, int8_narrow=True)),
}

# Every integer layer of those models, in graph order of first appearance: (kind, H, W, Cin, Cout, R, S, stride,
# pad top, pad left, P, Q, kernel, layers of that shape).  kind 'conv' runs pf_conv2d_u8_fwd on its TMA-fed kernel
# ('tma', where pf_conv2d_u8_supported holds) or its cp.async-fed one ('cp.async'); kind 'dw' runs pf_dwconv_u8_fwd
# on its row-blocked kernel ('rows': 3 x 3, equal strides, P >= 2) or its one-pixel kernel ('pixel').  The shapes do
# not depend on the batch.  tests/test_int8_edges_cpu.py checks these lists against int8.select on the graphs, and
# the kernel tests parametrize over them.
INT8_LAYERS = {
    'resnet20_narrow': [
        ('conv', 32, 32, 16, 16, 1, 1, 1, 0, 0, 32, 32, 'cp.async', 1),
        ('conv', 32, 32, 16, 16, 3, 3, 1, 1, 1, 32, 32, 'cp.async', 6),
        ('conv', 32, 32, 16, 32, 1, 1, 2, 0, 0, 16, 16, 'cp.async', 1),
        ('conv', 32, 32, 16, 32, 3, 3, 2, 1, 1, 16, 16, 'cp.async', 1),
        ('conv', 16, 16, 32, 32, 3, 3, 1, 1, 1, 16, 16, 'cp.async', 5),
        ('conv', 16, 16, 32, 64, 1, 1, 2, 0, 0, 8, 8, 'cp.async', 1),
        ('conv', 16, 16, 32, 64, 3, 3, 2, 1, 1, 8, 8, 'cp.async', 1),
        ('conv', 8, 8, 64, 64, 3, 3, 1, 1, 1, 8, 8, 'tma', 5),
    ],
    'resnet50': [
        ('conv', 56, 56, 64, 256, 1, 1, 1, 0, 0, 56, 56, 'tma', 4),
        ('conv', 56, 56, 64, 64, 1, 1, 1, 0, 0, 56, 56, 'tma', 1),
        ('conv', 56, 56, 64, 64, 3, 3, 1, 1, 1, 56, 56, 'tma', 3),
        ('conv', 56, 56, 256, 64, 1, 1, 1, 0, 0, 56, 56, 'tma', 2),
        ('conv', 56, 56, 256, 512, 1, 1, 2, 0, 0, 28, 28, 'tma', 1),
        ('conv', 56, 56, 256, 128, 1, 1, 1, 0, 0, 56, 56, 'tma', 1),
        ('conv', 56, 56, 128, 128, 3, 3, 2, 1, 1, 28, 28, 'tma', 1),
        ('conv', 28, 28, 128, 512, 1, 1, 1, 0, 0, 28, 28, 'tma', 4),
        ('conv', 28, 28, 512, 128, 1, 1, 1, 0, 0, 28, 28, 'tma', 3),
        ('conv', 28, 28, 128, 128, 3, 3, 1, 1, 1, 28, 28, 'tma', 3),
        ('conv', 28, 28, 512, 1024, 1, 1, 2, 0, 0, 14, 14, 'tma', 1),
        ('conv', 28, 28, 512, 256, 1, 1, 1, 0, 0, 28, 28, 'tma', 1),
        ('conv', 28, 28, 256, 256, 3, 3, 2, 1, 1, 14, 14, 'tma', 1),
        ('conv', 14, 14, 256, 1024, 1, 1, 1, 0, 0, 14, 14, 'tma', 6),
        ('conv', 14, 14, 1024, 256, 1, 1, 1, 0, 0, 14, 14, 'tma', 5),
        ('conv', 14, 14, 256, 256, 3, 3, 1, 1, 1, 14, 14, 'tma', 5),
        ('conv', 14, 14, 1024, 2048, 1, 1, 2, 0, 0, 7, 7, 'tma', 1),
        ('conv', 14, 14, 1024, 512, 1, 1, 1, 0, 0, 14, 14, 'tma', 1),
        ('conv', 14, 14, 512, 512, 3, 3, 2, 1, 1, 7, 7, 'tma', 1),
        ('conv', 7, 7, 512, 2048, 1, 1, 1, 0, 0, 7, 7, 'tma', 3),
        ('conv', 7, 7, 2048, 512, 1, 1, 1, 0, 0, 7, 7, 'tma', 2),
        ('conv', 7, 7, 512, 512, 3, 3, 1, 1, 1, 7, 7, 'tma', 2),
    ],
    'mobilenet_v1_depthwise': [
        ('dw', 112, 112, 32, 32, 3, 3, 1, 1, 1, 112, 112, 'rows', 1),
        ('dw', 112, 112, 64, 64, 3, 3, 2, 0, 0, 56, 56, 'rows', 1),
        ('conv', 56, 56, 64, 128, 1, 1, 1, 0, 0, 56, 56, 'tma', 1),
        ('dw', 56, 56, 128, 128, 3, 3, 1, 1, 1, 56, 56, 'rows', 1),
        ('conv', 56, 56, 128, 128, 1, 1, 1, 0, 0, 56, 56, 'tma', 1),
        ('dw', 56, 56, 128, 128, 3, 3, 2, 0, 0, 28, 28, 'rows', 1),
        ('conv', 28, 28, 128, 256, 1, 1, 1, 0, 0, 28, 28, 'tma', 1),
        ('dw', 28, 28, 256, 256, 3, 3, 1, 1, 1, 28, 28, 'rows', 1),
        ('conv', 28, 28, 256, 256, 1, 1, 1, 0, 0, 28, 28, 'tma', 1),
        ('dw', 28, 28, 256, 256, 3, 3, 2, 0, 0, 14, 14, 'rows', 1),
        ('conv', 14, 14, 256, 512, 1, 1, 1, 0, 0, 14, 14, 'tma', 1),
        ('dw', 14, 14, 512, 512, 3, 3, 1, 1, 1, 14, 14, 'rows', 5),
        ('conv', 14, 14, 512, 512, 1, 1, 1, 0, 0, 14, 14, 'tma', 5),
        ('dw', 14, 14, 512, 512, 3, 3, 2, 0, 0, 7, 7, 'rows', 1),
        ('conv', 7, 7, 512, 1024, 1, 1, 1, 0, 0, 7, 7, 'tma', 1),
        ('dw', 7, 7, 1024, 1024, 3, 3, 1, 1, 1, 7, 7, 'rows', 1),
        ('conv', 7, 7, 1024, 1024, 1, 1, 1, 0, 0, 7, 7, 'tma', 1),
    ],
    'mobilenet_v2_depthwise_narrow': [
        ('dw', 112, 112, 32, 32, 3, 3, 1, 1, 1, 112, 112, 'rows', 1),
        ('conv', 112, 112, 32, 16, 1, 1, 1, 0, 0, 112, 112, 'cp.async', 1),
        ('dw', 112, 112, 96, 96, 3, 3, 2, 0, 0, 56, 56, 'rows', 1),
        ('dw', 56, 56, 144, 144, 3, 3, 1, 1, 1, 56, 56, 'rows', 1),
        ('dw', 56, 56, 144, 144, 3, 3, 2, 0, 0, 28, 28, 'rows', 1),
        ('conv', 28, 28, 144, 32, 1, 1, 1, 0, 0, 28, 28, 'cp.async', 1),
        ('dw', 28, 28, 192, 192, 3, 3, 1, 1, 1, 28, 28, 'rows', 2),
        ('conv', 28, 28, 192, 32, 1, 1, 1, 0, 0, 28, 28, 'cp.async', 2),
        ('dw', 28, 28, 192, 192, 3, 3, 2, 0, 0, 14, 14, 'rows', 1),
        ('conv', 14, 14, 192, 64, 1, 1, 1, 0, 0, 14, 14, 'tma', 1),
        ('dw', 14, 14, 384, 384, 3, 3, 1, 1, 1, 14, 14, 'rows', 4),
        ('conv', 14, 14, 384, 64, 1, 1, 1, 0, 0, 14, 14, 'tma', 3),
        ('conv', 14, 14, 384, 96, 1, 1, 1, 0, 0, 14, 14, 'cp.async', 1),
        ('dw', 14, 14, 576, 576, 3, 3, 1, 1, 1, 14, 14, 'rows', 2),
        ('conv', 14, 14, 576, 96, 1, 1, 1, 0, 0, 14, 14, 'cp.async', 2),
        ('dw', 14, 14, 576, 576, 3, 3, 2, 0, 0, 7, 7, 'rows', 1),
        ('conv', 7, 7, 576, 160, 1, 1, 1, 0, 0, 7, 7, 'cp.async', 1),
        ('dw', 7, 7, 960, 960, 3, 3, 1, 1, 1, 7, 7, 'rows', 3),
        ('conv', 7, 7, 960, 160, 1, 1, 1, 0, 0, 7, 7, 'cp.async', 2),
        ('conv', 7, 7, 960, 320, 1, 1, 1, 0, 0, 7, 7, 'tma', 1),
    ],
}


def int8_graph(key, batch, weight_bits=8, activation_bits=8):
    """(graph, images, logits, int8 config) of INT8_MODELS[key]'s inference graph at `batch`, with FLAGS set as the
    uniform learner of that model would have them"""
    from pocketflow_b200 import int8
    net, flags, opts = INT8_MODELS[key]
    mod = importlib.import_module('pocketflow_b200.nets.' + net)
    importlib.import_module('pocketflow_b200.learners.uniform_quantization.learner')
    FLAGS.reset()
    for k, v in flags.items():
        setattr(FLAGS, k, v)
    FLAGS.uql_weight_bits, FLAGS.uql_activation_bits = weight_bits, activation_bits
    g, images, logits = C.build_eval_graph(mod.ModelHelper(), batch)
    return g, images, logits, dict(int8.config_from_flags(), **opts)
