"""The backward pass and the optimizer update of the benchmarked training steps, layer by layer, against float64.

The step tests compare gradients with a free-running oracle only where no activation level or ReLU gate differs
(test_bench_configs_gpu); at 8-bit activations that never happens, so the wiring of the backward pass — which dy planes
a dgrad reads, which levels a wgrad is fed, whether a residual gradient is accumulated, where the STE, the weight decay
and the momentum mask land — had no graph-level check.  Here one eager step runs with the executor's backward tapped
(no change to the engine: its `grad_of` / `grad_target` and the lowerings' wgrad / dgrad / BN backward are wrapped on
the instance), synchronising at every op boundary, and the backward is teacher-forced:
  * LOCAL: every op that has a gradient is rebuilt alone in float64 through autograd, with StepOracle's semantics for
    its type, from the device's own forward inputs as the op read them (operand planes as hi + lo, activation levels as
    scale x level, quantized weights from ex.QW) and the device's own upstream gradient as the op read it (the fp32
    gradient, or the dy planes of the BN backward where the lowering reads those).  Every discrete decision comes from
    the device: ReLU masks from the fp32 chain ((x - mean) * rstd) * gamma + beta on the saved statistics (bn_chain),
    ReLU masks of convolutions with a fused activation from their own output, the max-pool argmax, the dropout mask and
    the teacher's logits — so no flipped level or gate can make a difference and no comparison is gated on one.
    Bars: a gradient contribution to an activation within 2e-5 of max|float64|; a variable's gradient in ex.G after
    the step (split-K reduce, STE) within 2e-5 of the largest sum of |terms|; the dy operand a convolution's kernels
    read is bit for bit the gradient it was handed (times its ReLU mask), or the bf16 split of it.
  * CHAIN: the gradient each op read equals the sum of the contributions its output's consumers wrote, by the graph's
    semantics (Add / Reshape / Identity / a fused activation pass their gradient through), within 1e-6 of the sum of
    |terms| per element: this covers the plan-time Add aliases, the in-place shortcut accumulators, the dy planes that
    live in the fp32 gradient buffer's memory and the passthrough ops.
  * OPTIMIZER: given the device's final G and the state before the step, P, S1 and S2 are bit-exact per variable
    against oracle.pf_oracle.adam_step / momentum_step with the loss's own weight decay, the step's masks and the
    frozen codebooks; the BN moving statistics within 1e-6 of the float64 update from the device's batch statistics.
  * COVERAGE: every op of the executor that has a gradient is checked locally and every trainable variable's gradient
    is compared, except what EXEMPT lists with its reason.
  * CONTROLS (default workload, once): a dgrad referenced with the unquantized kernel, one convolution's gradient
    swapped with a same-shaped neighbour's and a dropped accumulate at a residual each miss their bar by more than 10x.
A second test checks that the multi-stream schedule does not change a bit of the benchmarked step (the tap above
synchronises, so it cannot see a side-stream race).
Worst errors go to parity_flips.json in $PF_PARITY_DIR (default: the system temp directory); DESIGN.md §4 quotes them.
"""
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

from oracle import pf_oracle as O  # noqa: E402
from test_bench_configs_gpu import record  # noqa: E402
from test_nn_variants_gpu import bn_chain  # noqa: E402
from test_tc_bench_layers_gpu import conv64  # noqa: E402
from pocketflow_b200 import ops  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
F32 = np.float32

BAR_DX = 2e-5          # of max|float64 reference|
BAR_W = 2e-5           # of the largest sum of |terms| of the reduction
BAR_CHAIN = 1e-6       # of the sum of |terms| per element
SPLIT = 2.0 ** -16     # |hi + lo - v| <= 2^-16 |v| for the bf16 split of an fp32 v (8 significant bits each)
# op types whose backward passes the gradient through unchanged (no launch)
THROUGH = ('Reshape', 'Identity', 'Dropout', 'Relu', 'Relu6')

# not compared, and why: {variable key in op.vars: reason}
EXEMPT = {
    'clusters': "codebooks in the non-uniform learner's 'weights' mode: frozen, so the step computes no gradient for "
                "them (cluster_grad runs only when they train); asserted: their gradient stays zero and the optimizer "
                "leaves them and their slots alone.  Trained codebooks are compared (Parity.codebook_terms)",
}


def dbl(t, shape):
    return t.reshape(-1)[:int(np.prod(shape))].double().view(shape)


def planes_value(pl, shape):
    n = int(np.prod(shape))
    return (pl.hi[:n].double() + pl.lo[:n].double()).view(shape)


def split_value(v):
    """hi + lo of the bf16 split of an fp32-valued float64 tensor, as the split kernels write it"""
    v = v.float()
    hi = v.to(torch.bfloat16)
    return hi.double() + (v - hi.float()).to(torch.bfloat16).double()


def max_rel(got, ref, slack=0.0):
    """max |got - ref| relative to max|ref|, after `slack` per element (the fp32 rounding of an accumulate)"""
    assert torch.isfinite(got).all(), 'non-finite gradient'
    return (((got - ref).abs() - slack).clamp_min(0.0).max() / ref.abs().max().clamp_min(1e-300)).item()


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
        from test_nn_variants_gpu import pool_dx_ref
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
                assert key_of[v] in EXEMPT, ('variable gradient not compared', v.name)
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


def free():
    gc.collect()
    torch.cuda.empty_cache()


def build(workload, batch, monkeypatch, **flags):
    import bench
    monkeypatch.setenv('PF_POISON', '1')
    if flags:
        net, size, learner, over, descr = bench.WORKLOADS[workload]
        monkeypatch.setitem(bench.WORKLOADS, workload, (net, size, learner, dict(over, **flags), descr))
    return bench.build_learner(workload, 1, batch)


@pytest.mark.parametrize('workload,batch,flags', [
    ('resnet50_uq8_dst_b128', 128, {}),
    ('resnet20_uq8_dst_b256', 256, {}),
    ('resnet50_uq8_dst_b128', 2, {'uql_activation_bits': 32}),
    ('resnet50_ws50_dst_b128', 2, {}),
    ('resnet50_nuq4_dst_b128', 2, {}),
    ('mobilenet_cpg50_b256', 2, {}),
    ('lenet_uq8_b128', 2, {}),
], ids=['resnet50_uq8_b128', 'resnet20_uq8_b256', 'resnet50_w8a32_b2', 'resnet50_ws50_b2', 'resnet50_nuq4_b2',
        'mobilenet_cpg50_b2', 'lenet_uq8_b2'])
def test_backward_and_update_match_float64_layer_by_layer(workload, batch, flags, monkeypatch):
    import bench
    lrn = build(workload, batch, monkeypatch, **flags)
    ex = lrn.sess_train
    frozen = ()
    if bench.WORKLOADS[workload][2] == 'non-uniform':
        frozen = tuple(op.vars['clusters'].name for op in ex.wq_ops if 'clusters' in op.vars)
        assert frozen and not ex.train_clusters
    name = '%s_b%d' % (workload.rsplit('_b', 1)[0], batch) + ''.join('_%s%s' % kv for kv in sorted(flags.items()))
    controls = workload == 'resnet50_uq8_dst_b128' and batch == 128 and not flags
    if controls:
        assert ex.act_lv and ex.w_lv and ex.bn_gplanes and any(ex.bn_gplanes_only.values())
    try:
        run_parity(name, lrn, frozen, controls)
    finally:
        del lrn, ex
        free()


def test_mobilenet_v2_uniform_backward_matches_float64_layer_by_layer(monkeypatch):
    """the linear-bottleneck BN + residual (bn_add) and dropout backward"""
    import importlib
    from pocketflow_b200.flags import FLAGS
    monkeypatch.setenv('PF_POISON', '1')
    FLAGS.reset()
    import pocketflow_b200.datasets.ilsvrc12_dataset as D
    importlib.reload(D)
    from pocketflow_b200.nets import mobilenet_at_ilsvrc12 as M
    importlib.reload(M)
    from pocketflow_b200.learners.learner_utils import create_learner
    import pocketflow_b200.learners.uniform_quantization.learner  # noqa: F401
    FLAGS.batch_size, FLAGS.learner, FLAGS.nb_classes, FLAGS.mobilenet_version = 2, 'uniform', 1001, 2
    FLAGS.uql_weight_bits, FLAGS.uql_activation_bits = 8, 8
    FLAGS.uql_use_buckets, FLAGS.uql_bucket_type = True, 'channel'
    lrn = create_learner(None, M.ModelHelper())
    ex = lrn.sess_train
    assert len(ex.bn_add) == 10 and len(ex.dropout) == 1
    try:
        run_parity('mobilenet_v2_uq8_b2', lrn)
    finally:
        del lrn, ex
        free()


def test_overlapped_step_is_bit_identical_to_serial_at_the_benchmarked_batch(monkeypatch):
    """resnet50_uq8_dst_b128 at batch 128: one eager step with PF_OVERLAP=0 and one with PF_OVERLAP=1 (teacher forward
    and weight gradients on side streams) from the same state and batch: P, O, S1, S2 and the losses bit for bit"""
    import bench
    out, start = [], None
    for overlap in ('0', '1'):
        monkeypatch.setenv('PF_OVERLAP', overlap)
        lrn = bench.build_learner('resnet50_uq8_dst_b128', 1, 128)
        ex = lrn.sess_train
        assert ex.overlap == (overlap == '1') and ex._graph is None
        if start is None:
            images, labels = lrn.iterator_train.next_batch()
            start = (ex.store.P.cpu(), ex.store.O.cpu(), ex.teacher.store.P.cpu(), ex.teacher.store.O.cpu(),
                     images.clone(), labels.clone())
        else:
            ex.store.P.copy_(start[0])
            ex.store.O.copy_(start[1])
            ex.teacher.store.P.copy_(start[2])
            ex.teacher.store.O.copy_(start[3])
            for f in ex.teacher.store.listeners:
                f()
        ex.buf[lrn.images].copy_(start[4])
        ex.buf[lrn.labels].copy_(start[5])
        ex.run_step(lrn.lrn_rate(0))
        torch.cuda.synchronize()
        out.append((ex.store.P.cpu(), ex.store.O.cpu(), ex.S1.cpu(), ex.S2.cpu(), ex.fetch_losses()))
        del lrn, ex                                   # one benchmarked learner on the device at a time
        free()
    (p0, o0, m0, v0, l0), (p1, o1, m1, v1, l1) = out
    assert torch.equal(p0, p1) and torch.equal(o0, o1) and torch.equal(m0, m1) and torch.equal(v0, v1)
    assert all(F32(l0[k]).view(np.uint32) == F32(l1[k]).view(np.uint32) for k in l0), (l0, l1)
