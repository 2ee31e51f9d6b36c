"""Executor: lowers a `graph.Graph` to launches of libpf_b200.so kernels (forward, backward,
gradient reduction, optimizer) and replays them through a CUDA graph.

This is the stand-in for `sess.run(train_op)` into TensorFlow's executor
(/root/reference/learners/uniform_quantization/learner.py:114-152): one call = one training step
on one GPU.  State layout: all trainable parameters, their gradients and the
optimizer slots live in FLAT fp32 buffers so that (a) the data-parallel gradient reduction is one
collective over one buffer (SURVEY §8e) and (b) the optimizer / mask / weight-decay work is a
handful of launches instead of ~110 per step.
"""
import contextlib
import os
from collections import OrderedDict

import numpy as np
import torch

from . import ops
from .utils.multi_gpu_wrapper import MultiGpuWrapper as mgw

F32 = np.float32
MATMUL_TYPES = ('Conv2D', 'MatMul', 'DepthwiseConv2dNative')
ACT_TYPES = {'Relu': 1, 'Relu6': 2}


def _align4(n):
    return (n + 3) // 4 * 4


class _ConvLowering:
    """How one Conv2D / MatMul runs, fixed at plan time; this class: the exact-fp32 CUDA-core kernels.
    wgrad writes dL/dW into `dw`, or (None) into the plan's target; dy_buf: bf16 buffer to split an external gy into."""
    side = False                     # the weight gradient may run on the side stream (both operands are planes)

    def __init__(self, ex, op):
        self.ex, self.op, self.d, self.x = ex, op, ex.desc[op], op.inputs[0]
        # the residual Add and the folded inference BN (_BnFolded) of the epilogue: tensor-core lowerings only
        self.res = ex.fused_add[op][1] if op in ex.fused_add else None
        self.bn_out = ex.batch_norm[ex.bn_fold[op]].bn_out if op in ex.bn_fold else None

    def _epilogue(self):
        """(bias, fused relu, output buffer) of the forward kernel"""
        op, ex = self.op, self.ex
        return ex.store.view(op.vars['bias']) if 'bias' in op.vars else None, op in ex.fused_act, ex.buf[op.output]

    def _target(self, dw):
        return dw if dw is not None else self.ex.store.view(self.op.vars['kernel'], self.ex.G)

    def prepare_weights(self):
        """refresh the tensor-core copy of the kernel (inference executors that own their parameters)"""

    def forward(self):
        with self.ex.timed('conv_fwd'):
            ops.conv2d_fwd(self.d, self.ex.T(self.x), self.ex.kernel_of(self.op), *self._epilogue())

    def wgrad(self, gy, ws, dw=None, dy_buf=None):
        ops.conv2d_wgrad(self.d, self.ex.T(self.x), gy, ws, self._target(dw))

    def dgrad(self, gy, gx, acc):
        ops.conv2d_dgrad(self.d, gy, self.ex.kernel_of(self.op), self.ex.wt_ws, acc, gx)


class _TcConv(_ConvLowering):
    """Tensor-core conv: x from its producer's planes (integer levels in training passes where it writes them) or fp32;
    with a tensor-core wgrad, dy from the BN backward's planes or split into the shared scratch, for wgrad and dgrad."""

    def __init__(self, ex, op):
        super().__init__(ex, op)
        self.tw, self.xp, self.w_lv = ex.tc[op], ex.planes_of(self.x), ex.w_lv.get(op)
        self.x_lv = ex.act_lv.get(ex._root(self.x).op) if self.xp is not None else None
        self.tc_wgrad = op in ex.tc_wgrad
        if self.tc_wgrad:
            self.xw = ops.Planes(self.x.numel, ex.device, ex.x_scratch.buf) if self.xp is None else self.xp
            self.dy_split = op not in ex.conv_dy_planes
            self.dy = ops.Planes(op.output.numel, ex.device, ex.dy_scratch.buf) if self.dy_split \
                else ex.conv_dy_planes[op]
            self.part = ex.wg_part.get(op)
            self.side = self.xp is not None and not self.dy_split

    def _levels(self):
        return self.ex._lv_on and self.x_lv is not None

    def _x_act(self):
        lv = self.x_lv
        return ops.tc_act(self.xp, lv['hdr'], lv['csum'], lv['nseg'])

    def _wt(self):
        lv = self.w_lv
        if lv is not None and self.ex.wq.bits[lv['index']] <= 8:
            return ops.tc_wt(self.tw.f_hi, None, lv['alpha'], lv['beta'], lv['ncols'] > 1, self.ex.wq.bits[lv['index']])
        return ops.tc_wt(self.tw.f_hi, self.tw.f_lo)

    def prepare_weights(self):
        self.tw.prepare(self.ex.kernel_of(self.op))

    def forward(self):
        ex = self.ex
        res = ex.T(self.res) if self.res is not None else None
        with ex.timed('conv_fwd'):
            if self._levels():
                ops.conv2d_tc_fwd_ex(self.d, self._x_act(), self._wt(), *self._epilogue(), res)
            elif self.xp is not None:
                ops.conv2d_tc_fwd_planes(self.d, self.xp, self.tw, *self._epilogue(), res, self.bn_out)
            else:
                ops.conv2d_tc_fwd(self.d, ex.T(self.x), self.tw, *self._epilogue(), res, self.bn_out)

    def wgrad(self, gy, ws, dw=None, dy_buf=None):
        if not self.tc_wgrad:
            return super().wgrad(gy, ws, dw)
        if self.xp is None:
            ops.split_bf16(self.ex.T(self.x), self.xw)
        dyp = self.dy if dy_buf is None else ops.Planes(self.op.output.numel, self.ex.device, dy_buf)
        if dy_buf is not None or self.dy_split:
            ops.split_bf16(gy, dyp)
        if dw is None and self.part is not None:
            ws = self.part                   # split-K partials, summed into the flat gradient after the backward pass
        else:
            dw = self._target(dw)
        if self._levels():
            ops.conv2d_tc_wgrad_ex(self.d, self._x_act(), ops.tc_act(dyp), ws, dw)
        else:
            ops.conv2d_tc_wgrad_planes(self.d, self.xw, dyp, ws, dw)

    def dgrad(self, gy, gx, acc):
        if self.tc_wgrad:
            ops.conv2d_tc_dgrad_planes(self.d, self.dy, self.tw, acc, gx)
        else:
            ops.conv2d_tc_dgrad(self.d, gy, self.tw, acc, gx)


class _StemConv(_ConvLowering):
    """First layer (its input is the image: no dgrad): a tensor-core conv over the columns / space-to-depth planes of
    ex.im2col[op], with the kernel re-arranged into that layout and its gradient mapped back."""

    def __init__(self, ex, op):
        super().__init__(ex, op)
        self.im = ex.im2col[op]
        self.s2d = self.im['mode'] == 's2d'

    def prepare_weights(self):
        im, wk = self.im, self.ex.kernel_of(self.op)
        if self.s2d:
            ops.gather_rows(wk, im['fwd_map'], im['wpad'], wk.shape[-1])
        else:
            ops.add(wk.reshape(-1), None, im['wpad'][:wk.numel()])       # rows >= R*S*C stay zero
        im['tw'].prepare(im['wpad'])

    def forward(self):
        ex, im = self.ex, self.im
        with ex.timed('conv_prep'):
            if im['compute']:
                x = ex.T(self.x)
                if self.s2d:
                    ops.s2d_planes(x, *self.op.attrs['pad'], im['d1'].h, im['d1'].w, im['d1'].c, im['cols'])
                else:
                    (ops.im2col_planes if im['planes'] else ops.im2col)(self.d, x, im['kpad'], im['cols'])
                if ex.cols_event is not None:
                    ex.cols_event.record()
            elif ex.cols_wait is not None:
                torch.cuda.current_stream().wait_event(ex.cols_wait)
            if not ex.static_weights:
                self.prepare_weights()
        with ex.timed('conv_fwd'):
            fwd = ops.conv2d_tc_fwd_planes if im['planes'] else ops.conv2d_tc_fwd
            fwd(im['d1'], im['cols'], im['tw'], *self._epilogue())

    def wgrad(self, gy, ws, dw=None, dy_buf=None):
        im, dw = self.im, self._target(dw)
        if im['planes']:
            dyp = ops.Planes(self.op.output.numel, self.ex.device, self.ex.dy_scratch.buf if dy_buf is None else dy_buf)
            ops.split_bf16(gy, dyp)
            if 'pair' in im:
                pr = im['pair']
                ops.conv2d_tc_wgrad_planes(pr['d'], im['cols'], dyp, ws, pr['dw'])
                ops.fold_diag_blocks(pr['dw'], pr['g'], im['kpad'], im['d1'].k, im['dwpad'])
            else:
                ops.conv2d_tc_wgrad_planes(im['d1'], im['cols'], dyp, ws, im['dwpad'])
        else:
            ops.conv2d_wgrad(im['d1'], im['cols'], gy, ws, im['dwpad'])
        if self.s2d:
            ops.gather_rows(im['dwpad'], im['bwd_map'], dw, dw.shape[-1])
        else:
            ops.add(im['dwpad'][:dw.numel()], None, dw.reshape(-1))


def _u8_operands(lo, layout):
    """an integer layer's operands (Executor.int_layers): the _U8Bn of its input's producer, and its weight levels in
    `layout`, scales and bits"""
    ex = lo.ex
    levels, alpha, beta, lo.bits = ex.int_layers[lo.op]
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(ex.device)
    lo.bn = ex.batch_norm[ex._root(lo.x).op]
    lo.wl, lo.alpha, lo.beta = up(layout(levels)), up(np.asarray(alpha, F32)), up(np.asarray(beta, F32))


class _U8Conv(_ConvLowering):
    """Integer layer: the u8 tensor-core conv (pf_conv2d_u8_fwd) from the levels of its input's producer and its own
    weight levels [Cout, R*S*Cin], with a tensor-core lowering's residual and folded BN; no split-bf16 weight copy."""

    def __init__(self, ex, op):
        super().__init__(ex, op)
        _u8_operands(self, lambda lv: lv.reshape(-1, lv.shape[-1]).T)

    def forward(self):
        ex, (bias, relu, y) = self.ex, self._epilogue()
        res = ex.T(self.res) if self.res is not None else None
        with ex.timed('conv_fwd'):
            ops.conv2d_u8_fwd(self.d, self.bn.levels, self.bn.hdr, self.bn.csum, self.wl, self.alpha, self.beta,
                              self.bits, y, bias, relu, res, self.bn_out)


class _DwConv:
    """How one DepthwiseConv2dNative runs, fixed at plan time; this class: the exact-fp32 CUDA-core kernels."""

    def __init__(self, ex, op):
        self.ex, self.op, self.d, self.x = ex, op, ex.desc[op], op.inputs[0]

    def forward(self):
        ex = self.ex
        with ex.timed('dwconv'):
            ops.dwconv_fwd(self.d, ex.T(self.x), ex.kernel_of(self.op), ex.buf[self.op.output])

    def backward(self, gy):
        ex = self.ex
        with ex.timed('dwconv'):
            ops.dwconv_wgrad(self.d, ex.T(self.x), gy, ex.wgrad_ws, ex.store.view(self.op.vars['kernel'], ex.G))
            if self.x.op.type != 'Placeholder':
                gx, acc = ex.grad_target(self.x)
                ops.dwconv_dgrad(self.d, gy, ex.kernel_of(self.op), acc, gx)


class _U8DwConv(_DwConv):
    """Integer depthwise layer: pf_dwconv_u8_fwd from the levels of its input's producer and its own weight levels
    [R*S, C]."""

    def __init__(self, ex, op):
        super().__init__(ex, op)
        _u8_operands(self, lambda lv: lv.reshape(-1, lv.shape[-2]))

    def forward(self):
        with self.ex.timed('dwconv'):
            ops.dwconv_u8_fwd(self.d, self.bn.levels, self.bn.hdr, self.wl, self.alpha, self.beta, self.bits,
                              self.ex.buf[self.op.output])


class _BnLowering:
    """How one FusedBatchNorm runs, fixed at plan time; this class: the apply, with the quantizer of its fused ReLU in
    the same pass (integer levels where it writes them).  `writes`: the op whose fp32 output / planes it writes."""

    def __init__(self, ex, op, writes=None):
        st, s = ex.store, ex.bn[op]
        self.ex, self.op, self.x = ex, op, op.inputs[0]
        c = op.output.shape[-1]
        m = op.output.numel // c
        gamma, beta = st.view(op.vars['gamma']), st.view(op.vars['beta'])
        mm, mv, eps = st.view(op.vars['moving_mean']), st.view(op.vars['moving_variance']), op.attrs['epsilon']
        momentum = op.attrs['momentum'] if ex.update_moving_stats else 1.0
        self.act = ex.fused_act.get(op, 0)
        self.y, (self.y_out, self.pl) = ex.buf[op.output], ex.outputs_of(writes or op)
        # the activation quantizer (an index into act_quant['bits'], which set_quant_bits changes) and its levels
        self.aq, self.lv = ex._aq_of_bn(op), ex.act_lv.get(op)
        self.slot = ex.aq_slots[self.aq] if self.aq is not None else None
        # launch arguments after x: statistics pass (which with a quantizer also yields the range of act(bn(x))),
        # batch-statistics apply (training), moving-statistics apply and its outputs (with a quantizer: fp32 + range)
        q = (gamma, beta, self.act, self.slot) if self.slot is not None else ()
        self.stats = (m, c, eps, momentum, s['mean'], s['var'], s['rstd'], mm, mv) + q
        self.batch = (m, c, s['mean'], s['rstd'], gamma, beta)
        self.moving = (m, c, mm, mv, eps, gamma, beta)
        self.eval_out = (self.y, self.slot, None) if self.slot is not None else (self.y_out, None, self.pl)
        if ex.train:
            self.dparams = st.view(op.vars['gamma'], ex.G), st.view(op.vars['beta'], ex.G)
            self.gp = ex.bn_gplanes.get(op)                          # the dy planes of the conv that reads dL/dx
            self.only = self.gp is not None and ex.bn_gplanes_only[op]

    def forward(self, training):
        """the one per-pass choice: batch statistics in training passes of a training-mode BN, else moving statistics"""
        ex, x = self.ex, self.ex.T(self.x)
        batch_stats = self.op.attrs['training'] and training
        if batch_stats and ex.aq_static and self.slot is not None:
            # bn_train_stats_range would fold this batch's range into the static range slot, which nothing resets
            raise RuntimeError('%s: a batch-statistics pass in an executor with static activation ranges' % self.op.name)
        if batch_stats:
            with ex.timed('bn_stats'):
                (ops.bn_train_stats if self.slot is None else ops.bn_train_stats_range)(x, *self.stats, ex.bn_ws)
        with ex.timed('bn_apply'):
            self._apply(x, batch_stats)
        if self.slot is not None and not batch_stats and not ex.aq_static:
            # the BN apply wrote fp32 (+ range), the quantizer the planes
            with ex.timed('act_quant'):
                ops.act_quant(self.y, self.y_out, self.slot, ex.act_quant['bits'][self.aq], self.pl)

    def _apply(self, x, batch_stats):
        bits = self.ex.act_quant['bits'][self.aq] if self.slot is not None else None
        if not batch_stats and self.slot is not None and self.ex.aq_static:    # calibrated range: one clamping pass
            ops.bn_apply_eval_quant_static(x, *self.moving, self.act, self.slot, bits, self.y_out, self.pl)
        elif not batch_stats:
            ops.bn_apply_eval(x, *self.moving, self.act, *self.eval_out)
        elif self.slot is None:
            ops.bn_apply(x, *self.batch, self.act, self.y_out, None, self.pl)
        elif self.ex._lv_on and self.lv is not None:
            ops.bn_apply_quant_levels(x, *self.batch, self.act, self.slot, bits, self.y_out, self.pl, self.lv['hdr'],
                                      self.lv['csum'])
        else:
            ops.bn_apply_quant(x, *self.batch, self.act, self.slot, bits, self.y_out, self.pl)

    def backward(self, gy):
        gx, acc = self.ex.grad_target(self.x)
        assert not (self.only and acc)
        with self.ex.timed('bn_bwd'):
            ops.bn_bwd(gy, self.ex.T(self.x), *self.batch, self.act, *self.dparams, None if self.only else gx, acc,
                       self.ex.bn_ws, self.gp)


class _BnAdd(_BnLowering):
    """Linear bottleneck (Executor.bn_add): bn(x) + shortcut, written as the residual Add's output."""

    def __init__(self, ex, op):
        add_op, self.other = ex.bn_add[op]
        super().__init__(ex, op, add_op)

    def _apply(self, x, batch_stats):
        if batch_stats:
            ops.bn_apply_add(x, *self.batch, self.ex.T(self.other), self.y_out, self.pl)
        else:
            ops.bn_apply_add_eval(x, *self.moving, self.ex.T(self.other), self.y_out, self.pl)


class _BnGather(_BnLowering):
    """BN (+ activation) that writes the channel gather reading it (Executor.bn_gather).  Its backward is the base
    class's: the gather's own backward has scattered dL/dy into this BN's full-width gradient buffer by then."""

    def __init__(self, ex, op):
        super().__init__(ex, op, ex.bn_gather[op])
        self.idx = ex.gather_idx[ex.bn_gather[op]]

    def _apply(self, x, batch_stats):
        if batch_stats:
            ops.bn_apply_gather(x, *self.batch, self.act, self.idx, self.y_out, self.pl)
        else:
            ops.bn_apply_eval_gather(x, *self.moving, self.act, self.idx, self.y_out, self.pl)


class _BnFolded(_BnLowering):
    """Inference-mode BN that the conv producing its input applies in its epilogue (Executor.bn_fold), from `bn_out`."""

    def __init__(self, ex, op):
        super().__init__(ex, op)
        self.bn_out = ops.TcBnOut(*self.moving[2:], self.act, self.y_out, self.pl)

    def forward(self, training):
        """applied by the producing conv's epilogue"""


class _U8Bn:
    """Inference BN + quantized ReLU that feeds integer layers: writes the u8 levels, header and channel sums they read
    (pf_bn_eval_levels_u8; pf_bn_eval_levels_u8_static in one pass with a calibrated range), after its fake-quant
    lowering `base` when other readers need the fp32 tensor or planes."""

    def __init__(self, ex, op, base):
        self.ex, self.op, self.base, self.others = ex, op, base, ex.u8_others[op]
        c = op.output.shape[-1]
        self.levels = torch.empty(op.output.numel, dtype=torch.uint8, device=ex.device)
        self.hdr = torch.zeros(2, dtype=torch.int32, device=ex.device)
        self.csum = torch.empty(op.output.numel // c * ((c + 127) // 128), dtype=torch.float32, device=ex.device)

    def forward(self, training):
        ex, base = self.ex, self.base
        if self.others:
            base.forward(training)
        x, bits = ex.T(self.op.inputs[0]), ex.act_quant['bits'][base.aq]
        with ex.timed('act_quant'):
            if ex.aq_static:
                ops.bn_eval_levels_u8_static(x, *base.moving, base.act, bits, base.slot, self.levels, self.hdr,
                                             self.csum)
            else:
                ops.bn_eval_levels_u8(x, *base.moving, base.act, bits, base.slot, self.levels, self.hdr, self.csum,
                                      have_range=self.others)


class ParamStore:
    """Flat storage for the trainable variables of one model scope (+ separate non-trainable store).

    Order: maskable variables first, then by weight-decay coefficient, so that the optimizer runs
    over at most a few contiguous ranges."""

    def __init__(self, variables, device, wd_of=None, maskable=None, seed=1, frozen=None):
        """frozen: trainable variables the optimizer must NOT update (they still count in the weight-decay loss and
        receive gradients): the codebooks in the non-uniform learner's 'weights' mode, everything but the codebooks in
        its 'cluster' mode (learners/nonuniform_quantization/learner.py:252-268).  They form their own ranges."""
        self.device = device
        wd_of = wd_of or {}
        maskable = set(maskable or [])
        frozen = set(frozen or [])
        train = [v for v in variables if v.trainable]
        other = [v for v in variables if not v.trainable]
        key = lambda v: (0 if v in maskable else 1, 1 if v in frozen else 0, -float(wd_of.get(v, 0.0)))
        order = sorted(range(len(train)), key=lambda i: (key(train[i]), i))
        self.train_vars = [train[i] for i in order]
        self.other_vars = other
        self.offset, self.ranges = {}, []      # ranges: (start, end, masked, wd)
        self.frozen_ranges = set()             # (start, end) of the ranges the optimizer skips
        pos = 0
        cur = None

        def close(cur, pos):
            self.ranges.append((cur[0], pos, cur[2], cur[3]))
            if cur[4]:
                self.frozen_ranges.add((cur[0], pos))
        for v in self.train_vars:
            k = (v in maskable, float(wd_of.get(v, 0.0)), v in frozen)
            if cur is None or cur[2:] != k:
                if cur is not None:
                    close(cur, pos)
                cur = (pos, None) + k
            self.offset[v] = pos
            pos += _align4(v.numel)
        if cur is not None:
            close(cur, pos)
        self.n_train = max(pos, 4)
        self.n_masked = max([e for (s, e, m, w) in self.ranges if m] + [0])
        opos = 0
        for v in other:
            self.offset[v] = opos
            opos += _align4(v.numel)
        self.n_other = max(opos, 4)
        self.P = torch.zeros(self.n_train, dtype=torch.float32, device=device)
        self.O = torch.zeros(self.n_other, dtype=torch.float32, device=device)
        self.listeners = []                     # called after every bulk (re)load of the parameters
        self.init(seed)

    def init(self, seed):
        rng = np.random.default_rng(seed)
        hp = np.zeros(self.n_train, F32)
        for v in sorted(self.train_vars, key=lambda v: v.name):
            hp[self.offset[v]:self.offset[v] + v.numel] = v.initializer(rng, v.shape).reshape(-1)
        ho = np.zeros(self.n_other, F32)
        for v in self.other_vars:
            ho[self.offset[v]:self.offset[v] + v.numel] = v.initializer(rng, v.shape).reshape(-1)
        self.P.copy_(torch.from_numpy(hp))
        self.O.copy_(torch.from_numpy(ho))
        for f in self.listeners:
            f()

    def view(self, v, flat=None):
        buf = flat if flat is not None else (self.P if v.trainable else self.O)
        o = self.offset[v]
        return buf[o:o + v.numel].view(v.shape)

    def state_dict(self):
        d = OrderedDict()
        for v in self.train_vars + self.other_vars:
            d[v.name] = self.view(v).detach().cpu().numpy().copy()
        return d

    def load_state_dict(self, d, strict=True, require=None, optional=()):
        """Copy the variables `d` names into the store.  Returns (trainable variables found, trainable variables).
        strict: every variable must be present.  require ('any' | 'all' | None) applies to the TRAINABLE variables of a
        non-strict load: a checkpoint of another net / scope matches nothing and must not pass for a restore;
        variables whose name contains one of the `optional` substrings are not required."""
        found = 0
        for v in self.train_vars + self.other_vars:
            if v.name in d:
                a = np.asarray(d[v.name], F32)
                if a.size != v.numel:
                    raise ValueError('checkpoint variable %s has %d elements, the model\'s has %d'
                                     % (v.name, a.size, v.numel))
                self.view(v).copy_(torch.from_numpy(a.reshape(v.shape)))
                found += 1 if v.trainable else 0
            elif strict:
                raise KeyError('missing variable in checkpoint: ' + v.name)
        needed = [v for v in self.train_vars if not any(o in v.name for o in optional)]
        total = len(needed)
        found = sum(1 for v in needed if v.name in d)
        if require is not None and total > 0:
            if found == 0 or (require == 'all' and found < total):
                missing = [v.name for v in needed if v.name not in d][:5]
                raise ValueError('checkpoint matches %d of the model\'s %d trainable variables (e.g. missing %s; the '
                                 'checkpoint holds %s ...)' % (found, total, missing, sorted(d)[:3]))
        for f in self.listeners:
            f()
        return found, total


class Executor:
    """Forward (+ backward + update) of one graph on one GPU."""

    def __init__(self, graph, images, logits, device, store=None, train=True, loss=None, labels=None,
                 optimizer=None, weight_quant=None, act_quant=None, maskable=None, teacher=None,
                 seed=1, exact_ste=True, grad_scale=1.0, scope=None, conv_path=None, fuse_add=True,
                 update_moving_stats=True, frozen=None, int_layers=None):
        self.g, self.device, self.train = graph, device, train
        # int_layers (inference only, int8.IntModel): {Conv2D / depthwise op: (weight levels uint8 HWIO, alpha, beta,
        # bits)} of the layers that run on the u8 kernels, from the u8 levels their batch norm + ReLU producer writes
        if int_layers and train:
            raise ValueError('integer layers run only in an inference executor (train=False)')
        self.int_layers = dict(int_layers or {})
        # fuse_add=False: every Conv2D output is materialised on its own (the channel-pruning learner regresses conv
        # outputs of a pruned model onto those of the full model, learners/channel_pruning_gpu/learner.py:339-354);
        # update_moving_stats=False: training-mode BN without the moving-average update ops (the FULL model of that
        # learner runs forward_train but only the pruned model's update ops are ever executed, :283-286)
        self.fuse_add, self.update_moving_stats = bool(fuse_add), bool(update_moving_stats)
        self.images, self.logits_t, self.labels_t = images, logits, labels
        self.loss, self.teacher = loss, teacher
        self.optimizer = optimizer or {}
        self.exact_ste, self.grad_scale = exact_ste, float(grad_scale)
        # 'tc': tensor-core (wgmma) split-bf16 conv where the shape allows (Cin, Cout multiples of 16), exact-fp32
        # CUDA-core kernels elsewhere; 'fp32': exact-fp32 everywhere (the on-device reference)
        import os as _os
        self.conv_path = conv_path or _os.environ.get('PF_CONV_PATH', 'tc')
        self.seed = int(seed)
        self.ops = self._reachable_ops(logits)
        variables = []
        for op in self.ops:
            for v in op.vars.values():
                if v not in variables:
                    variables.append(v)
        self.variables = variables
        wd_of = dict(loss.l2) if loss is not None else {}
        self.wd_of = wd_of
        self.maskable = [v for v in (maskable or []) if v in variables]
        # an inference-only executor that owns its parameters (the distillation teacher): the split-bf16 weight
        # copies are prepared once and refreshed only when the store is (re)loaded
        self.static_weights = (not train) and store is None
        self._static_ready = False
        self.store = store or ParamStore(variables, device, wd_of, self.maskable, seed, frozen=frozen)
        if self.static_weights:
            self.store.listeners.append(self._invalidate_static)
        self.weight_quant, self.act_quant = weight_quant, act_quant
        self.prof = None
        # multi-stream overlap inside one step (captured into the CUDA graph as parallel branches): the teacher's
        # forward runs beside the student's, and the weight-gradient kernels run beside dgrad + BN-backward, so that
        # tensor-bound and HBM-bound kernels share the GPU (a BN kernel's CTAs fit next to a persistent conv CTA)
        self.overlap = _os.environ.get('PF_OVERLAP', '1') != '0' and device.type == 'cuda'
        self.side = torch.cuda.Stream(device=device) if self.overlap else None
        self.side2 = torch.cuda.Stream(device=device) if self.overlap else None
        self._shares_cols = False
        self._side_active = False
        self.cols_event = None          # recorded after this executor's im2col (shared columns)
        self.cols_wait = None           # event to wait for before reading shared columns
        self._plan()
        self._graph = None
        self.step_count = 0

    def _invalidate_static(self):
        """Parameters were (re)loaded: refresh the prepared weight copies now (a captured CUDA graph that contains
        this executor's forward does not re-run the preparation)."""
        self._static_ready = False
        if hasattr(self, 'conv'):
            self.prepare_static_weights()

    def prepare_static_weights(self):
        for lo in self.conv.values():
            lo.prepare_weights()
        self._static_ready = True

    # ------------------------------------------------------------------ planning
    def _reachable_ops(self, out):
        seen, order = set(), []

        def visit(t):
            if t.op in seen:
                return
            seen.add(t.op)
            for i in t.op.inputs:
                visit(i)
            order.append(t.op)
        import sys
        sys.setrecursionlimit(max(10000, sys.getrecursionlimit()))
        visit(out)
        pos = {op: i for i, op in enumerate(self.g.ops)}
        return sorted(order, key=lambda o: pos[o])

    def _consumers(self, t):
        return [c for c in t.consumers if c in self._opset]

    def _plan(self):
        dev = self.device
        self._opset = set(self.ops)
        st = self.store
        # PF_POISON=1 (debugging): every scratch / activation buffer starts as NaN, so that a read of memory no kernel
        # has written this step shows up in the losses instead of depending on what the allocator recycled
        poison = os.environ.get('PF_POISON', '0') == '1'
        E = (lambda shape: torch.full(shape, float('nan'), dtype=torch.float32, device=dev)) if poison else \
            (lambda shape: torch.empty(shape, dtype=torch.float32, device=dev))
        self.buf, self.alias = {}, {}
        self.fused_act, self.fused_into = {}, {}
        # ---- fusion: BN -> Relu/Relu6 and Conv/MatMul(bias) -> Relu with a single consumer
        for op in self.ops:
            if op.type in ACT_TYPES:
                src = op.inputs[0].op
                if src.type in ('FusedBatchNorm', 'Conv2D', 'MatMul') and len(self._consumers(src.output)) == 1:
                    if src.type == 'FusedBatchNorm' or op.type == 'Relu':
                        self.fused_act[src] = ACT_TYPES[op.type]
                        self.fused_into[op] = src
                        continue
                raise NotImplementedError('activation %s is not preceded by a fusable producer' % op.name)
        # ---- quantization marks
        self.wq_ops = list(self.weight_quant['ops']) if self.weight_quant else []
        self.aq_ops = list(self.act_quant['ops']) if self.act_quant else []
        self.aq_index = {op: i for i, op in enumerate(self.aq_ops)}
        self.aq_slots = torch.zeros(max(len(self.aq_ops), 1), 2, dtype=torch.int32, device=dev)
        # act_quant['ranges'] (inference only, int8.calibrate): a static (lo, hi) per quantized activation, in the same
        # slots, written once here; every quantizer then clamps to it in one pass and no range is computed per batch
        self.aq_static = bool(self.act_quant and self.act_quant.get('ranges') is not None)
        if self.aq_static:
            if self.train:
                raise ValueError('static activation ranges are for inference executors only (train=False)')
            if len(self.act_quant['ranges']) != len(self.aq_ops):
                raise ValueError('one activation range per quantized activation expected (%d)' % len(self.aq_ops))
            self.aq_slots = ops.range_slots(self.act_quant['ranges'], dev)
        self.aq_out = {}           # relu op -> out-of-place quantized buffer (producer is not BN)
        # quantized weights live in a flat buffer with the same offsets as the parameters
        self.QW = torch.zeros(st.n_train, dtype=torch.float32, device=dev) if self.wq_ops else None
        self.wq, self.train_clusters = None, False
        if self.wq_ops:
            kvars = [op.vars['kernel'] for op in self.wq_ops]
            srcs = [st.view(v) for v in kvars]
            dsts = [st.view(v, self.QW) for v in kvars]
            wq = self.weight_quant
            if wq.get('kind', 'uniform') == 'uniform':
                self.wq = ops.UniformWeightQuantizer(srcs, dsts, wq['bits'], wq.get('use_buckets', False),
                                                     wq.get('bucket_type', 'channel'), wq.get('bucket_size', 256))
            else:
                # codebooks: the reference's trainable `clusters` variables when the graph carries them (then they
                # live in the parameter store), else a private table of the quantizer
                cvars = [op.vars.get('clusters') for op in self.wq_ops]
                self.train_clusters = bool(wq.get('train_clusters', False)) and self.train
                # bucketed codebooks (utils.py:196-243): one [2^bits, nb] codebook matrix per tensor
                bkw = dict(use_buckets=True, bucket_type=wq.get('bucket_type', 'split'),
                           bucket_size=wq.get('bucket_size', 256)) if wq.get('use_buckets', False) else {}
                if all(c is not None for c in cvars):
                    self.wq = ops.CodebookWeightQuantizer(srcs, dsts, wq['bits'], keep_index=self.train_clusters,
                                                          cluster_views=[st.view(c) for c in cvars], cluster_base=st.P,
                                                          **bkw)
                else:
                    if self.train_clusters:
                        raise ValueError('training the codebooks needs `clusters` variables on the quantized ops')
                    self.wq = ops.CodebookWeightQuantizer(srcs, dsts, wq['bits'], **bkw)
        self.qvars = {op: op.vars['kernel'] for op in self.wq_ops}
        # ---- dropout (slim.dropout): per training-mode Dropout op a mask, a Philox stream index (its position among the
        # graph's Dropout ops) and a device-side step counter (row of drop_state) that the forward kernel advances, so a
        # replayed CUDA graph draws a fresh mask each step; an inference-mode Dropout is the identity (an alias).  A
        # Dropout of a compact graph (attrs 'layout', 'full_width': compact.build_graph) draws the masked full-width
        # model's mask gathered by its layout (drop_layout)
        self.dropout, self.drop_stream, self.drop_layout = {}, {}, {}
        for op in self.ops:
            if op.type == 'Dropout' and op.attrs['training']:
                mask = torch.empty(op.output.numel, dtype=torch.uint8, device=dev)
                if poison:
                    mask.fill_(0xff)
                self.drop_stream[op] = len(self.dropout)
                self.dropout[op] = mask
                if 'layout' in op.attrs:
                    self.drop_layout[op] = torch.as_tensor(np.asarray(op.attrs['layout'], np.int32), device=dev)
        self.drop_state = torch.zeros(len(self.dropout), 2, dtype=torch.int64, device=dev) if self.dropout else None
        self.drop_key = (self.seed, mgw.rank())
        self._drop_on = False          # set per forward(): masks only in training-mode passes
        # ---- tensors
        for op in self.ops:
            t = op.output
            if op.type == 'Placeholder':
                self.buf[t] = E(t.shape)
                self.buf[t].zero_()
            elif self._passthrough(op):
                self.alias[t] = op.inputs[0]
            elif op in self.fused_into:
                self.alias[t] = op.inputs[0]
            else:
                self.buf[t] = E(t.shape)
            if op in self.aq_index and self.fused_into.get(op) is not None and \
                    self.fused_into[op].type != 'FusedBatchNorm':
                self.aq_out[op] = E(t.shape)
        # ---- per-op scratch
        self.bn = {}
        self.tc_conv = set()       # convs with a tensor-core lowering (_TcConv, or _U8Conv for an integer layer)
        self.tc = {}               # their split-bf16 weight copies (not an integer layer's)
        self.tc_wgrad = set()
        self.im2col = {}
        self.pool_argmax = {}
        max_ws, max_wt, max_bnws = 4, 4, 4
        max_x = max_dy = 8             # the x / dy operands split into planes (shared scratch)
        self.desc = {}
        for op in self.ops:
            if op.type == 'FusedBatchNorm':
                c = op.output.shape[-1]
                self.bn[op] = dict(mean=E((c,)), var=E((c,)), rstd=E((c,)))
                max_bnws = max(max_bnws, 5 * c * ops.BN_MAX_SPLITS)
            if op.type in ('Conv2D', 'MatMul'):
                x, y = op.inputs[0], op.output
                if op.type == 'Conv2D':
                    n, h, w, c = x.shape
                    _, p, q, k = y.shape
                    (kh, kw), (sh, sw), (pt, pl) = op.attrs['ksize'], op.attrs['strides'], op.attrs['pad']
                    d = ops.conv_desc(n, h, w, c, k, kh, kw, p, q, sh, sw, pt, pl)
                else:
                    n, c = x.shape
                    k = y.shape[1]
                    d = ops.conv_desc(n, 1, 1, c, k, 1, 1, 1, 1, 1, 1, 0, 0)
                self.desc[op] = d
                if self.conv_path == 'tc' and op.type == 'Conv2D' and not ops.conv2d_tc_supported(d) \
                        and k % 16 == 0 and c % 16 != 0 and x.op.type == 'Placeholder':
                    # first layer (Cin = 3): explicit im2col into kpad channels, then a 1x1 tensor-core conv
                    kdim = kh * kw * c
                    kpad = (kdim + 15) // 16 * 16
                    d1 = ops.conv_desc(n, p, q, kpad, k, 1, 1, p, q, 1, 1, 0, 0)
                    # columns directly in operand planes when every consumer is a tensor-core kernel
                    as_planes = (not self.train) or ops.conv2d_tc_wgrad_supported(d1)
                    mode = 'im2col'
                    # fewer than 64 output channels (MobileNet's 3 -> 32 stem): the tensor-core wgrad wants Cout % 64 == 0,
                    # so g = 64 / Cout pixels share one GEMM row — cols [pixels, kpad] and dy [pixels, k] are read as
                    # [pixels / g, g kpad] and [pixels / g, g k]; the weight gradient is the sum of the g diagonal
                    # kpad x k blocks of the (g kpad) x (g k) result (the exact-fp32 CUDA-core wgrad of this layer is
                    # slow: one output channel block per CTA over every pixel)
                    pair = None
                    if self.train and not as_planes and k in (16, 32) and (kpad * (64 // k)) % 64 == 0 \
                            and (p * q) % (64 // k) == 0:
                        g_ = 64 // k
                        dp = ops.conv_desc(n, 1, p * q // g_, kpad * g_, k * g_, 1, 1, 1, p * q // g_, 1, 1, 0, 0)
                        if ops.conv2d_tc_wgrad_supported(dp):
                            pair, as_planes = dict(g=g_, d=dp), True
                    if sh == 2 and sw == 2 and 4 * c <= 16 and os.environ.get('PF_STEM_S2D', '1') != '0':
                        # stride-2 stem: space-to-depth instead of im2col — a stride-1 conv over 16 channels that the
                        # tensor-core kernels gather themselves (no 2 GB column matrix)
                        r2, s2, fwd_map, bwd_map = ops.s2d_weight_maps(kh, kw, c, 16)
                        d2 = ops.conv_desc(n, p + r2 - 1, q + s2 - 1, 16, k, r2, s2, p, q, 1, 1, 0, 0)
                        if ops.conv2d_tc_supported(d2) and ((not self.train) or ops.conv2d_tc_wgrad_supported(d2)):
                            mode, d1, as_planes, kpad = 's2d', d2, True, r2 * s2 * 16
                    self.im2col[op] = dict(kdim=kdim, kpad=kpad, d1=d1, compute=True, planes=as_planes, mode=mode,
                                           cols=ops.Planes(n * d1.h * d1.w * d1.c, dev) if as_planes else E((n * p * q, kpad)),
                                           wpad=torch.zeros(kpad * k, dtype=torch.float32, device=dev),
                                           tw=ops.TcWeights(d1, dev, need_dgrad=False))
                    if mode == 's2d':
                        self.im2col[op]['fwd_map'] = torch.from_numpy(fwd_map).to(dev)
                        self.im2col[op]['bwd_map'] = torch.from_numpy(bwd_map).to(dev)
                    if self.train:
                        self.im2col[op]['dwpad'] = torch.zeros(kpad * k, dtype=torch.float32, device=dev)
                        if as_planes:                      # dy is split into planes for the tensor-core wgrad
                            max_dy = max(max_dy, n * p * q * k)
                        if pair is not None and mode == 'im2col':
                            pair['dw'] = torch.zeros(pair['g'] * kpad * pair['g'] * k, dtype=torch.float32, device=dev)
                            self.im2col[op]['pair'] = pair
                            max_ws = max(max_ws, ops.conv2d_tc_wgrad_planes_workspace_floats(pair['d']))
                        if ops.conv2d_tc_wgrad_supported(d1):
                            max_ws = max(max_ws, ops.conv2d_tc_wgrad_planes_workspace_floats(d1))
                        max_ws = max(max_ws, ops.conv2d_wgrad_workspace_floats(d1))
                if self.conv_path == 'tc' and ops.conv2d_tc_supported(d):
                    self.tc_conv.add(op)
                    if op not in self.int_layers:
                        self.tc[op] = ops.TcWeights(d, dev, need_dgrad=self.train and x.op.type != 'Placeholder')
                elif op in self.int_layers:
                    raise ValueError('%s: an integer layer needs a tensor-core lowering (conv path %r) for its '
                                     'residual and folded batch norm' % (op.name, self.conv_path))
                if self.train:
                    if op in self.tc and ops.conv2d_tc_wgrad_supported(d):
                        self.tc_wgrad.add(op)
                        max_ws = max(max_ws, ops.conv2d_tc_wgrad_planes_workspace_floats(d))
                    max_ws = max(max_ws, ops.conv2d_wgrad_workspace_floats(d))
                    max_wt = max(max_wt, op.vars['kernel'].numel)
            if op.type == 'DepthwiseConv2dNative':
                x, y = op.inputs[0], op.output
                n, h, w, c = x.shape
                _, p, q, _ = y.shape
                (kh, kw), (sh, sw), (pt, pl) = op.attrs['ksize'], op.attrs['strides'], op.attrs['pad']
                self.desc[op] = ops.conv_desc(n, h, w, c, c, kh, kw, p, q, sh, sw, pt, pl)
                if self.train:
                    max_ws = max(max_ws, ops.dwconv_wgrad_workspace_floats(self.desc[op]))
            if op.type == 'MaxPool':
                x, y = op.inputs[0], op.output
                n, h, w, c = x.shape
                _, p, q, _ = y.shape
                (kh, kw), (sh, sw), (pt, pl) = op.attrs['ksize'], op.attrs['strides'], op.attrs['pad']
                self.desc[op] = ops.conv_desc(n, h, w, c, c, kh, kw, p, q, sh, sw, pt, pl)
                if self.train:
                    self.pool_argmax[op] = torch.empty(y.shape, dtype=torch.uint8, device=dev)
        # ---- residual Add fused into the epilogue of the tensor-core conv that produces one of its inputs:
        # the conv writes conv(x) + shortcut straight into the Add's buffer (one pass instead of three)
        self.fused_add = {}        # conv op -> (add op, other input tensor)
        self.add_fused = set()
        for op in self.ops:
            if op.type != 'Add' or not self.fuse_add:
                continue
            for i, x_t in enumerate(op.inputs):
                src, other = x_t.op, op.inputs[1 - i]
                if src.type == 'Conv2D' and src in self.tc_conv and x_t not in self.alias \
                        and src not in self.fused_act and 'bias' not in src.vars and len(self._consumers(x_t)) == 1 \
                        and self.g.ops.index(other.op) < self.g.ops.index(src):
                    self.fused_add[src] = (op, other)
                    self.add_fused.add(op)
                    self.buf[x_t] = self.buf[op.output]       # the conv output IS the add output
                    break
        self._plan_bn_add()
        readers = self._plan_operand_planes()
        self._plan_bn_gather()
        self._plan_levels(readers, E)
        # one launch refreshes the split-bf16 copies of all (trainable) conv kernels
        self.tc_batch = None
        if self.tc and not self.static_weights:
            tc_ops = [op for op in self.ops if op in self.tc]
            levels = {}
            for j, op in enumerate(tc_ops):
                if op in self.w_lv:
                    lv = self.w_lv[op]
                    levels[j] = (self.store.view(op.vars['kernel']), lv['alpha'], lv['beta'], lv['ralpha'], lv['ncols'],
                                 self.wq.bits[lv['index']])
                    lv['batch_index'] = j
            self.tc_batch = ops.TcWeightsBatch([(self.tc[op], self.kernel_of(op)) for op in tc_ops], dev, levels)
        self._lv_on = False            # set per forward(): levels only in training-mode passes
        if self.labels_t is not None and self.labels_t not in self.buf:
            self.buf[self.labels_t] = torch.zeros(self.labels_t.shape, dtype=torch.float32, device=dev)
        self.bn_ws = E((max_bnws,))
        n_rows = self.logits_t.shape[0]
        self.loss_out = torch.zeros(8, dtype=torch.float32, device=dev)
        self.row_ws = E((4 * n_rows,))
        if self.train:
            self.G = torch.zeros(st.n_train, dtype=torch.float32, device=dev)
            self.S1 = torch.zeros(st.n_train, dtype=torch.float32, device=dev)
            self.S2 = torch.zeros(st.n_train, dtype=torch.float32, device=dev) \
                if self.optimizer.get('kind') == 'adam' else None
            self.hp = torch.zeros(4, dtype=torch.float32, device=dev)
            # per-step scalars (lr, Adam beta powers) travel through a RING of pinned slots: the async upload of step
            # i must have executed before the host rewrites its slot (a single slot let step i pick up step i+1's
            # beta powers whenever the host ran ahead of the GPU)
            self.hp_ring = torch.zeros(16, 4, dtype=torch.float32).pin_memory() if dev.type == 'cuda' else torch.zeros(16, 4)
            self.hp_events, self._hp_i = [None] * 16, 0
            self.wgrad_ws = E((max_ws,))
            self.wgrad_ws2 = E((max_ws,)) if self.overlap else None
            self.wt_ws = E((max_wt,))
            self.l2_out = torch.zeros(4, dtype=torch.float32, device=dev)
            self.l2_ws = E((ops.L2_PARTIALS,))
            self.gbuf, self.galias = {}, {}
            self.relu_scratch = {}
            # d(out)/d(in) of a residual Add is the identity, so an input can SHARE the Add output's gradient buffer
            # (no copy kernel):
            #  - an input consumed only by the Add (the conv3 / projection branch) is a pure reader of it;
            #  - the identity shortcut x (also consumed by the next BN) turns the buffer into an in-place
            #    accumulator: x's other consumers add their dx into it.  That is safe when every reader of the Add
            #    output's gradient runs (in backward order) before every such writer, i.e. comes LATER in forward
            #    order — checked below.
            pos = {op: i for i, op in enumerate(self.ops)}
            add_alias = {}

            def root_of(t):
                while t in add_alias or t in self.alias:
                    t = add_alias[t] if t in add_alias else self.alias[t]
                return t
            for op in self.ops:
                if op.type != 'Add':
                    continue
                for x_t in op.inputs:
                    root = x_t
                    while root in self.alias:
                        root = self.alias[root]
                    if root.op.type == 'Placeholder' or root in add_alias or root is op.output:
                        continue
                    single = len(self._consumers(x_t)) == 1
                    chain_single = True
                    tt = x_t
                    while tt in self.alias:
                        tt = self.alias[tt]
                        chain_single = chain_single and len(self._consumers(tt)) == 1
                    if single and chain_single:
                        add_alias[root] = op.output
                        continue
                    if x_t in self.alias:
                        continue
                    # readers of g(Add out): ops whose output gradient lives in that buffer
                    key = root_of(op.output)
                    readers = [o for o in self.ops if o.type != 'Placeholder' and o is not op and root_of(o.output) is key]
                    writers = [c for c in self._consumers(x_t) if c is not op]
                    if all(pos[r] > pos[w] for r in readers for w in writers) and all(pos[w] < pos[op] for w in writers):
                        add_alias[root] = op.output
            for op in self.ops:
                t = op.output
                if op.type == 'Placeholder':
                    continue
                if t in self.alias:
                    self.galias[t] = self.alias[t]
                elif t in add_alias:
                    self.galias[t] = add_alias[t]
                else:
                    self.gbuf[t] = E(t.shape)
                if op.type in ('Conv2D', 'MatMul') and op in self.fused_act:
                    self.relu_scratch[op] = E(t.shape)
            self._plan_dy_planes(pos)
            # split-K partials of every tensor-core wgrad get their own buffer; ONE reduction launch at the end of the
            # backward pass sums them into the flat gradient buffer (fixed order: deterministic)
            self.wg_part, red_items = {}, []
            for op in self.ops:
                if op in self.tc_wgrad:
                    splits = ops.conv2d_tc_wgrad_splits(self.desc[op])
                    if splits > 1:
                        gk = st.view(op.vars['kernel'], self.G)
                        self.wg_part[op] = E((splits * gk.numel(),))
                        red_items.append((self.wg_part[op], gk, splits))
            self._red_items = red_items
            self.wg_reduce = ops.TcWgradReduceBatch(red_items, dev) if red_items else None
            # the x / dy operands of the tensor-core convs that no producer writes as planes are split into these
            self.x_scratch = ops.Planes(max([max_x] + [op.inputs[0].numel for op in self.tc if op not in self.im2col
                                                       and self.planes_of(op.inputs[0]) is None]), dev)
            self.dy_scratch = ops.Planes(max([max_dy] + [op.output.numel for op in self.tc_wgrad
                                                         if op not in self.conv_dy_planes]), dev)
            if self.maskable:
                self.MASK = torch.ones(st.n_masked, dtype=torch.float32, device=dev)
                self.BKUP = st.P[:st.n_masked].clone()
                mv = self.maskable
                # (the builder takes device pointers: planning-only executors on the CPU — tests — do without)
                self.mask_builder = ops.MaskBuilder([st.view(v) for v in mv],
                                                    [st.view(v, self.BKUP) for v in mv],
                                                    [st.view(v, self.MASK) for v in mv]) if dev.type == 'cuda' else None
            else:
                self.MASK = None
            if self.exact_ste and self.wq is not None and isinstance(self.wq, ops.UniformWeightQuantizer):
                self._ste_grads = [st.view(v, self.G) for v in [op.vars['kernel'] for op in self.wq_ops]]
            else:
                self._ste_grads = None
            self.beta1_power = F32(self.optimizer.get('beta1', 0.9))
            self.beta2_power = F32(self.optimizer.get('beta2', 0.999))
        self.bn_fold = self._plan_bn_fold()
        # ---- how each FusedBatchNorm, Conv2D / MatMul and depthwise conv runs forward, backward and in layer_wgrad
        self.batch_norm = {}
        for op in self.ops:
            if op.type == 'FusedBatchNorm':
                lo = (_BnAdd if op in self.bn_add else _BnFolded if op in self.bn_fold.values() else
                      _BnGather if op in self.bn_gather else _BnLowering)(self, op)
                self.batch_norm[op] = _U8Bn(self, op, lo) if op in self.u8_others else lo
        self.conv = {op: (_U8Conv if op in self.int_layers else _StemConv if op in self.im2col else
                          _TcConv if op in self.tc else _ConvLowering)(self, op)
                     for op in self.ops if op.type in ('Conv2D', 'MatMul')}
        self.depthwise = {op: (_U8DwConv if op in self.int_layers else _DwConv)(self, op)
                          for op in self.ops if op.type == 'DepthwiseConv2dNative'}

    def _plan_bn_add(self):
        """Linear bottleneck: a BatchNorm without activation whose only consumer is a residual Add (MobileNet-v2's
        projection, conv_blocks.py:289-313) writes bn(x) + shortcut straight into the Add's buffer (and / or the Add's
        operand planes) — one pass instead of BN apply + add + split."""
        self.bn_add = {}           # BN op -> (add op, other input tensor)
        fuse_bn_add = os.environ.get('PF_FUSE_BN_ADD', '1') != '0'
        for op in self.ops:
            if op.type != 'Add' or op in self.add_fused or not fuse_bn_add:
                continue
            for i, x_t in enumerate(op.inputs):
                src, other = x_t.op, op.inputs[1 - i]
                if src.type == 'FusedBatchNorm' and src not in self.fused_act and x_t not in self.alias \
                        and self._consumers(x_t) == [op] and other is not x_t \
                        and self.g.ops.index(other.op) < self.g.ops.index(src):
                    self.bn_add[src] = (op, other)
                    self.add_fused.add(op)
                    self.buf[x_t] = self.buf[op.output]       # the BN output IS the add output
                    break

    def _plan_operand_planes(self):
        """Split-bf16 operand planes (tensor-core path): the BN apply / activation quantizer / gather that produces a
        conv input writes it directly in the operand format of the tensor-core kernels (x = hi + lo, two bf16 planes);
        the fp32 copy is only written when some other consumer needs it.  An integer layer reads its producer's u8
        levels (_U8Bn): it is neither a planes nor an fp32 reader, and `u8_others` says whether such a producer also
        writes its planes or fp32 output for other readers.  Returns {producer: the convs reading its planes}."""
        bn_adds = {a for a, _ in self.bn_add.values()}
        self.xplanes, self.bn_need_f32, readers = {}, {}, {}
        for op in self.ops:
            if op in self.tc and op not in self.im2col:
                r = self._root(op.inputs[0])
                if r is not None and (r.op.type in ('FusedBatchNorm', 'GatherChannels') or r.op in bn_adds) \
                        and r.numel % 8 == 0:
                    if r.op not in self.xplanes:
                        self.xplanes[r.op] = ops.Planes(r.numel, self.device)
                    readers.setdefault(r.op, []).append(op)
        u8_src = dict.fromkeys(self._root(op.inputs[0]).op for op in self.ops if op in self.int_layers)
        self.u8_others = {}
        for bn_op in dict.fromkeys(list(self.xplanes) + list(u8_src)):
            ts = [bn_op.output] + [c.output for c in self._consumers(bn_op.output) if c in self.fused_into]
            # a reader that is not the fused activation, an integer layer nor a planes conv
            f32 = any(self.fused_into.get(c) is not bn_op and c not in self.int_layers and
                      not (c in self.tc and c not in self.im2col and (not self.train or c in self.tc_wgrad))
                      for t in ts for c in self._consumers(t))
            if bn_op in self.xplanes:
                self.bn_need_f32[bn_op] = f32
            if bn_op in u8_src:
                self.u8_others[bn_op] = f32 or bn_op in self.xplanes
        return readers

    def _plan_bn_gather(self):
        """Channel gathers of a compact (channel-pruned) graph, compact.py: a GatherChannels op writes its consumer's
        operand planes; when it is the only reader of a BN (+ activation), the BN apply writes the gathered tensor
        itself and the full-width BN output is never materialised (a training-mode BN only in a training executor:
        pf_bn_apply_gather).  A training executor also holds each gather's inverse table, for its backward."""
        self.gather_idx, self.bn_gather, self.scatter_inv = {}, {}, {}
        for op in self.ops:
            if op.type != 'GatherChannels':
                continue
            t = op.inputs[0]
            if len(op.attrs['index']) % 4 or (self.train and t.shape[-1] % 4):
                raise ValueError('%s: the channel gather / scatter kernels need widths that are multiples of 4 (%d -> %d)'
                                 % (op.name, t.shape[-1], len(op.attrs['index'])))
            self.gather_idx[op] = torch.from_numpy(np.ascontiguousarray(op.attrs['index'], np.int32)).to(self.device)
            if self.train:
                self.scatter_inv[op] = torch.from_numpy(ops.scatter_table(op.attrs['index'], t.shape[-1])).to(self.device)
            bn = t.op.inputs[0].op if t.op in self.fused_into else t.op
            if bn.type == 'FusedBatchNorm' and (self.train or not bn.attrs['training']) and bn not in self.bn_add \
                    and bn not in self.xplanes and self._consumers(t) == [op] \
                    and (t.op is bn or self._consumers(bn.output) == [t.op]) and t.op not in self.aq_index:
                self.bn_gather[bn] = op
        self.gather_fused = set(self.bn_gather.values())

    def _plan_levels(self, readers, E):
        """Integer-level operands (TMA-fed kernels, SURVEY §7 hard part 1b): a <= 8-bit fake-quantized tensor is
        exactly scale * level, and the levels are exact in bf16 — one operand plane instead of hi + lo, one MMA per
        k-slice instead of three (two against a split gradient).  Activation side: the fused BN + ReLU + fake-quant pass
        writes levels + a device header + per-pixel channel sums when EVERY reader of its planes is a TMA-fed kernel.
        Weight side: the preparation launch derives the levels from the unquantized kernel with the quantizer's own op
        chain; needs per-layer / per-output-channel buckets and the input's channel sums."""
        self.act_lv, self.w_lv = {}, {}
        if os.environ.get('PF_TC_LEVELS', '1') == '0' or not (self.train and self.aq_ops) or self.device.type != 'cuda':
            return
        for bn_op, users in readers.items():
            c = bn_op.output.shape[-1]
            if self._aq_of_bn(bn_op) is not None and bn_op.attrs['training'] and c >= 16 and not c & (c - 1) \
                    and all(ops.conv2d_tc_tma_supported(self.desc[u], 0) and u in self.tc_wgrad
                            and ops.conv2d_tc_tma_supported(self.desc[u], 2) for u in users):
                m = bn_op.output.numel // c
                nseg = (c + 127) // 128
                self.act_lv[bn_op] = dict(hdr=torch.zeros(2, dtype=torch.int32, device=self.device),
                                          csum=E((m * nseg,)), nseg=nseg)
        wq = self.weight_quant
        if self.wq is not None and isinstance(self.wq, ops.UniformWeightQuantizer) and \
                (not wq.get('use_buckets', False) or wq.get('bucket_type', 'channel') == 'channel'):
            nbk = self.wq.n_buckets
            lv_readers = {u for bn_op in self.act_lv for u in readers[bn_op]}
            for i, op in enumerate(self.wq_ops):
                if op in lv_readers and op.type == 'Conv2D' and 1 <= self.wq.bits[i] <= 8:
                    b0, ncols = int(self.wq.segs[i]['bucket0']), int(self.wq.segs[i]['ncols'])
                    sc = self.wq.scales
                    self.w_lv[op] = dict(index=i, ncols=ncols, alpha=sc[b0:b0 + ncols], beta=sc[nbk + b0:nbk + b0 + ncols],
                                         ralpha=sc[2 * nbk + b0:2 * nbk + b0 + ncols])

    def _plan_dy_planes(self, pos):
        """dy operand planes.  For every tensor-core conv, the LAST op that writes the gradient of its output before
        the conv's own backward runs; when that is a BatchNorm backward or a channel scatter (the backward of a
        GatherChannels), it also emits the gradient as split-bf16
        planes (dgrad + wgrad operands) instead of a separate split pass.  If the BN is the only writer and the conv the
        only reader, the fp32 copy is dropped and the planes live in its memory."""
        grad_writers = {}
        for op in self.ops:
            if op.type == 'Placeholder' or self._passthrough(op) or op in self.fused_into:
                continue
            ins = op.inputs if op.type == 'Add' else op.inputs[:1]
            for x_t in ins:
                k = self.gkey(x_t)
                if x_t.op.type != 'Placeholder' and not (op.type == 'Add' and k is self.gkey(op.output)):
                    grad_writers.setdefault(k, []).append(op)
        self.bn_gplanes, self.bn_gplanes_only, self.conv_dy_planes = {}, {}, {}
        for op in self.ops:
            if op not in self.tc_wgrad or op in self.fused_act or 'bias' in op.vars or op.output.numel % 8:
                continue
            k = self.gkey(op.output)
            later = [w for w in grad_writers.get(k, []) if pos[w] > pos[op]]
            lw = min(later, key=lambda w: pos[w]) if later else None
            if lw is None or lw.type not in ('FusedBatchNorm', 'GatherChannels') or lw.inputs[0].numel != op.output.numel:
                continue
            if lw not in self.bn_gplanes:
                readers = [o for o in self.ops if o.type != 'Placeholder' and self.gkey(o.output) is k]
                only = len(grad_writers[k]) == 1 and readers == [op]
                self.bn_gplanes_only[lw] = only
                self.bn_gplanes[lw] = ops.Planes(op.output.numel, self.device,
                                                 self.gbuf[k].view(-1).view(torch.bfloat16) if only else None)
            self.conv_dy_planes[op] = self.bn_gplanes[lw]

    def _plan_bn_fold(self):
        """{tensor-core conv op: inference-mode BatchNorm op} of the BNs applied in the epilogue of the conv that
        produces their input (the conv's own output, or the residual Add fused into it): the BN apply pass, which reads
        the conv's fp32 output back, is not launched.  Only in inference executors on the GPU (the distillation teacher,
        evaluation); training executors, and executors planned on the CPU (the golden plan snapshots), fold nothing.
        Excluded: the stem (its output is not a tensor-core conv's) and BNs that already have a fused form (bn_add,
        bn_gather) or feed an activation quantizer."""
        fold = {}
        if self.train or self.device.type != 'cuda':
            return fold
        add_conv = {a: c for c, (a, _) in self.fused_add.items()}
        for op in self.ops:
            if op.type != 'FusedBatchNorm' or op.attrs['training'] or op in self.bn_add or op in self.bn_gather:
                continue
            x, r = op.inputs[0], self._root(op.inputs[0])         # through Identity / Reshape / a fused ReLU
            if r is None or r.shape[-1] != x.shape[-1]:
                continue
            conv = r.op if r.op.type == 'Conv2D' else add_conv.get(r.op)
            if conv is None or conv not in self.tc_conv or conv in self.im2col or conv in fold \
                    or self._aq_of_bn(op) is not None:
                continue
            fold[conv] = op
        return fold

    # ------------------------------------------------------------------ profiling (bench.py roofline)
    class _Timed:
        def __init__(self, ex, cat):
            self.ex, self.cat = ex, cat

        def __enter__(self):
            if self.ex.prof is not None:
                self.a = torch.cuda.Event(enable_timing=True)
                self.a.record()

        def __exit__(self, *exc):
            if self.ex.prof is not None:
                b = torch.cuda.Event(enable_timing=True)
                b.record()
                self.ex.prof.setdefault(self.cat, []).append((self.a, b))

    def timed(self, cat):
        return Executor._Timed(self, cat)

    def profile_step(self, lr, allreduce=None):
        """One EAGER step with every launch group bracketed by CUDA events on the launching stream.
        Returns {category: milliseconds}.  (Not the timed region: the benchmark replays a CUDA graph.)"""
        self.prof = {}
        if self.teacher is not None:
            self.teacher.prof = self.prof
        self.set_hyper(lr)
        self.device_step(allreduce)
        torch.cuda.synchronize()
        out = {k: sum(a.elapsed_time(b) for a, b in v) for k, v in self.prof.items()}
        self.prof = None
        if self.teacher is not None:
            self.teacher.prof = None
        self.advance_optimizer_state()
        return out

    # ------------------------------------------------------------------ helpers
    def T(self, t):
        """Buffer that holds tensor t as seen by its consumers."""
        shape = t.shape
        while t in self.alias:
            op = t.op
            if op in self.aq_out:
                return self.aq_out[op].view(shape)
            t = self.alias[t]
        if t.op in self.dropout and not self._drop_on:
            return self.T(t.op.inputs[0]).view(shape)         # inference-mode pass: dropout is the identity
        b = self.buf[t]
        return b if b.shape == shape else b.view(shape)

    def _passthrough(self, op):
        """ops that launch nothing and whose output (and gradient) buffer is their input's"""
        return op.type in ('Reshape', 'Identity') or (op.type == 'Dropout' and op not in self.dropout)

    def _aq_of_bn(self, bn_op):
        """the activation quantizer (index into aq_ops) that reads the Relu / Relu6 fused into bn_op, else None"""
        relu_op = self._consumers(bn_op.output)[0] if bn_op in self.fused_act else None
        return self.aq_index.get(relu_op)

    def _root(self, t):
        """The tensor whose buffer holds t (following Reshape / fused-activation aliases); None when t is
        held by an out-of-place quantized buffer."""
        while t in self.alias:
            if t.op in self.aq_out:
                return None
            t = self.alias[t]
        return t

    def outputs_of(self, op):
        """(fp32 output or None, operand planes or None) of a BN / bn_add Add / gather: fp32 if no planes or a reader"""
        pl = self.xplanes.get(op)
        return (self.buf[op.output] if pl is None or self.bn_need_f32[op] else None), pl

    def planes_of(self, t):
        r = self._root(t)
        return self.xplanes.get(r.op) if r is not None else None

    def gkey(self, t):
        while t in self.galias:
            t = self.galias[t]
        return t

    def grad_target(self, t):
        """(buffer, accumulate) for writing a contribution to dL/dt."""
        k = self.gkey(t)
        acc = k in self._gwritten
        self._gwritten.add(k)
        return self.gbuf[k], acc

    def grad_of(self, t):
        k = self.gkey(t)
        return self.gbuf[k] if k in self._gwritten else None

    def kernel_of(self, op):
        v = op.vars['kernel']
        if op in self.qvars:
            return self.store.view(v, self.QW)
        return self.store.view(v)

    # ------------------------------------------------------------------ forward
    def forward(self, training=None, upto=None):
        """upto: stop after this op has run (its output buffer is the result wanted)."""
        training = self.train if training is None else training
        if self.aq_ops and not self.aq_static:
            ops.minmax_reset(self.aq_slots)
        if self.wq is not None:
            with self.timed('weight_quant'):
                self.wq.forward()
        if self.static_weights and not self._static_ready:
            self.prepare_static_weights()
        self._lv_on = bool(training and (self.act_lv or self.w_lv))
        self._drop_on = bool(training)
        if self.tc_batch is not None:
            with self.timed('conv_prep'):
                self.tc_batch.prepare(levels=self._lv_on)
        prev = None
        for op in self.ops:
            if prev is not None and prev is upto:
                return None
            prev = op
            ty = op.type
            if ty == 'Placeholder' or self._passthrough(op):
                continue
            if ty in ('Conv2D', 'MatMul'):
                self.conv[op].forward()
            elif ty == 'DepthwiseConv2dNative':
                self.depthwise[op].forward()
            elif ty == 'FusedBatchNorm':
                self.batch_norm[op].forward(training)
            elif ty == 'GatherChannels':
                if op in self.gather_fused:
                    continue                               # written by the producing BN apply
                with self.timed('gather'):
                    ops.gather_channels(self.T(op.inputs[0]), self.gather_idx[op], *self.outputs_of(op))
            elif ty in ACT_TYPES:
                if op in self.aq_out:                      # a quantized ReLU whose producer is not a BN
                    y, i = self.buf[self.fused_into[op].output], self.aq_index[op]
                    with self.timed('act_quant'):
                        if self.aq_static:
                            ops.act_quant_static(y, self.aq_out[op], self.aq_slots[i], self.act_quant['bits'][i])
                        else:
                            ops.act_minmax(y, self.aq_slots[i])
                            ops.act_quant(y, self.aq_out[op], self.aq_slots[i], self.act_quant['bits'][i])
            elif ty == 'MaxPool':
                with self.timed('pool'):
                    ops.maxpool_fwd(self.desc[op], self.T(op.inputs[0]), self.buf[op.output], self.pool_argmax.get(op))
            elif ty == 'Mean':
                x = op.inputs[0]
                n, h, w, c = x.shape
                with self.timed('pool'):
                    ops.global_avgpool_fwd(self.T(x), n, h * w, c, self.buf[op.output])
            elif ty == 'Dropout':
                if training:
                    with self.timed('dropout'):
                        i = self.drop_stream[op]
                        ops.dropout_fwd(self.T(op.inputs[0]), op.attrs['keep_prob'], self.drop_key[0], self.drop_key[1],
                                        self.drop_state[i], self.buf[op.output], self.dropout[op], stream_id=i,
                                        layout=self.drop_layout.get(op), full_width=op.attrs.get('full_width'))
            elif ty == 'Add':
                if op in self.add_fused:
                    continue                               # computed by the producing conv's / BN's epilogue
                with self.timed('add_fwd'):
                    ops.add(self.T(op.inputs[0]), self.T(op.inputs[1]), self.buf[op.output])
            elif ty == 'Softmax':
                ops.softmax_fwd(self.T(op.inputs[0]), self.buf[op.output])
            else:
                raise NotImplementedError('op type %s' % ty)
        return self.T(self.logits_t)

    # ------------------------------------------------------------------ gradient buckets of the data-parallel step
    def _bucket_plan(self):
        """The flat gradient buffer is summed over the workers in TWO all-reduces instead of one (SURVEY §8e): the
        kernels of the LAST layers — about half of the first (weight-decayed) range of the parameter store, which is laid
        out in forward order — are complete long before the backward pass ends (stage 4 + the dense layer of ResNet-50
        hold 2/3 of its parameters and take ~10 % of its backward time), so their all-reduce runs on a communication
        stream underneath the rest of the backward pass.  Returns None when the split does not apply."""
        if hasattr(self, '_bk'):
            return self._bk
        self._bk = None
        st = self.store
        if os.environ.get('PF_AR_BUCKETS', '2') == '1' or not self.overlap or self.train_clusters \
                or not st.ranges:
            return None
        s0, e0 = st.ranges[0][0], st.ranges[0][1]
        pos = {op: i for i, op in enumerate(self.ops)}
        owners = sorted((st.offset[v], v.numel, pos[op]) for op in self.ops for v in op.vars.values()
                        if v.trainable and s0 <= st.offset[v] < e0)
        if len(owners) < 4 or any(b[2] < a[2] for a, b in zip(owners, owners[1:])):
            return None                                    # store order is not the forward order: no valid split
        acc, cut = 0, None
        for i in range(len(owners) - 1, 0, -1):
            acc += owners[i][1]
            if acc >= 0.5 * (e0 - s0) and owners[i][2] > owners[i - 1][2]:
                cut = i
                break
        if cut is None:
            return None
        split, bpos = owners[cut][0], owners[cut][2]
        off = lambda t: (t.data_ptr() - self.G.data_ptr()) // 4
        hi = [it for it in self._red_items if off(it[1]) >= split]
        lo = [it for it in self._red_items if off(it[1]) < split]
        ste_hi = ste_lo = None
        if self._ste_grads is not None:
            ste_hi = [i for i, g in enumerate(self._ste_grads) if off(g) >= split]
            ste_lo = [i for i, g in enumerate(self._ste_grads) if off(g) < split]
        self._bk = dict(split=split, end=e0, pos=bpos, stream=torch.cuda.Stream(device=self.device),
                        red_hi=ops.TcWgradReduceBatch(hi, self.device) if hi else None,
                        red_lo=ops.TcWgradReduceBatch(lo, self.device) if lo else None, ste_hi=ste_hi, ste_lo=ste_lo)
        return self._bk

    def _bucket_hi(self, bk, allreduce):
        """the last layers' gradients are final: reduce their split-K partials, apply their STE, start their all-reduce —
        all on the communication stream, behind what the main and the weight-gradient streams have enqueued so far"""
        cs, main = bk['stream'], torch.cuda.current_stream()
        cs.wait_stream(main)
        if self._side_active:
            cs.wait_stream(self.side2)
        with torch.cuda.stream(cs):
            if bk['red_hi'] is not None:
                bk['red_hi'].reduce()
            if bk['ste_hi']:
                self.wq.ste_backward_(self._ste_grads, bk['ste_hi'])
            allreduce(self.G[bk['split']:bk['end']])

    # ------------------------------------------------------------------ loss + backward
    def loss_and_backward(self, allreduce=None):
        """allreduce (data-parallel step): callable summing a contiguous range of the flat gradient buffer over the
        workers on the current stream; called for every range of the buffer before this method returns."""
        st = self.store
        L = self.loss
        self._gwritten = set()
        self._side_active = self.overlap and self.prof is None
        bk = self._bucket_plan() if (allreduce is not None and self._side_active) else None
        bk_fired = False
        op_pos = {op: i for i, op in enumerate(self.ops)} if bk is not None else None
        labels = self.T(self.labels_t)
        ce_logits = L.ce[1]
        teacher_logits, w_dst, T_dst = None, 0.0, 1.0
        if L.dst is not None:
            teacher_logits = self.teacher.T(self.teacher.logits_t)
            w_dst, T_dst = L.dst[2], L.dst[3]
        gl, _ = self.grad_target(ce_logits)
        ops.softmax_ce(self.T(ce_logits), labels, teacher_logits, T_dst, w_dst, gl.view(ce_logits.shape),
                       self.loss_out[:4], self.row_ws)
        for op in reversed(self.ops):
            if bk is not None and not bk_fired and op_pos[op] < bk['pos']:
                bk_fired = True
                self._bucket_hi(bk, allreduce)
            ty = op.type
            if ty == 'Placeholder':
                continue
            gy = self.grad_of(op.output)
            if gy is None:
                continue
            if self._passthrough(op) or op in self.fused_into:
                continue                                   # gradient buffer is shared with the input
            if ty in ('Conv2D', 'MatMul'):
                lo, x_t = self.conv[op], op.inputs[0]
                y = self.buf[op.output]
                m, k = y.numel() // y.shape[-1], y.shape[-1]
                if op in self.fused_act:
                    dz = self.relu_scratch[op]
                    ops.relu_bwd(gy, y, dz, self.fused_act[op])
                    gy = dz
                if 'bias' in op.vars:
                    ops.colsum(gy, m, k, st.view(op.vars['bias'], self.G))
                with self.timed('conv_wgrad'):
                    if lo.side and self._side_active:
                        # the weight gradient runs on the side stream, beside the dgrad / BN-backward chain that
                        # continues on the main stream
                        self.side2.wait_stream(torch.cuda.current_stream())
                        with torch.cuda.stream(self.side2):
                            lo.wgrad(gy, self.wgrad_ws2)
                    else:
                        lo.wgrad(gy, self.wgrad_ws)
                if x_t.op.type != 'Placeholder':
                    gx, acc = self.grad_target(x_t)
                    with self.timed('conv_dgrad'):
                        lo.dgrad(gy, gx, acc)
            elif ty == 'DepthwiseConv2dNative':
                self.depthwise[op].backward(gy)
            elif ty == 'FusedBatchNorm':
                self.batch_norm[op].backward(gy)
            elif ty == 'GatherChannels':
                # also the backward of a gather fused into its BN: the scatter fills that BN's dy buffer
                gp = self.bn_gplanes.get(op)
                only = gp is not None and self.bn_gplanes_only[op]
                gx, acc = self.grad_target(op.inputs[0])
                assert not (only and acc)
                with self.timed('scatter'):
                    ops.scatter_channels(gy, self.scatter_inv[op], None if only else gx, acc, gp)
            elif ty == 'MaxPool':
                x_t = op.inputs[0]
                gx, acc = self.grad_target(x_t)
                with self.timed('pool'):
                    ops.maxpool_bwd(self.desc[op], gy, self.pool_argmax[op], gx, acc)
            elif ty == 'Dropout':
                gx, acc = self.grad_target(op.inputs[0])
                with self.timed('dropout'):
                    ops.dropout_bwd(gy, self.dropout[op], op.attrs['keep_prob'], gx, acc)
            elif ty == 'Mean':
                x_t = op.inputs[0]
                n, h, w, c = x_t.shape
                gx, acc = self.grad_target(x_t)
                with self.timed('pool'):
                    ops.global_avgpool_bwd(gy, n, h * w, c, gx, acc)
            elif ty == 'Add':
                for x_t in op.inputs:
                    if self.gkey(x_t) is self.gkey(op.output):
                        continue                           # gradient buffer shared with the output (plan-time alias)
                    gx, acc = self.grad_target(x_t)
                    with self.timed('add_bwd'):
                        ops.add(gy, None, gx, acc)
            elif ty == 'Softmax':
                x_t = op.inputs[0]
                gx, acc = self.grad_target(x_t)
                assert not acc
                ops.softmax_bwd(gy, self.buf[op.output], gx)
            else:
                raise NotImplementedError('backward of %s' % ty)
        if self._side_active:
            torch.cuda.current_stream().wait_stream(self.side2)
        if bk is not None and bk_fired:
            # the rest of the buffer: [0, split) of the first range and everything behind it (BN scales / offsets, ...)
            if bk['red_lo'] is not None:
                bk['red_lo'].reduce()
            if bk['ste_lo']:
                self.wq.ste_backward_(self._ste_grads, bk['ste_lo'])
            allreduce(self.G[:bk['split']])
            if bk['end'] < self.G.numel():
                allreduce(self.G[bk['end']:])
            torch.cuda.current_stream().wait_stream(bk['stream'])
            return
        if self.wg_reduce is not None:
            with self.timed('conv_wgrad'):
                self.wg_reduce.reduce()
        if self._ste_grads is not None:
            self.wq.ste_backward_(self._ste_grads)
        if self.train_clusters:
            # codebook gradients from the gradients w.r.t. the quantized kernels (which stay, unchanged, as the kernels'
            # own gradients: the straight-through estimator of utils.py:303-306)
            with self.timed('weight_quant'):
                self.wq.cluster_grad([st.view(op.vars['kernel'], self.G) for op in self.wq_ops], self.G)

    @contextlib.contextmanager
    def standalone_forward(self):
        """forward() calls outside device_step (layer-wise regression passes): an executor that shares the first layer's
        im2col columns with the distillation teacher normally lets the teacher's forward fill them — here it fills
        them itself."""
        saved = {op: im['compute'] for op, im in self.im2col.items()}
        for im in self.im2col.values():
            im['compute'] = True
        try:
            yield self
        finally:
            for op, c in saved.items():
                self.im2col[op]['compute'] = c

    def layer_wgrad(self, op, gy, dw):
        """dW of ONE Conv2D / MatMul for an externally supplied gradient `gy` of its output, after a training-mode
        forward() of this executor: the weight gradient of the layer-wise regression loss of the channel-pruning
        learner (learners/channel_pruning_gpu/learner.py:370, :391 — compute_gradients(reg_loss_i, [kernel_i])).
        Same kernels as the step's own backward; `dw` is an fp32 tensor of the kernel's shape."""
        # own dy planes: the step's dy_scratch is only sized for the layers whose gradient is split in a separate pass
        lw = getattr(self, '_lw_planes', None)
        if lw is None or lw.numel < op.output.numel:
            lw = self._lw_planes = ops.Planes(op.output.numel, self.device)
        with self.timed('conv_wgrad'):
            self.conv[op].wgrad(gy, self.wgrad_ws, dw, lw.buf)

    def forward_eval_loss(self):
        """Evaluation pass: BN in inference mode, quantizers active, losses/metrics only."""
        if self.teacher is not None:
            self.teacher.forward()
        self.forward(training=False)
        L = self.loss
        teacher_logits, w_dst, T_dst = None, 0.0, 1.0
        if L.dst is not None:
            teacher_logits = self.teacher.T(self.teacher.logits_t)
            w_dst, T_dst = L.dst[2], L.dst[3]
        scratch = self.gbuf[self.gkey(L.ce[1])]
        ops.softmax_ce(self.T(L.ce[1]), self.T(self.labels_t), teacher_logits, T_dst, w_dst,
                       scratch.view(L.ce[1].shape), self.loss_out[:4], self.row_ws)
        self.l2_value()

    def l2_value(self):
        first = True
        for (s, e, masked, wd) in self.store.ranges:
            if wd != 0.0:
                ops.l2_loss(self.store.P[s:e], wd, self.l2_out, self.l2_ws, accumulate=not first)
                first = False
        if first:
            self.l2_out.zero_()

    def apply_gradients(self):
        st, o = self.store, self.optimizer
        for (s, e, masked, wd) in st.ranges:
            if e <= s or (s, e) in st.frozen_ranges:
                continue
            if o['kind'] == 'momentum':
                mask = self.MASK[s:e] if (masked and self.MASK is not None) else None
                ops.momentum_step(st.P[s:e], self.S1[s:e], self.G[s:e], mask, self.hp, o.get('momentum', 0.9), wd,
                                  self.grad_scale)
            else:
                ops.adam_step(st.P[s:e], self.S1[s:e], self.S2[s:e], self.G[s:e], self.hp, o.get('beta1', 0.9),
                              o.get('beta2', 0.999), o.get('eps', 1e-8), wd, self.grad_scale)

    def share_im2col_from(self, other):
        """The teacher and the student read the same image batch: reuse the teacher's im2col of the first
        layer (it runs first inside device_step) instead of recomputing it."""
        for op, im in self.im2col.items():
            for op2, im2 in other.im2col.items():
                if op.inputs[0] is op2.inputs[0] and im['kpad'] == im2['kpad'] and im['planes'] == im2['planes'] \
                        and im['mode'] == im2['mode'] \
                        and all(op.attrs[a] == op2.attrs[a] for a in ('ksize', 'strides', 'pad')):
                    im['cols'] = im2['cols']
                    im['compute'] = False
                    self._shares_cols = True

    # ------------------------------------------------------------------ one training step
    def device_step(self, allreduce=None):
        """Everything that runs on the GPU for one step (CUDA-graph capturable)."""
        par = self.overlap and self.prof is None and self.teacher is not None
        if par:
            main = torch.cuda.current_stream()
            self.side.wait_stream(main)
            if self._shares_cols:
                self.teacher.cols_event = self.cols_wait = torch.cuda.Event()
            with torch.cuda.stream(self.side):
                self.teacher.forward()
            self.forward()
            main.wait_stream(self.side)
            self.teacher.cols_event = self.cols_wait = None
        else:
            if self.teacher is not None:
                self.teacher.forward()
            self.forward()
        self.loss_and_backward(allreduce)
        if allreduce is not None and not (self._side_active and self._bucket_plan() is not None):
            with self.timed('allreduce'):
                allreduce(self.G)
        with self.timed('optimizer'):
            self.l2_value()
            self.apply_gradients()

    def set_hyper(self, lr):
        i = self._hp_i % self.hp_ring.shape[0]
        self._hp_i += 1
        if self.hp_events[i] is not None:
            self.hp_events[i].synchronize()            # slot's previous upload has executed (16 steps ago: no wait)
        slot = self.hp_ring[i]
        slot[0] = float(lr)
        slot[1] = float(self.beta1_power)
        slot[2] = float(self.beta2_power)
        self.hp.copy_(slot, non_blocking=True)
        if self.hp.device.type == 'cuda':
            ev = torch.cuda.Event()
            ev.record()
            self.hp_events[i] = ev

    def advance_optimizer_state(self):
        if self.optimizer.get('kind') == 'adam':
            self.beta1_power = F32(self.beta1_power * F32(self.optimizer.get('beta1', 0.9)))
            self.beta2_power = F32(self.beta2_power * F32(self.optimizer.get('beta2', 0.999)))
        self.step_count += 1

    def reset_optimizer_slots(self):
        """tf.variables_initializer(optimizer.variables()) — run after every mask update
        (weight_sparsification/learner.py:128,217)."""
        self.S1.zero_()
        if self.S2 is not None:
            self.S2.zero_()

    def reset_optimizer_state(self):
        """A fresh optimizer: zero slots, Adam's beta powers and the step counter back to their initial values."""
        self.reset_optimizer_slots()
        self.beta1_power = F32(self.optimizer.get('beta1', 0.9))
        self.beta2_power = F32(self.optimizer.get('beta2', 0.999))
        self.step_count = 0

    def set_quant_bits(self, w_bits=None, a_bits=None):
        """New bit-widths for the quantized layers / activations.  The reference feeds them through placeholders on
        every sess.run (uniform_quantization/learner.py:330-337); here they are launch arguments (the weight
        quantizer's segment table, the activation kernels' `bits`), so a captured step graph is dropped and the next
        steps run eagerly until `capture` is called again."""
        if w_bits is not None:
            if self.wq is None:
                raise ValueError('this executor has no weight quantizer')
            self.wq.set_bits(list(w_bits))
            self.weight_quant['bits'] = list(w_bits)
            if self.tc_batch is not None and self.w_lv:
                self.tc_batch.set_bits({lv['batch_index']: self.wq.bits[lv['index']] for lv in self.w_lv.values()})
        if a_bits is not None:
            if len(a_bits) != len(self.aq_ops):
                raise ValueError('one bit-width per quantized activation expected (%d)' % len(self.aq_ops))
            if any(int(b) < 1 or int(b) > 32 for b in a_bits):
                raise ValueError('bit-widths must be in [1, 32]')
            if self.act_quant:
                self.act_quant['bits'] = [int(b) for b in a_bits]
        self._graph = None

    def capture(self, allreduce=None):
        """Capture device_step into a CUDA graph (after one eager warm-up on a side stream)."""
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            self.device_step(allreduce)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        self._graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self._graph):
            self.device_step(allreduce)
        return self._graph

    def run_step(self, lr, allreduce=None):
        self.set_hyper(lr)
        if self._graph is not None:
            self._graph.replay()
        else:
            self.device_step(allreduce)
        self.advance_optimizer_state()

    def fetch_losses(self):
        """(hard CE, distillation, l2, total, top1, top5) of the last step — one small D2H read."""
        dev_vals = torch.cat([self.loss_out[:4], self.l2_out[:1]])
        self.last_d2h_bytes = dev_vals.numel() * dev_vals.element_size()      # what this call reads back
        o = dev_vals.cpu().numpy()
        hard, dst, top1, top5, l2 = [F32(x) for x in o]
        total = F32(F32(hard + l2) + dst)
        return dict(model_loss=F32(hard + l2), dst_loss=dst, l2=l2, ce=hard, loss=total, acc_top1=top1,
                    acc_top5=top5)
