"""Uniformly quantized models at inference on the 8-bit integer tensor cores.

The uniform-quantization learner (`--learner uniform`) trains a network whose convolutions see fake-quantized operands:
weights w_q = alpha_w[n] * q_w / k_w + beta_w[n] with levels q_w in [0, k_w] (one (alpha, beta) per layer, or per
output channel with `channel` buckets), and every ReLU / ReLU6 output a_q = alpha_a * q_a / k_a + beta_a with its range
taken from the current batch (learners/uniform_quantization/utils.py).  Evaluated as it is trained, such a model still
runs in fp32 on split-bf16 operands.  This module runs it as integers where it can: a convolution whose weights have
<= 8 bits and whose input is a quantized ReLU / ReLU6 output with <= 8 bits computes

    y[m, n] = (alpha_a alpha_w[n] / (k_a k_w)) * sum_K q_a q_w  +  (alpha_a beta_w[n] / k_a) * sum_K q_a

(beta_a = min(act) = 0 after a ReLU) with one u8 x u8 -> s32 tensor-core MMA per 32-wide k-slice, exact, and the
rank-1 term from the activation's per-pixel level sums (pf_conv2d_u8_fwd).  The batch norm + ReLU that produces its
input writes the u8 levels instead of split-bf16 planes (pf_bn_eval_levels_u8).

Which convolutions run as integers is decided from what the graph and the quantizer settings show (`select`): weight
bits, the producer of the input and its activation bits, and the shape the u8 kernel takes (Cin and Cout multiples of
64).  Every other layer keeps the fake-quant inference kernels: the stem and the dense layer, first and last layers
unless all layers are quantized, depthwise convolutions, `split` buckets.

With `cfg['int8_depthwise']` (opt-in; `config_from_flags` leaves it out) the depthwise convolutions that meet the same
conditions run on u8 levels too (pf_dwconv_u8_fwd, CUDA cores: exact window sums S = sum q_a q_w and J = sum q_a per
channel, then the same affine epilogue), fed by the same batch norm + ReLU level producer.  Their sidecar carries
version 2, which loaders before this option refuse.

With `cfg['int8_narrow']` (opt-in, like `int8_depthwise`) the shape conditions widen to channel counts that are
multiples of 16: a convolution qualifies where `ops.conv2d_u8_narrow_supported` holds (pf_conv2d_u8_fwd picks its
cp.async-fed kernel for the shapes the TMA-fed one does not take), a depthwise layer at any input C % 16 == 0, and the
level producer writes any such C.  ResNet-20's 16- and 32-channel stages and MobileNet-v2's depthwise layers and
projections then run on integers.  The sidecar records the option in its config and keeps its version (1, or 2 with
depthwise integer layers): a loader that does not know the option selects fewer integer layers than the file holds
levels for, and IntModel refuses that with its coverage ValueError instead of building a different model.

Calibrated activation ranges (opt-in): `calibrate` runs the fake-quantized model over a few batches and returns a
static (lo, hi) per quantized activation, the float64 mean of the per-batch min / max ('mean', the default: the learner
trained with per-batch ranges) or their extremes ('max').  With `act_ranges`, every quantized activation of the model is
clamped to its range and quantized with lo / hi in place of the batch's min / max, in one pass: the u8 level producer
(pf_bn_eval_levels_u8_static) and the fake-quant BN + act (pf_bn_apply_eval_quant_static) and activation quantizers
(pf_uq_act_quant_static) compute no range, so an image's logits no longer depend on the rest of its batch.  A consumer
whose calibrated input range does not start at 0 keeps fake-quant (the u8 convolution has no term for an activation
offset).  The sidecar of a calibrated model carries the ranges under version 3; one without them is written as before.

select() decides from the graph (and the ranges) alone.  IntModel hands the selected layers and their weight levels to the executor
(`int_layers`), whose plan lowers them (engine._U8Conv, _U8DwConv) and the batch norms feeding them (_U8Bn) beside
every other layer.  A u8 convolution takes the residual and folded batch norm a tensor-core lowering of the layer would
take, and owns no split-bf16 weight copy.  Every selected shape has that lowering on the default conv path (Cin, Cout
% 16 == 0); with another path (PF_CONV_PATH) the executor's plan fails with a ValueError naming the layer, rather than
the layer falling back to fake-quant.

    im = IntModel.from_checkpoint(graph, images, logits, state, cfg)   # the learner's checkpoint (unquantized weights)
    logits = im.forward(images_tensor)
    r = calibrate(graph, images, logits, state, cfg, batches)          # optional: static activation ranges
    im = IntModel.from_checkpoint(graph, images, logits, state, cfg, act_ranges=r)
    im.export(path)                                                    # integer checkpoint + sidecar
    im2 = IntModel.load(graph, images, logits, path)
`graph` / `images` / `logits` are the network's inference graph (compact.build_eval_graph); `cfg` the quantizer settings
(`config_from_flags`).
"""
import json
import os

import numpy as np

from . import compact

F32 = np.float32
SIDECAR_VERSION = 2          # written when depthwise layers run as integers; version 1 otherwise
SIDECAR_VERSION_RANGES = 3   # written when the model has calibrated activation ranges
SIDECAR_VERSIONS = (1, 2, 3)  # what load() reads
STATS = ('mean', 'max')      # calibrate()'s statistics
CFG_KEYS = ('weight_bits', 'activation_bits', 'quantize_all_layers', 'use_buckets', 'bucket_type', 'bucket_size')


def config_from_flags():
    """The uniform learner's quantizer settings (its --uql_* flags)."""
    from .flags import FLAGS
    import pocketflow_b200.learners.uniform_quantization.learner  # noqa: F401  (defines the --uql_* flags)
    return dict(weight_bits=int(FLAGS.uql_weight_bits), activation_bits=int(FLAGS.uql_activation_bits),
                quantize_all_layers=bool(FLAGS.uql_quantize_all_layers), use_buckets=bool(FLAGS.uql_use_buckets),
                bucket_type=str(FLAGS.uql_bucket_type), bucket_size=int(FLAGS.uql_bucket_size))


def quant_marks(graph, cfg):
    """(quantized Conv2D / MatMul / depthwise ops, quantized Relu / Relu6 ops) of `graph`, as the learner marks them
    (UniformQuantization.search_matmul_op / search_activation_op)."""
    from .learners.uniform_quantization.utils import UniformQuantization
    uq = UniformQuantization(graph, cfg['bucket_size'], cfg['use_buckets'], cfg['bucket_type'])
    mm = uq.search_matmul_op(cfg['quantize_all_layers'])
    acts = [op for op in uq.search_activation_op() if op.type in ('Relu', 'Relu6')]
    return list(mm), acts


def weight_levels(kernel, bits, per_channel):
    """The weight quantizer's levels and scales of one kernel (the arithmetic of oracle.pf_oracle.uniform_quantize):
    alpha = (max - min) + 1e-10, beta = min per bucket, q = rint(((w - beta) / alpha) * k) in fp32.  Returns
    (levels uint8 with the kernel's shape, alpha [buckets], beta [buckets])."""
    w = np.ascontiguousarray(kernel, F32)
    cols = w.reshape(-1, w.shape[-1]) if per_channel else w.reshape(-1, 1)
    mx, mn = cols.max(axis=0), cols.min(axis=0)
    alpha = (mx - mn).astype(F32) + F32(1e-10)
    beta = mn.astype(F32)
    k = F32(2 ** bits - 1)
    q = np.rint((((cols - beta) / alpha).astype(F32) * k).astype(F32))
    return q.astype(np.uint8).reshape(w.shape), alpha.astype(F32), beta


def dequantize(levels, alpha, beta, bits):
    """alpha * (q / k) + beta in fp32, op by op (uq_inv_scale): the fake-quantized weight the levels stand for."""
    q = np.asarray(levels, F32)
    cols = q.reshape(-1, alpha.shape[0])
    k = F32(2 ** bits - 1)
    return ((alpha * (cols / k).astype(F32)).astype(F32) + beta).astype(F32).reshape(q.shape)


def _conv_desc(op):
    from . import ops
    n, h, w, c = op.inputs[0].shape
    _, p, q, k = op.output.shape
    (kh, kw), (sh, sw), (pt, pl) = op.attrs['ksize'], op.attrs['strides'], op.attrs['pad']
    return ops.conv_desc(n, h, w, c, k, kh, kw, p, q, sh, sw, pt, pl)


def range_stats(per_batch, stat='mean'):
    """{name: (lo, hi)} in fp32 from per-batch ranges [{name: (lo, hi)}, ...]: 'mean' = the float64 mean of the
    per-batch min and max (with one batch, that batch's range bit for bit), 'max' = the extremes over the batches."""
    if stat not in STATS:
        raise ValueError('calibration statistic %r (one of %s)' % (stat, ', '.join(STATS)))
    if not per_batch:
        raise ValueError('calibration needs at least one batch')
    out = {}
    for name in per_batch[0]:
        r = np.array([b[name] for b in per_batch], np.float64)
        lo, hi = (r.mean(axis=0) if stat == 'mean' else (r[:, 0].min(), r[:, 1].max()))
        out[name] = (F32(lo), F32(hi))
    return out


def executor_ranges(ex, batches, stat='mean'):
    """range_stats of the per-batch ranges an inference executor's activation quantizers write into their slots, over
    `batches` (an iterable of image tensors of its input's shape, each read once, in turn)"""
    from . import ops
    if ex.aq_static:
        raise ValueError('the executor already quantizes with static ranges: it computes none per batch')
    per_batch = []
    for x in batches:
        ex.buf[ex.images].copy_(x)
        ex.forward(training=False)
        r = ops.decode_ordered(ex.aq_slots.cpu().numpy().view(np.uint32)).reshape(-1, 2)
        per_batch.append({op.name: (r[i, 0], r[i, 1]) for i, op in enumerate(ex.aq_ops)})
    return range_stats(per_batch, stat)


def calibrate(graph, images, logits, state, cfg, batches, stat='mean', device=None):
    """Static activation ranges {Relu / Relu6 op name: (lo, hi) fp32} of every activation quant_marks returns: the
    fake-quantized model (fake_quant_executor, the learner's checkpoint `state`) run over `batches`, its per-batch
    ranges combined by `stat` (range_stats)."""
    import torch
    device = device or torch.device('cuda', torch.cuda.current_device())
    full = compact.map_state(graph, compact.reachable_ops(graph, logits), state)
    return executor_ranges(fake_quant_executor(graph, images, logits, full, cfg, device), batches, stat)


def _ranges(graph, cfg, act_ranges):
    """act_ranges normalised to {name: (F32 lo, F32 hi)}, checked to cover every quantized activation"""
    if act_ranges is None:
        return None
    names = [op.name for op in quant_marks(graph, cfg)[1]]
    missing = [n for n in names if n not in act_ranges]
    if missing:
        raise ValueError('no calibrated range for the quantized activations %s' % missing)
    out = {n: (F32(act_ranges[n][0]), F32(act_ranges[n][1])) for n in names}
    bad = [n for n, (lo, hi) in out.items() if not lo <= hi]
    if bad:
        raise ValueError('calibrated ranges with lo > hi (or NaN): %s' % bad)
    return out


def select(graph, logits, cfg, act_ranges=None):
    """[(op name, None or the reason it keeps the fake-quant kernels)] for every Conv2D / MatMul / depthwise op in
    graph order; None = it runs on a u8 kernel.  Depthwise ops are considered only with cfg['int8_depthwise'];
    cfg['int8_narrow'] admits channel counts that are multiples of 16; with calibrated `act_ranges` ({activation name:
    (lo, hi)}) a layer whose input range does not start at 0 keeps fake-quant."""
    from . import ops
    mm, acts = quant_marks(graph, cfg)
    mm, acts = set(mm), set(acts)
    act_ranges = _ranges(graph, cfg, act_ranges)
    depthwise = bool(cfg.get('int8_depthwise', False))
    narrow = bool(cfg.get('int8_narrow', False))
    out = []
    for op in compact.reachable_ops(graph, logits):
        if op.type not in ('Conv2D', 'MatMul', 'DepthwiseConv2dNative'):
            continue
        x = op.inputs[0]
        dw = op.type == 'DepthwiseConv2dNative'
        why = None
        if op not in mm:
            why = 'weights not quantized (first / last layer)'
        elif dw and not depthwise:
            why = 'depthwise convolution'
        elif op.type == 'MatMul':
            why = 'dense layer'
        elif cfg['use_buckets'] and cfg['bucket_type'] != 'channel':
            why = '%s buckets' % cfg['bucket_type']
        elif cfg['weight_bits'] > 8:
            why = 'weight bits %d > 8' % cfg['weight_bits']
        elif x.op not in acts or x.op.inputs[0].op.type != 'FusedBatchNorm' or len(x.op.inputs[0].consumers) != 1:
            why = 'input is not a quantized batch norm + ReLU output'
        elif cfg['activation_bits'] > 8:
            why = 'activation bits %d > 8' % cfg['activation_bits']
        elif act_ranges is not None and act_ranges[x.op.name][0] != 0:
            why = 'calibrated activation range does not start at 0'
        else:
            c = x.shape[-1]
            if dw and (c < 16 or (c % 16 if narrow else c & (c - 1))):
                why = 'input channels %d: the level producer needs %s' % (
                    c, 'a multiple of 16' if narrow else 'a power of two >= 16')
            elif dw:
                if not ops.dwconv_u8_supported(_conv_desc(op)):
                    (kh, kw), (sh, sw) = op.attrs['ksize'], op.attrs['strides']
                    why = 'depthwise %dx%d stride %dx%d over %d channels (the u8 depthwise kernel needs C %% 16 == 0, ' \
                          '<= 9 taps, strides 1 or 2)' % (kh, kw, sh, sw, c)
            elif narrow:
                if not ops.conv2d_u8_narrow_supported(_conv_desc(op)):
                    why = 'shape %d -> %d channels (the u8 kernels need multiples of 16)' % (c, op.output.shape[-1])
            elif c < 16 or c & (c - 1):
                why = 'input channels %d not a power of two' % c
            elif not ops.conv2d_u8_supported(_conv_desc(op)):
                why = 'shape %d -> %d channels (the u8 kernel needs multiples of 64)' % (c, op.output.shape[-1])
        out.append((op.name, why))
    return out


def report_lines(sel):
    """What tools/export_uq_int8.py prints: one line per layer."""
    def path(name, why):
        if why is not None:
            return 'fake-quant (%s)' % why
        return 'u8 depthwise (CUDA cores)' if name.rsplit('/', 1)[-1] == 'depthwise' else 'u8 x u8 tensor cores'
    lines = ['%s: %s' % (name, path(name, why)) for name, why in sel]
    n = sum(1 for _, why in sel if why is None)
    lines.append('%d of %d layers run as integers' % (n, len(sel)))
    return lines


def _specs(graph, cfg, exclude=(), act_ranges=None):
    """the Executor's weight_quant / act_quant specs of the fake-quant model, less the weight quantizers of `exclude`;
    with act_ranges ({name: (lo, hi)}, _ranges) the activation quantizers take them as static ranges"""
    mm, acts = quant_marks(graph, cfg)
    mm = [op for op in mm if op.name not in exclude]
    wq = dict(kind='uniform', ops=mm, bits=[cfg['weight_bits']] * len(mm), use_buckets=cfg['use_buckets'],
              bucket_type=cfg['bucket_type'], bucket_size=cfg['bucket_size']) if mm else None
    aq = dict(ops=acts, bits=[cfg['activation_bits']] * len(acts)) if acts else None
    if aq and act_ranges is not None:
        aq['ranges'] = [act_ranges[op.name] for op in acts]
    return wq, aq


def _load(ex, state):
    """Load an inference executor's parameters and prepare its tensor-core weight copies from the QUANTIZED kernels:
    an inference executor prepares them once, when its store is loaded, and the weight quantizer has not run by then."""
    ex.store.load_state_dict(state, strict=True)
    if ex.wq is not None:
        ex.wq.forward()
    ex.prepare_static_weights()


def fake_quant_executor(graph, images, logits, state, cfg, device, act_ranges=None):
    """The fake-quantized model as the learner evaluates it, on `graph` in inference mode (engine.Executor); with
    act_ranges (calibrate) its activations are quantized with those static ranges instead of each batch's."""
    from .engine import Executor
    wq, aq = _specs(graph, cfg, act_ranges=_ranges(graph, cfg, act_ranges))
    ex = Executor(graph, images, logits, device, train=False, weight_quant=wq, act_quant=aq)
    _load(ex, state)
    return ex


class IntModel:
    """A uniformly quantized model whose eligible convolutions run on the u8 kernels: an inference engine.Executor
    given them as its `int_layers`, whose plan lowers them and the batch norms feeding them to the u8 kernels."""

    # None, or the static {activation name: (lo, hi)} it quantizes with (calibrate); a class default as well, so that
    # export() answers for subclasses that fill the model's fields without this __init__
    act_ranges = None

    def __init__(self, graph, images, logits, cfg, state, wlevels, device=None, act_ranges=None):
        """state: {variable name: fp32 array} of every variable but the integer layers' kernels; wlevels: {conv op
        name: (levels uint8 HWIO, alpha, beta)} of the integer layers; act_ranges: None (each batch's ranges) or the
        static {activation name: (lo, hi)} of every quantized activation (calibrate)"""
        import torch
        from .engine import Executor
        self.graph, self.images, self.logits, self.cfg = graph, images, logits, dict(cfg)
        self.act_ranges = _ranges(graph, cfg, act_ranges)
        self.sel = select(graph, logits, cfg, self.act_ranges)
        ints = [name for name, why in self.sel if why is None]
        if sorted(ints) != sorted(wlevels):
            raise ValueError('the weight levels do not cover the integer layers: %s' % sorted(set(ints) ^ set(wlevels)))
        self.wlevels = wlevels
        self.state = dict(state)
        bits = cfg['weight_bits']
        byname = {op.name: op for op in compact.reachable_ops(graph, logits)}
        full, int_layers = dict(state), {}
        for name, (lv, al, be) in wlevels.items():                 # the executor's copy: the fake-quantized kernel
            full[byname[name].vars['kernel'].name] = dequantize(lv, al, be, bits)
            int_layers[byname[name]] = (lv, al, be, bits)
        self.device = device or torch.device('cuda', torch.cuda.current_device())
        wq, aq = _specs(graph, cfg, exclude=set(ints), act_ranges=self.act_ranges)
        self.ex = Executor(graph, images, logits, self.device, train=False, weight_quant=wq, act_quant=aq,
                           int_layers=int_layers)
        _load(self.ex, full)

    @classmethod
    def from_checkpoint(cls, graph, images, logits, state, cfg, device=None, act_ranges=None):
        """From the uniform learner's checkpoint (unquantized weights under any one scope, compact.map_state), with
        calibrated activation ranges or without."""
        full = compact.map_state(graph, compact.reachable_ops(graph, logits), state)
        per_channel = cfg['use_buckets'] and cfg['bucket_type'] == 'channel'
        byname = {op.name: op for op in compact.reachable_ops(graph, logits)}
        wlevels = {}
        for name, why in select(graph, logits, cfg, act_ranges):
            if why is None:
                kname = byname[name].vars['kernel'].name
                wlevels[name] = weight_levels(full.pop(kname), cfg['weight_bits'], per_channel)
        return cls(graph, images, logits, cfg, full, wlevels, device, act_ranges)

    def calibrate(self, batches, stat='mean'):
        """Static activation ranges {name: (lo, hi)} measured on this (per-batch) integer model's own activations over
        `batches`, combined by `stat` (range_stats): with the batch that is then evaluated, a model built with them
        computes what this one computes."""
        return executor_ranges(self.ex, batches, stat)

    def forward(self, images=None):
        """Logits (device tensor, the executor's own buffer) of `images` (or of what the input buffer holds)."""
        if images is not None:
            self.ex.buf[self.images].copy_(images)
        return self.ex.forward(training=False)

    def export(self, path):
        """Write the integer checkpoint `path`.npz (the other variables in fp32 under their names; per integer layer
        `<kernel>/levels` uint8 HWIO, `<kernel>/alpha` and `<kernel>/beta`) and the sidecar `path`.int8.json (quantizer
        settings and the layer selection).  Returns the checkpoint's file name."""
        os.makedirs(os.path.dirname(path) or '.', exist_ok=True)
        byname = {op.name: op for op in compact.reachable_ops(self.graph, self.logits)}
        arrays = {k.replace('/', '|'): v for k, v in self.state.items()}
        for name, (lv, al, be) in self.wlevels.items():
            k = byname[name].vars['kernel'].name[:-2]
            arrays[(k + '/levels').replace('/', '|')] = lv
            arrays[(k + '/alpha').replace('/', '|')] = al
            arrays[(k + '/beta').replace('/', '|')] = be
        fn = path + '.npz'
        np.savez(fn, **arrays)
        version = SIDECAR_VERSION if any(byname[n].type == 'DepthwiseConv2dNative' for n in self.wlevels) else 1
        rec = dict(version=version, config=self.cfg, layers=[[n, w] for n, w in self.sel])
        if self.act_ranges is not None:      # fp32 -> JSON double -> fp32 is exact
            rec.update(version=SIDECAR_VERSION_RANGES,
                       act_ranges={n: [float(lo), float(hi)] for n, (lo, hi) in self.act_ranges.items()})
        with open(path + '.int8.json', 'w') as f:
            json.dump(rec, f)
        return fn

    @classmethod
    def load(cls, graph, images, logits, path, device=None):
        """Rebuild the integer model from what export(path) wrote."""
        with open(path + '.int8.json') as f:
            rec = json.load(f)
        if rec.get('version') not in SIDECAR_VERSIONS:
            raise ValueError('%s.int8.json: unsupported sidecar version %r (this loader reads %s)'
                             % (path, rec.get('version'), ', '.join(map(str, SIDECAR_VERSIONS))))
        if (rec['version'] == SIDECAR_VERSION_RANGES) != ('act_ranges' in rec):
            raise ValueError('%s.int8.json: unsupported sidecar version %r with%s act_ranges (version %d carries them)'
                             % (path, rec['version'], '' if 'act_ranges' in rec else 'out', SIDECAR_VERSION_RANGES))
        cfg = {k: rec['config'][k] for k in CFG_KEYS}
        for opt in ('int8_depthwise', 'int8_narrow'):
            if rec['config'].get(opt):
                cfg[opt] = True
        d = np.load(path + '.npz')
        arrays = {k.replace('|', '/'): d[k] for k in d.files}
        byname = {op.name: op for op in compact.reachable_ops(graph, logits)}
        wlevels = {}
        for name, why in rec['layers']:
            if why is None:
                k = byname[name].vars['kernel'].name[:-2]
                wlevels[name] = (arrays.pop(k + '/levels'), arrays.pop(k + '/alpha'), arrays.pop(k + '/beta'))
        kw = dict(act_ranges=rec['act_ranges']) if 'act_ranges' in rec else {}
        return cls(graph, images, logits, cfg, arrays, wlevels, device, **kw)
