"""Channel-pruned networks at their pruned width.

The channel-pruning learners (`chn-pruned-gpu`, `chn-pruned-rmt`) end with a masked model at full width: the pruned
input channels of every convolution are zero rows of its kernel, and are still loaded, multiplied and stored.  This
module turns such a masked model into a compact one, the counterpart of the reference's
tools/conversion/export_chn_pruned_tflite_model.py (`insert_alt_routines`: `gather(x, nnzs)` followed by a conv on
`kernel[:, :, nnzs, :]`), carried through the whole inference graph:

1. Input set of every Conv2D: the channels with `sum(|kernel|, axis=(0, 1, 3)) != 0`, the reference's `nnzs`, computed
   with the same numpy reduction.  A MatMul (the dense layer) needs all its inputs.
2. Backward liveness: the live channels of a tensor are the union of what its consumers need.  Per-channel ops
   (BN, ReLU / ReLU6, depthwise conv, pooling, squeeze, Identity, Dropout, Add) pass their output's live set to their
   input(s); a Conv2D's output channels shrink to its output's live set; the logits are all live.  A dead channel only
   ever meets zero kernel rows, so dropping it is exact.
3. Layouts: every tensor of the compact graph holds a list of full-width channel indices, -1 for a zero padding
   channel.  A Conv2D / Add output holds its live set, padded with zero channels to a multiple of 16 when the full
   width is a multiple of 16 (so a convolution that ran on the tensor cores at full width still does), else to a
   multiple of 4 (the vector width of the BN / depthwise / pooling kernels).  A per-channel op keeps its input's layout.
   The image is never narrowed.  A layer whose whole input is dead keeps one padding group of zero channels.
4. Where a consumer needs a strict subset of a tensor's channels, a `GatherChannels` op (attrs['index']: positions in
   its input's layout, -1 for padding) narrows it; engine.Executor lowers it to pf_gather_channels, or fuses it into the
   inference-mode BN apply that produces its input (pf_bn_apply_eval_gather).

Padding channels carry zero kernel rows and columns, zero bias, and BN gamma = beta = moving mean = 0, moving
variance = 1, so they stay exactly zero through every op.

The same plan applies to the TRAINING graph of a ModelHelper (forward_train): training-mode BN, Dropout and the
linear-bottleneck BN + Add are per-channel ops too.  `CompactTrainer` builds the training step of a channel-pruning
learner at the pruned width from the learner's masked full-width step executor: parameters, optimizer slots and masks
are sliced into it (`slice_state`) and expanded back (`expand_state`), so the learner keeps writing its masked
full-width checkpoints.  A padding channel also stays exactly zero through a training step: its activations are 0, so
its batch mean and variance are 0 and BN gives ((0 - 0) * rstd) * 0 + 0 = 0; the BN backward multiplies dx by gamma = 0
and forms dgamma from xhat = 0; dbeta and a bias gradient are column sums of a gradient that is 0 because every
consumer reads the channel through zero kernel rows (dgrad) or never gathers it (scatter); the weight gradient of a
padding row is a sum of 0 * dy and of a padding column a sum of x * 0; with zero weight, slot and gradient the Momentum
update acc = m * acc + (g + wd * 0), w -= lr * acc leaves 0, and the sliced mask is 0 there besides.
"""
import json
import os
from collections import OrderedDict

import numpy as np

from . import graph as G

PER_CHANNEL = ('FusedBatchNorm', 'Relu', 'Relu6', 'DepthwiseConv2dNative', 'MaxPool', 'Mean', 'Identity', 'Dropout')
SIDECAR_VERSION = 1


def conv_input_channels(kernel):
    """The reference's `nnzs` of a conv kernel [kh, kw, cin, cout] (export_chn_pruned_tflite_model.py:249)."""
    return np.nonzero(np.sum(np.abs(kernel), axis=(0, 1, 3)))[0]


def fake_prune(graph, logits, state, ratio, seed):
    """The reference export tool's --enbl_fake_prune (apply_fake_pruning, export_chn_pruned_tflite_model.py:186-203):
    after np.random.seed(seed), every Conv2D kernel in graph order loses int(cin * ratio) randomly shuffled input
    channels.  For speed measurements without a trained model.  Returns a new state dict; `state` is keyed by the
    graph's variable names."""
    out = dict(state)
    np.random.seed(seed)
    for op in reachable_ops(graph, logits):
        if op.type != 'Conv2D':
            continue
        k = np.array(state[op.vars['kernel'].name], np.float32, copy=True)
        nb_chns = k.shape[2]
        idxs_all = np.arange(nb_chns)
        np.random.shuffle(idxs_all)
        k[:, :, idxs_all[:int(nb_chns * ratio)], :] = 0.0
        out[op.vars['kernel'].name] = k
    return out


def _per_channel(op):
    if op.type in PER_CHANNEL:
        return True
    # a squeeze of [N, 1, 1, C] keeps the channel axis; a flatten of a spatial map does not
    return op.type == 'Reshape' and op.inputs[0].shape[-1] == op.output.shape[-1] and \
        int(np.prod(op.inputs[0].shape[1:-1])) == 1


def padded_width(n, full):
    """Channels a compact tensor of `n` live channels (of `full`) holds."""
    q = 16 if full % 16 == 0 else 4 if full % 4 == 0 else 1
    return min(full, max(q, (n + q - 1) // q * q))


def canonical_layout(channels, full):
    keep = sorted(int(c) for c in channels)
    return keep + [-1] * (padded_width(len(keep), full) - len(keep))


def reachable_ops(graph, logits):
    seen, stack = set(), [logits.op]
    while stack:
        op = stack.pop()
        if op in seen:
            continue
        seen.add(op)
        stack.extend(t.op for t in op.inputs)
    return [op for op in graph.ops if op in seen]


def map_state(graph, ops_, state):
    """{variable name of `graph`: array} from a checkpoint of the same net under any single scope (the learners write
    'pruned_model/...'; a full-precision checkpoint 'model/...').  Every variable of the graph must be matched, with
    its shape."""
    scopes = sorted({k.split('/', 1)[0] for k in state if '/' in k})
    prefer = 'pruned_model' if 'pruned_model' in scopes else None
    by_suffix = {}
    for k, v in state.items():
        if '/' not in k:
            continue
        scope, rest = k.split('/', 1)
        if prefer is not None and scope != prefer:
            continue
        if rest in by_suffix:
            raise ValueError('checkpoint holds %s under more than one scope (%s)' % (rest, scopes))
        by_suffix[rest] = v
    out = {}
    for op in ops_:
        for v in op.vars.values():
            rest = v.name.split('/', 1)[1]
            if rest not in by_suffix:
                raise KeyError('missing variable in checkpoint: ' + v.name)
            a = np.asarray(by_suffix[rest], np.float32)
            if a.shape != v.shape:
                raise ValueError('checkpoint variable %s has shape %s, the model\'s has %s' % (v.name, a.shape, v.shape))
            out[v.name] = a
    return out


def plan(graph, logits, state):
    """Liveness + layouts of the compact graph.  Returns the JSON-able record {'tensors': {tensor name: layout},
    'gathers': {'<consumer op>:<input>': layout}, 'convs': {conv op: reference nnzs}}; `state` is the masked full-width
    state dict keyed by the graph's variable names."""
    ops_ = reachable_ops(graph, logits)
    opset = set(ops_)
    need, live, nnz = {}, {}, {}
    for op in reversed(ops_):
        t = op.output
        w = t.shape[-1]
        if t is logits:
            live[t] = set(range(w))
        else:
            s = set()
            for c in t.consumers:
                if c in opset:
                    for i, x in enumerate(c.inputs):
                        if x is t:
                            s |= need[(c, i)]
            live[t] = s
        for i, x in enumerate(op.inputs):
            if op.type == 'Conv2D':
                nz = conv_input_channels(state[op.vars['kernel'].name])
                nnz[op.name] = [int(c) for c in nz]
                need[(op, i)] = set(nnz[op.name])
            elif op.type == 'Add' or _per_channel(op):
                need[(op, i)] = set(live[t])
            else:
                need[(op, i)] = set(range(x.shape[-1]))
    layout, gathers = {}, {}
    for op in ops_:
        t = op.output
        w = t.shape[-1]
        if op.type == 'Placeholder':
            layout[t] = list(range(w))
        elif op.type in ('Conv2D', 'MatMul', 'Add'):
            layout[t] = canonical_layout(live[t], w)
        elif _per_channel(op):
            layout[t] = list(layout[op.inputs[0]])
        else:
            layout[t] = list(range(w))
        for i, x in enumerate(op.inputs):
            have = layout[x]
            real = {c for c in have if c >= 0}
            want = None
            if op.type == 'Conv2D' and x.op.type != 'Placeholder' and real != need[(op, i)]:
                want = canonical_layout(need[(op, i)], x.shape[-1])
            elif op.type == 'Add':
                want = layout[t]
            elif not _per_channel(op) and op.type != 'Conv2D' and have != list(range(x.shape[-1])):
                raise AssertionError('%s needs every channel of %s' % (op.name, x.name))
            if want is not None and want != have:
                gathers['%s:%d' % (op.name, i)] = want
    return dict(version=SIDECAR_VERSION, tensors={t.name: l for t, l in layout.items()}, gathers=gathers, convs=nnz)


def _positions(have, want):
    pos = {c: j for j, c in enumerate(have) if c >= 0}
    return np.array([pos[c] if c >= 0 else -1 for c in want], np.int32)


def _input_layouts(op, rec):
    return [rec['gathers'].get('%s:%d' % (op.name, i), rec['tensors'][x.name]) for i, x in enumerate(op.inputs)]


def build_graph(graph, images, logits, rec):
    """The compact graph.Graph of `rec`: same op and variable names, sliced shapes, GatherChannels ops where a consumer
    reads a narrower layout.  Returns (graph, images tensor, logits tensor)."""
    ops_ = reachable_ops(graph, logits)
    # the gathers of a tensor follow its producer directly (one per distinct layout), so that a residual Add whose
    # shortcut is narrowed can still be fused into the epilogue of the conv that produces its other operand
    wanted = {}
    for op in ops_:
        for i, x in enumerate(op.inputs):
            want = rec['gathers'].get('%s:%d' % (op.name, i))
            if want is not None:
                wanted.setdefault(x.name, []).append((op.name, i, tuple(want)))
    g = G.Graph()
    tmap, gmap = {}, {}
    with g.as_default():
        for op in ops_:
            ins = []
            for i, x in enumerate(op.inputs):
                want = rec['gathers'].get('%s:%d' % (op.name, i))
                ins.append(tmap[x] if want is None else gmap[(x.name, tuple(want))])
            wout = len(rec['tensors'][op.output.name])
            vs = {}
            for role, v in op.vars.items():
                if op.type == 'Conv2D' and role == 'kernel':
                    shape = v.shape[:2] + (ins[0].shape[-1], wout)
                elif op.type == 'MatMul' and role == 'kernel':
                    shape = (ins[0].shape[-1], wout)
                elif op.type == 'DepthwiseConv2dNative':
                    shape = v.shape[:2] + (wout, 1)
                else:
                    shape = (wout,)
                vs[role] = g.get_variable(v.name[:-2], shape, v.initializer, v.trainable)
            attrs = dict(op.attrs)
            if op.type == 'Dropout':
                # the compact mask is the full-width one gathered by the layout (pf_dropout_fwd_mapped)
                attrs.update(layout=np.asarray(rec['tensors'][op.output.name], np.int32),
                             full_width=op.output.shape[-1])
            nop = g.add_op(op.type, op.type, ins, vs, attrs, op.output.shape[:-1] + (wout,), name=op.name)
            if op.type == 'Placeholder':
                g.placeholders[nop.name] = nop.output
            tmap[op.output] = nop.output
            for cname, i, want in wanted.get(op.output.name, []):
                if (op.output.name, want) not in gmap:
                    idx = _positions(rec['tensors'][op.output.name], want)
                    gmap[(op.output.name, want)] = g.add_op(
                        'GatherChannels', 'GatherChannels', [nop.output], {}, dict(index=idx),
                        nop.output.shape[:-1] + (len(want),),
                        name=cname + '/GatherChannels' + ('_%d' % i if i else '')).output
    return g, tmap[images], tmap[logits]


def _take(a, axis, lay, fill=0.0):
    idx = np.asarray(lay, np.int64)
    r = np.take(a, np.where(idx >= 0, idx, 0), axis=axis)
    r = np.moveaxis(r, axis, 0)
    r[idx < 0] = fill
    return np.ascontiguousarray(np.moveaxis(r, 0, axis))


def slice_state(graph, logits, rec, state, partial=False):
    """Compact state dict (same variable names) of the masked full-width `state`.  partial: `state` may hold only some
    of the variables (per-variable views of an optimizer slot, the masks of the maskable kernels)."""
    out = {}
    for op in reachable_ops(graph, logits):
        if not op.vars:
            continue
        lout = rec['tensors'][op.output.name]
        lin = _input_layouts(op, rec)[0] if op.inputs else None
        for role, v in op.vars.items():
            if partial and v.name not in state:
                continue
            a = state[v.name]
            if op.type == 'Conv2D' and role == 'kernel':
                a = _take(_take(a, 2, lin), 3, lout)
            elif op.type == 'MatMul' and role == 'kernel':
                a = _take(_take(a, 0, lin), 1, lout)
            elif op.type == 'DepthwiseConv2dNative':
                a = _take(a, 2, lout)
            else:
                a = _take(a, 0, lout, 1.0 if role == 'moving_variance' else 0.0)
            out[v.name] = a.astype(np.float32)
    return out


def expand_state(graph, logits, rec, compact_state, full_state):
    """The inverse of slice_state: a copy of `full_state` whose kept entries (non-negative positions of the layouts)
    come from `compact_state`; dead producer channels and the zero kernel rows keep what `full_state` holds.  Variables
    missing from `compact_state` are copied unchanged.  expand_state(slice_state(s), s) == s bit for bit."""
    out = {k: np.array(v, np.float32, copy=True) for k, v in full_state.items()}
    for op in reachable_ops(graph, logits):
        if not op.vars:
            continue
        lout = np.asarray(rec['tensors'][op.output.name], np.int64)
        lin = np.asarray(_input_layouts(op, rec)[0], np.int64) if op.inputs else None
        jo = np.nonzero(lout >= 0)[0]
        for role, v in op.vars.items():
            if v.name not in compact_state:
                continue
            a, f = np.asarray(compact_state[v.name], np.float32), out[v.name]
            if op.type in ('Conv2D', 'MatMul') and role == 'kernel':
                ji = np.nonzero(lin >= 0)[0]
                f[..., lin[ji][:, None], lout[jo][None, :]] = a[..., ji[:, None], jo[None, :]]
            elif op.type == 'DepthwiseConv2dNative':
                f[:, :, lout[jo], :] = a[:, :, jo, :]
            else:
                f[lout[jo]] = a[jo]
    return out


def check_widths(graph, logits):
    """Every narrowed shape must be one the kernels run: the BN / depthwise / pooling kernels move 4 channels at a time
    (the executor checks the gathers' own widths when it plans them; a convolution runs at any width, on the CUDA cores
    where the tensor-core kernels do not take it — CompactTrainer.report names those).  Raises a ValueError naming the
    first layer that is not."""
    for op in reachable_ops(graph, logits):
        if op.type in ('FusedBatchNorm', 'DepthwiseConv2dNative', 'MaxPool', 'Mean', 'Add') \
                and (op.output.shape[-1] % 4 or op.inputs[0].shape[-1] % 4):
            raise ValueError('%s: %d -> %d channels at the pruned width; the per-channel kernels need multiples of 4'
                             % (op.name, op.inputs[0].shape[-1], op.output.shape[-1]))


class CompactTrainer:
    """The fine-tune step of a channel-pruning learner at the pruned width.

        ct = CompactTrainer(ex)      # ex: the learner's masked full-width step Executor, channels already chosen
        ct.ex.run_step(lr, allreduce)
        ct.push()                    # parameters, moving statistics and optimizer slots back into `ex`
    The compact executor shares `ex`'s image and label buffers, its distillation teacher (which stays at full width),
    optimizer and grad_scale; its flat gradient buffer (what a data-parallel step all-reduces) has the compact size.
    A compact Dropout draws the masked step's mask gathered by its layout (pf_dropout_fwd_mapped; its step counter moves
    with the state in pull / push), so the two steps drop the same activations.
    Deviations from the masked step: a producer channel that no consumer reads is frozen at the value it has when the
    trainer is built instead of decaying under weight decay, and the reported L2 loss omits it (it cannot reach the
    logits either way); a narrowed K dimension is summed in another fp32 order, so logits agree to rounding."""

    def __init__(self, ex):
        from .engine import Executor
        self.full = ex
        g, logits = ex.g, ex.logits_t
        self.rec = plan(g, logits, ex.store.state_dict())
        self.graph, self.images, self.logits = build_graph(g, ex.images, logits, self.rec)
        check_widths(self.graph, self.logits)
        cvar, L = self.graph.variables, ex.loss
        loss = G.LossSpec()
        loss.ce = (L.ce[0], self.logits, L.ce[2])
        loss.l2 = OrderedDict((cvar[v.name], c) for v, c in L.l2.items())
        if L.dst is not None:
            loss.dst = (self.logits,) + tuple(L.dst[1:])
        self.ex = Executor(self.graph, self.images, self.logits, ex.device, train=True, loss=loss, labels=ex.labels_t,
                           optimizer=ex.optimizer, maskable=[cvar[v.name] for v in ex.maskable], teacher=ex.teacher,
                           seed=ex.seed, grad_scale=ex.grad_scale, conv_path=ex.conv_path, fuse_add=ex.fuse_add)
        self.ex.buf[self.images] = ex.buf[ex.images]              # one mini-batch feeds both executors
        self.ex.buf[ex.labels_t] = ex.buf[ex.labels_t]
        self.pull()

    def _flat_pairs(self):
        """(full flat buffer, compact flat buffer, variables of the full executor held in it)"""
        f, c = self.full, self.ex
        pairs = [(f.S1, c.S1, f.store.train_vars), (f.MASK, c.MASK, f.maskable)]
        if f.S2 is not None:
            pairs.append((f.S2, c.S2, f.store.train_vars))
        return [p for p in pairs if p[0] is not None]

    def pull(self):
        """full-width learner state -> compact executor: parameters, moving statistics, slots, masks, step count,
        dropout step counters"""
        f, c = self.full, self.ex
        g, lg, cvar = f.g, f.logits_t, self.graph.variables
        c.store.load_state_dict(slice_state(g, lg, self.rec, f.store.state_dict()), strict=True)
        for fb, cb, vs in self._flat_pairs():
            part = slice_state(g, lg, self.rec, {v.name: f.store.view(v, fb).cpu().numpy() for v in vs}, partial=True)
            for name, a in part.items():
                c.store.view(cvar[name], cb).copy_(_to_device(a, cb))
        c.step_count, c.beta1_power, c.beta2_power = f.step_count, f.beta1_power, f.beta2_power
        self._copy_drop_state(f, c)

    def _copy_drop_state(self, src, dst):
        """the dropout step counters (a Dropout op keeps its name and its stream index in the compact graph)"""
        if src.drop_state is None:
            return
        for op, i in src.drop_stream.items():
            j = [k for o, k in dst.drop_stream.items() if o.name == op.name]
            assert j == [i], (op.name, i, j)
        dst.drop_state.copy_(src.drop_state)

    def push(self):
        """compact executor -> full-width learner state (the masks do not change while fine-tuning)"""
        f, c = self.full, self.ex
        g, lg = f.g, f.logits_t
        f.store.load_state_dict(expand_state(g, lg, self.rec, c.store.state_dict(), f.store.state_dict()), strict=True)
        for fb, cb, vs in self._flat_pairs():
            if fb is f.MASK:
                continue
            comp = {v.name: c.store.view(self.graph.variables[v.name], cb).cpu().numpy() for v in vs}
            full = expand_state(g, lg, self.rec, comp, {v.name: f.store.view(v, fb).cpu().numpy() for v in vs})
            for v in vs:
                f.store.view(v, fb).copy_(_to_device(full[v.name], fb))
        f.step_count, f.beta1_power, f.beta2_power = c.step_count, c.beta1_power, c.beta2_power
        self._copy_drop_state(c, f)

    def report(self):
        """what tools/export_chn_pruned.py prints: every conv's kept input channels, and the parameter counts"""
        lines = ['%s: reducing %d channels to %d' % (op.name, op.inputs[0].shape[-1], len(self.rec['convs'][op.name]))
                 for op in reachable_ops(self.full.g, self.full.logits_t) if op.type == 'Conv2D']
        n_full = sum(v.numel for v in self.full.variables)
        n_comp = sum(v.numel for v in self.ex.variables)
        lines.append('parameters: %d -> %d (%.1f %%)' % (n_full, n_comp, 100.0 * n_comp / n_full))
        cops = {op.name: op for op in self.ex.ops}
        lost = [op.name for op in self.full.ops if op in self.full.tc_wgrad and cops[op.name] not in self.ex.tc_wgrad]
        if lost:
            lines.append('%d convolutions leave the tensor-core weight-gradient kernel at the pruned width: %s'
                         % (len(lost), ', '.join(lost)))
        return lines


def _to_device(a, like):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(like.device)


def build_eval_graph(model_helper, batch_size, scope='model'):
    """A ModelHelper's inference graph at `batch_size`: (graph, images, logits)."""
    g = G.Graph()
    with g.as_default():
        with G.variable_scope('data'):
            images = G.placeholder((batch_size,) + tuple(model_helper.dataset_eval.image_shape), 'images')
        with G.variable_scope(scope):
            logits = model_helper.forward_eval(images)
    return g, images, logits


def build_train_graph(model_helper, batch_size, scope='model'):
    """A ModelHelper's training graph (forward_train) at `batch_size`: (graph, images, logits)."""
    g = G.Graph()
    with g.as_default():
        with G.variable_scope('data'):
            images = G.placeholder((batch_size,) + tuple(model_helper.dataset_train.image_shape), 'images')
        with G.variable_scope(scope):
            logits = model_helper.forward_train(images)
    return g, images, logits


class CompactModel:
    """A channel-pruned model at its pruned width, run by engine.Executor in inference mode.

        cm = CompactModel.from_masked(graph, images, logits, state)     # masked full-width state dict
        logits = cm.forward(images_tensor)
        cm.export(path)                                                 # compact checkpoint + channel sidecar
        cm2 = CompactModel.load(graph, images, logits, path)
    `graph` / `images` / `logits` are the full-width inference graph (build_eval_graph)."""

    def __init__(self, graph, images, logits, rec, state, device=None, conv_path=None):
        import torch
        from .engine import Executor
        self.full = (graph, images, logits)
        self.rec = rec
        self.graph, self.images, self.logits = build_graph(graph, images, logits, rec)
        self.state = slice_state(graph, logits, rec, state)
        self.device = device or torch.device('cuda', torch.cuda.current_device())
        self.ex = Executor(self.graph, self.images, self.logits, self.device, train=False, conv_path=conv_path)
        self.ex.store.load_state_dict(self.state, strict=True)

    @classmethod
    def from_masked(cls, graph, images, logits, state, device=None, conv_path=None):
        full = map_state(graph, reachable_ops(graph, logits), state)
        return cls(graph, images, logits, plan(graph, logits, full), full, device, conv_path)

    def forward(self, images=None):
        """Logits (device tensor, the executor's own buffer) of `images` (or of what the input buffer holds)."""
        if images is not None:
            self.ex.buf[self.images].copy_(images)
        return self.ex.forward(training=False)

    def conv_report(self):
        """[(conv op name, full input channels, kept input channels)] in graph order (the reference's
        'reducing %d channels to %d')."""
        g, _, lg = self.full
        return [(op.name, op.inputs[0].shape[-1], len(self.rec['convs'][op.name]))
                for op in reachable_ops(g, lg) if op.type == 'Conv2D']

    def export(self, path, fmt='npz'):
        """Write the compact checkpoint (`path`.npz, or a TensorFlow V2 bundle at `path` with fmt='tf') and its
        sidecar `path`.channels.json: every tensor's kept channel indices (-1: zero padding), the gathers and each
        conv's input set.  Returns the checkpoint's file name."""
        from .utils import tf_bundle
        os.makedirs(os.path.dirname(path) or '.', exist_ok=True)
        if fmt == 'tf':
            fn = tf_bundle.save(path, {k[:-2]: v for k, v in self.state.items()})
        elif fmt == 'npz':
            fn = path + '.npz'
            np.savez(fn, **{k.replace('/', '|'): v for k, v in self.state.items()})
        else:
            raise ValueError('unknown checkpoint format %r (npz | tf)' % fmt)
        shapes = {k: list(v.shape) for k, v in self.state.items()}
        with open(path + '.channels.json', 'w') as f:
            json.dump(dict(self.rec, format=fmt, shapes=shapes), f)
        return fn

    @classmethod
    def load(cls, graph, images, logits, path, device=None, conv_path=None):
        """Rebuild a compact model from what export(path) wrote."""
        from .utils import tf_bundle
        with open(path + '.channels.json') as f:
            rec = json.load(f)
        if rec.get('version') != SIDECAR_VERSION:
            raise ValueError('%s.channels.json: unsupported sidecar version %r' % (path, rec.get('version')))
        if rec['format'] == 'npz':
            d = np.load(path + '.npz')
            compact = {k.replace('|', '/'): d[k] for k in d.files}
        else:
            compact = {k + ':0': v for k, v in tf_bundle.load(path).items()}
        self = cls.__new__(cls)
        import torch
        from .engine import Executor
        self.full, self.rec = (graph, images, logits), rec
        self.graph, self.images, self.logits = build_graph(graph, images, logits, rec)
        names = {v.name for op in reachable_ops(self.graph, self.logits) for v in op.vars.values()}
        missing = sorted(names - set(compact))
        if missing:
            raise KeyError('missing variable in compact checkpoint: ' + missing[0])
        self.state = {k: np.asarray(compact[k], np.float32) for k in names}
        self.device = device or torch.device('cuda', torch.cuda.current_device())
        self.ex = Executor(self.graph, self.images, self.logits, self.device, train=False, conv_path=conv_path)
        self.ex.store.load_state_dict(self.state, strict=True)
        return self
