"""Pruned-width fine-tuning (--enbl_compact_ft) of MobileNet-v2, LeNet and with distillation, on the GPU.

* pf_dropout_fwd_mapped bit for bit: the compact Dropout's mask is the masked full-width model's mask gathered by the
  layout, on odd sizes and misaligned views, unsorted layouts with padding, two streams, an advancing step and a CUDA
  graph replay; with a NULL map it is pf_dropout_fwd on both of its paths.
* For each configuration of CONFIGS, one compact training step against float64 layer by layer (the CompactParity tap
  of tests/test_compact_train_gpu.py at its bars), the compact forward layer-local against the float64 oracle (with a
  GatherChannels handler), and the compact step against the masked step from the same state and batch: logits,
  cross-entropy, the distillation term, the dropout mask after k masked steps, padding through three steps, and the
  push / slice round trip.
* Under PF_POISON=1, a MobileNet-v2 compact step at batch 64: finite losses, graph replay equal to the eager step.
* chn-pruned-gpu on MobileNet-v2 and both learners on ResNet-8 with --enbl_dst, with and without the flag.
* A final test fails if a path the configurations are there for was never taken."""
import gc
import types

import numpy as np
import pytest
import torch

from oracle.mbv2_oracle import DropoutStepOracle
from pocketflow_b200 import compact as C
from pocketflow_b200 import lib, ops
from support import BAR_FWD, QUIET, free, local_parity, make, mapped_mask, ref_mask, snapshot, tapped_step

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
F32 = np.float32
KEEP = 0.8

SEEN = {}                     # path -> first configuration that took it


@pytest.fixture(autouse=True)
def _release():
    yield
    from pocketflow_b200.flags import FLAGS
    FLAGS.reset()
    free()


def seen(path, where):
    SEEN.setdefault(path, where)


# ------------------------------------------------------------------------------------------ the mapped dropout kernel
def _mapped(x, layout, cfull, state, y, mask, seed=11, rank=0, stream_id=0):
    lay = torch.tensor(layout, dtype=torch.int32, device=DEV)
    ops.dropout_fwd(x, KEEP, seed, rank, state, y, mask, stream_id=stream_id, layout=lay, full_width=cfull)


def _want_y(x, m):
    return (x.cpu().numpy() / F32(KEEP)) * m.reshape(x.shape)


@pytest.mark.parametrize('rows,cfull,layout,offset', [
    (64, 1280, 'half', 0),                           # MobileNet-v2 x1.0 at 0.5, batch 64
    (3, 7, [6, 0, -1, 3, 5], 1),                     # cfull % 4 != 0, unsorted, padding, misaligned views
    (5, 16, [15, -1, 2, 9, -1, -1, 0], 3),           # n % 4 != 0
    (2, 9, list(range(8, -1, -1)), 0),               # every channel, reversed
])
def test_mapped_dropout_is_the_full_width_draw_gathered(rows, cfull, layout, offset):
    if layout == 'half':
        layout = sorted(np.random.RandomState(0).permutation(cfull)[:cfull // 2].tolist())
    c = len(layout)
    lay = np.asarray(layout)
    g = torch.Generator().manual_seed(rows * cfull)
    xf = torch.randn(rows, cfull, generator=g).to(DEV)
    xbuf = torch.randn(rows * c + offset, generator=g).to(DEV)
    x = xbuf[offset:].view(rows, c)                  # a view `offset` floats into its buffer
    x.copy_(torch.where(torch.from_numpy(lay >= 0).to(DEV), xf[:, np.maximum(lay, 0)], 0.0))
    ybuf = torch.full((rows * c + offset,), float('nan'), device=DEV)
    y = ybuf[offset:].view(rows, c)
    mbuf = torch.full((rows * c + offset,), 0xee, dtype=torch.uint8, device=DEV)
    mask = mbuf[offset:]
    yf, mf = torch.empty_like(xf), torch.empty(rows * cfull, dtype=torch.uint8, device=DEV)
    for stream_id in (0, 3):
        sf = torch.tensor([5, 0], dtype=torch.int64, device=DEV)
        sc = sf.clone()
        for step in (5, 6, 7):                       # the counter advances once per launch
            ops.dropout_fwd(xf, KEEP, 11, 2, sf, yf, mf, stream_id=stream_id)
            _mapped(x, layout, cfull, sc, y, mask, 11, 2, stream_id)
            torch.cuda.synchronize()
            full = mf.view(rows, cfull).cpu().numpy().astype(F32)
            want = np.where(lay[None, :] >= 0, full[:, np.maximum(lay, 0)], 0.0).astype(F32)
            got = mask.cpu().numpy().astype(F32).reshape(rows, c)
            assert np.array_equal(got, want), (stream_id, step)
            assert np.array_equal(got, mapped_mask(rows, layout, cfull, KEEP, 11, 2, step, stream_id))
            assert np.array_equal(y.cpu().numpy().view(np.uint32), _want_y(x, got).view(np.uint32))
            assert sc.cpu().tolist() == sf.cpu().tolist() == [step + 1, 0]
        # nothing outside the view was written
        assert torch.isnan(ybuf[:offset]).all() and (mbuf[:offset] == 0xee).all()
    seen('mapped dropout', 'kernel')


def test_mapped_dropout_graph_replay_draws_the_eager_masks():
    rows, cfull = 16, 1280
    layout = [-1, -1] + sorted(np.random.RandomState(1).permutation(cfull)[:500].tolist())[::-1]
    x = torch.randn(rows, len(layout), device=DEV)
    y, mask = torch.empty_like(x), torch.empty(x.numel(), dtype=torch.uint8, device=DEV)
    state = torch.zeros(2, dtype=torch.int64, device=DEV)
    lay = torch.tensor(layout, dtype=torch.int32, device=DEV)
    eager = []
    for _ in range(3):
        ops.dropout_fwd(x, KEEP, 7, 1, state, y, mask, layout=lay, full_width=cfull)
        eager.append(mask.cpu().numpy().copy())
    assert not np.array_equal(eager[0], eager[1])
    state.zero_()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        ops.dropout_fwd(x, KEEP, 7, 1, state, y, mask, layout=lay, full_width=cfull)
    torch.cuda.synchronize()
    assert state.cpu().tolist() == [0, 0]
    for i in range(3):
        graph.replay()
        torch.cuda.synchronize()
        assert np.array_equal(mask.cpu().numpy(), eager[i]), i
        assert np.array_equal(eager[i].reshape(rows, -1).astype(F32), mapped_mask(rows, layout, cfull, KEEP, 7, 1, i))


@pytest.mark.parametrize('n,offset', [(64 * 1280, 0), (10_003, 1)])    # the vector path, the scalar path
def test_mapped_dropout_without_a_map_is_the_unmapped_kernel(n, offset):
    xbuf = torch.randn(n + offset, device=DEV)
    x = xbuf[offset:]
    outs = []
    for mapped in (False, True):
        ybuf = torch.full((n + offset,), float('nan'), device=DEV)
        mbuf = torch.zeros(n + offset, dtype=torch.uint8, device=DEV)
        y, mask = ybuf[offset:], mbuf[offset:]
        state = torch.tensor([9, 0], dtype=torch.int64, device=DEV)
        if mapped:
            lib.check(lib.load().pf_dropout_fwd_mapped(ops._p(x), n, KEEP, 3, 0, 1, None, 0, 0, ops._p(state),
                                                        ops._p(y), ops._p(mask), ops._stream()), 'pf_dropout_fwd_mapped')
        else:
            ops.dropout_fwd(x, KEEP, 3, 0, state, y, mask, stream_id=1)
        torch.cuda.synchronize()
        outs.append((y.cpu().numpy().view(np.uint32), mask.cpu().numpy(), state.cpu().tolist()))
    (y0, m0, s0), (y1, m1, s1) = outs
    assert np.array_equal(y0, y1) and np.array_equal(m0, m1) and s0 == s1 == [10, 0]
    assert np.array_equal(m0.astype(F32), ref_mask(n, KEEP, 3, 0, 9, 1))


# ------------------------------------------------------------------------------------------ compact training steps
V2 = 'mobilenet_at_ilsvrc12'
CIFAR = dict(nb_classes=10)
# (id, net module, net flags, batch, conv path, --enbl_dst)
CONFIGS = [
    ('v2_x1.0_tc', V2, dict(mobilenet_version=2), 4, 'tc', False),
    ('v2_x1.0_fp32', V2, dict(mobilenet_version=2), 4, 'fp32', False),
    ('v2_x0.35_tc', V2, dict(mobilenet_version=2, mobilenet_depth_mult=0.35), 4, 'tc', False),
    ('v2_x0.75_tc', V2, dict(mobilenet_version=2, mobilenet_depth_mult=0.75), 4, 'tc', False),
    ('lenet_tc', 'lenet_at_cifar10', CIFAR, 16, 'tc', False),
    ('lenet_fp32', 'lenet_at_cifar10', CIFAR, 16, 'fp32', False),
    ('resnet20_dst_tc', 'resnet_at_cifar10', dict(CIFAR, resnet_size=20), 16, 'tc', True),
    ('resnet20_dst_fp32', 'resnet_at_cifar10', dict(CIFAR, resnet_size=20), 16, 'fp32', True),
    ('resnet50_dst_b32_tc', 'resnet_at_ilsvrc12', dict(resnet_size=50), 32, 'tc', True),
]
BUILD = dict(QUIET, nb_classes=1001)   # what every learner below is built with besides its own flags
K_MASKED = 2                  # masked steps before the compact trainer is built


def prune_all(lrn, ratio, seed):
    """C.fake_prune on the learner's masked model: int(cin * ratio) random input channels of every conv kernel but the
    first, the logits conv included, zeroed; the masks set from them"""
    ex = lrn.sess_train
    lrn.init_from_full()
    rng = np.random.RandomState(seed)
    for v in lrn.maskable_vars[1:]:
        w = ex.store.view(v)
        if w.dim() != 4:
            continue
        cin = w.shape[2]
        w[:, :, torch.from_numpy(rng.permutation(cin)[:int(cin * ratio)]).to(DEV), :] = 0.0
    for v in lrn.maskable_vars:
        ops.cpg_channel_mask(ex.store.view(v), ex.store.view(v, ex.MASK))
    ex.reset_optimizer_state()


class CompactOracle(DropoutStepOracle):
    """the oracle's forward of a compact graph: DropoutStepOracle with each GatherChannels (y[..., j] = x[..., index[j]],
    0 where index[j] < 0) stated as a 1x1 convolution with a 0/1 selection kernel, which is exact"""

    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        self.select, ops_ = {}, []
        for op in self.ops:
            if op.type == 'GatherChannels':
                idx = np.asarray(op.attrs['index'])
                sel = np.zeros((1, 1, op.inputs[0].shape[-1], len(idx)), F32)
                sel[0, 0, idx[idx >= 0], np.nonzero(idx >= 0)[0]] = 1.0
                kname = op.name + '/select:0'
                self.select[kname] = sel
                op = types.SimpleNamespace(type='Conv2D', name=op.name, inputs=op.inputs, output=op.output,
                                           vars={'kernel': types.SimpleNamespace(name=kname)},
                                           attrs=dict(ksize=(1, 1), strides=(1, 1), pad=(0, 0)))
            ops_.append(op)
        self.ops = ops_

    def forward(self, params, images, *args, **kw):
        dt = next(iter(params.values())).dtype
        params = dict(params, **{k: torch.from_numpy(v).to(dt) for k, v in self.select.items()})
        return super().forward(params, images, *args, **kw)


def compact_forward_parity(name, cex, ct, state, img):
    """the compact training forward against float64, every op on the device's own inputs (local_parity)"""
    masks = {op.name: cex.dropout[op].view(op.output.shape).cpu().numpy() for op in cex.dropout}
    orc = CompactOracle(cex.ops, cex.logits_t, ct.images, cex.labels_t, cex.loss, masks=masks)
    worst, where, _, _, _ = local_parity(cex, orc, state, img, True)
    print('%s: compact forward worst %.2e (%s)' % (name, worst, where))
    assert worst <= BAR_FWD, (name, where, worst)
    return worst


def record_paths(name, ex, cex, par):
    full_tc = {op.name for op in ex.ops if op in ex.tc}
    for op in cex.ops:
        if op.type == 'Conv2D' and op in cex.tc and op.name not in full_tc:
            seen('conv on the tensor cores only at the compact width', name)
    cops = {op.name: op for op in cex.ops}
    if any(op in ex.tc_wgrad and cops[op.name] not in cex.tc_wgrad for op in ex.ops):
        seen('conv that left the tensor-core wgrad', name)
    for bn, (add, other) in cex.bn_add.items():
        if other.op.type == 'GatherChannels':
            seen('fused BN + Add with a gathered shortcut', name)
    for op in cex.scatter_inv:
        if op.inputs[0].op.type == 'Add':
            seen('gather reading a fused Add output', name)
    for op, acc, gpl, planes_only in par.scatters:
        seen('scatter: accumulating' if acc else 'scatter: whole buffer', name)
        if gpl:
            seen('scatter: emitting dy planes', name)
    if cex.drop_layout:
        seen('mapped dropout in a compact step', name)


@pytest.mark.parametrize('cfg', CONFIGS, ids=[c[0] for c in CONFIGS])
def test_compact_step_matches_float64_and_the_masked_step(cfg, monkeypatch):
    """One compact step after K_MASKED masked ones: backward and update layer by layer against float64 (2e-5 per
    gradient contribution and variable, 1e-6 chain, Momentum update bit for bit), the forward layer-local against
    float64 at the sweep's bar (4e-5, DESIGN §4), and against the masked step from the same state and batch: logits and
    cross-entropy (1e-5 exact fp32, 2e-4 split bf16, DESIGN §8), the distillation term, the dropout mask gathered;
    then padding exactly zero through three steps and the push / slice round trip."""
    name, mod, nflags, batch, path, dst = cfg
    monkeypatch.setenv('PF_CONV_PATH', path)
    torch.cuda.reset_peak_memory_stats()
    lrn = make(mod, 'chn-pruned-gpu', batch, **dict(BUILD, **nflags, enbl_dst=dst))
    ex = lrn.sess_train
    assert (ex.teacher is not None) == dst
    prune_all(lrn, 0.5, 3)
    g, lg = ex.g, ex.logits_t
    images, labels = lrn.iterator_train.next_batch()
    ex.buf[lrn.images].copy_(images)
    ex.buf[lrn.labels].copy_(labels)
    lr = 0.05
    for _ in range(K_MASKED):
        ex.run_step(lr)
    ct = C.CompactTrainer(ex)
    cex = ct.ex
    assert cex.step_count == ex.step_count == K_MASKED
    two = {k: np.full_like(v, 2.0) for k, v in ex.store.state_dict().items()}
    pad = {k: v != 2.0 for k, v in C.slice_state(g, lg, ct.rec, two).items()}
    state = cex.store.state_dict()
    dw = []
    orig = ops.dwconv_fwd

    def dw_rec(*a, **kw):
        orig(*a, **kw)
        dw.append((a[1].shape[-1], ops.dwconv_last_variant()))
    ex.run_step(lr)
    monkeypatch.setattr(ops, 'dwconv_fwd', dw_rec)
    par = tapped_step(cex, lr)
    monkeypatch.setattr(ops, 'dwconv_fwd', orig)
    record_paths(name, ex, cex, par)
    for c, variant in dw:
        if c % 16:
            seen('depthwise with C %% 16 != 0 (%s)' % variant, name)
            seen('depthwise with C % 16 != 0', name)
    # ---- the compact step against the masked one
    lf, lc = ex.T(lg).cpu().numpy(), cex.T(ct.logits).cpu().numpy()
    bar = 1e-5 if path == 'fp32' else 2e-4
    err = float(np.abs(lf - lc).max() / np.abs(lf).max())
    rf, rc = ex.fetch_losses(), cex.fetch_losses()
    print('%s: logits %.2e of max, ce %.3g / %.3g, dst %.4g / %.4g' % (name, err, rf['ce'], rc['ce'], rf['dst_loss'],
                                                                         rc['dst_loss']))
    assert err <= bar, (name, err)
    assert abs(rf['ce'] - rc['ce']) <= bar * abs(rf['ce'])
    if dst:
        assert rf['dst_loss'] > 0 and abs(rf['dst_loss'] - rc['dst_loss']) <= bar * abs(rf['dst_loss'])
        seen('distillation term in a compact step', name)
    for fop, i in ex.drop_stream.items():
        cop, = [o for o in cex.dropout if o.name == fop.name]
        lay = np.asarray(cop.attrs['layout'])
        rows = cop.output.numel // len(lay)
        full = ex.dropout[fop].view(rows, -1).cpu().numpy()
        got = cex.dropout[cop].view(rows, -1).cpu().numpy()
        assert np.array_equal(got, np.where(lay >= 0, full[:, np.maximum(lay, 0)], 0)), name
        assert np.array_equal(got.astype(F32), mapped_mask(rows, lay, cop.attrs['full_width'], KEEP, ex.drop_key[0],
                                                           ex.drop_key[1], K_MASKED, i))
        assert got.shape[1] < full.shape[1]
        assert ex.drop_state.tolist() == cex.drop_state.tolist() == [[K_MASKED + 1, 0]]
    # ---- the forward, layer-local, from the state the step read
    compact_forward_parity(name, cex, ct, state, images.cpu().numpy() if torch.is_tensor(images) else images)
    if cex.bn_gather:
        seen('fused BN + gather checked layer-local', name)
    del par
    # ---- padding stays exactly zero; the expanded state is the compact one
    for _ in range(2):
        cex.run_step(lr)
    assert all(np.isfinite(v) for v in cex.fetch_losses().values())
    npad = 0
    for v in cex.store.train_vars:
        p = pad[v.name]
        npad += int(p.sum())
        for flat in (cex.store.P, cex.S1, cex.G):
            assert not cex.store.view(v, flat).cpu().numpy()[p].any(), v.name
    assert npad > 0 or mod == 'lenet_at_cifar10'           # LeNet's widths are not multiples of 4: no padding
    ct.push()
    after = ex.store.state_dict()
    assert ex.step_count == cex.step_count == K_MASKED + 3
    if ex.drop_state is not None:
        assert ex.drop_state.tolist() == cex.drop_state.tolist() == [[K_MASKED + 3, 0]]
    again, now = C.slice_state(g, lg, ct.rec, after), cex.store.state_dict()
    for k in now:
        assert np.array_equal(again[k][~pad[k]], now[k][~pad[k]]), k
    print('%s: peak %.1f GB' % (name, torch.cuda.max_memory_allocated() / 2 ** 30))


def test_v2_compact_step_under_poison_is_finite_and_replays_bit_identically(monkeypatch):
    """every buffer filled with NaN at allocation (PF_POISON=1): a buffer some kernel forgets to write reaches the loss"""
    monkeypatch.setenv('PF_POISON', '1')
    lrn = make(V2, 'chn-pruned-gpu', 64, **BUILD, mobilenet_version=2)
    ex = lrn.sess_train
    prune_all(lrn, 0.5, 5)
    images, labels = lrn.iterator_train.next_batch()
    ex.buf[lrn.images].copy_(images)
    ex.buf[lrn.labels].copy_(labels)
    ct = C.CompactTrainer(ex)
    cex = ct.ex
    snap = snapshot(cex)
    drop = cex.drop_state.clone()
    cex.run_step(0.05)
    losses = cex.fetch_losses()
    assert all(np.isfinite(v) for v in losses.values()), losses
    eager = [cex.store.P.clone(), cex.S1.clone(), cex.T(cex.logits_t).clone(), next(iter(cex.dropout.values())).clone()]

    def restore():
        cex.store.P.copy_(snap['P'])
        cex.store.O.copy_(snap['O'])
        cex.S1.copy_(snap['S1'])
        cex.drop_state.copy_(drop)
    restore()
    cex.capture()                                       # (its warm-up runs one real step)
    restore()
    cex.run_step(0.05)
    torch.cuda.synchronize()
    for a, b in zip(eager, (cex.store.P, cex.S1, cex.T(cex.logits_t), next(iter(cex.dropout.values())))):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------ the learners end to end
def resnet8(learner, **flags):
    """ResNet-8 on CIFAR-10 at batch 16, as tests/test_compact_train_gpu.py builds it"""
    return make('resnet_at_cifar10', learner, 16, reload='cifar10_dataset', **dict(QUIET, resnet_size=8, **flags))


def _losses(lrn, nb_iters):
    out = []
    step = lrn.train_step

    def logged():
        step()
        out.append(lrn.sess_step.fetch_losses())
    lrn.train_step = logged
    lrn.train(nb_iters=nb_iters)
    return out


def _rel_diffs(masked, compact, key):
    return [abs(float(a[key]) - float(b[key])) / max(abs(float(a[key])), 1e-30) for a, b in zip(masked, compact)]


# The learners' 5-step loss trajectories with and without the flag, from the same selection on the same batches.  The
# first fine-tune step starts from the same state in both runs, so its cross-entropy agrees at the one-step bars (1e-5
# exact fp32, 2e-4 split bf16).  After that the two runs part by rounding alone, and on MobileNet-v2 at batch 4 rounding
# is amplified quickly: a 1e-6 relative perturbation of the masked run's parameters moves its cross-entropy by up to
# 6e-3 after one step and 3.4e-2 after five on an H100 (the rounding-perturbation test below, DESIGN §8).  Later steps
# are held to 0.1, above that control.
FIRST_STEP_BAR = {'fp32': 1e-5, 'tc': 2e-4}
LATER_STEPS_BAR = 0.1


@pytest.mark.parametrize('path', ['fp32', 'tc'])
def test_v2_compact_steps_track_the_masked_steps_as_closely_as_a_rounding_perturbation(monkeypatch, path):
    """MobileNet-v2 x1.0 at batch 4, five steps on five batches at the learner's rate from one pruned state: the masked
    steps, the masked steps from parameters perturbed by 1e-6 relative (a control: how far rounding alone carries two
    runs apart), and the compact steps.  The compact cross-entropy must stay as close to the masked one as the control
    does (within 10x, or 1e-5), and the first step must agree at the one-step bars."""
    monkeypatch.setenv('PF_CONV_PATH', path)
    lrn = make(V2, 'chn-pruned-gpu', 4, **BUILD, mobilenet_version=2)
    ex = lrn.sess_train
    prune_all(lrn, 0.5, 3)
    batches = [tuple(t.clone() if torch.is_tensor(t) else t for t in lrn.iterator_train.next_batch()) for _ in range(5)]
    s0, d0 = snapshot(ex), ex.drop_state.clone()

    def restore():
        ex.store.P.copy_(s0['P'])
        ex.store.O.copy_(s0['O'])
        ex.S1.copy_(s0['S1'])
        ex.drop_state.copy_(d0)
        ex.step_count = 0

    def run(exe):
        ce = []
        for images, labels in batches:
            ex.buf[lrn.images].copy_(images)                 # the compact executor shares these buffers
            ex.buf[lrn.labels].copy_(labels)
            exe.run_step(lrn.lrn_rate(exe.step_count))
            ce.append(float(exe.fetch_losses()['ce']))
        return np.array(ce)
    masked = run(ex)
    restore()
    g = torch.Generator(device=DEV).manual_seed(0)
    ex.store.P.mul_(1.0 + 1e-6 * torch.randn(ex.store.P.shape, generator=g, device=DEV))   # zeros stay zero
    control = run(ex)
    restore()
    compact = run(C.CompactTrainer(ex).ex)
    dc, dk = np.abs(compact - masked) / np.abs(masked), np.abs(control - masked) / np.abs(masked)
    print('v2 %s, 5 steps: ce masked %s; relative difference compact %s, perturbed control %s'
          % (path, masked.tolist(), ['%.2e' % x for x in dc], ['%.2e' % x for x in dk]))
    assert dc[0] <= (1e-5 if path == 'fp32' else 2e-4)
    assert dc.max() <= max(10 * dk.max(), 1e-5), (dc, dk)


@pytest.mark.parametrize('path', ['fp32', 'tc'])
def test_chn_pruned_gpu_on_v2_tracks_the_masked_losses(tmp_path, monkeypatch, path):
    """chn-pruned-gpu on MobileNet-v2 (batch 4), 5 fine-tune steps with and without --enbl_compact_ft: the first step's
    cross-entropy agrees at the one-step bar, the later ones within what rounding alone explains (FIRST_STEP_BAR,
    LATER_STEPS_BAR).  The learner's selection keeps every input channel of the logits conv, so the Dropout keeps its
    full width here: the narrowed, mapped draw is checked by the step tests above, which prune the logits conv."""
    monkeypatch.setenv('PF_CONV_PATH', path)
    runs = {}
    for ft in (False, True):
        lrn = make(V2, 'chn-pruned-gpu', 4, **BUILD, mobilenet_version=2, enbl_compact_ft=ft, cpg_nb_iters_layer=2,
                   cpg_save_path=str(tmp_path / ('c' if ft else 'm') / 'model.ckpt'))
        runs[ft] = _losses(lrn, 5)
        if ft:
            assert lrn.compact.ex.drop_layout and lrn.compact.ex.step_count == lrn.sess_train.step_count == 5
            assert lrn.compact.ex.drop_state.tolist() == lrn.sess_train.drop_state.tolist()
        del lrn
        gc.collect()
    d = _rel_diffs(runs[False], runs[True], 'ce')
    print('v2 chn-pruned-gpu, %s: ce per step %s, relative differences %s'
          % (path, [(float(a['ce']), float(b['ce'])) for a, b in zip(runs[False], runs[True])],
             ['%.2e' % x for x in d]))
    assert all(np.isfinite(r['loss']) for r in runs[True])
    assert d[0] <= FIRST_STEP_BAR[path] and max(d[1:]) <= LATER_STEPS_BAR, d


@pytest.mark.parametrize('learner', ['chn-pruned-gpu', 'chn-pruned-rmt'])
def test_learners_fine_tune_resnet8_with_distillation_at_the_pruned_width(tmp_path, learner):
    """ResNet-8 with --enbl_dst, 5 fine-tune steps with and without --enbl_compact_ft from the same selection on the
    same batches: the cross-entropy and the distillation term track per step at the 2e-3 of the ResNet-8 test of
    tests/test_compact_train_gpu.py; the compact executor shares the full-width teacher"""
    base = dict(enbl_dst=True, cpr_save_path_ws=str(tmp_path / 'ws' / 'model.ckpt'), cpg_nb_iters_layer=2,
                cpr_nb_smpls=40, cpr_nb_crops_per_smpl=3, cpr_ista_nb_iters=30, cpr_lstsq_nb_iters=10)
    if learner == 'chn-pruned-rmt':
        # one selection leaves the warm-start file both fine-tune runs start from
        sel = resnet8(learner, **base)
        sel.choose_channels()
        del sel
    runs = {}
    for ft in (False, True):
        sub = tmp_path / ('c' if ft else 'm')
        lrn = resnet8(learner, **dict(
            base, enbl_compact_ft=ft, cpr_warm_start=learner == 'chn-pruned-rmt',
            cpg_save_path=str(sub / 'cpg' / 'model.ckpt'), cpr_save_path=str(sub / 'cpr' / 'model.ckpt'),
            cpr_save_path_eval=str(sub / 'eval' / 'model.ckpt')))
        runs[ft] = _losses(lrn, 5)
        ex = lrn.sess_train
        assert ex.teacher is not None
        if ft:
            cex = lrn.compact.ex
            assert cex.teacher is ex.teacher and cex.loss.dst is not None and cex.step_count == ex.step_count == 5
        del lrn, ex
        gc.collect()
    dce, ddst = _rel_diffs(runs[False], runs[True], 'ce'), _rel_diffs(runs[False], runs[True], 'dst_loss')
    print('resnet8 %s + dst: relative differences ce %s, dst %s'
          % (learner, ['%.2e' % x for x in dce], ['%.2e' % x for x in ddst]))
    assert all(r['dst_loss'] > 0 and np.isfinite(r['loss']) for r in runs[True])
    assert max(dce) <= 2e-3 and max(ddst) <= 2e-3, (dce, ddst)
    seen('distillation term in a learner\'s compact step', learner)


# ------------------------------------------------------------------------------------------ coverage
REQUIRED = frozenset([
    'mapped dropout',
    'mapped dropout in a compact step',
    'fused BN + Add with a gathered shortcut',
    'gather reading a fused Add output',
    'scatter: accumulating',
    'scatter: whole buffer',
    'scatter: emitting dy planes',
    'depthwise with C % 16 != 0',
    'conv on the tensor cores only at the compact width',
    'conv that left the tensor-core wgrad',
    'distillation term in a compact step',
    'fused BN + gather checked layer-local',
])


def test_every_path_was_taken():
    """run with the tests above (the same session): each path the configurations exist for was taken by one of them"""
    if not SEEN:
        pytest.skip('run together with the tests above')
    for k, v in sorted(SEEN.items()):
        print('%-60s %s' % (k, v))
    assert not sorted(REQUIRED - set(SEEN))
