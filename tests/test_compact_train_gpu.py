"""Fine-tuning channel-pruned models at their pruned width on the GPU: pf_scatter_channels and pf_bn_apply_gather against
torch / the unfused kernels, one training step of the compact model against the masked full-width step from the same
state and batch, padding channels through three steps, eager step against CUDA-graph replay, and both channel-pruning
learners end to end with and without --enbl_compact_ft."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from pocketflow_b200 import compact as C
from pocketflow_b200 import ops
from pocketflow_b200.flags import FLAGS
from support import QUIET, free, make, prune_interior, tapped_step

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)


@pytest.fixture(autouse=True)
def release_device_memory():
    """the ResNet-50 case holds two benchmarked steps at batch 128: hand the cached blocks back for the tests (and their
    child processes) that follow"""
    yield
    free()


def _idx(kept, cout):
    return torch.tensor(list(kept) + [-1] * (cout - len(kept)), dtype=torch.int32, device=DEV)


def _split(x):
    p = ops.Planes(x.numel(), DEV)
    ops.split_bf16(x.contiguous(), p)
    return p


def _same_planes(a, b):
    return torch.equal(a.hi.view(torch.int16), b.hi.view(torch.int16)) and \
        torch.equal(a.lo.view(torch.int16), b.lo.view(torch.int16))


# (rows, full width, kept channels in gather order, compact width)
SCATTER_CASES = [
    ((2, 4, 5), 24, [1, 2, 3, 5, 20, 23], 8),                       # odd runs, padding indices
    ((2, 4, 5), 64, list(range(16, 48)), 32),                       # 4-aligned runs: the 128-bit path
    ((2, 8), 260, list(range(0, 260, 3)), 96),                      # odd width, element by element
    ((2, 8), 64, list(range(64)), 64),                              # all kept
    ((2, 8), 64, [], 16),                                           # none kept
    ((2, 8), 32, [7, 6, 5, 4, 12, 13, 14, 15], 8),                  # a gather need not be sorted
    ((128, 28, 28), 512, sorted(np.random.RandomState(0).permutation(512)[:256].tolist()), 256),   # ResNet-50, batch 128
]


@pytest.mark.parametrize('accumulate', [False, True])
@pytest.mark.parametrize('rows,cin,kept,cout', SCATTER_CASES)
def test_scatter_channels_is_exact(rows, cin, kept, cout, accumulate):
    g = torch.Generator().manual_seed(cin + cout)
    dy = torch.randn(*rows, cout, generator=g).to(DEV)
    prev = torch.randn(*rows, cin, generator=g).to(DEV)
    idx = _idx(kept, cout)
    inv = torch.from_numpy(ops.scatter_table(idx.cpu().numpy(), cin)).to(DEV)
    ref = prev.clone() if accumulate else torch.zeros_like(prev)
    if kept:
        k = torch.tensor(kept, device=DEV)
        ref[..., k] += dy[..., :len(kept)]
    dx = prev.clone() if accumulate else torch.full_like(prev, float('nan'))
    pl = ops.Planes(dx.numel(), DEV)
    pl.buf.fill_(float('nan'))
    ops.scatter_channels(dy, inv, dx, accumulate, pl)
    torch.cuda.synchronize()
    assert torch.equal(dx, ref)
    assert _same_planes(pl, _split(ref))
    # fp32 alone; planes alone (no accumulate: nothing to add into)
    dx2 = prev.clone() if accumulate else torch.full_like(prev, float('nan'))
    ops.scatter_channels(dy, inv, dx2, accumulate)
    assert torch.equal(dx2, ref)
    if not accumulate:
        pl2 = ops.Planes(dx.numel(), DEV)
        ops.scatter_channels(dy, inv, None, False, pl2)
        assert _same_planes(pl2, pl)
    else:
        with pytest.raises(ValueError, match='accumulate needs the fp32 dx'):
            ops.scatter_channels(dy, inv, None, True, pl)


@pytest.mark.parametrize('act', [0, 1, 2])
@pytest.mark.parametrize('c,kept,cout', [(24, [1, 2, 3, 5, 20, 23], 8), (64, list(range(16, 48)), 32),
                                         (260, list(range(0, 260, 3)), 96), (64, [0, 1, 2, 3, 8, 9, 10, 11, 60], 16)])
def test_bn_apply_gather_equals_bn_apply_then_gather(c, kept, cout, act):
    g = torch.Generator().manual_seed(act * 7 + c)
    x = (3 * torch.randn(4, 6, 6, c, generator=g)).to(DEV)
    ga, be = torch.randn(c, generator=g).to(DEV), torch.randn(c, generator=g).to(DEV)
    m = x.numel() // c
    mean, var, rstd = (torch.empty(c, device=DEV) for _ in range(3))
    mm, mv = torch.zeros(c, device=DEV), torch.ones(c, device=DEV)
    ws = torch.empty(5 * c * ops.BN_MAX_SPLITS, device=DEV)
    ops.bn_train_stats(x, m, c, 1e-3, 0.9, mean, var, rstd, mm, mv, ws)
    full, fullp = torch.empty_like(x), ops.Planes(x.numel(), DEV)
    ops.bn_apply(x, m, c, mean, rstd, ga, be, act, full)
    ops.bn_apply(x, m, c, mean, rstd, ga, be, act, full, None, fullp)
    idx = _idx(kept, cout)
    ref, refp = torch.empty(4, 6, 6, cout, device=DEV), ops.Planes(m * cout, DEV)
    ops.gather_channels(full, idx, ref, refp)
    y = torch.full(ref.shape, float('nan'), device=DEV)
    yp = ops.Planes(ref.numel(), DEV)
    ops.bn_apply_gather(x, m, c, mean, rstd, ga, be, act, idx, y, yp)
    torch.cuda.synchronize()
    assert torch.equal(y, ref) and _same_planes(yp, refp)
    assert torch.equal(y[..., len(kept):], torch.zeros_like(y[..., len(kept):]))


# ------------------------------------------------------------------ one training step, compact against masked
# net -> (net module, dataset module reloaded with it, batch, net flags)
NETS = {'mobilenet': ('mobilenet_at_ilsvrc12', 'ilsvrc12_dataset', 4, dict(nb_classes=1001)),
        'resnet50': ('resnet_at_ilsvrc12', 'ilsvrc12_dataset', 128, dict(resnet_size=50, nb_classes=1001)),
        'resnet20': ('resnet_at_cifar10', 'cifar10_dataset', 16, dict(resnet_size=20)),
        'resnet8': ('resnet_at_cifar10', 'cifar10_dataset', 16, dict(resnet_size=8))}


def make_learner(net, learner, **flags):
    mod, data, batch, nflags = NETS[net]
    return make(mod, learner, batch, reload=data, **dict(dict(QUIET, **nflags), **flags))


@pytest.mark.parametrize('net,learner,conv_path', [
    ('resnet20', 'chn-pruned-gpu', 'fp32'), ('resnet20', 'chn-pruned-gpu', 'tc'), ('mobilenet', 'chn-pruned-rmt', 'fp32'),
    ('mobilenet', 'chn-pruned-rmt', 'tc'), ('resnet50', 'chn-pruned-gpu', 'tc')])
def test_compact_step_equals_the_masked_step(monkeypatch, net, learner, conv_path):
    """From the same state and batch (ResNet-20 at batch 16, MobileNet-v1 at batch 4, ResNet-50 at the benchmarked batch
    128): the compact logits and cross-entropy against the masked full-width ones, and the compact step's backward and
    update layer by layer against float64 (CompactParity) at the bars of tests/test_backward_parity_gpu.py: 2e-5 for
    every gradient contribution and every variable's gradient, 1e-6 for the chain, the Momentum update with the sliced
    masks bit for bit.  The compact gradients are not compared with the masked ones end to end: both differ from
    float64 by ReLU gates that flip under rounding, which a layer-by-layer reference does not see.  The exact-fp32
    logits differ by the order of the narrowed K sums only (1e-5 of max|logit|); split-bf16 operands carry 16 mantissa
    bits per convolution, in both models, through up to 53 layers of training-mode BN (2e-4)."""
    monkeypatch.setenv('PF_CONV_PATH', conv_path)
    lrn = make_learner(net, learner)
    ex = lrn.sess_train
    prune_interior(lrn, 0.5, 3)
    g, lg = ex.g, ex.logits_t
    images, labels = lrn.iterator_train.next_batch()
    ex.buf[lrn.images].copy_(images)
    ex.buf[lrn.labels].copy_(labels)
    ct = C.CompactTrainer(ex)
    cex = ct.ex
    assert cex.G.numel() < ex.G.numel() and cex.buf[ct.images] is ex.buf[lrn.images]
    assert (net == 'mobilenet') == (not cex.scatter_inv)              # MobileNet-v1 needs no gather
    lr = 0.05
    two = {k: np.full_like(v, 2.0) for k, v in ex.store.state_dict().items()}
    pad = {k: v != 2.0 for k, v in C.slice_state(g, lg, ct.rec, two).items()}          # padding entries of each variable
    ex.run_step(lr)
    par = tapped_step(cex, lr)
    lf, lc = ex.T(lg).cpu().numpy(), cex.T(ct.logits).cpu().numpy()
    bar = 1e-5 if conv_path == 'fp32' else 2e-4
    assert np.abs(lf - lc).max() <= bar * np.abs(lf).max()
    rf, rc = ex.fetch_losses(), cex.fetch_losses()
    assert abs(rf['ce'] - rc['ce']) <= bar * abs(rf['ce'])
    if net != 'mobilenet':
        # the paths the gathers add were taken: BN apply + gather fused, scatters that write a whole buffer and
        # scatters that accumulate into a shared residual gradient
        assert cex.bn_gather and len(par.scatters) == len(cex.scatter_inv)
        assert {a for _, a, _, _ in par.scatters} == {False, True}, par.scatters
        assert all(bn.attrs['training'] for bn in cex.bn_gather)
    if net == 'resnet50':
        # two gathers read one pre-activation; a scatter hands the convolution in front of it its dy planes
        assert any(len([c for c in cex._consumers(op.inputs[0]) if c.type == 'GatherChannels']) >= 2 for op in cex.scatter_inv)
        assert any(pl for _, _, pl, _ in par.scatters), 'no scatter emitted dy planes'
        assert any(op in cex.tc_wgrad for op in cex.ops)
    del par
    # ---- two more steps: padding stays exactly zero, masked rows too; the expanded state is the compact one
    for _ in range(2):
        cex.run_step(lr)
    npad = 0
    for v in cex.store.train_vars:
        p = pad[v.name]
        npad += int(p.sum())
        for flat in (cex.store.P, cex.S1, cex.G):
            assert not cex.store.view(v, flat).cpu().numpy()[p].any(), v.name
    del lf, lc
    assert npad > 0 or net == 'mobilenet'
    before = ex.store.state_dict()
    ct.push()
    after = ex.store.state_dict()
    assert ex.step_count == cex.step_count == 3
    again = C.slice_state(g, lg, ct.rec, after)
    now = cex.store.state_dict()
    for name in now:
        keep = ~pad[name]
        assert np.array_equal(again[name][keep], now[name][keep]), name
    for v in lrn.maskable_vars:
        m = ex.store.view(v, ex.MASK).cpu().numpy()
        assert not after[v.name][m == 0].any()
    changed = sum(int((after[k] != before[k]).sum()) for k in after)
    assert 0 < changed <= sum(a.size for a in now.values())


def test_eager_step_and_graph_replay_are_identical():
    lrn = make_learner('resnet20', 'chn-pruned-gpu')
    ex = lrn.sess_train
    prune_interior(lrn, 0.5, 4)
    images, labels = lrn.iterator_train.next_batch()
    ex.buf[lrn.images].copy_(images)
    ex.buf[lrn.labels].copy_(labels)
    cex = C.CompactTrainer(ex).ex
    snap = [t.clone() for t in (cex.store.P, cex.store.O, cex.S1)]

    def restore():
        for t, s in zip((cex.store.P, cex.store.O, cex.S1), snap):
            t.copy_(s)
    cex.run_step(0.05)
    eager = [cex.store.P.clone(), cex.store.O.clone(), cex.S1.clone(), cex.T(cex.logits_t).clone()]
    restore()
    cex.capture()                                       # (its warm-up runs one real step)
    restore()
    cex.run_step(0.05)
    torch.cuda.synchronize()
    for a, b in zip(eager, (cex.store.P, cex.store.O, cex.S1, cex.T(cex.logits_t))):
        assert torch.equal(a, b)


# ------------------------------------------------------------------ the learners end to end
def _dead_l2(lrn, state):
    """the L2 term of the entries the compact model does not hold (frozen dead producer channels)"""
    ex = lrn.sess_train
    rec = lrn.compact.rec
    kept = C.expand_state(ex.g, ex.logits_t, rec, C.slice_state(ex.g, ex.logits_t, rec, {k: np.ones_like(v) for k, v in state.items()}),
                          {k: np.zeros_like(v) for k, v in state.items()})
    return sum(c * 0.5 * float((np.asarray(state[v.name], np.float64)[kept[v.name] == 0] ** 2).sum())
               for v, c in ex.loss.l2.items())


@pytest.mark.parametrize('learner', ['chn-pruned-gpu', 'chn-pruned-rmt'])
def test_learner_fine_tunes_at_the_pruned_width_and_writes_the_masked_checkpoint(tmp_path, capsys, learner):
    def run(compact_ft, warm=False):
        sub = tmp_path / ('c' if compact_ft else 'm')
        flags = dict(enbl_compact_ft=compact_ft, cpg_save_path=str(sub / 'cpg' / 'model.ckpt'),
                     cpr_save_path=str(sub / 'cpr' / 'model.ckpt'), cpr_save_path_eval=str(sub / 'eval' / 'model.ckpt'),
                     cpr_save_path_ws=str(tmp_path / 'ws' / 'model.ckpt'), cpr_warm_start=warm, cpg_nb_iters_layer=2,
                     cpr_nb_smpls=40, cpr_nb_crops_per_smpl=3, cpr_ista_nb_iters=30, cpr_lstsq_nb_iters=10)
        lrn = make_learner('resnet8', learner, **flags)
        losses = []
        step = lrn.train_step

        def logged():
            step()
            losses.append(lrn.sess_step.fetch_losses())
        lrn.train_step = logged
        lrn.train(nb_iters=5)
        return lrn, losses, str(sub / ('cpg' if learner == 'chn-pruned-gpu' else 'cpr'))
    # chn-pruned-rmt: one selection leaves the warm-start file both fine-tune runs start from, on the same batches
    if learner == 'chn-pruned-rmt':
        sel = make_learner('resnet8', learner, cpr_save_path_ws=str(tmp_path / 'ws' / 'model.ckpt'), cpr_nb_smpls=40,
                           cpr_nb_crops_per_smpl=3, cpr_ista_nb_iters=30, cpr_lstsq_nb_iters=10)
        sel.choose_channels()
        del sel
    lrn_m, loss_m, _ = run(False, warm=learner == 'chn-pruned-rmt')
    assert lrn_m.compact is None
    start = lrn_m.sess_train.store.state_dict()                                   # (5 steps of decay: < 1e-3)
    del lrn_m
    capsys.readouterr()
    lrn_c, loss_c, ckpt_dir = run(True, warm=learner == 'chn-pruned-rmt')
    out = capsys.readouterr().out
    assert out.count('reducing ') == lrn_c.nb_layers and 'parameters: ' in out
    ex, cex = lrn_c.sess_train, lrn_c.compact.ex
    assert cex.step_count == ex.step_count == 5 and cex.G.numel() < ex.G.numel()
    # same selected model (chn-pruned-gpu: the same selection from the same seed on the same batches), same fine-tune
    # batches: the losses track once the frozen channels' L2 term is added back
    dead = _dead_l2(lrn_c, start)
    for a, b in zip(loss_m, loss_c):
        assert abs(a['ce'] - b['ce']) <= 2e-3 * abs(a['ce']), (a, b)
        assert abs(a['l2'] - (b['l2'] + dead)) <= 2e-3 * abs(a['l2']), (a, b, dead)
    assert all(np.isfinite(r['loss']) for r in loss_c)
    # the checkpoint is the masked full-width one: a fresh full-width learner evaluates it to the compact model's loss
    from pocketflow_b200.datasets.abstract_dataset import POOL_SIZE
    from pocketflow_b200.learners.abstract_learner import latest_checkpoint, load_checkpoint
    saved = load_checkpoint(latest_checkpoint(ckpt_dir))
    now = ex.store.state_dict()
    assert all(np.array_equal(saved[k], now[k]) for k in now)
    for v in lrn_c.maskable_vars:
        assert not now[v.name][ex.store.view(v, ex.MASK).cpu().numpy() == 0].any()
    trained = lrn_c.evaluate(nb_iters=POOL_SIZE)[0]
    comp = []
    for _ in range(POOL_SIZE):
        lrn_c.feed(ex, lrn_c.eval_iterator())
        cex.forward_eval_loss()
        comp.append(cex.fetch_losses()['ce'] + ex.fetch_losses()['l2'])
    flags = {k: v for k, v in FLAGS._values.items() if k != 'learner'}
    del lrn_c
    fresh = make_learner('resnet8', learner, **dict(flags, exec_mode='eval', enbl_compact_ft=False))
    got = fresh.evaluate(nb_iters=POOL_SIZE)[0]
    assert abs(got - trained) <= 1e-6 * abs(trained)
    assert abs(float(np.mean(comp)) - trained) <= 1e-4 * abs(trained)
    del fresh
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'export_chn_pruned.py'), '--net', 'resnet_at_cifar10',
                        '--resnet_size', '8', '--ckpt_dir', ckpt_dir, '--out', str(tmp_path / 'exp' / 'model'),
                        '--no_time'], capture_output=True, text=True)
    assert r.returncode == 0 and 'reducing ' in r.stdout, r.stdout + r.stderr
