"""The LASSO channel-pruning learner (`--learner channel`) on the GPU: its sampling, design-matrix and normal-equation
kernels against float64 at ResNet-50 and MobileNet-v1 layer shapes, then whole selections of ResNet-20 and MobileNet-v1
against the float64 oracle (tests/cp_oracle.py) fed the same samples, masked fine-tuning and the export at the pruned
width."""
import importlib
import json
import os
import re
import sys

import numpy as np
import pytest
import torch

from pocketflow_b200 import ops
from pocketflow_b200.flags import FLAGS

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cp_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu
F32 = np.float32


def cuda(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(device='cuda', dtype=dtype)


# ------------------------------------------------------------------------------------------------------------ kernels
# (N, H, W, C, K, kh, stride, pads, P, Q): ResNet-50's 3x3 512 -> 512 at 7x7 and strided 3x3 at 14x14 (explicit pads),
# MobileNet-v1's 1x1 512 -> 512 at 14x14
SHAPES = [(3, 7, 7, 512, 512, 3, 1, (1, 1), 7, 7), (2, 14, 14, 256, 256, 3, 2, (0, 0), 6, 6),
          (3, 14, 14, 512, 512, 1, 1, (0, 0), 14, 14)]


@pytest.mark.parametrize('shape', SHAPES, ids=['rn50_3x3', 'rn50_3x3_s2', 'mbv1_1x1'])
@pytest.mark.parametrize('residual', [False, True])
@pytest.mark.parametrize('feed', ['fp32', 'planes'])
def test_sample_gram_and_normal_equations_against_float64(shape, residual, feed):
    """feed 'planes': the conv input is read as hi + lo of the split-bf16 operand planes the tensor-core path keeps"""
    n, h, w, c, k, kh, st, pads, p, q = shape
    rng = np.random.RandomState(7)
    x = rng.randn(n, h, w, c).astype(F32)
    planes, x_in = None, cuda(x)
    if feed == 'planes':
        pad = (x.size + 7) // 8 * 8
        planes = ops.Planes(pad, torch.device('cuda'))
        ops.split_bf16(cuda(np.concatenate([x.reshape(-1), np.zeros(pad - x.size, F32)])), planes)
        x_in = None
        x = (planes.hi.float() + planes.lo.float()).cpu().numpy()[:x.size].reshape(x.shape)
    y = rng.randn(n, p, q, k).astype(F32)
    bias = rng.randn(k).astype(F32)
    af, ac = rng.randn(n, p, q, k).astype(F32), rng.randn(n, p, q, k).astype(F32)
    nb_pts, nb_b = 5, 2
    d = ops.conv_desc(n, h, w, c, k, kh, kh, p, q, st, st, pads[0], pads[1])
    from pocketflow_b200.learners.channel_pruning.learner import sample_rows
    nrows = n * nb_pts * nb_b
    X = torch.full((nrows, kh * kh * c), float('nan'), dtype=torch.float32, device='cuda')
    Y = torch.full((nrows, k), float('nan'), dtype=torch.float64, device='cuda')
    Xr, Yr = [], []
    for b in range(nb_b):
        pos = (rng.randint(0, p, nb_pts), rng.randint(0, q, nb_pts))
        pos_add = (rng.randint(0, p, nb_pts), rng.randint(0, q, nb_pts))
        rows = sample_rows(pos, pos_add if residual else None, n, b * n * nb_pts)
        ops.cp_sample(d, x_in, cuda(y), cuda(rows, torch.int32), X, Y, planes=planes, bias=cuda(bias),
                      res_full=cuda(af) if residual else None, res_cur=cuda(ac) if residual else None)
        xr, yr = O.sample(x, (y - bias).astype(F32), pos, kh, kh, (st, st), pads,
                          af if residual else None, ac if residual else None, pos_add)
        Xr.append(xr)
        Yr.append(yr)
    Xr, Yr = np.vstack(Xr), np.vstack(Yr)
    # the sampled rows bit for bit: the patches are copies, Y is (y - b) + (full - cur) in float64 as the oracle forms it
    assert np.array_equal(X.cpu().numpy().astype(np.float64), Xr)
    assert np.array_equal(Y.cpu().numpy(), Yr)
    # design matrix Gram in float64
    W2 = (rng.randn(kh, kh, c, k) * 0.05).astype(F32)
    samples = rng.randint(0, nrows, max(nrows // 3, 1))
    g = torch.empty((c + 1) ** 2 + 1, dtype=torch.float64, device='cuda')
    ops.cp_gram(X, Y, cuda(samples, torch.int32), cuda(W2), g, chunk_rows=4)
    G = g[:(c + 1) ** 2].view(c + 1, c + 1).cpu().numpy()
    P, yv = O.design_matrix(Xr, W2, Yr, samples)
    Pa = np.concatenate([P, yv[:, None]], 1)
    ref = Pa.T.dot(Pa)
    assert np.abs(G - ref).max() <= 1e-12 * np.abs(ref).max(), np.abs(G - ref).max() / np.abs(ref).max()
    assert np.array_equal(G, G.T)
    # normal equations of the kept columns
    kept = np.sort(rng.choice(c, c // 3, replace=False))
    cols = (np.arange(kh * kh)[:, None] * c + kept[None, :]).reshape(-1)
    m = cols.size + k
    g2 = torch.empty(m * m + 1, dtype=torch.float64, device='cuda')
    ops.cp_normal_eq(X, Y, cuda(cols, torch.int32), g2, chunk_rows=7)
    A = g2[:m * m].view(m, m).cpu().numpy()
    Za = np.concatenate([Xr[:, cols], Yr], 1)
    ref2 = Za.T.dot(Za)
    assert np.abs(A - ref2).max() <= 1e-12 * np.abs(ref2).max()


# ------------------------------------------------------------------------------------------------------------ learner
def make(net, batch, **flags):
    FLAGS.reset()
    importlib.import_module('pocketflow_b200.learners.channel_pruning.learner')
    importlib.reload(importlib.import_module('pocketflow_b200.datasets.ilsvrc12_dataset'))
    mod = importlib.reload(importlib.import_module('pocketflow_b200.nets.' + net))
    from pocketflow_b200.learners.learner_utils import create_learner
    FLAGS.learner, FLAGS.batch_size = 'channel', batch
    base = dict(cp_prune_option='uniform', cp_nb_points_per_layer=10, summ_step=10 ** 9,
                save_step=10 ** 9)
    base.update(flags)
    for k, v in base.items():
        setattr(FLAGS, k, v)
    return create_learner(None, mod.ModelHelper())


# enough rows that every refit is overdetermined (N >= 2 x the kept columns)
NETS = {'resnet20': ('resnet_at_cifar10', 8, dict(resnet_size=20, cp_nb_batches=10)),
        'mobilenet_v1': ('mobilenet_at_ilsvrc12', 2, dict(nb_classes=1001, cp_nb_batches=30, cp_nb_points_per_layer=24))}


@pytest.mark.parametrize('net,conv_path', [('mobilenet_v1', 'fp32'), ('resnet20', 'fp32'), ('resnet20', 'default')])
def test_selection_matches_the_oracle_then_finetune_and_export(net, conv_path, tmp_path, monkeypatch, capsys):
    """every selected layer against the oracle fed the same X / Y and the same row draws: identical kept channel sets,
    refit W2 within 1e-6 of its magnitude, pruned channels exactly zero in W2, W1 and W1's bias; then 3 masked
    fine-tuning steps keep every zero, and the saved checkpoint, exported at the pruned width by
    tools/export_chn_pruned.py, gives the masked model's logits within 1e-4 of their magnitude.  conv_path 'default':
    the tensor-core convs, whose split-bf16 operand planes the sampler reads"""
    if conv_path == 'fp32':
        monkeypatch.setenv('PF_CONV_PATH', 'fp32')
    else:
        monkeypatch.delenv('PF_CONV_PATH', raising=False)
    module, bs, flags = NETS[net]
    paths = dict(save_path=str(tmp_path / 'ft' / 'model.ckpt'),
                 cp_channel_pruned_path=str(tmp_path / 'sel' / 'model.ckpt'))
    lrn = make(module, bs, **paths, **flags)
    from pocketflow_b200.learners.channel_pruning import learner as L
    store = lrn.sess_train.store
    seen = []
    sample_layer = lrn.sample_layer

    def capture(idx_layer, cached, ex_f, ex_p):
        X, Y = sample_layer(idx_layer, cached, ex_f, ex_p)
        seen.append((idx_layer, X.cpu().numpy().astype(np.float64), Y.cpu().numpy(), store.state_dict()))
        return X, Y
    lrn.sample_layer = capture
    lrn.choose_channels()
    assert len(seen) == lrn.nb_layers - 2 and len(lrn.selection_log) == len(seen)
    final = store.state_dict()
    for (i, X, Y, before), rec in zip(seen, lrn.selection_log):
        op = lrn.conv_ops_prnd[i]
        kname = op.vars['kernel'].name
        W2 = before[kname]
        idxs, w_ref, log = O.select_layer(X, Y, W2, rec['c_new'], rec['samples'])
        assert np.array_equal(idxs, rec['kept']), (i, log, rec['search'])
        assert [a for a in log] == rec['search']
        for later in lrn.selection_log:                            # later layers' prune_W1 of this conv
            if later['layer'] > i and later['father'] == op.name:
                w_ref[:, :, :, ~later['kept']] = 0
        bar = 1e-6 * np.abs(w_ref).max()
        assert np.abs(final[kname] - w_ref).max() <= bar, (i, np.abs(final[kname] - w_ref).max(), bar)
        assert np.all(final[kname][:, :, ~idxs, :] == 0)
        father = L.w1_target(op)
        if father is not None:
            fk = final[father.vars['kernel'].name]
            assert np.all(fk[:, :, :, ~idxs] == 0) if father.type == 'Conv2D' else np.all(fk[:, :, ~idxs, :] == 0)
            if 'bias' in father.vars:
                assert np.all(final[father.vars['bias'].name][~idxs] == 0)
    assert lrn.pr_maskable() > 0.2
    # masked fine-tuning keeps the zeros
    zeros = {v.name: final[v.name] == 0 for v in lrn.maskable_vars}
    lrn.choose_channels = lambda *a, **k: None                     # (selection already done and saved)
    lrn.train(nb_iters=3)
    ex = lrn.sess_train
    assert ex.step_count == 3 and np.isfinite(ex.fetch_losses()['loss'])
    now = ex.store.state_dict()
    for v in lrn.maskable_vars:
        assert np.all(now[v.name][zeros[v.name]] == 0), v.name
        assert not np.array_equal(now[v.name], final[v.name]), v.name
    # the saved masked checkpoint exports at the pruned width, and its logits are the masked model's
    out = str(tmp_path / 'compact' / 'model')
    js = str(tmp_path / 'export.json')
    argv = ['--net', module, '--ckpt_dir', str(tmp_path / 'ft'), '--out', out, '--batch_size_eval', str(bs),
            '--nb_repts_warmup', '1', '--nb_repts', '1', '--nb_rounds', '1', '--json', js]
    for k in ('resnet_size',):
        if k in flags:
            argv += ['--' + k, str(flags[k])]
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tools'))
    import export_chn_pruned
    capsys.readouterr()
    assert export_chn_pruned.main(argv) == 0
    printed = capsys.readouterr().out
    with open(js) as f:
        res = json.load(f)
    assert res['logits_max_rel_diff'] <= 1e-4, res['logits_max_rel_diff']
    assert res['params_compact'] < res['params_full']
    reduced = [tuple(int(v) for v in m) for m in re.findall(r'reducing (\d+) channels to (\d+)', printed)]
    assert reduced and any(kept < cin for cin, kept in reduced), printed
    assert os.path.exists(out + '.channels.json')
