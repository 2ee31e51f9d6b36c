"""The remastered channel-pruning learner (chn-pruned-rmt) on the GPU: each selection kernel (pf_cpr.cu) against the
numpy oracle (oracle/cpr_oracle.py) on the same inputs, then the learner on ResNet-8 and MobileNet-v1."""
import os

import numpy as np
import pytest
import torch

from oracle import cpr_oracle as C
from pocketflow_b200 import ops
from pocketflow_b200.flags import FLAGS
from pocketflow_b200.learners.channel_pruning_rmt import learner as L
from support import check_selection

pytestmark = pytest.mark.gpu
F32 = np.float32
DEV = torch.device('cuda', 0)


class FixedRng(object):
    """randint stand-in that hands out a given sequence (every output position, in order)"""

    def __init__(self, seq):
        self.seq = list(seq)

    def randint(self, n):
        v = self.seq.pop(0)
        assert 0 <= v < n
        return v


def cuda(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dtype)


# ---------------------------------------------------------------------------------------------------------- sampler
SAMPLER_CASES = [
    # (n, h, w, c, k, r, s, stride, padding)
    (3, 7, 7, 5, 6, 3, 3, 1, 'SAME'),         # odd size, stride 1
    (2, 8, 8, 4, 3, 3, 3, 2, 'SAME'),         # even size, stride 2 (pad 0 at the top, 1 at the bottom)
    (2, 9, 7, 3, 4, 3, 3, 2, 'SAME'),         # odd size, stride 2
    (2, 6, 7, 4, 5, 3, 3, 1, 'VALID'),
    (3, 5, 6, 8, 7, 1, 1, 1, 'SAME'),         # 1x1
    (2, 9, 9, 3, 4, 7, 7, 2, 'SAME'),         # 7x7 stem-like
]


@pytest.mark.parametrize('case', SAMPLER_CASES)
@pytest.mark.parametrize('feed', ['fp32', 'planes'])
def test_sampler_bit_exact(case, feed):
    n, h, w, c, k, r, s, st, padding = case
    rng = np.random.RandomState(1)
    p = (h - 1) // st + 1 if padding == 'SAME' else (h - r) // st + 1
    q = (w - 1) // st + 1 if padding == 'SAME' else (w - s) // st + 1
    pt, pl = C.cpr_pads(h, w, r, s, st, st, padding)
    x = rng.randn(n, h, w, c).astype(F32)
    y = rng.randn(n, p, q, k).astype(F32)
    bias = rng.randn(k).astype(F32)
    d = ops.conv_desc(n, h, w, c, k, r, s, p, q, st, st, pt, pl)
    if feed == 'planes':
        pad = (x.size + 7) // 8 * 8
        pl_ = ops.Planes(pad, DEV)
        ops.split_bf16(cuda(np.concatenate([x.reshape(-1), np.zeros(pad - x.size, F32)])), pl_)
        x_in = None
        x_ref = (pl_.hi.float() + pl_.lo.float()).cpu().numpy()[:x.size].reshape(x.shape)
    else:
        pl_, x_in, x_ref = None, cuda(x), x
    pos = [(a, b) for a in range(p) for b in range(q)]              # every output position: every ragged edge
    seq = [v for ab in pos for v in ab]
    kern = np.zeros((r, s, c, k), F32)
    X_ref, Y_ref, got_pos, _ = C.cpr_sample(FixedRng(seq), kern, kern, x_ref, x_ref, y, y, (st, st), padding,
                                            len(pos))
    assert got_pos == pos
    nrow = len(pos) * n
    dst = rng.permutation(nrow + 5)[:nrow] - 5                        # a few rows dropped (< 0), the rest scattered
    kept = dst >= 0
    X = torch.full((nrow, r * s * c), float('nan'), device=DEV)
    Y = torch.full((nrow, k), float('nan'), device=DEV)
    rows = cuda(L.sample_rows(pos, n, dst), torch.int32)
    ops.cpr_sample(d, x_in, cuda(y), rows, X, Y, planes=pl_)
    Xg, Yg = X.cpu().numpy(), Y.cpu().numpy()
    assert np.array_equal(Xg[dst[kept]], X_ref[kept].astype(F32))
    assert np.array_equal(Yg[dst[kept]], Y_ref[kept].astype(F32))
    assert np.isnan(Xg[np.setdiff1d(np.arange(nrow), dst[kept])]).all()   # dropped rows: nothing written
    # a fused bias is subtracted from the gathered outputs
    ops.cpr_sample(d, x_in, cuda(y), rows, X, Y, planes=pl_, bias=cuda(bias))
    assert np.array_equal(Y.cpu().numpy()[dst[kept]], (Y_ref[kept].astype(F32) - bias).astype(F32))


# ---------------------------------------------------------------------------------------------------------- Gram
@pytest.mark.parametrize('rs,cin,cout,n,chunk', [(9, 24, 16, 300, 37), (1, 70, 130, 200, 64), (1, 3, 5, 50, None),
                                                 (4, 129, 8, 120, 50)])
def test_gram_float64(rs, cin, cout, n, chunk):
    rng = np.random.RandomState(2)
    X = rng.randn(n, rs * cin).astype(F32)
    Y = rng.randn(n, cout).astype(F32)
    w = (rng.randn(1, rs, cin, cout) * 0.3).astype(F32)
    idxs = rng.choice(n, size=C.cpr_secondary_rows(n, cout), replace=False)
    g_ref, b_ref, nrm = C.cpr_gram(X, Y, w, idxs)
    g = torch.full(((cin + 1) ** 2 + 1,), float('nan'), dtype=torch.float64, device=DEV)
    gf = torch.empty(cin * cin, device=DEV)
    bf = torch.empty(cin, device=DEV)
    ops.cpr_gram(cuda(X), cuda(Y), cuda(idxs, torch.int32), cuda(w), g, gf, bf, chunk_rows=chunk)
    gg = g.cpu().numpy()
    G = gg[:(cin + 1) ** 2].reshape(cin + 1, cin + 1)
    assert np.abs(G[:cin, :cin] - g_ref).max() <= 1e-12 * np.abs(g_ref).max()
    assert np.abs(G[:cin, cin] - b_ref[:, 0]).max() <= 1e-12 * np.abs(b_ref).max()
    assert abs(gg[-1] - nrm) <= 1e-12 * nrm
    assert np.array_equal(G[:cin, :cin], G[:cin, :cin].T)                     # exactly symmetric
    assert np.array_equal(gf.cpu().numpy().reshape(cin, cin), G[:cin, :cin].astype(F32))
    assert np.array_equal(bf.cpu().numpy(), G[:cin, cin].astype(F32))
    # deterministic: a second run gives the same bits
    g2 = torch.empty_like(g)
    ops.cpr_gram(cuda(X), cuda(Y), cuda(idxs, torch.int32), cuda(w), g2, gf, bf, chunk_rows=chunk)
    assert torch.equal(g, g2)


# ---------------------------------------------------------------------------------------------------------- ISTA
def lasso_problem(rng, n, cin, cout, keep=None, rs=1):
    """a regression problem; keep: the channels that carry the response (planted sparsity)"""
    X = rng.randn(n, rs * cin).astype(F32)
    w = (rng.randn(1, rs, cin, cout) * 0.3).astype(F32)
    if keep is None:
        Y = rng.randn(n, cout).astype(F32)
    else:
        Xk = X.reshape(n, rs, cin).copy()
        Xk[:, :, [c for c in range(cin) if c not in keep]] = 0
        Y = (Xk.reshape(n, -1) @ w.reshape(-1, cout)).astype(F32)
    idxs = np.arange(n)
    g, b, _ = C.cpr_gram(X, Y, w, idxs)
    return X, Y, w, g, b


@pytest.mark.parametrize('cin,gamma', [(40, 0.05), (300, 0.02), (7, 0.3)])
def test_ista_one_solve(cin, gamma):
    rng = np.random.RandomState(3)
    _, _, _, g, b = lasso_problem(rng, 400, cin, 8)
    m0 = rng.uniform(size=(cin, 1))
    m_ref, nnz_ref = C.cpr_ista(g, b, m0, gamma, 1e-2, 100)
    gf, bf, m0d = cuda(g.astype(F32)), cuda(b.astype(F32).reshape(-1)), cuda(m0.astype(F32).reshape(-1))
    m = torch.full((cin,), float('nan'), device=DEV)
    ws, nnz = torch.empty(2 * cin, device=DEV), torch.full((1,), -7, dtype=torch.int32, device=DEV)
    ops.cpr_ista(gf, bf, m0d, 1e-2, gamma, 100, m, ws, nnz)
    got = m.cpu().numpy()
    assert np.abs(got - m_ref[:, 0]).max() <= 1e-5 * max(np.abs(m_ref).max(), 1e-30)
    assert int(nnz.item()) == nnz_ref == int(np.count_nonzero(got))
    assert 0 < nnz_ref < cin or cin == 7
    m2 = torch.empty_like(m)
    ops.cpr_ista(gf, bf, m0d, 1e-2, gamma, 100, m2, ws, nnz)
    assert torch.equal(m, m2)                                              # fixed reduction order
    ops.cpr_ista(gf, bf, m0d, 1e-2, gamma, 0, m2, ws, nnz)                # zero iterations: m0 itself
    assert torch.equal(m2, m0d) and int(nnz.item()) == cin


def test_gamma_search_planted_sparse():
    """channels 0..cin-1 of which `keep` carry the response: the device search keeps the same channels with the same
    number of solves as the oracle's search"""
    rng = np.random.RandomState(4)
    cin, keep = 32, [1, 4, 5, 9, 12, 17, 20, 22, 27, 30, 31, 8, 3, 14, 25, 19]
    _, _, _, g, b = lasso_problem(rng, 600, cin, 8, keep=keep)
    m0 = rng.uniform(size=(cin, 1))
    target = len(keep)
    mask_ref, log_ref = C.cpr_gamma_search(lambda x: C.cpr_ista(g, b, m0, x, 1e-2, 100), target)
    gf, bf, m0d = cuda(g.astype(F32)), cuda(b.astype(F32).reshape(-1)), cuda(m0.astype(F32).reshape(-1))
    m, ws, nnz = torch.empty(cin, device=DEV), torch.empty(2 * cin, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV)

    def solve(x):
        ops.cpr_ista(gf, bf, m0d, 1e-2, x, 100, m, ws, nnz)
        return int(nnz.item())
    log = L.gamma_search(solve, target)
    assert len(log) == len(log_ref) and log[-1][1] == log_ref[-1][1] == target, (log, log_ref)
    assert [a[1] for a in log] == [a[1] for a in log_ref]
    assert sorted(np.flatnonzero(m.cpu().numpy())) == sorted(np.flatnonzero(mask_ref[:, 0]))


# ---------------------------------------------------------------------------------------------------------- refit
@pytest.mark.parametrize('conv_path,shape', [('fp32', (3, 3, 16, 64)), ('tc', (3, 3, 16, 64)), ('fp32', (1, 1, 6, 10)),
                                             ('tc', (1, 1, 64, 128)), ('tc', (1, 1, 64, 48))])
def test_lstsq_refit(conv_path, shape):
    kh, kw, cin, cout = shape
    rng = np.random.RandomState(5)
    n, iters, lr, wd = 512, 20, 1e-3, 4e-5
    X = rng.randn(n, kh * kw * cin).astype(F32)
    w = (rng.randn(*shape) * 0.2).astype(F32)
    Y = (X @ (w + 0.05 * rng.randn(*shape).astype(F32)).reshape(-1, cout)).astype(F32)
    mask = rng.uniform(-1, 1, size=cin).astype(F32)
    mask[rng.choice(cin, cin // 2, replace=False)] = 0
    w_ref = C.cpr_lstsq(X, Y, w, (np.abs(mask) > 0).astype(F32), lr, iters, wd)
    Xd, wd_ = cuda(X), cuda(w)
    md = cuda(mask)
    ops.cpr_mask_channels(Xd, md, kh * kw, cin, 1)
    x_m = (X.reshape(n, kh * kw, cin) * (np.abs(mask) > 0)).reshape(n, -1).astype(F32)
    assert np.array_equal(Xd.cpu().numpy(), x_m)
    lst = ops.CprLstsq(Xd, cuda(Y), conv_path)
    assert lst.tc_fwd == (conv_path == 'tc')
    assert lst.tc_wgrad == (conv_path == 'tc' and cout % 64 == 0)     # (the tensor-core wgrad wants Cout % 64 == 0)
    l0, l1 = lst.run(wd_, iters, lr, wd)
    ops.cpr_mask_channels(wd_, md, kh * kw, cin, cout)
    got = wd_.cpu().numpy()
    assert np.all(got[:, :, np.abs(mask) == 0, :] == 0)
    # every Adam step moves a weight by about lr: the bar is a fraction of the total path lr * iters
    bar = (2e-3 if conv_path == 'fp32' else 2e-2) * lr * iters
    assert np.abs(got - w_ref).max() <= bar, np.abs(got - w_ref).max()
    assert l1 < l0


# ---------------------------------------------------------------------------------------------------------- learner
def make_resnet(**flags):
    FLAGS.reset()
    from pocketflow_b200.nets import resnet_at_cifar10 as R
    from pocketflow_b200.learners.learner_utils import create_learner
    FLAGS.resnet_size, FLAGS.batch_size, FLAGS.learner = 8, 16, 'chn-pruned-rmt'
    base = dict(cpr_nb_smpls=40, cpr_nb_crops_per_smpl=3, cpr_ista_nb_iters=30, cpr_lstsq_nb_iters=10,
                summ_step=10 ** 9, save_step=10 ** 9)
    base.update(flags)
    for k, v in base.items():
        setattr(FLAGS, k, v)
    return create_learner(None, R.ModelHelper())


def make_mobilenet(**flags):
    FLAGS.reset()
    import importlib
    import pocketflow_b200.datasets.ilsvrc12_dataset as D
    importlib.reload(D)
    from pocketflow_b200.nets import mobilenet_at_ilsvrc12 as M
    importlib.reload(M)
    from pocketflow_b200.learners.learner_utils import create_learner
    FLAGS.batch_size, FLAGS.learner, FLAGS.nb_classes = 2, 'chn-pruned-rmt', 1001
    base = dict(cpr_nb_smpls=4, cpr_nb_crops_per_smpl=4, cpr_ista_nb_iters=30, cpr_lstsq_nb_iters=5,
                summ_step=10 ** 9, save_step=10 ** 9)
    base.update(flags)
    for k, v in base.items():
        setattr(FLAGS, k, v)
    return create_learner(None, M.ModelHelper())


@pytest.mark.parametrize('poison', [False, True])
def test_resnet8_selection_finetune_warm_start_and_eval(monkeypatch, tmp_path, poison):
    if poison:
        monkeypatch.setenv('PF_POISON', '1')
    paths = dict(cpr_save_path=str(tmp_path / 'cpr' / 'model.ckpt'), cpr_save_path_ws=str(tmp_path / 'ws' / 'model.ckpt'),
                 cpr_save_path_eval=str(tmp_path / 'eval' / 'model.ckpt'))
    lrn = make_resnet(**paths)
    assert len(lrn.maskable_vars) == 10                                      # 7 3x3 convs + 2 projections + the stem
    assert lrn.prune_ratios[0] == 0.0 and lrn.prune_ratios[-1] == 0.5
    ex = lrn.sess_train
    lrn.train(nb_iters=3)                          # selection, save / restore ws, masks, 3 masked Momentum steps
    check_selection(lrn, lrn.store_full.state_dict())
    for rec, v in zip(lrn.selection_log, lrn.maskable_vars):
        # masks = the selected channels; the masked weights stayed zero through the fine-tuning steps
        w, m = ex.store.view(v).cpu().numpy(), ex.store.view(v, ex.MASK).cpu().numpy()
        keep = (rec['mask'] != 0).astype(F32)
        assert np.array_equal(m, np.broadcast_to(keep[None, None, :, None], m.shape)), v.name
        assert np.all(w[m == 0] == 0)
    assert ex.step_count == 3 and np.isfinite(ex.fetch_losses()['loss'])
    if poison:
        return
    from pocketflow_b200.learners.abstract_learner import latest_checkpoint, load_checkpoint
    ws_state = load_checkpoint(latest_checkpoint(str(tmp_path / 'ws')))
    from pocketflow_b200.datasets.abstract_dataset import POOL_SIZE
    trained = lrn.evaluate(nb_iters=POOL_SIZE)[0]                     # (the whole synthetic pool: the same batches)
    del lrn
    # --exec_mode eval restores the fine-tuned model
    fresh = make_resnet(exec_mode='eval', **paths)
    assert abs(fresh.evaluate(nb_iters=POOL_SIZE)[0] - trained) <= 1e-6 * abs(trained)
    del fresh
    # warm start: no selection, the selected model is restored from cpr_save_path_ws (its training run then writes
    # its own checkpoints to cpr_save_path)
    warm = make_resnet(cpr_warm_start=True, **paths)
    warm.choose_channels = lambda *a, **k: pytest.fail('cpr_warm_start must skip the channel selection')
    warm.train(nb_iters=0)
    now = warm.sess_train.store.state_dict()
    for k, v in ws_state.items():
        assert np.array_equal(now[k], v), k


def test_mobilenet_selection_keeps_the_target_counts(tmp_path):
    lrn = make_mobilenet(cpr_save_path_ws=str(tmp_path / 'ws' / 'model.ckpt'))
    assert len(lrn.maskable_vars) == 15                                      # stem, 13 pointwise, the logits conv
    assert 'Logits' in lrn.maskable_vars[-1].name and lrn.prune_ratios[-1] == 0.5
    lrn.choose_channels()
    check_selection(lrn, lrn.store_full.state_dict())
    assert os.path.exists(str(tmp_path / 'ws' / 'model.ckpt.npz'))
    for rec in lrn.selection_log:
        assert set(rec['times']) == {'sample', 'gram', 'search', 'refit'}


def test_selection_matches_the_layer_by_layer_oracle(monkeypatch, tmp_path):
    """one full selection of ResNet-8 (exact-fp32 convs) against the oracle driven layer by layer on the same cached
    batches with the same seed: the draws, the γ sequence and the kept channels exactly, the kernels within the refit's
    tolerance"""
    from oracle.step_oracle import StepOracle
    monkeypatch.setenv('PF_CONV_PATH', 'fp32')
    lrn = make_resnet(cpr_save_path_ws=str(tmp_path / 'ws' / 'model.ckpt'), cpr_nb_smpls=32, cpr_nb_crops_per_smpl=2)
    ex = lrn.sess_train
    cached = lrn.cache_batches()
    lrn.init_from_full()
    g = lrn.graph_train
    orc_f = StepOracle([op for op in g.ops if op.name.startswith('model/')], lrn.logits_full, lrn.images)
    orc_p = StepOracle([op for op in g.ops if op.name.startswith('pruned_model/')], ex.logits_t, lrn.images)
    st_f, st_p = lrn.store_full.state_dict(), ex.store.state_dict()
    rng = np.random.RandomState(lrn.seed)
    images = [c.cpu().numpy() for c in cached]
    nb_min = FLAGS.cpr_nb_crops_per_smpl * FLAGS.cpr_nb_smpls
    ref = []
    for i, (op_f, op_p) in enumerate(zip(lrn.conv_ops_full, lrn.conv_ops_prnd)):
        kname = op_p.vars['kernel'].name
        xs, ys, nb = [], [], 0
        for im in images:
            pf = {k: torch.from_numpy(np.array(v, F32)) for k, v in st_f.items()}
            pp = {k: torch.from_numpy(np.array(v, F32)) for k, v in st_p.items()}
            with torch.no_grad():
                tf_ = orc_f.forward(pf, torch.from_numpy(im), True, {})
                tp_ = orc_p.forward(pp, torch.from_numpy(im), True, {})
            x_f, y_f = tf_[op_f.inputs[0].name].numpy(), tf_[op_f.output.name].numpy()
            x_p, y_p = tp_[op_p.inputs[0].name].numpy(), tp_[op_p.output.name].numpy()
            X, Y, _, err = C.cpr_sample(rng, st_f[op_f.vars['kernel'].name], st_p[kname], x_f, x_p, y_f, y_p,
                                        op_f.attrs['strides'], op_f.attrs['padding'], FLAGS.cpr_nb_crops_per_smpl,
                                        pads=op_f.attrs['pad'])
            assert max(err) < 1e-6
            xs.append(X)
            ys.append(Y)
            nb += len(Y)
            if nb > nb_min:
                break
        idxs = rng.choice(nb, size=(nb_min), replace=False)
        X, Y = np.vstack(xs)[idxs], np.vstack(ys)[idxs]
        w_new, log, mask = C.cpr_solve_sparse_regression(
            rng, X, Y, st_p[kname], lrn.prune_ratios[i], FLAGS.cpr_ista_lrn_rate, FLAGS.cpr_ista_nb_iters,
            FLAGS.cpr_lstsq_lrn_rate, FLAGS.cpr_lstsq_nb_iters, FLAGS.loss_w_dcy)
        ref.append((log, mask, w_new))
        st_p[kname] = w_new
    lrn.choose_channels(cached=cached)
    for i, (rec, (log, mask, w_new)) in enumerate(zip(lrn.selection_log, ref)):
        assert [a[1] for a in rec['search']] == [a[1] for a in log], (i, rec['search'], log)
        assert np.allclose([a[0] for a in rec['search']], [a[0] for a in log], rtol=0, atol=0)
        assert np.array_equal(rec['mask'] != 0, mask[:, 0] != 0), i
        w = ex.store.view(lrn.maskable_vars[i]).cpu().numpy()
        assert np.abs(w - w_new).max() <= 2e-3 * FLAGS.cpr_lstsq_lrn_rate * FLAGS.cpr_lstsq_nb_iters + \
            1e-4 * np.abs(w_new).max(), i
