"""CPU tests of the remastered channel-pruning learner's host loop (learners/channel_pruning_rmt/learner.py): the random
draws, the row tables of the sampler, the γ search and the layer ratios, driven by stand-ins and compared with the
numpy oracle (oracle/cpr_oracle.py), plus the flag defaults; then the oracle and the host loop against the reference's
own code, executed under a numpy stub of tensorflow (tests/golden/ref_executed_cpr_v1.json)."""
import ast
import hashlib
import importlib.util
import json
import os

import numpy as np

from oracle import cpr_oracle as C
from pocketflow_b200.learners.channel_pruning_rmt import learner as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


def test_flag_defaults():
    tree = ast.parse(open(os.path.join(ROOT, 'pocketflow_b200', 'learners', 'channel_pruning_rmt', 'learner.py')).read())
    mine = {}
    for node in ast.walk(tree):
        if isinstance(node, ast.Call) and getattr(node.func, 'id', '').startswith('DEFINE_'):
            mine[ast.literal_eval(node.args[0])] = ast.literal_eval(node.args[1])
    assert mine == C.FLAG_DEFAULTS


def test_layer_ratios():
    names = ['pruned_model/conv%d/kernel:0' % i for i in range(6)]
    for frst in (True, False):
        for last in (True, False):
            for skip in (None, 'conv2', 'conv1,conv4/kernel', 'nothing'):
                got = L.prune_ratio_list(names, 0.7, frst, last, skip)
                assert got == C.cpr_prune_ratios(names, 0.7, frst, last, skip)
    assert L.prune_ratio_list(names, 0.5, True, True, 'conv3') == [0.0, 0.5, 0.5, 0.0, 0.5, 0.0]


def test_draws_and_rows_replay_the_oracle_sampling():
    """the learner draws every batch's crops up front, then the kept instances; the oracle draws them batch by batch
    inside the sampling loop, as the reference does — same RandomState, same numbers, same rows"""
    bs, nb_crops, p, q, c = 5, 3, 6, 4, 2
    for nb_smpls, nb_mbtcs in ((7, 2), (10, 2), (9, 4)):
        nb_min = nb_crops * nb_smpls
        rng_l, rng_o = np.random.RandomState(11), np.random.RandomState(11)
        draws, dst = L.draw_samples(rng_l, nb_mbtcs, bs, p, q, nb_crops, nb_min)
        x = np.random.RandomState(0).randn(nb_mbtcs, bs, p, q, c)
        k = np.zeros((1, 1, c, c), F32)
        xs, nb = [], 0
        for b in range(nb_mbtcs):
            X, _, pos, _ = C.cpr_sample(rng_o, k, k, x[b], x[b], x[b], x[b], (1, 1), 'SAME', nb_crops)
            assert pos == draws[b]
            xs.append(X)
            nb += len(X)
            if nb > nb_min:
                break
        assert len(draws) == len(xs)
        idxs = rng_o.choice(nb, size=nb_min, replace=False)
        ref = np.vstack(xs)[idxs]
        # what the device gather writes: row dst[g] of X holds instance g (batch offset + crop * bs + n)
        got = np.full_like(ref, np.nan)
        for b, pos in enumerate(draws):
            rows = L.sample_rows(pos, bs, dst[b * bs * nb_crops:(b + 1) * bs * nb_crops])
            for n_, oh, ow, d in rows:
                if d >= 0:
                    got[d] = x[b, n_, oh, ow]
        assert np.array_equal(got, ref)
        assert rng_l.randint(1 << 30) == rng_o.randint(1 << 30)             # the streams stay in step


def test_gamma_search_matches_the_oracle():
    """the learner's γ search driven by the oracle's ISTA: the same (γ, nnz) sequence, for targets met by doubling,
    by bisection, a target of every channel (ratio 0) and one that bisection cannot meet exactly"""
    rng = np.random.RandomState(5)
    cin, n, cout = 24, 300, 6
    X = rng.randn(n, cin).astype(F32)
    w = (rng.randn(1, 1, cin, cout) * 0.3).astype(F32)
    Y = (X @ w.reshape(cin, cout) + 0.1 * rng.randn(n, cout)).astype(F32)
    g, b, _ = C.cpr_gram(X, Y, w, np.arange(n))
    m0 = rng.uniform(size=(cin, 1))
    for target in (cin, 20, 12, 5, 1, 0):
        masks = []

        def solve(x):
            m, nnz = C.cpr_ista(g, b, m0, x, 1e-2, 50)
            masks.append(m)
            return nnz
        log = L.gamma_search(solve, target)
        mask_ref, log_ref = C.cpr_gamma_search(lambda x: C.cpr_ista(g, b, m0, x, 1e-2, 50), target)
        assert log == log_ref, (target, log, log_ref)
        assert np.array_equal(masks[-1], mask_ref)
        assert log[0][0] == 0.1 and all(x[1] <= cin for x in log)


def test_oracle_lstsq_reduces_the_residual():
    rng = np.random.RandomState(6)
    n, kh, kw, cin, cout = 200, 3, 3, 4, 5
    X = rng.randn(n, kh * kw * cin).astype(F32)
    w = (rng.randn(kh, kw, cin, cout) * 0.2).astype(F32)
    Y = (X @ (w * 1.5).reshape(-1, cout)).astype(F32)
    bnry = np.array([1, 0, 1, 1], F32)
    w2 = C.cpr_lstsq(X, Y, w, bnry, 1e-2, 50, 0.0)
    xm = (X.reshape(n, kh * kw, cin) * bnry).reshape(n, -1)
    r0 = np.square(xm @ (w * bnry[None, None, :, None]).reshape(-1, cout) - Y).sum()
    r1 = np.square(xm @ w2.reshape(-1, cout) - Y).sum()
    assert r1 < r0 and np.all(w2[:, :, 1, :] == 0)


# ---------------------------------------------------------------------------------------------------------- golden
# tests/golden/ref_executed_cpr_v1.json: the reference's own __smpl_inputs_n_outputs, __solve_sparse_regression (on its
# meta LASSO / least-square graphs) and __choose_channels, executed under a numpy stub of tensorflow
# (tests/golden/make_golden_cpr.py, whose case tables and input generators are reused here)

_spec = importlib.util.spec_from_file_location('make_golden_cpr', os.path.join(ROOT, 'tests', 'golden', 'make_golden_cpr.py'))
MG = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MG)
GOLD = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'ref_executed_cpr_v1.json')))


def sha(a, dtype):
    return hashlib.sha256(np.ascontiguousarray(a, dtype).tobytes()).hexdigest()


def test_golden_flag_defaults_and_ratios():
    assert GOLD['flag_defaults'] == C.FLAG_DEFAULTS
    assert len(GOLD['ratios']) == len(MG.RATIO_CASES)
    for g in GOLD['ratios']:
        args = (g['names'], g['cpr_prune_ratio'], g['cpr_skip_frst_layer'], g['cpr_skip_last_layer'], g['cpr_skip_op_names'])
        assert L.prune_ratio_list(*args) == g['ratios'] == C.cpr_prune_ratios(*args), g


def gather_rows(x, rows, k, stride, pt, pl, n_rows):
    """numpy stand-in of pf_cpr_sample's patch gather (include/pf_b200.h): X[dst, (r*S+s)*C + c]"""
    bs, ih, iw, ic = x.shape
    X = np.full((n_rows, k * k * ic), np.nan, F32)
    for n_, oh, ow, d in rows:
        if d < 0:
            continue
        patch = np.zeros((k, k, ic), F32)
        for r in range(k):
            for s in range(k):
                a, b = oh * stride - pt + r, ow * stride - pl + s
                if 0 <= a < ih and 0 <= b < iw:
                    patch[r, s] = x[n_, a, b]
        X[d] = patch.reshape(-1)
    return X


def test_golden_sampling():
    """positions, pruned patches and full outputs of the reference's sampler: the oracle bit for bit, and the learner's
    draws + row table through a numpy stand-in of the gather"""
    assert len(GOLD['sample']) == len(MG.SAMPLE_CASES)
    for g, case in zip(GOLD['sample'], MG.SAMPLE_CASES):
        assert g['case'] == list(case)
        seed, bs, ih, iw, ic, oc, k, stride, padding, nb_crops = case
        x_f, x_p, w_f, w_p, y_f, y_p = MG.sample_inputs(seed, bs, ih, iw, ic, oc, k, stride, padding)
        X, Y, pos, err = C.cpr_sample(np.random.RandomState(seed), w_f, w_p, x_f, x_p, y_f, y_p, (stride, stride),
                                      padding, nb_crops)
        assert [list(p) for p in pos] == g['positions']
        assert sha(X, np.float64) == g['x_sha256'] and sha(Y, np.float64) == g['y_sha256']
        assert max(err) < 1e-6
        n = bs * nb_crops
        draws, dst = L.draw_samples(np.random.RandomState(seed), 1, bs, y_f.shape[1], y_f.shape[2], nb_crops, n)
        assert [list(p) for p in draws[0]] == g['positions'] and sorted(dst) == list(range(n))
        pt, pl = C.cpr_pads(ih, iw, k, k, stride, stride, padding)
        rows = L.sample_rows(draws[0], bs, np.arange(n))
        assert sha(gather_rows(x_p, rows, k, stride, pt, pl, n), np.float64) == g['x_sha256']
        assert sha(np.stack([y_f[r[0], r[1], r[2]] for r in rows]), np.float64) == g['y_sha256']


def test_golden_sparse_regression():
    """the reference's secondary sample, initial mask, normalised G / b, (γ, nnz) of every solve, kept channels and
    final kernel: the oracle (indices, γ sequence and kept channels exactly; G and b by SHA-256; the kernel, whose
    float32 matmul order is not pinned, within 1e-5 of its largest entry) and the learner's host loop (its draws, and
    its γ search replaying the reference's nnz)"""
    rf = GOLD['run_flags']
    assert len(GOLD['regression']) == len(MG.REGRESSION_CASES)
    for g, case in zip(GOLD['regression'], MG.REGRESSION_CASES):
        assert g['case'] == list(case)
        seed, n, kh, kw, ic, oc, ratio, planted = case
        X, Y, w = MG.regression_inputs(seed, n, kh, kw, ic, oc, planted)
        # the learner's draws
        idxs, m0 = L.draw_regression(np.random.RandomState(seed), n, ic, oc)
        assert [int(i) for i in idxs] == g['idxs'] and sha(m0, np.float64) == g['m0_sha256']
        # the oracle's G / b
        gg, bb, _ = C.cpr_gram(X, Y, w, idxs)
        assert sha(gg, np.float64) == g['g_sha256']
        assert np.array_equal(bb.reshape(-1), np.array(g['b']))
        # the oracle's whole regression
        kern, log, mask = C.cpr_solve_sparse_regression(
            np.random.RandomState(seed), X, Y, w, ratio, rf['cpr_ista_lrn_rate'], rf['cpr_ista_nb_iters'],
            rf['cpr_lstsq_lrn_rate'], rf['cpr_lstsq_nb_iters'], rf['loss_w_dcy'])
        assert [list(e) for e in log] == g['solves'], (log, g['solves'])
        assert [int(c) for c in np.flatnonzero(mask[:, 0])] == g['kept']
        ref = np.array(g['kernel'], F32).reshape(w.shape)
        assert np.array_equal(ref == 0, kern == 0)
        assert np.abs(kern - ref).max() <= 1e-5 * np.abs(ref).max()
        # the learner's γ search, its solves replaying the reference's
        it = iter(g['solves'])

        def solve(gamma, it=it):
            want_gamma, nnz = next(it)
            assert gamma == want_gamma
            return nnz
        assert [list(e) for e in L.gamma_search(solve, g['nnz_target'])] == g['solves']
