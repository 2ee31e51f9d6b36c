"""The LASSO channel-pruning learner (`--learner channel`) without a GPU: the LARS-Lasso solver (KKT conditions, and
sklearn's LassoLars where sklearn is installed), the reference's alpha bisection, the refit, the W1 / W2 prunability rules
against a golden file, the preserve ratios, and create_learner."""
import importlib
import json
import os

import numpy as np
import pytest

from pocketflow_b200.flags import FLAGS
from pocketflow_b200.learners.channel_pruning import lars
from pocketflow_b200.learners.channel_pruning import learner as L

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'cp_fathers_v1.json')


def problem(seed, n, c, noise=0.5):
    rng = np.random.RandomState(seed)
    P = rng.randn(n, c) * rng.uniform(0.1, 3.0, c)
    b = np.zeros(c)
    on = rng.choice(c, max(c // 3, 1), replace=False)
    b[on] = rng.randn(on.size)
    return P, P.dot(b) + noise * rng.randn(n)


PROBLEMS = [(0, 400, 30), (1, 2000, 64), (2, 3000, 128), (3, 5000, 256)]
FRACTIONS = (0.9, 0.5, 0.1, 0.01, 1e-3)


@pytest.mark.parametrize('seed,n,c', PROBLEMS)
def test_lars_meets_the_lasso_kkt_conditions(seed, n, c):
    P, y = problem(seed, n, c)
    G, xy = P.T.dot(P), P.T.dot(y)
    path = lars.LarsLassoPath(G, xy, n)
    amax = np.abs(xy).max() / n
    for f in FRACTIONS:
        alpha = amax * f
        b = path.coef_at(alpha)
        corr = (xy - G.dot(b)) / n                                    # P^T (y - P b) / n
        on = b != 0
        assert on.any()
        assert np.all(np.abs(corr) <= alpha * (1 + 1e-9)), (f, np.abs(corr).max() / alpha)
        assert np.allclose(np.abs(corr[on]), alpha, rtol=1e-9, atol=0), f
        assert np.array_equal(np.sign(corr[on]), np.sign(b[on])), f


@pytest.mark.parametrize('seed,n,c', PROBLEMS)
def test_lars_matches_sklearn_lassolars(seed, n, c):
    sklm = pytest.importorskip('sklearn.linear_model')
    import warnings
    P, y = problem(seed, n, c)
    path = lars.LarsLassoPath(P.T.dot(P), P.T.dot(y), n)
    amax = np.abs(P.T.dot(y)).max() / n
    for f in FRACTIONS:
        alpha = amax * f
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            ref = sklm.LassoLars(alpha=alpha, fit_intercept=False, max_iter=3000).fit(P, y).coef_
        got = path.coef_at(alpha)
        assert np.array_equal(ref != 0, got != 0), f
        assert np.abs(got - ref).max() <= 1e-8 * np.abs(ref).max(), f


def channel_problem(seed, S=60, cin=48, cout=16):
    """a design matrix as compute_pruned_kernel forms it: rows (s, o), one column per input channel"""
    rng = np.random.RandomState(seed)
    X = rng.randn(S, 9, cin) * rng.uniform(0.2, 2.0, cin)
    W2 = rng.randn(9, cin, cout) * 0.1
    P = np.einsum('shc,hco->soc', X, W2).reshape(S * cout, cin)
    y = P.dot(rng.uniform(0.5, 1.5, cin)) + 0.1 * rng.randn(S * cout)
    return P, y


@pytest.mark.parametrize('seed,c_new,quadruple', [(0, 20, False), (1, 29, False), (2, 10, True), (3, 33, True),
                                                    (4, 1, False)])
def test_bisection_matches_the_reference_loop_on_sklearn(seed, c_new, quadruple):
    """the package's bisection on the Gram path and the reference's loop driving sklearn's LassoLars on P: the same
    alphas, counts and kept channels"""
    sklm = pytest.importorskip('sklearn.linear_model')
    import warnings
    P, y = channel_problem(seed)
    cin = P.shape[1]

    def sk_solve(alpha):
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            return sklm.LassoLars(alpha=alpha, fit_intercept=False, max_iter=3000).fit(P, y).coef_
    ref_idxs, ref_log = lars.select_channels(sk_solve, cin, c_new, quadruple=quadruple)
    idxs, log = lars.lasso_select(P.T.dot(P), P.T.dot(y), P.shape[0], c_new, quadruple=quadruple)
    assert log == ref_log
    assert np.array_equal(idxs, ref_idxs)


# the reference loop (channel_pruner.py:496-565) driving sklearn 1.9's LassoLars on channel_problem(5, cin=64) with
# c_new = 32: its solves (alpha, nnz) and the kept channels, recorded once so that the check runs without sklearn
REF_LOG_5 = [(0.0001, 64), (0.0002, 64), (0.0004, 64), (0.0008, 64), (0.0016, 64), (0.0032, 63), (0.0064, 63),
             (0.0128, 60), (0.0256, 50), (0.0512, 45), (0.1024, 34), (0.2048, 15), (0.0001, 64), (0.102425, 34),
             (0.12801875000000001, 25), (0.10882343750000001, 30), (0.09442695312500002, 37), (0.10522431640625002, 32)]
REF_KEPT_5 = [0, 1, 2, 6, 7, 8, 9, 12, 14, 16, 20, 21, 22, 23, 26, 31, 32, 33, 35, 39, 40, 44, 46, 47, 50, 52, 54, 59,
              60, 61, 62, 63]


def test_bisection_returns_the_reference_kept_count():
    """a seeded problem: exactly the solves, the kept count and the kept channels of the reference loop on sklearn"""
    P, y = channel_problem(5, cin=64)
    idxs, log = lars.lasso_select(P.T.dot(P), P.T.dot(y), P.shape[0], 32)
    assert log == REF_LOG_5
    assert int(idxs.sum()) == 32 and list(np.where(idxs)[0]) == REF_KEPT_5
    assert lars.lasso_select(P.T.dot(P), P.T.dot(y), P.shape[0], 64)[0].all()


def test_refit_matches_linear_regression():
    sklm = pytest.importorskip('sklearn.linear_model')
    rng = np.random.RandomState(3)
    X = rng.randn(900, 120) * rng.uniform(0.5, 2.0, 120)
    Y = X.dot(rng.randn(120, 24)) + 0.1 * rng.randn(900, 24)
    ref = sklm.LinearRegression(fit_intercept=False).fit(X, Y).coef_.T
    got, how = lars.solve_normal_equations(X.T.dot(X), X.T.dot(Y))
    assert how == 'cholesky'
    assert np.abs(got - ref).max() <= 1e-8 * np.abs(ref).max()


def test_refit_of_a_rank_deficient_input_is_the_minimum_norm_solution():
    rng = np.random.RandomState(4)
    X = rng.randn(300, 40)
    X[:, 7] = 0.0                                                      # a dead input channel
    Y = rng.randn(300, 5)
    got, how = lars.solve_normal_equations(X.T.dot(X), X.T.dot(Y))
    assert how == 'lstsq'
    ref = np.linalg.lstsq(X, Y, rcond=None)[0]
    assert np.all(got[7] == 0) or np.abs(got[7]).max() <= 1e-12
    assert np.abs(got - ref).max() <= 1e-8 * np.abs(ref).max()


def test_refit_of_collinear_constant_channels_is_the_minimum_norm_solution():
    """two constant input channels (relu(beta) of producer channels another consumer pruned) are collinear: A factors
    with a rounding-sized pivot, which the relative pivot test sends to lstsq"""
    rng = np.random.RandomState(5)
    X = np.maximum(rng.randn(400, 30), 0)
    X[:, 3], X[:, 11] = 0.7, 1.4
    Y = rng.randn(400, 4)
    got, how = lars.solve_normal_equations(X.T.dot(X), X.T.dot(Y))
    ref = np.linalg.lstsq(X, Y, rcond=None)[0]
    assert how == 'lstsq'
    assert np.abs(got - ref).max() <= 1e-8 * np.abs(ref).max()


def test_l1_selection_keeps_the_largest_input_channels():
    rng = np.random.RandomState(0)
    w = rng.randn(3, 3, 10, 4)
    norms = np.abs(w).sum((0, 1, 3))
    kept = lars.l1_select(w, 4)
    assert kept.sum() == 4 and set(np.where(kept)[0]) == set(np.argsort(-norms)[:4])


# ---------------------------------------------------------------------------------------------------- learner plumbing
def test_flag_defaults():
    assert FLAGS.cp_prune_option == 'auto' and FLAGS.cp_prune_list_file == 'ratio.list'
    assert FLAGS.cp_uniform_preserve_ratio == 0.6 and FLAGS.cp_preserve_ratio == 0.5
    assert FLAGS.cp_lasso is True and FLAGS.cp_quadruple is False
    assert FLAGS.cp_nb_points_per_layer == 10 and FLAGS.cp_nb_batches == 30
    assert FLAGS.cp_channel_pruned_path == './models/pruned_model.ckpt' and FLAGS.cp_list_group == 1000


def test_preserve_ratios(tmp_path):
    assert L.preserve_ratios(5, 'uniform', 0.6, None) == [1.0, 0.6, 0.6, 0.6, 1.0]
    f = tmp_path / 'ratio.list'
    f.write_text('0.3\n0.4\n0.5\n')
    assert L.preserve_ratios(5, 'list', 0.6, str(f)) == [1.0, 0.4, 0.5, 1.0, 1.0]
    with pytest.raises(ValueError, match='cp_prune_option uniform'):
        L.preserve_ratios(5, 'auto', 0.6, None)
    assert L.kept_count(64, 0.6) == 38 and L.kept_count(3, 0.1) == 1


def test_list_groups_are_refused():
    L.refuse_list_groups(22, 'list', 1000, False, False)
    L.refuse_list_groups(22, 'list', 22, False, False)
    L.refuse_list_groups(22, 'uniform', 5, False, False)               # (uniform mode has no groups)
    with pytest.raises(ValueError, match='cp_list_group'):
        L.refuse_list_groups(22, 'list', 21, False, False)
    for ft, rt in ((True, False), (False, True)):
        with pytest.raises(ValueError, match='cp_finetune / --cp_retrain'):
            L.refuse_list_groups(22, 'uniform', 1000, ft, rt)


def test_sampling_draws_replay_in_the_reference_order():
    rng, ref = np.random.RandomState(1), np.random.RandomState(1)
    draws = L.draw_positions(rng, 2, [(8, 8), (4, 6)], 3)
    for b in range(2):
        for t, (h, w) in enumerate([(8, 8), (4, 6)]):
            assert np.array_equal(draws[b][t][0], ref.randint(0, h, 3))
            assert np.array_equal(draws[b][t][1], ref.randint(0, w, 3))
    rows = L.sample_rows(draws[0][0], draws[0][1], 2, 6)
    assert rows.shape == (6, 8) and list(rows[:, 3]) == list(range(6, 12))
    assert list(rows[:, 0]) == [0, 0, 0, 1, 1, 1]                    # n-major, then the point
    assert list(rows[:3, 1]) == list(draws[0][0][0]) and list(rows[3:, 4]) == list(draws[0][1][0])


@pytest.mark.parametrize('net', ['resnet20', 'resnet50', 'mobilenet_v1', 'mobilenet_v2'])
def test_prunability_rules_match_the_golden_file(net):
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
    import make_cp_fathers
    with open(GOLDEN) as f:
        ref = json.load(f)[net]
    assert make_cp_fathers.rules(net) == ref


def test_golden_fathers_follow_the_block_structure():
    with open(GOLDEN) as f:
        g = json.load(f)
    count = lambda k, i: sum(r[i] is not None for r in g[k])
    # ResNet v2: the second conv of every basic block, the stride-1 convs of the first block (stem-fed); bottleneck:
    # every last 1x1, every stride-1 3x3, the first block's 1x1 and projection (max-pool-fed)
    assert (len(g['resnet20']), count('resnet20', 1), count('resnet20', 3)) == (22, 11, 12)
    assert (len(g['resnet50']), count('resnet50', 1), count('resnet50', 3)) == (53, 31, 20)
    # MobileNet-v1: every pointwise conv, through its depthwise conv to the previous pointwise conv
    v1 = g['mobilenet_v1']
    assert count('mobilenet_v1', 1) == 13 and count('mobilenet_v1', 3) == 0
    for name, father, target, _ in v1[1:-1]:
        assert father.endswith('/depthwise') and target.endswith('/Conv2D')


def make(**flags):
    FLAGS.reset()
    importlib.import_module('pocketflow_b200.learners.channel_pruning.learner')
    mod = importlib.reload(importlib.import_module('pocketflow_b200.nets.resnet_at_cifar10'))
    from pocketflow_b200.learners.learner_utils import create_learner
    FLAGS.batch_size, FLAGS.resnet_size = 2, 20
    for k, v in flags.items():
        setattr(FLAGS, k, v)
    return create_learner(None, mod.ModelHelper())


def test_create_learner():
    lrn = make(learner='channel', cp_prune_option='uniform')
    assert type(lrn).__name__ == 'ChannelPrunedLearner'
    assert len(lrn.maskable_vars) == 22 and lrn.prune_ratios[0] == lrn.prune_ratios[-1] == 1.0
    with pytest.raises(ValueError, match='cp_prune_option auto'):
        make(learner='channel')
    for name in ('dis-chn-pruned', 'uniform-tf'):
        with pytest.raises(ValueError, match='outside the hot-path scope'):
            make(learner=name)
    with pytest.raises(ValueError, match='cp_list_group'):
        make(learner='channel', cp_prune_option='list', cp_list_group=4)
    with pytest.raises(ValueError, match='cp_finetune'):
        make(learner='channel', cp_prune_option='uniform', cp_finetune=True)
    with pytest.raises(ValueError, match='enbl_compact_ft'):
        make(learner='channel', cp_prune_option='uniform', enbl_compact_ft=True)
