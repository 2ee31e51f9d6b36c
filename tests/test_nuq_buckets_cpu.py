"""Bucketed codebooks (--nuql_use_buckets) without a GPU: the oracle against the reference's own __bucket_quantize
(tests/golden/ref_executed_nuq_buckets_v1.json, made by tests/golden/make_golden_nuq_buckets.py), the host-side work
tables of the bucketed kernels, and the flag checks."""
import hashlib
import json
import os

import numpy as np
import pytest

from oracle import nuq_bucket_oracle as B
from oracle import pf_oracle as O

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_executed_nuq_buckets_v1.json')


def _gold():
    with open(GOLD) as f:
        return json.load(f)


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _input(c):
    rng = np.random.default_rng(c['seed'])
    x = (rng.standard_normal(c['shape']) * rng.choice([1e-2, 1.0, 9.0])).astype(np.float32)
    if c['tie_runs']:
        x.reshape(-1)[: x.size // 3] = x.reshape(-1)[0]
    if c['constant']:
        x[...] = x.reshape(-1)[0]
    return x


def test_golden_covers_the_layouts_and_bits():
    cases = _gold()['cases']
    kinds = set()
    for c in cases:
        n = int(np.prod(c['shape']))
        if c['bucket_type'] == 'split':
            kinds.add('split<' if n < c['bucket_size'] else ('split=' if n % c['bucket_size'] == 0 else 'split%'))
        else:
            kinds.add('dense' if len(c['shape']) == 2 else ('depthwise' if c['shape'][-1] == 1 else 'conv'))
    assert kinds == {'split<', 'split=', 'split%', 'conv', 'dense', 'depthwise'}
    assert {c['bits'] for c in cases} == {1, 2, 4, 8}
    assert any(c['constant'] for c in cases) and any(c['tie_runs'] for c in cases)


@pytest.mark.parametrize('i', range(32))
def test_oracle_reproduces_the_reference_bucket_quantize(i):
    c = _gold()['cases'][i]
    x = _input(c)
    qx, clusters, idx, _, _ = B.nonuniform_quantize_buckets(x, c['bits'], c['bucket_type'], c['bucket_size'])
    assert list(clusters.shape) == c['clusters_shape']
    assert _sha(qx) == c['qx']
    assert _sha(clusters) == c['clusters']
    assert _sha(idx.astype(np.int64)) == c['idx']
    shape = tuple(c['shape'])
    assert B.bucket_storage_bits([shape], c['bucket_type'], c['bucket_size']) == c['bucket_storage']


def test_bucket_storage_matches_the_reference():
    from pocketflow_b200 import ops
    for r in _gold()['bucket_storage']:
        shapes = [tuple(s) for s in r['shapes']]
        assert B.bucket_storage_bits(shapes, r['bucket_type'], r['bucket_size']) == r['bits']
        assert sum(64 * ops.uq_bucket_layout(s, True, r['bucket_type'], r['bucket_size'])[0] for s in shapes) == r['bits']


def test_reference_cannot_run_uniform_init_with_buckets():
    assert all(r['raises'] for r in _gold()['uniform_init'])


def test_quantile_positions_are_the_oracle_order_statistics():
    from pocketflow_b200 import ops
    rng = np.random.default_rng(5)
    for rows in (1, 2, 7, 64, 100, 4608, 9216):
        col = rng.standard_normal((rows, 1)).astype(np.float32)
        s = np.sort(col[:, 0])
        for bits in (1, 2, 4, 8):
            k = 1 << bits
            pos = ops.nuq_bucket_quantile_positions(rows, bits)
            ref = O.nuq_quantile_init(col, k, axis=0)[:, 0]
            assert np.array_equal(s[pos[:k]], ref)


@pytest.mark.parametrize('bits', [1, 4, 8])
def test_bucket_work_tables_cover_every_element_once(bits):
    from pocketflow_b200 import ops
    shapes = [((3, 3, 512, 512), 'channel', 0), ((2048, 1000), 'channel', 0), ((3, 3, 32, 1), 'channel', 0),
              ((3, 3, 64, 64), 'split', 256), ((1, 1, 8, 5), 'split', 64), ((5, 5, 3, 7), 'split', 100)]
    segs = np.zeros(len(shapes), dtype=ops.UQ_SEG)
    for i, (s, bt, bs) in enumerate(shapes):
        nb, padded = ops.uq_bucket_layout(s, True, bt, bs)
        segs[i]['numel'], segs[i]['padded'], segs[i]['ncols'], segs[i]['bits'] = int(np.prod(s)), padded, nb, bits
    tiles, finals, n_partial = ops.nuq_bucket_works(segs)
    tw = ops.nuq_bucket_tile_width(bits)
    assert (1 << bits) * tw <= ops.NUQ_BUCKET_SMEM_FLOATS and tw <= 256
    for i, seg in enumerate(segs):
        nb, rows = int(seg['ncols']), int(seg['padded']) // int(seg['ncols'])
        cover = np.zeros((rows, nb), np.int32)
        for t in tiles[tiles['seg'] == i]:
            assert t['ncol_tile'] <= tw
            cover[t['start']:t['start'] + t['count'], t['c0']:t['c0'] + t['ncol_tile']] += 1
        assert (cover == 1).all()
    # the finals list each tile's row items in order; partial ranges are disjoint and fill the workspace
    seen = []
    for f in finals:
        items = tiles[f['start']:f['start'] + f['count']]
        assert (items['seg'] == f['seg']).all() and (items['c0'] == f['c0']).all()
        assert list(items['start']) == sorted(items['start'])
        seen.extend(range(f['start'], f['start'] + f['count']))
    assert seen == list(range(len(tiles)))
    ends = tiles['reserved'] + (1 << bits) * tiles['ncol_tile']
    assert tiles['reserved'][0] == 0 and (tiles['reserved'][1:] == ends[:-1]).all() and ends[-1] == n_partial


def test_flag_checks_refuse_what_cannot_run():
    from pocketflow_b200.learners.nonuniform_quantization.utils import NonUniformQuantization, check_bucket_args
    with pytest.raises(ValueError, match='A.6-6'):
        NonUniformQuantization(None, 256, True, 'uniform', 'split')
    with pytest.raises(ValueError, match='A.6-6'):
        check_bucket_args('uniform', 'channel', 0)
    with pytest.raises(ValueError, match='nuql_bucket_size'):
        NonUniformQuantization(None, 0, True, 'quantile', 'split')
    NonUniformQuantization(None, 0, True, 'quantile', 'channel')          # channel ignores the bucket size
    NonUniformQuantization(None, 256, False, 'uniform', 'split')          # per-layer uniform init stays allowed


@pytest.mark.parametrize('extra', [['--nuql_init_style', 'uniform'],
                                   ['--nuql_bucket_type', 'split', '--nuql_bucket_size', '0']])
def test_run_script_returns_1_on_refused_bucket_flags(extra, capsys):
    import importlib
    from pocketflow_b200.flags import FLAGS
    from pocketflow_b200.nets import run_utils
    FLAGS.reset()
    try:
        mod = importlib.import_module('pocketflow_b200.nets.resnet_at_cifar10_run')
        assert run_utils.run(mod.ModelHelper, ['--learner', 'non-uniform', '--nuql_use_buckets'] + extra) == 1
        assert 'ValueError' in capsys.readouterr().err
    finally:
        FLAGS.reset()
