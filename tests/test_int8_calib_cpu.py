"""Host side of calibrated activation ranges (int8.calibrate / act_ranges): the two calibration statistics on hand-made
ranges, the clamped static-range quantizer against hand-computed levels, select()'s reason for a range that does not
start at 0, the version 3 sidecar round trip, the encoding of the static range slots, and that files without ranges
are written, read and selected exactly as before."""
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from oracle import pf_oracle as O  # noqa: E402
from pocketflow_b200 import compact, int8, ops  # noqa: E402
from support import int8_graph  # noqa: E402

F32 = np.float32


def static_quantize(x, bits, lo, hi):
    """(levels, values) of the activation quantizer (O.uniform_quantize, mode='activation') with its min / max replaced
    by a static range [lo, hi] and x clamped to it first"""
    y = np.clip(np.asarray(x, F32), F32(lo), F32(hi)).astype(F32)
    alpha, beta, k = (F32(hi) - F32(lo)).astype(F32) + F32(1e-10), F32(lo), O.uq_k(bits)
    lv = np.rint((((y - beta) / alpha).astype(F32) * k).astype(F32)).astype(F32)
    return lv, O.uq_inv_scale((lv / k).astype(F32), alpha, beta)


def test_static_quantizer_hand_levels():
    x = np.array([-1.0, 0.0, 0.4, 0.6, 1.5, 2.9, 3.0, 7.0, 1e30], F32)
    lv, v = static_quantize(x, 2, 0.0, 3.0)                    # k = 3, alpha = 3: level = rint(clamp(x))
    assert lv.tolist() == [0, 0, 0, 1, 2, 3, 3, 3, 3]           # 1.5 rounds half to even; above hi -> k
    assert v.tolist() == [0, 0, 0, 1, 2, 3, 3, 3, 3]
    lv, _ = static_quantize(np.array([0.0, 0.5, 1.0, 6.0], F32), 8, 0.0, 1.0)
    assert lv.tolist() == [0, 128, 255, 255]
    # with the tensor's own range the static quantizer is the per-batch one
    rng = np.random.default_rng(0)
    a = np.maximum(rng.standard_normal(4096), 0).astype(F32)
    for bits in (2, 5, 8):
        _, v = static_quantize(a, bits, a.min(), a.max())
        assert np.array_equal(v.view(np.uint32), O.uniform_quantize(a, bits, mode='activation').view(np.uint32))


def test_range_stats():
    per = [{'a': (F32(0), F32(1.0)), 'b': (F32(-1), F32(2))},
           {'a': (F32(0), F32(2.0)), 'b': (F32(-3), F32(5))},
           {'a': (F32(0.5), F32(4.0)), 'b': (F32(0), F32(1))}]
    m = int8.range_stats(per, 'mean')
    assert m == {'a': (F32(0.5 / 3), F32(7.0 / 3)), 'b': (F32(-4.0 / 3), F32(8.0 / 3))}
    assert all(type(v) is F32 for r in m.values() for v in r)
    assert int8.range_stats(per, 'max') == {'a': (F32(0), F32(4)), 'b': (F32(-3), F32(5))}
    assert int8.range_stats(per) == m
    # the float64 mean rounded once to fp32
    big = [{'a': (F32(0), F32(2 ** 24 + 2))}] + [{'a': (F32(0), F32(1))}] * 2
    assert int8.range_stats(big)['a'][1] == F32((2 ** 24 + 4) / 3)
    # one batch: that batch's range bit for bit
    one = {'r': (F32(0.1), F32(np.pi)), 's': (F32(0), F32(6.0))}
    assert int8.range_stats([one], 'mean') == one == int8.range_stats([one], 'max')
    with pytest.raises(ValueError, match='statistic'):
        int8.range_stats(per, 'median')
    with pytest.raises(ValueError, match='at least one batch'):
        int8.range_stats([], 'mean')


def test_range_slots_encoding():
    """range_slots writes the ordered-uint encoding (pf_enc) the kernels decode, and decode_ordered inverts it"""
    import torch
    r = [(0.0, 1.5), (-2.25, 6.0), (-0.0, 3.0e-38), (F32(0.1), F32(np.pi))]
    s = ops.range_slots(r, torch.device('cpu'))
    assert s.dtype == torch.int32 and tuple(s.shape) == (4, 2)
    u = s.numpy().view(np.uint32)
    assert u[0, 0] == 0x80000000 and u[0, 1] == 0x80000000 | np.float32(1.5).view(np.uint32)
    assert u[1, 0] == ~np.float32(-2.25).view(np.uint32) & 0xFFFFFFFF
    got = ops.decode_ordered(u).reshape(-1, 2)
    assert np.array_equal(got.view(np.uint32), np.asarray(r, F32).view(np.uint32))
    # the order of the encoding is the order of the floats
    assert u[1, 0] < u[0, 0] < u[0, 1] < u[1, 1]


def _ranges(g, cfg, lo=0.0):
    return {op.name: (F32(lo), F32(6.0)) for op in int8.quant_marks(g, cfg)[1]}


@pytest.mark.parametrize('key', ['resnet20_narrow', 'resnet50', 'mobilenet_v1_depthwise', 'mobilenet_v2_depthwise_narrow'])
def test_select_with_ranges(key):
    """ranges that start at 0 select what select() without ranges does; a consumer whose input range starts elsewhere
    keeps fake-quant with the reason, every other layer keeps its selection"""
    g, _, lg, cfg = int8_graph(key, 2)
    base = int8.select(g, lg, cfg)
    r = _ranges(g, cfg)
    assert int8.select(g, lg, cfg, r) == base
    byname = {op.name: op for op in compact.reachable_ops(g, lg)}
    ints = [n for n, w in base if w is None]
    moved = byname[ints[len(ints) // 2]].inputs[0].op.name        # the activation feeding one integer layer
    r[moved] = (F32(0.25), F32(6.0))
    sel = int8.select(g, lg, cfg, r)
    changed = [(n, w) for (n, w), (_, w0) in zip(sel, base) if w != w0]
    assert changed and all(w == 'calibrated activation range does not start at 0' for _, w in changed)
    assert all(byname[n].inputs[0].op.name == moved for n, _ in changed)
    assert int8.report_lines(sel)[-1] == '%d of %d layers run as integers' % (len(ints) - len(changed), len(sel))
    # a negative lo, too; ranges must cover every quantized activation and be ordered
    r[moved] = (F32(-1.0), F32(6.0))
    assert int8.select(g, lg, cfg, r) == sel
    del r[moved]
    with pytest.raises(ValueError, match='no calibrated range'):
        int8.select(g, lg, cfg, r)
    r[moved] = (F32(2.0), F32(1.0))
    with pytest.raises(ValueError, match='lo > hi'):
        int8.select(g, lg, cfg, r)


class _Probe(int8.IntModel):
    """IntModel without the executor: what load() hands the constructor, and what export() writes"""

    def __init__(self, graph, images, logits, cfg, state, wlevels, device=None, act_ranges=None):
        self.graph, self.images, self.logits, self.cfg = graph, images, logits, dict(cfg)
        self.act_ranges = int8._ranges(graph, cfg, act_ranges)
        self.sel = int8.select(graph, logits, cfg, self.act_ranges)
        self.state, self.wlevels = dict(state), wlevels


def _probe(g, images, lg, cfg, act_ranges=None):
    byname = {op.name: op for op in compact.reachable_ops(g, lg)}
    wl = {}
    for n, why in int8.select(g, lg, cfg, act_ranges):
        if why is None:
            wl[n] = (np.zeros(byname[n].vars['kernel'].shape, np.uint8), np.ones(1, F32), np.zeros(1, F32))
    return _Probe(g, images, lg, cfg, {'other/var': np.ones(3, F32)}, wl, act_ranges=act_ranges)


@pytest.mark.parametrize('key', ['resnet20_narrow', 'mobilenet_v1_depthwise'])
def test_sidecar_v3_round_trip(key, tmp_path):
    """with ranges: version 3 and every range read back bit for bit (values no short decimal holds included); the
    selection the ranges change travels with them"""
    g, images, lg, cfg = int8_graph(key, 2)
    rng = np.random.default_rng(3)
    r = {n: (F32(0), F32(rng.uniform(0.1, 7.0))) for n in _ranges(g, cfg)}
    first = next(iter(r))
    r[first] = (F32(np.nextafter(F32(0), F32(1))), F32(1) / F32(3))   # a denormal lo: not 0, keeps fake-quant
    path = str(tmp_path / 'm')
    p0 = _probe(g, images, lg, cfg, r)
    p0.export(path)
    rec = json.load(open(path + '.int8.json'))
    assert rec['version'] == int8.SIDECAR_VERSION_RANGES == 3
    assert sorted(rec['act_ranges']) == sorted(r)
    p = _Probe.load(g, images, lg, path)
    assert p.cfg == cfg and p.sel == p0.sel and sorted(p.wlevels) == sorted(p0.wlevels)
    for n, (lo, hi) in r.items():
        glo, ghi = p.act_ranges[n]
        assert type(glo) is F32 and glo.view(np.uint32) == lo.view(np.uint32) and ghi.view(np.uint32) == hi.view(np.uint32)
    assert any(w == 'calibrated activation range does not start at 0' for _, w in p.sel)
    # a version 3 record without ranges, and ranges under an older version, are refused
    for v, drop in ((3, True), (1, False), (2, False)):
        bad = dict(rec, version=v)
        if drop:
            del bad['act_ranges']
        with open(path + '.int8.json', 'w') as f:
            json.dump(bad, f)
        with pytest.raises(ValueError, match='unsupported sidecar version'):
            _Probe.load(g, images, lg, path)


@pytest.mark.parametrize('key', ['resnet20_narrow', 'resnet50', 'mobilenet_v1_depthwise', 'mobilenet_v2_depthwise_narrow'])
def test_files_without_ranges_unchanged(key, tmp_path):
    """no ranges: the sidecar has exactly the keys and version it had before, and loads and selects as before"""
    g, images, lg, cfg = int8_graph(key, 2)
    path = str(tmp_path / 'm')
    _probe(g, images, lg, cfg).export(path)
    rec = json.load(open(path + '.int8.json'))
    dw = any(w is None and n.endswith('/depthwise') for n, w in int8.select(g, lg, cfg))
    assert sorted(rec) == ['config', 'layers', 'version'] and rec['version'] == (2 if dw else 1)
    p = _Probe.load(g, images, lg, path)
    assert p.act_ranges is None and p.sel == int8.select(g, lg, cfg)
    assert [list(x) for x in p.sel] == rec['layers']


def test_executor_refuses_static_ranges_in_training():
    import torch
    from pocketflow_b200.engine import Executor
    g, images, lg, cfg = int8_graph('resnet20_narrow', 2)
    wq, aq = int8._specs(g, cfg, act_ranges=_ranges(g, cfg))
    with pytest.raises(ValueError, match='inference executors only'):
        Executor(g, images, lg, torch.device('cpu'), train=True, weight_quant=wq, act_quant=aq)
    aq['ranges'] = aq['ranges'][:-1]
    with pytest.raises(ValueError, match='one activation range per quantized activation'):
        Executor(g, images, lg, torch.device('cpu'), train=False, weight_quant=wq, act_quant=aq)


RANGE_PASS = {'pf_minmax_reset', 'pf_uq_act_minmax', 'pf_uq_act_quant', 'pf_uq_act_quant_planes', 'pf_bn_eval_levels_u8'}


def _forward_launches():
    """{case: (per-batch forward launches, calibrated forward launches)} of the integer models of
    tests/golden/make_launch_trace_int8.py, recorded without running a kernel; the calibrated model's ranges are [0, 6]"""
    import gc

    import torch
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
    import make_launch_trace_int8 as T
    out = {}
    with pytest.MonkeyPatch.context() as mp:
        rec = T.install(mp)
        for key in T.CASES:
            im = T.model(key, 'cpu')
            r = {op.name: (F32(0), F32(6)) for op in int8.quant_marks(im.graph, im.cfg)[1]}
            imc = int8.IntModel(im.graph, im.images, im.logits, im.cfg, im.state, im.wlevels, torch.device('cpu'),
                                act_ranges=r)
            got = []
            for m in (im, imc):
                rec.reset()
                m.forward()
                got.append(list(rec.launches))
            out[key] = got
            del im, imc
            gc.collect()
    return out


def test_calibrated_forward_launches_no_range_pass():
    """the calibrated model's forward launches no range reset, range pass or separate activation quantizer, no BN apply
    that accumulates a range, and fewer kernels than the per-batch model, whose forward is otherwise the same: each
    per-batch quantizer launch group becomes one static-range launch"""
    import subprocess
    argv = [sys.executable, '-B'] + (['-s'] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), '--trace']
    res = subprocess.run(argv, cwd=ROOT, env=dict(os.environ, CUDA_VISIBLE_DEVICES=''), capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    traces = json.loads(res.stdout)
    assert len(traces) == 4
    for key, (per_batch, calib) in traces.items():
        names_p, names_c = [x[0] for x in per_batch], [x[0] for x in calib]
        assert not RANGE_PASS & set(names_c), (key, RANGE_PASS & set(names_c))
        # pf_bn_apply_eval's minmax argument (last before the stream) is NULL: no range accumulated
        assert all(x[-2] == 0 for x in calib if x[0] == 'pf_bn_apply_eval'), key
        n_static = sum(n in ('pf_bn_eval_levels_u8_static', 'pf_bn_apply_eval_quant_static', 'pf_uq_act_quant_static')
                       for n in names_c)
        assert n_static > 0 and 'pf_bn_eval_levels_u8_static' in names_c, key
        # every launch that is not a quantizer's is the same, in the same order
        quant = RANGE_PASS | {'pf_bn_apply_eval', 'pf_bn_eval_levels_u8_static', 'pf_bn_apply_eval_quant_static',
                              'pf_uq_act_quant_static'}
        assert [n for n in names_p if n not in quant] == [n for n in names_c if n not in quant], key
        # kernels: pf_bn_eval_levels_u8 without a range launches three (reset, range pass, levels), the static one one
        kern = lambda names: len(names) + 2 * sum(n == 'pf_bn_eval_levels_u8' and x[12] == 0 for n, x in
                                                  zip(names, per_batch if names is names_p else calib))
        assert kern(names_c) < kern(names_p), (key, kern(names_c), kern(names_p))
        print(key, 'forward entry points: per-batch %d, calibrated %d' % (len(names_p), len(names_c)))


if __name__ == '__main__' and '--trace' in sys.argv:
    sys.stdout.write(json.dumps(_forward_launches(), default=str))


def _write_cifar(d, n_files=2, per_file=40):
    rng = np.random.default_rng(5)
    for f in range(n_files):
        lab = rng.integers(0, 10, size=per_file).astype(np.uint8)
        img = rng.integers(0, 256, size=(per_file, 3 * 32 * 32)).astype(np.uint8)
        np.concatenate([lab[:, None], img], axis=1).tofile(os.path.join(d, 'data_batch_%d.bin' % (f + 1)))


@pytest.mark.parametrize('real', [True, False])
def test_export_tool_calibrates_on_distinct_batches(real, tmp_path, monkeypatch):
    """tools/export_uq_int8.py --int8_calibrate N with N > POOL_SIZE hands int8.calibrate N distinct batches, real
    (streamed from --data_dir_local) or synthetic, even when calibrate keeps every batch it was given"""
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    import export_uq_int8 as tool
    from pocketflow_b200.datasets.abstract_dataset import POOL_SIZE
    from pocketflow_b200.flags import FLAGS
    n = POOL_SIZE + 4
    argv = ['--net', 'resnet_at_cifar10', '--resnet_size', '20', '--batch_size_eval', '4', '--int8_calibrate', str(n)]
    if real:
        _write_cifar(str(tmp_path))
        argv += ['--data_dir_local', str(tmp_path)]
    args = tool.parse(argv)
    try:
        _, _, _, cfg = tool.setup(args)
        seen = []
        monkeypatch.setattr(int8, 'calibrate', lambda g, i, l, s, c, batches, stat: seen.extend(batches) or {})
        tool.calibration_ranges(args, cfg, {})
    finally:
        FLAGS.reset()
    assert len(seen) == n and all(tuple(b.shape) == (4, 32, 32, 3) for b in seen)
    flat = {b.numpy().tobytes() for b in seen}
    assert len(flat) == n


def test_static_ranges_refuse_a_batch_statistics_pass(monkeypatch):
    """an inference executor with static ranges whose graph holds a training-mode BN feeding a quantized activation
    refuses forward(training=True): its statistics pass would fold the batch's range into the static slot"""
    import torch
    from pocketflow_b200.engine import Executor
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
    import make_launch_trace as T
    g, images, lg, cfg = int8_graph('resnet20_narrow', 2)
    wq, aq = int8._specs(g, cfg, act_ranges=_ranges(g, cfg))
    T.install(monkeypatch)
    ex = Executor(g, images, lg, torch.device('cpu'), train=False, weight_quant=wq, act_quant=aq)
    bn = next(op for op in ex.ops if op.type == 'FusedBatchNorm' and ex._aq_of_bn(op) is not None)
    ex.forward(training=True)                               # every BN in inference mode: nothing to refuse
    monkeypatch.setitem(bn.attrs, 'training', True)
    with pytest.raises(RuntimeError, match='batch-statistics pass'):
        ex.forward(training=True)
    ex.forward(training=False)
