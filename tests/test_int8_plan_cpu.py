"""The integer inference model's launches against the trace tests/golden/make_launch_trace_int8.py recorded
(tests/golden/launches_int8_v1.json): what building int8.IntModel launches and what its forward() launches, for
ResNet-20 with `int8_narrow`, ResNet-50, MobileNet-v1 with `int8_depthwise` and MobileNet-v2 with both, launch by
launch with normalised arguments.  Also that the plan allocates nothing the integer layers do not read: no split-bf16
weight copies of an integer convolution, and no operand planes of a batch norm that only integer layers read."""
import functools
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
WANT = json.load(open(os.path.join(GOLDEN, 'launches_int8_v1.json')))


@functools.lru_cache(maxsize=None)
def _traced():
    """traced in a child process that sees no CUDA device, as the fixture was"""
    code = ('import sys, json; sys.path.insert(0, %r); import make_launch_trace_int8 as T; '
            'sys.stdout.write(json.dumps(T.snapshot()))' % GOLDEN)
    argv = [sys.executable, '-B'] + (['-s'] if sys.flags.no_user_site else []) + ['-c', code]
    out = subprocess.run(argv, cwd=ROOT, env=dict(os.environ, CUDA_VISIBLE_DEVICES=''), capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
    return json.loads(out.stdout)


def test_int_model_launches_exactly_as_recorded():
    got, _ = _traced()
    assert sorted(got) == sorted(WANT)
    for key in WANT:
        for i, (a, b) in enumerate(zip(got[key], WANT[key])):
            assert a == b, (key, i, a, b)
        assert len(got[key]) == len(WANT[key]), key


def test_int_model_owns_no_unread_buffers():
    """building the model prepares the split-bf16 weight copies of every other tensor-core layer and of no integer
    layer, which owns none; no batch norm read only by integer layers owns operand planes"""
    _, own = _traced()
    for case, o in own.items():
        ints = set(o['ints'])
        assert ints, case
        assert not ints & set(o['tc']), case
        assert set(o['prep']) == set(o['tc']) | set(o['stem']), case
        assert not set(o['only_int']) & set(o['planes']), case
    assert all(own[case]['only_int'] for case in ('resnet50', 'mobilenet_v1_depthwise'))


def test_int_layers_need_an_inference_executor_and_a_tensor_core_lowering(monkeypatch):
    """a training executor refuses integer layers; on the exact-fp32 conv path the integer model's plan fails naming
    the first integer convolution, which has no tensor-core lowering whose residual and folded batch norm it takes"""
    import importlib.util

    import pytest
    import torch

    from pocketflow_b200.engine import Executor
    spec = importlib.util.spec_from_file_location('make_launch_trace_int8',
                                                  os.path.join(GOLDEN, 'make_launch_trace_int8.py'))
    T = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(T)
    T.install(monkeypatch)
    im = T.model('resnet20_narrow', 'cpu')
    with pytest.raises(ValueError, match='inference executor'):
        Executor(im.graph, im.images, im.logits, torch.device('cpu'), train=True, int_layers=im.ex.int_layers)
    monkeypatch.setenv('PF_CONV_PATH', 'fp32')
    with pytest.raises(ValueError, match='^model/resnet_model/conv2d_1/Conv2D: an integer layer needs a tensor-core'):
        T.model('resnet20_narrow', 'cpu')
