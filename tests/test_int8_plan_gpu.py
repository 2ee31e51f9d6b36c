"""The integer inference model's launches on a CUDA device against the trace tests/golden/make_launch_trace_int8.py
recorded (tests/golden/launches_int8_gpu_v1.json): the cases of tests/test_int8_plan_cpu.py planned on cuda:0, where
the inference batch norms that follow a u8 convolution are folded into its epilogue, launch by launch with normalised
arguments and stream placement.  Nothing runs: every launch entry point is replaced by a recorder."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
WANT = json.load(open(os.path.join(GOLDEN, 'launches_int8_gpu_v1.json')))


@pytest.mark.gpu
def test_int_model_launches_on_gpu_exactly_as_recorded():
    """traced in a child process, so that the caching allocator starts empty as it did for the fixture"""
    code = ('import sys, json; sys.path.insert(0, %r); import make_launch_trace_int8 as T; '
            'sys.stdout.write(json.dumps(T.snapshot("cuda:0")))' % GOLDEN)
    argv = [sys.executable, '-B'] + (['-s'] if sys.flags.no_user_site else []) + ['-c', code]
    out = subprocess.run(argv, cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
    got, _ = json.loads(out.stdout)
    assert sorted(got) == sorted(WANT)
    for key in WANT:
        for i, (a, b) in enumerate(zip(got[key], WANT[key])):
            assert a == b, (key, i, a, b)
        assert len(got[key]) == len(WANT[key]), key
    # the folded batch norm is reached
    assert any(launch[0] == 'pf_conv2d_u8_fwd' and launch[-2] != 0 for key in WANT if key.endswith('/forward')
               for launch in WANT[key])
