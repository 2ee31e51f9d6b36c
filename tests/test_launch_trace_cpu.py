"""The executor's kernel launches against the trace tests/golden/make_launch_trace.py recorded
(tests/golden/launches_v1.json): forward, backward and layer_wgrad of the benchmarked networks and of the variants that
reach every conv lowering, launch by launch with normalised arguments."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
WANT = json.load(open(os.path.join(GOLDEN, 'launches_v1.json')))

# the conv and batch-norm lowerings the trace has to reach (the level operands, the side-stream weight gradient and
# the folded batch norm need a CUDA device: tests/test_launch_trace_gpu.py covers them)
COVERED = ('pf_conv2d_tc_fwd', 'pf_conv2d_tc_fwd_planes', 'pf_conv2d_fwd', 'pf_conv2d_tc_dgrad',
           'pf_conv2d_tc_dgrad_planes', 'pf_conv2d_dgrad', 'pf_conv2d_tc_wgrad_planes', 'pf_conv2d_wgrad', 'pf_im2col',
           'pf_im2col_planes', 'pf_s2d_planes', 'pf_gather_rows', 'pf_fold_diag_blocks', 'pf_split_bf16',
           'pf_bn_apply_add_eval', 'pf_uq_act_quant_planes', 'pf_uq_act_quant', 'pf_uq_act_minmax')


def test_trace_reaches_every_conv_lowering():
    names = {launch[0] for case in WANT.values() for launch in case}
    assert not [n for n in COVERED if n not in names]


def test_executor_launches_exactly_as_recorded():
    """traced in a child process that sees no CUDA device, as the fixture was: the split-K partition of a weight
    gradient follows the SM count of the current device"""
    code = ('import sys; sys.path.insert(0, %r); import make_launch_trace as T; sys.stdout.write(T.dumps(T.snapshot()))'
            % GOLDEN)
    argv = [sys.executable, '-B'] + (['-s'] if sys.flags.no_user_site else []) + ['-c', code]
    out = subprocess.run(argv, cwd=ROOT, env=dict(os.environ, CUDA_VISIBLE_DEVICES=''), capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
    got = json.loads(out.stdout)
    assert sorted(got) == sorted(WANT)
    for key in WANT:
        for i, (a, b) in enumerate(zip(got[key], WANT[key])):
            assert a == b, (key, i, a, b)
        assert len(got[key]) == len(WANT[key]), key
    assert out.stdout == open(os.path.join(GOLDEN, 'launches_v1.json')).read()
