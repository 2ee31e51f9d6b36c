"""The executor's kernel launches on a CUDA device against the trace tests/golden/make_launch_trace.py recorded
(tests/golden/launches_gpu_v1.json): the forms that are only planned on a GPU (integer-level operands, the side-stream
weight gradient, batch norms folded into the conv epilogue), launch by launch with normalised arguments and stream
placement.  Nothing runs: every launch entry point is replaced by a recorder."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
WANT = json.load(open(os.path.join(GOLDEN, 'launches_gpu_v1.json')))

# the entry points only an executor planned on a CUDA device reaches
COVERED = ('pf_bn_apply_quant_levels', 'pf_conv2d_tc_fwd_ex', 'pf_conv2d_tc_wgrad_ex', 'pf_conv2d_tc_fwd_planes_bn')

# entry points of the lowerings that neither trace reaches, with the reason
NOT_REACHED = {
    'pf_conv2d_tc_fwd_bn': 'in the traced networks every conv whose batch norm is folded reads its input as planes; '
                           'tests/test_teacher_bn_fold_gpu.py checks the fp32-input kernel against the unfused pair',
}

# every entry point a batch-norm or conv lowering of engine.Executor can call: each is reached by this trace or the
# CPU one (tests/golden/launches_v1.json), or listed in NOT_REACHED
LOWERING_ENTRY_POINTS = (
    'pf_conv2d_fwd', 'pf_conv2d_dgrad', 'pf_conv2d_wgrad', 'pf_conv2d_tc_fwd', 'pf_conv2d_tc_fwd_planes',
    'pf_conv2d_tc_fwd_bn', 'pf_conv2d_tc_fwd_planes_bn', 'pf_conv2d_tc_fwd_ex', 'pf_conv2d_tc_dgrad',
    'pf_conv2d_tc_dgrad_planes', 'pf_conv2d_tc_wgrad_planes', 'pf_conv2d_tc_wgrad_ex', 'pf_conv2d_tc_prep_weight',
    'pf_split_bf16', 'pf_im2col', 'pf_im2col_planes', 'pf_s2d_planes', 'pf_gather_rows', 'pf_add',
    'pf_fold_diag_blocks', 'pf_bn_train_stats', 'pf_bn_train_stats_range', 'pf_bn_apply', 'pf_bn_apply_planes',
    'pf_bn_apply_quant', 'pf_bn_apply_quant_levels', 'pf_bn_apply_eval', 'pf_bn_apply_add', 'pf_bn_apply_add_eval',
    'pf_bn_apply_eval_gather', 'pf_bn_bwd', 'pf_bn_bwd_planes', 'pf_gather_channels', 'pf_uq_act_quant',
    'pf_uq_act_quant_planes', 'pf_uq_act_minmax')


def names(trace):
    return {launch[0] for case in trace.values() for launch in case}


def test_trace_reaches_every_lowering_entry_point():
    got = names(WANT['cases'])
    assert not [n for n in COVERED if n not in got]
    got |= names(json.load(open(os.path.join(GOLDEN, 'launches_v1.json'))))
    assert not [n for n in LOWERING_ENTRY_POINTS if n not in got and n not in NOT_REACHED]
    assert not [n for n in NOT_REACHED if n in got]


@pytest.mark.gpu
def test_executor_launches_on_gpu_exactly_as_recorded():
    """traced in a child process, so that the caching allocator starts empty as it did for the fixture"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if sms != WANT['sm_count']:
        pytest.skip('the fixture was recorded on a device with %d SMs, this one has %d: the split-K partition of the '
                    'weight gradients follows the SM count' % (WANT['sm_count'], sms))
    code = ('import sys; sys.path.insert(0, %r); import make_launch_trace as T; '
            'sys.stdout.write(T.dumps_gpu(T.snapshot_gpu()))' % GOLDEN)
    argv = [sys.executable, '-B'] + (['-s'] if sys.flags.no_user_site else []) + ['-c', code]
    out = subprocess.run(argv, cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
    got = json.loads(out.stdout)['cases']
    want = WANT['cases']
    assert sorted(got) == sorted(want)
    for key in want:
        for i, (a, b) in enumerate(zip(got[key], want[key])):
            assert a == b, (key, i, a, b)
        assert len(got[key]) == len(want[key]), key
    assert out.stdout == open(os.path.join(GOLDEN, 'launches_gpu_v1.json')).read()
