"""Every tensor-core convolution of one training step of the benchmarked workloads, at the benchmarked batch, against
float64.

bench.py measures its workloads at batch 128 (ResNet-50) and 256 (ResNet-20, MobileNet) (DESIGN.md §8); the other step
tests run ResNet-50 at batch 2, where no CTA of the persistent kernels ever sees a second tile.  Here the learner of a
workload is built at the benchmarked batch under PF_POISON=1 (activation and scratch buffers start as NaN) and one
eager step runs with the tensor-core entry points of `ops` wrapped: each call is passed through unchanged, then
  * its output must be finite, and its launch plan (pf_conv2d_tc_last_plan) is collected;
  * the first call of each (entry point, geometry, operand form, epilogue) is compared with a float64 convolution of
    exactly the operands it was fed — split planes as hi + lo, activation levels as scale x level, weight levels as
    alpha / k * level + beta — with its own epilogue (bias, ReLU, residual, accumulate) and, for a deferred weight
    gradient, the sum of its split-K partials.  Bars as DESIGN.md §6: 2e-5 of max|ref| with a split-bf16 operand,
    1e-5 for levels x levels.  Repeated geometries are checked once: the float64 references of every layer would
    dominate the run time.
Finally every plan the step used must be one the kernel-variant sweep (test_tc_variants_gpu.py) proves it reaches,
so the small-shape sweep covers what the benchmark runs."""

import pytest
import torch

from support import TcRecorder, after_step, geom, run_workload

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')


def tc_recorder(monkeypatch, lrn):
    """a Recorder expecting what the executors planned: every convolution they put on the tensor cores, student and
    teacher, makes at least one forward call, at its own geometry (the first layer's lowered one)"""
    geoms = []
    for ex in (lrn.sess_train, lrn.sess_train.teacher):
        for op in (set(ex.tc) | set(ex.im2col) if ex is not None else ()):
            geoms.append(geom(ex.im2col[op]['d1'] if op in ex.im2col else ex.desc[op]))
    return TcRecorder(monkeypatch, len(geoms), set(geoms))


def test_resnet50_uq8_bench_layers_at_batch_128(monkeypatch):
    run_workload('resnet50_uq8_dst_b128', 128, monkeypatch, tc_recorder)


def test_mobilenet_cpg50_bench_layers_at_batch_256(monkeypatch):
    run_workload('mobilenet_cpg50_b256', 256, monkeypatch, tc_recorder)


@pytest.mark.parametrize('workload,batch', [('resnet50_ws50_dst_b128', 128), ('resnet50_nuq4_dst_b128', 128),
                                            ('resnet20_uq8_dst_b256', 256), ('resnet20_ws50_dst_b256', 256)])
def test_bench_tc_convs(workload, batch, monkeypatch):
    run_workload(workload, batch, monkeypatch, tc_recorder, after=after_step(workload))
