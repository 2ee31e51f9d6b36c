"""The layers between the tensor-core convolutions, in one training step of the benchmarked workloads at the
benchmarked batch, against float64 or bit for bit.

The harness is test_tc_bench_layers_gpu.run_workload: the learner is built at the batch bench.py measures, under
PF_POISON=1, and one eager step runs with entry points of `ops` wrapped.  Each call passes through unchanged; then
  * its output must be finite;
  * the first call of each (entry point, geometry, form, flags) is compared on exactly the operands it was given, with
    "prior" outputs (accumulate targets, moving statistics, range slots) cloned before the call:
      - batch-norm statistics: mean within 1e-6 of |mean| + std, var 1e-5 relative, rstd within one ulp of
        fp32(1 / sqrt(fl(var + eps))), moving statistics 1e-6 of float64 from the prior (the mean at the scale
        |prior| momentum + (|mean| + std)(1 - momentum), and bit-exact as the fp32 chain of the batch mean), the range
        slot bit-exact;
      - BN apply, fake-quant, planes, levels and range slots: bit-exact against the fp32 op chain
        ((x - mean) * rstd) * gamma + beta and the quantizer's op chain (test_nn_variants_gpu);
      - BN backward: mask from that fp32 chain, dgamma / dbeta within 1e-6 of the sum of |terms| per channel, dx 1e-5
        of max|ref| on the fed fp32 statistics, planes == split(fp32 dx);
      - depthwise fwd / dgrad 1e-5 of max|ref|; wgrad against max|ref|, the sum of |terms| and an fp32 reference;
      - max-pool: y and argmax (first maximum) bit-exact, dx 1e-6; the rest float64 at 1e-5 or bit-exact.
The weight-sparse and codebook workloads also run what their learners do besides the step (run_workload's `after`):
      - mask rebuild: masks, weights (as uint32: -0.0 counts), backups and thresholds bit-exact against
        oracle.ws_build_mask at the ratios passed in;
      - codebook forward: quantized weights (and kept indices, ties to the first centroid) bit-exact against
        oracle.nonuniform_quantize with the device codebook; quantile init: every codebook bit-exact against
        oracle.nuq_quantile_init of the normalised tensor, entries past 2^bits zero; order statistics (pf_select_desc)
        bit-exact against a sort; codebook gradient within 1e-6 of each centroid's sum of |terms| of float64
        oracle.nuq_grads, and the same bits on a second call.
      Each of them must cover every tensor its object holds.
Every public callable of `ops` is wrapped: the test fails when the step calls one that is neither a tensor-core entry
point (test_tc_bench_layers_gpu), nor checked here, nor in EXEMPT with its reason."""

import pytest
import torch

from pocketflow_b200 import ops
from support import RUNS, NnRecorder, after_step, run_workload

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')



def expected_checks(workload, lrn):
    """the checks the learner's plan calls for: {tag: tensors each run must cover, or None where the tag only has to
    appear} — the weight-sparse mask rebuild over every maskable variable, the codebook checks over every quantized
    kernel, and the producer of each first layer that computes its own operand (the stem's folded weight gradient
    included)"""
    import bench
    ex = lrn.sess_train
    want = {}
    if bench.WORKLOADS[workload][2] == 'weight-sparse':
        want['mask rebuild'] = len(ex.maskable)
    if isinstance(ex.wq, ops.CodebookWeightQuantizer):
        for tag in ('codebook forward', 'codebook quantile values', 'codebook quantile init'):
            want[tag] = len(ex.wq_ops)
        if ex.train_clusters:
            want['codebook gradient'] = len(ex.wq_ops)
    for e in (ex, ex.teacher):
        for im in (e.im2col.values() if e is not None else ()):
            if im['compute']:
                want['s2d_planes' if im['mode'] == 's2d' else ('im2col_planes' if im['planes'] else 'im2col')] = None
            if e.train and 'pair' in im:
                want['fold_diag_blocks / sum|terms|'] = None
    return want


@pytest.mark.parametrize('workload,batch,flags', [
    pytest.param(w, b, f, id='%s-%d' % (w, b) + ''.join('-%s' % v for _, v in sorted((f or {}).items())))
    for w, b, f in RUNS])
def test_bench_layers_besides_the_tc_convs(workload, batch, flags, monkeypatch):
    run_workload(workload, batch, monkeypatch, lambda mp, lrn: NnRecorder(mp, expected_checks(workload, lrn)),
                 flags=flags, after=after_step(workload))
