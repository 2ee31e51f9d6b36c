"""Kernel launches of engine.Executor, recorded on the CPU (no kernel runs): every launch entry point of
libpf_b200.so is replaced by a recorder, the query entry points (shape support, workspace sizes, split counts) still
answer from the library.  `snapshot()` traces forward / backward / layer_wgrad of the benchmarked networks and of the
variants that reach the other conv lowerings (quantized operands, unfused residual adds, the paired-pixel stem weight
gradient, compact graphs); tests/test_launch_trace_cpu.py holds the executor to the trace this script wrote
(tests/golden/launches_v1.json), so a change to the executor that alters a launch, its arguments, their aliasing or
the launch order is caught.

Arguments are normalised: a pointer becomes the ordinal of its address's first appearance in the case's trace (NULL
is 0), a ConvDesc / TcAct / TcWt passed by reference becomes its name and fields, numbers stay as they are.

    python tests/golden/make_launch_trace.py        # rewrites tests/golden/launches_v1.json
    python tests/golden/make_launch_trace.py --gpu  # rewrites tests/golden/launches_gpu_v1.json (on an H100)
"""
import ctypes
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import make_plan_snapshot as SNAP  # noqa: E402

OUT = os.path.join(HERE, 'launches_v1.json')
OUT_GPU = os.path.join(HERE, 'launches_gpu_v1.json')

# entry points that launch nothing: answered by the library itself
QUERIES = {'pf_abi_version', 'pf_last_error', 'pf_conv2d_tc_supported', 'pf_conv2d_tc_weight_elems',
           'pf_conv2d_tc_wgrad_supported', 'pf_conv2d_tc_wgrad_workspace_bytes',
           'pf_conv2d_tc_wgrad_planes_workspace_bytes', 'pf_conv2d_tc_wgrad_splits', 'pf_conv2d_tc_tma_supported',
           'pf_conv2d_wgrad_workspace_bytes', 'pf_dwconv_wgrad_workspace_bytes'}


class Recorder:
    """Stands in for the loaded library: launch entry points append (name, normalised arguments) and return 0."""

    def __init__(self, real):
        self.real = real
        self.reset()

    def reset(self):
        self.launches, self.ptrs = [], {}

    def _ptr(self, v):
        return self.ptrs.setdefault(v, len(self.ptrs) + 1) if v else 0

    def _arg(self, a):
        if a is None:
            return 0
        if isinstance(a, ctypes.c_void_p):
            return self._ptr(a.value)
        if type(a).__name__ == 'CArgObject':            # ctypes.byref(struct)
            s = a._obj
            return [type(s).__name__] + [self._ptr(getattr(s, f)) if t is ctypes.c_void_p else getattr(s, f)
                                         for f, t in s._fields_]
        if isinstance(a, float):
            return a
        return int(a)

    def __getattr__(self, name):
        if name in QUERIES:
            return getattr(self.real, name)
        if not name.startswith('pf_'):
            raise AttributeError(name)

        def launch(*args):
            self.launches.append([name] + [self._arg(a) for a in args])
            return 0
        return launch


def install(mp, streams=False):
    """Route every library call through a Recorder (mp: a pytest MonkeyPatch).  Returns the recorder.
    streams: launches keep the current stream's handle (the default stream is NULL, other streams get pointer
    ordinals), so stream placement is part of the trace."""
    from pocketflow_b200 import lib, ops
    rec = Recorder(lib.load())
    mp.setattr(lib, '_lib', rec)
    mp.setattr(lib, 'load', lambda: rec)
    if not streams:
        mp.setattr(ops, '_stream', lambda: None)
    mp.setattr(ops, '_check_f32', lambda *ts: None)
    return rec


MOBILENET_V2 = ('mobilenet_at_ilsvrc12', dict(batch_size=64, mobilenet_version=2))


def uq8(g):
    """8-bit per-channel weights and 8-bit activations, marked as the uniform quantization learner marks them"""
    from pocketflow_b200.learners.uniform_quantization.utils import UniformQuantization
    uq = UniformQuantization(g, 256, True, 'channel')
    uq.insert_quant_op_for_weights({op.name: 8 for op in uq.search_matmul_op(False)})
    uq.insert_quant_op_for_activations({op.name: 8 for op in uq.search_activation_op()})
    return dict(weight_quant=uq.weight_quant_spec(), act_quant=uq.act_quant_spec())


def compact_executor(net, device='cpu'):
    """the compact inference executor of a fake-pruned network (as tests/test_chn_compact_cpu.py builds it)"""
    import numpy as np
    import torch

    import make_golden_chn_export as X
    from pocketflow_b200 import compact as C
    from pocketflow_b200.engine import Executor
    g, im, lg = X.eval_graph(net)
    rng = np.random.default_rng(0)
    st = {v.name: v.initializer(rng, v.shape) for op in C.reachable_ops(g, lg) for v in op.vars.values()}
    st = C.fake_prune(g, lg, st, 0.5, 1)
    cg, ci, cl = C.build_graph(g, im, lg, C.plan(g, lg, st))
    return Executor(cg, ci, cl, torch.device(device), train=False)


def trace_step(rec, ex):
    rec.reset()
    ex.forward()
    if ex.train:
        ex.loss_and_backward()
    return rec.launches


def trace_eval(rec, ex):
    """the evaluation pass of a training executor: BN in inference mode, quantizers active"""
    rec.reset()
    ex.forward(training=False)
    return rec.launches


def trace_layer_wgrad(rec, ex):
    import torch
    convs = [op for op in ex.ops if op.type in ('Conv2D', 'MatMul')]
    gys = [torch.empty(op.output.shape, device=ex.device) for op in convs]
    dws = [torch.empty(op.vars['kernel'].shape, device=ex.device) for op in convs]
    rec.reset()
    ex.forward()
    for op, gy, dw in zip(convs, gys, dws):
        ex.layer_wgrad(op, gy, dw)
    return rec.launches


def snapshot():
    import pytest
    out = {}
    with pytest.MonkeyPatch.context() as mp:
        rec = install(mp)
        for key, (net, flags, teacher) in SNAP.CASES.items():
            out[key] = trace_step(rec, SNAP.build(net, flags))
            if teacher:
                out[key + '_teacher'] = trace_step(rec, SNAP.build(net, flags, train=False))
        ex = SNAP.build(*SNAP.CASES['resnet20_b256'][:2], edit=uq8)
        out['resnet20_uq8_b256'] = trace_step(rec, ex)
        out['resnet20_uq8_b256_eval'] = trace_eval(rec, ex)
        out['resnet50_uq8_b128'] = trace_step(rec, SNAP.build(*SNAP.CASES['resnet50_b128'][:2], edit=uq8))
        out['resnet20_b256_unfused_add'] = trace_step(rec, SNAP.build(*SNAP.CASES['resnet20_b256'][:2], fuse_add=False))
        ex = SNAP.build(*MOBILENET_V2)
        out['mobilenet_v2_b64'] = trace_step(rec, ex)
        out['mobilenet_v2_b64_eval'] = trace_eval(rec, ex)
        out['mobilenet_v2_b64_inference'] = trace_step(rec, SNAP.build(*MOBILENET_V2, train=False))
        out['lenet_uq8_b128'] = trace_step(rec, SNAP.build(*SNAP.CASES['lenet_b128'][:2], edit=uq8))
        with mp.context() as env:
            env.setenv('PF_STEM_S2D', '0')
            out['mobilenet_v1_b256_no_s2d'] = trace_step(rec, SNAP.build(*SNAP.CASES['mobilenet_v1_b256'][:2]))
        for key in ('resnet20_b256', 'mobilenet_v1_b256', 'lenet_b128'):
            out[key + '_layer_wgrad'] = trace_layer_wgrad(rec, SNAP.build(*SNAP.CASES[key][:2]))
        for net in ('resnet20', 'resnet50', 'mobilenet_v1'):
            out[net + '_compact_b2'] = trace_step(rec, compact_executor(net))
    return out


def snapshot_gpu():
    """The forms only an executor planned on a CUDA device takes (integer-level operands, the side-stream weight
    gradient, batch norms folded into the conv epilogue), traced on cuda:0 with stream placement.  Nothing is
    launched; executors are freed one by one to bound device memory.  Returns {'sm_count': .., 'cases': {..}}: the
    split-K partition of a weight gradient follows the device's SM count."""
    import gc

    import pytest
    import torch
    out = {}

    def done():
        gc.collect()
        torch.cuda.empty_cache()
    with pytest.MonkeyPatch.context() as mp:
        rec = install(mp, streams=True)
        for key in ('resnet50_b128', 'resnet20_b256'):
            net, flags, _ = SNAP.CASES[key]
            uq = key.replace('_b', '_uq8_b')
            ex = SNAP.build(net, flags, edit=uq8, device='cuda:0')
            out[uq] = trace_step(rec, ex)
            out[uq + '_eval'] = trace_eval(rec, ex)
            if key == 'resnet20_b256':
                out[uq + '_layer_wgrad'] = trace_layer_wgrad(rec, ex)
            del ex
            done()
            out[key + '_teacher'] = trace_step(rec, SNAP.build(net, flags, train=False, device='cuda:0'))
            done()
        for net in ('resnet50', 'mobilenet_v1'):
            out[net + '_compact_b2'] = trace_step(rec, compact_executor(net, 'cuda:0'))
            done()
        out['mobilenet_v2_b64_inference'] = trace_step(rec, SNAP.build(*MOBILENET_V2, train=False, device='cuda:0'))
        done()
    return dict(sm_count=torch.cuda.get_device_properties(0).multi_processor_count, cases=out)


def dumps_gpu(snap):
    return '{"sm_count": %d,\n"cases": %s}\n' % (snap['sm_count'], dumps(snap['cases']).rstrip('\n'))


def dumps(trace):
    """one launch per line"""
    cases = ['%s: [\n%s\n]' % (json.dumps(k), ',\n'.join(json.dumps(l, separators=(',', ':')) for l in v))
             for k, v in sorted(trace.items())]
    return '{\n' + ',\n'.join(cases) + '\n}\n'


if __name__ == '__main__':
    if '--gpu' in sys.argv:       # needs cuda:0; the fixture is only valid for devices with its SM count
        with open(OUT_GPU, 'w') as f:
            f.write(dumps_gpu(snapshot_gpu()))
        print('wrote', OUT_GPU)
    else:
        with open(OUT, 'w') as f:
            f.write(dumps(snapshot()))
        print('wrote', OUT)
