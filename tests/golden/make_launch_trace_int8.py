"""Kernel launches of int8.IntModel, recorded with make_launch_trace's recorder (no kernel runs): what building the
integer model launches and what its forward() launches, for ResNet-20 with `int8_narrow`, ResNet-50, MobileNet-v1 with
`int8_depthwise` and MobileNet-v2 with both, at batch 8.  The u8 shape queries answer from the library as well.  A
split-bf16 weight preparation (pf_conv2d_tc_prep_weight) is not traced but noted by the layer whose copy it wrote
(`owners`), so that which layers own such copies is checked apart from the rest of the trace.
tests/test_int8_plan_cpu.py holds IntModel to the CPU trace (tests/golden/launches_int8_v1.json),
tests/test_int8_plan_gpu.py to the trace on cuda:0 (tests/golden/launches_int8_gpu_v1.json), where the inference
batch norms folded into the u8 convolution's epilogue are planned too.

    python tests/golden/make_launch_trace_int8.py        # rewrites tests/golden/launches_int8_v1.json
    python tests/golden/make_launch_trace_int8.py --gpu  # rewrites tests/golden/launches_int8_gpu_v1.json (on a GPU)
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import make_launch_trace as T  # noqa: E402

OUT = os.path.join(HERE, 'launches_int8_v1.json')
OUT_GPU = os.path.join(HERE, 'launches_int8_gpu_v1.json')

U8_QUERIES = {'pf_conv2d_u8_supported', 'pf_conv2d_u8_narrow_supported', 'pf_dwconv_u8_supported'}
BATCH = 8

# case: (net module, flags, int8 options)
CASES = {
    'resnet20_narrow': ('resnet_at_cifar10', dict(resnet_size=20), dict(int8_narrow=True)),
    'resnet50': ('resnet_at_ilsvrc12', dict(resnet_size=50), {}),
    'mobilenet_v1_depthwise': ('mobilenet_at_ilsvrc12', {}, dict(int8_depthwise=True)),
    'mobilenet_v2_depthwise_narrow': ('mobilenet_at_ilsvrc12', dict(mobilenet_version=2),
                                      dict(int8_depthwise=True, int8_narrow=True)),
}


class Recorder(T.Recorder):
    """make_launch_trace's recorder; a weight preparation is noted by the raw address of its forward hi plane"""

    def reset(self):
        super().reset()
        self.prep = []

    def __getattr__(self, name):
        if name == 'pf_conv2d_tc_prep_weight':
            return lambda d, w, f_hi, *rest: self.prep.append(f_hi.value) or 0
        return super().__getattr__(name)


def install(mp, streams=False):
    mp.setattr(T, 'Recorder', Recorder)
    mp.setattr(T, 'QUERIES', T.QUERIES | U8_QUERIES)
    return T.install(mp, streams)


def model(key, device, batch=BATCH):
    """the case's integer model (IntModel.from_checkpoint) from seed-initialised weights, 8-bit per-channel weights and
    8-bit activations"""
    import importlib

    import numpy as np
    import torch

    from pocketflow_b200 import compact, int8
    from pocketflow_b200.flags import FLAGS
    net, flags, opts = CASES[key]
    mod = importlib.import_module('pocketflow_b200.nets.' + net)
    import pocketflow_b200.learners.uniform_quantization.learner  # noqa: F401  (defines the --uql_* flags)
    FLAGS.reset()
    for k, v in flags.items():
        setattr(FLAGS, k, v)
    FLAGS.uql_weight_bits, FLAGS.uql_activation_bits = 8, 8
    FLAGS.uql_use_buckets, FLAGS.uql_bucket_type = True, 'channel'
    g, images, logits = compact.build_eval_graph(mod.ModelHelper(), batch)
    rng = np.random.default_rng(0)
    state = {v.name: v.initializer(rng, v.shape) for op in compact.reachable_ops(g, logits) for v in op.vars.values()}
    return int8.IntModel.from_checkpoint(g, images, logits, state, dict(int8.config_from_flags(), **opts),
                                         torch.device(device))


def prep_names(im, addrs):
    """the layer names of the weight copies at `addrs` (raw addresses of split-bf16 forward hi planes)"""
    ex = im.ex
    owner = {tw.f_hi.data_ptr(): op.name for op, tw in ex.tc.items()}
    owner.update({im_['tw'].f_hi.data_ptr(): op.name for op, im_ in ex.im2col.items()})
    return [owner.get(a, '?') for a in addrs]


def trace(rec, key, device):
    """({'build': launches, 'forward': launches}, the layers whose weight copies the build prepared, the model)"""
    rec.reset()
    im = model(key, device)
    out, prep = dict(build=rec.launches), prep_names(im, rec.prep)
    rec.reset()
    im.forward()
    out['forward'] = rec.launches
    return out, prep, im


def owners(im, prep):
    """which layers are integer, which batch norms only integer layers read (through their ReLU), which layers own
    split-bf16 weight copies, which were prepared and which producers own operand planes"""
    ex = im.ex
    ints = sorted(n for n, why in im.sel if why is None)
    only_int = []
    for op in ex.ops:
        if op.type == 'FusedBatchNorm':
            relu = op.output.consumers
            if len(relu) == 1 and relu[0].type in ('Relu', 'Relu6') and relu[0].output.consumers \
                    and all(c.name in ints for c in relu[0].output.consumers):
                only_int.append(op.name)
    return dict(ints=ints, only_int=sorted(only_int), tc=sorted(op.name for op in ex.tc), prep=prep,
                stem=sorted(op.name for op in ex.im2col), planes=sorted(op.name for op in ex.xplanes))


def snapshot(device='cpu'):
    """({case/part: ...}, {case: owners}) of every case; on a CUDA device with stream placement, models freed one by
    one"""
    import gc

    import pytest
    import torch
    out, own = {}, {}
    with pytest.MonkeyPatch.context() as mp:
        rec = install(mp, streams=device != 'cpu')
        for key in CASES:
            got, prep, im = trace(rec, key, device)
            out.update({key + '/' + part: v for part, v in got.items()})
            own[key] = owners(im, prep)
            del im
            gc.collect()
            if device != 'cpu':
                torch.cuda.empty_cache()
    return out, own


if __name__ == '__main__':
    gpu = '--gpu' in sys.argv
    with open(OUT_GPU if gpu else OUT, 'w') as f:
        f.write(T.dumps(snapshot('cuda:0' if gpu else 'cpu')[0]))
    print('wrote', OUT_GPU if gpu else OUT)
