"""Launch plans of the networks the benchmark runs, as the planner of engine.Executor lays them out on the CPU
(no kernel runs).  `plan_record` names, per op, the kernel family it lowers to and the operand forms it reads and
writes; tests/test_mbv2_cpu.py holds the planner to the snapshot this script wrote (tests/golden/plans_v1.json), so
a planner change that alters an existing network's launches is caught.

    python tests/golden/make_plan_snapshot.py        # rewrites tests/golden/plans_v1.json
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

OUT = os.path.join(ROOT, 'tests', 'golden', 'plans_v1.json')

# (net module, flags) of every bench.py workload's network at the workload's batch; the distillation teacher (an
# inference executor) is planned as well where the workload enables distillation
CASES = {
    'resnet50_b128': ('resnet_at_ilsvrc12', dict(resnet_size=50, batch_size=128), True),
    'resnet20_b256': ('resnet_at_cifar10', dict(resnet_size=20, batch_size=256), True),
    'mobilenet_v1_b256': ('mobilenet_at_ilsvrc12', dict(batch_size=256), False),
    'lenet_b128': ('lenet_at_cifar10', dict(batch_size=128), False),
}


def build(net, flags, train=True, edit=None, device='cpu', **kw):
    """edit(graph) -> extra Executor arguments (quantization specs); kw: further Executor arguments"""
    import importlib

    import torch

    from pocketflow_b200 import graph as G
    from pocketflow_b200.engine import Executor
    from pocketflow_b200.flags import FLAGS
    FLAGS.reset()
    mod = importlib.import_module('pocketflow_b200.nets.' + net)
    for k, v in flags.items():
        setattr(FLAGS, k, v)
    mh = mod.ModelHelper()
    g = G.Graph()
    with g.as_default():
        with G.variable_scope('data'):
            im, lab = mh.build_dataset_train().get_next()
        with G.variable_scope('model'):
            out = mh.forward_train(im) if train else mh.forward_eval(im)
            tv = [v for v in g.variables.values() if v.name.startswith('model/') and v.trainable]
            loss, _ = mh.calc_loss(lab, out, tv)
    if edit is not None:
        kw.update(edit(g))
    if not train:
        return Executor(g, im, out, torch.device(device), train=False, **kw)
    return Executor(g, im, out, torch.device(device), train=True, loss=loss, labels=lab,
                    optimizer=dict(kind='momentum', momentum=0.9), **kw)


def plan_record(ex):
    """{op name: [op type, {decision: value}]} for every op the executor runs."""
    def name(t):
        return t.name if t is not None else None

    rec = {}
    for op in ex.ops:
        d = {}
        t = op.output
        d['buf'] = t in ex.buf
        d['alias'] = name(ex.alias.get(t))
        if op in ex.fused_act:
            d['act'] = ex.fused_act[op]
        if op in ex.fused_into:
            d['fused_into'] = ex.fused_into[op].name
        if op.type in ('Conv2D', 'MatMul'):
            d['tc'] = op in ex.tc
            d['tc_wgrad'] = op in ex.tc_wgrad
            if op in ex.im2col:
                im = ex.im2col[op]
                d['im2col'] = [im['mode'], bool(im['planes']), int(im['kpad']), 'pair' in im]
            d['x_planes'] = ex.planes_of(op.inputs[0]) is not None
            if op in ex.fused_add:
                d['fused_add'] = [ex.fused_add[op][0].name, ex.fused_add[op][1].name]
            if ex.train:
                d['dy_planes'] = op in ex.conv_dy_planes
                d['wg_part'] = op in ex.wg_part
        if op.type == 'FusedBatchNorm':
            d['planes'] = op in ex.xplanes
            d['need_f32'] = bool(ex.bn_need_f32.get(op, True))
            d['act_lv'] = op in ex.act_lv
            if ex.train:
                d['gplanes'] = op in ex.bn_gplanes
                d['gplanes_only'] = bool(ex.bn_gplanes_only.get(op, False))
        if op.type == 'Add':
            d['fused'] = op in ex.add_fused
        if ex.train and op.type != 'Placeholder':
            d['grad'] = name(ex.gkey(t))
        rec[op.name] = [op.type, d]
    return rec


def snapshot():
    out = {}
    for key, (net, flags, teacher) in CASES.items():
        out[key] = plan_record(build(net, flags))
        if teacher:
            out[key + '_teacher'] = plan_record(build(net, flags, train=False))
    return out


if __name__ == '__main__':
    with open(OUT, 'w') as f:
        json.dump(snapshot(), f, indent=0, sort_keys=True)
        f.write('\n')
    print('wrote', OUT)
