"""Writes cp_fathers_v1.json: for every Conv2D of ResNet-20, ResNet-50, MobileNet-v1 and MobileNet-v2, in `thisconvs`
order, the producer conv (is_W1_prunable's father), the conv whose output channels prune_W1 zeroes (through depthwise
producers), and the Add of get_Add_if_is_last_in_resblock.

Provenance: the file is written by the package's own restatement of the reference's model_wrapper rules
(learners/channel_pruning/learner.py: producer_conv, w1_target, add_after), not by the reference, which needs
TensorFlow.  It pins those rules against regressions.  Its agreement with the reference rests on the hand-derived
counts that tests/test_cp_cpu.py checks from the block structure: on ResNet v2 the second conv of every basic block,
every bottleneck's last 1x1 and stride-1 3x3, and the first block's stem-fed convs (strided convs sit behind the
reference's tf.pad); every MobileNet-v1 pointwise conv through its depthwise conv.

    python tests/golden/make_cp_fathers.py"""
import importlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

NETS = {'resnet20': ('resnet_at_cifar10', dict(resnet_size=20)),
        'resnet50': ('resnet_at_ilsvrc12', dict(resnet_size=50)),
        'mobilenet_v1': ('mobilenet_at_ilsvrc12', dict(nb_classes=1001, mobilenet_version=1)),
        'mobilenet_v2': ('mobilenet_at_ilsvrc12', dict(nb_classes=1001, mobilenet_version=2))}


def rules(key):
    from pocketflow_b200 import graph as G
    from pocketflow_b200.flags import FLAGS
    from pocketflow_b200.learners.channel_pruning import learner as L
    module, flags = NETS[key]
    FLAGS.reset()
    importlib.reload(importlib.import_module('pocketflow_b200.datasets.ilsvrc12_dataset'))
    mod = importlib.reload(importlib.import_module('pocketflow_b200.nets.' + module))
    for k, v in flags.items():
        setattr(FLAGS, k, v)
    FLAGS.batch_size = 2
    helper = mod.ModelHelper()
    g = G.Graph()
    with g.as_default():
        images, _ = helper.build_dataset_train().get_next()
        helper.forward_train(images)
    name = lambda op: op.name if op is not None else None
    return [[op.name, name(L.producer_conv(op)), name(L.w1_target(op)), name(L.add_after(op))]
            for op in g.ops if op.type == 'Conv2D']


if __name__ == '__main__':
    out = {key: rules(key) for key in NETS}
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'cp_fathers_v1.json'), 'w') as f:
        json.dump(out, f, indent=1)
