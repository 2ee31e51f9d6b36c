#!/usr/bin/env python
"""Time the LASSO channel-pruning learner's selection (`--learner channel`) layer by layer: sampling (pf_cp_sample and
the two models' forward passes), the design matrix's Gram (pf_cp_gram), the LARS-Lasso bisection on the host and the
refit (pf_cp_normal_eq + the float64 solve).  Synthetic data and seed-initialised weights; the selection runs once
after a warm-up selection of the first prunable layer.

    python tools/bench_cp.py --net resnet_at_ilsvrc12 --resnet_size 50 --batch_size 32 --json /tmp/cp_rn50.json
    python tools/bench_cp.py --net mobilenet_at_ilsvrc12 --batch_size 32
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def parse(argv=None):
    p = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    p.add_argument('--net', default='resnet_at_ilsvrc12')
    p.add_argument('--resnet_size', type=int, default=None)
    p.add_argument('--mobilenet_version', type=int, default=None)
    p.add_argument('--batch_size', type=int, default=32)
    p.add_argument('--cp_nb_batches', type=int, default=30)
    p.add_argument('--cp_nb_points_per_layer', type=int, default=10)
    p.add_argument('--cp_uniform_preserve_ratio', type=float, default=0.6)
    p.add_argument('--layers', type=int, default=0, help='time only the first N prunable layers (0: all)')
    p.add_argument('--json', default=None)
    return p.parse_args(argv)


def main(argv=None):
    args = parse(argv)
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError('bench_cp times the selection on the GPU: no CUDA device found')
    from pocketflow_b200.flags import FLAGS
    FLAGS.reset()
    importlib.import_module('pocketflow_b200.learners.channel_pruning.learner')
    importlib.reload(importlib.import_module('pocketflow_b200.datasets.ilsvrc12_dataset'))
    mod = importlib.reload(importlib.import_module('pocketflow_b200.nets.' + args.net))
    from pocketflow_b200.learners.learner_utils import create_learner
    from pocketflow_b200.learners.channel_pruning.learner import draw_positions
    FLAGS.learner, FLAGS.batch_size, FLAGS.cp_prune_option = 'channel', args.batch_size, 'uniform'
    FLAGS.cp_nb_batches, FLAGS.cp_nb_points_per_layer = args.cp_nb_batches, args.cp_nb_points_per_layer
    FLAGS.cp_uniform_preserve_ratio = args.cp_uniform_preserve_ratio
    FLAGS.save_path = os.path.join('/tmp', 'bench_cp_%d' % os.getpid(), 'model.ckpt')
    FLAGS.cp_channel_pruned_path = os.path.join('/tmp', 'bench_cp_%d' % os.getpid(), 'sel', 'model.ckpt')
    for k in ('resnet_size', 'mobilenet_version'):
        if getattr(args, k) is not None:
            setattr(FLAGS, k, getattr(args, k))
    if 'mobilenet' in args.net:
        FLAGS.nb_classes = 1001
    lrn = create_learner(None, mod.ModelHelper())
    lrn.init_from_full()
    rng = np.random.RandomState(lrn.seed)
    cached = lrn.cache_batches()
    shapes = [(op.output.shape[1], op.output.shape[2]) for op in lrn.sampled_prnd]
    positions = draw_positions(rng, len(cached), shapes, FLAGS.cp_nb_points_per_layer)
    lrn.positions = positions
    ex_f, ex_p = lrn.selection_executors()
    lrn.selection_log = []
    layers = [i for i in range(lrn.nb_layers) if lrn.prune_ratios[i] != 1]
    if args.layers:
        layers = layers[:args.layers]
    lrn.select_layer(layers[0], np.random.RandomState(0), cached, ex_f, ex_p)     # warm-up (modules, allocator)
    lrn.init_from_full()
    lrn.positions = positions
    lrn.selection_log = []
    for i in layers:
        lrn.select_layer(i, rng, cached, ex_f, ex_p)
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    rows = []
    print('GPU: %s' % gpu)
    print('%-55s %14s %8s %8s %8s %8s %8s' % ('layer', 'shape', 'kept', 'sample', 'gram', 'solve', 'refit'))
    for rec in lrn.selection_log:
        v = lrn.maskable_vars[rec['layer']]
        t = rec['times']
        rows.append(dict(layer=v.name, shape=list(v.shape), kept=int(rec['kept'].sum()), **t))
        print('%-55s %14s %8d %8.3f %8.3f %8.3f %8.3f' % (v.name[-55:], 'x'.join(map(str, v.shape)),
                                                          rows[-1]['kept'], t['sample'], t['gram'], t['solve'],
                                                          t['refit']))
    tot = {k: sum(r[k] for r in rows) for k in ('sample', 'gram', 'solve', 'refit')}
    print('total (s): ' + ', '.join('%s %.2f' % kv for kv in tot.items()))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(dict(gpu=gpu, args=vars(args), layers=rows, total=tot), f, indent=1)
    return 0


if __name__ == '__main__':
    sys.exit(main())
