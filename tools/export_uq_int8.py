#!/usr/bin/env python
"""Export a uniformly quantized model as an integer model, and time it against the fake-quantized model.

The latest checkpoint of a `--learner uniform` run (npz or TF bundle) is turned into an integer model
(pocketflow_b200/int8.py): u8 weight levels with their per-layer or per-channel alpha / beta for every convolution that
runs on the u8 x u8 tensor cores, every other variable (batch-norm constants included) in fp32, plus a sidecar JSON of
the quantizer settings and the layer selection.  Each layer is reported with the path it runs on, and why.  Then the
inference forward of both models is timed as CUDA-graph replays at --batch_size_eval, alternating in one process.

    python tools/export_uq_int8.py --net resnet_at_ilsvrc12 --resnet_size 50 --ckpt_dir ./uql_quant_models \\
        --uql_weight_bits 8 --uql_activation_bits 8 --uql_use_buckets --batch_size_eval 128 --out ./rn50_int8/model

Without --ckpt_dir the model keeps its seed initialisation (for speed measurements only).

With --int8_calibrate N the fake-quantized model is run over N fresh batches of the net's training set (--data_dir_local:
real data, with the training augmentation, so that the ranges are not fitted to the evaluation images; otherwise the
learners' synthetic batches) and the exported model carries static activation ranges (int8.calibrate,
--int8_calib_stat mean | max): its logits no longer depend on the rest of the batch.  The tool prints every range and
also times the integer model with per-batch ranges ('integer') against the calibrated one ('integer_calibrated').
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
sys.path.insert(0, os.path.join(ROOT, 'tools'))


def parse(argv=None):
    p = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    p.add_argument('--net', default='resnet_at_ilsvrc12', help='pocketflow_b200.nets module with a ModelHelper')
    p.add_argument('--resnet_size', type=int, default=None)
    p.add_argument('--mobilenet_version', type=int, default=None)
    p.add_argument('--ckpt_dir', default=None, help='directory of the uniform learner\'s checkpoint (default: seed init)')
    p.add_argument('--out', default='./models_uq_int8/model', help='integer checkpoint path prefix')
    p.add_argument('--uql_weight_bits', type=int, default=8)
    p.add_argument('--uql_activation_bits', type=int, default=8)
    p.add_argument('--uql_use_buckets', action='store_true')
    p.add_argument('--uql_bucket_type', default='channel', choices=('channel', 'split'))
    p.add_argument('--uql_bucket_size', type=int, default=256)
    p.add_argument('--uql_quantize_all_layers', action='store_true')
    p.add_argument('--int8_depthwise', action='store_true',
                   help='depthwise layers on u8 levels too (pf_dwconv_u8_fwd); also times the integer model without them')
    p.add_argument('--int8_narrow', action='store_true',
                   help='channel counts that are multiples of 16 too (the cp.async-fed u8 kernel, any C %% 16 level '
                        'producer); also times the integer model without them')
    p.add_argument('--int8_calibrate', type=int, default=0, metavar='N',
                   help='calibrate static activation ranges on N batches and export the calibrated model')
    p.add_argument('--int8_calib_stat', default='mean', choices=('mean', 'max'),
                   help='mean: the mean of the per-batch min / max; max: their extremes')
    p.add_argument('--batch_size_calib', type=int, default=None, help='calibration batch size (default: batch_size_eval)')
    p.add_argument('--data_dir_local', default=None,
                   help='the net\'s dataset on disk; calibration reads its training split with the training augmentation '
                        '(default: synthetic batches)')
    p.add_argument('--batch_size_eval', type=int, default=100)
    p.add_argument('--nb_repts_warmup', type=int, default=20, help='graph replays before timing')
    p.add_argument('--nb_repts', type=int, default=50, help='graph replays per timed window')
    p.add_argument('--nb_rounds', type=int, default=5, help='alternating (fake-quant, integer[, ...]) timed windows')
    p.add_argument('--no_time', action='store_true', help='export only')
    p.add_argument('--json', default=None, help='write the measurements here')
    return p.parse_args(argv)


def setup(args):
    """(graph, images, logits, quantizer config) of the net's inference graph at --batch_size_eval"""
    from pocketflow_b200 import compact, int8
    from pocketflow_b200.flags import FLAGS
    net = importlib.import_module('pocketflow_b200.nets.' + args.net)           # defines the net's flags
    import pocketflow_b200.learners.uniform_quantization.learner  # noqa: F401  (the --uql_* flags)
    FLAGS.reset()
    if args.resnet_size is not None:
        FLAGS.resnet_size = args.resnet_size
    if args.mobilenet_version is not None:
        FLAGS.mobilenet_version = args.mobilenet_version
    FLAGS.batch_size_eval = args.batch_size_eval
    for k in ('uql_weight_bits', 'uql_activation_bits', 'uql_use_buckets', 'uql_bucket_type', 'uql_bucket_size',
              'uql_quantize_all_layers'):
        setattr(FLAGS, k, getattr(args, k))
    graph, images, logits = compact.build_eval_graph(net.ModelHelper(), args.batch_size_eval)
    cfg = int8.config_from_flags()
    for opt in ('int8_depthwise', 'int8_narrow'):
        if getattr(args, opt, False):
            cfg[opt] = True
    return graph, images, logits, cfg


def load_state(args, graph, logits):
    from pocketflow_b200 import compact
    from pocketflow_b200.learners.abstract_learner import latest_checkpoint, load_checkpoint
    if args.ckpt_dir:
        fn = latest_checkpoint(args.ckpt_dir) if os.path.isdir(args.ckpt_dir) else None
        if fn is None:
            raise ValueError('no checkpoint found in ' + args.ckpt_dir)
        print('quantized model restored from ' + fn)
        return load_checkpoint(fn)
    rng = np.random.default_rng(1)
    return {v.name: v.initializer(rng, v.shape) for op in compact.reachable_ops(graph, logits) for v in op.vars.values()}


def calibration_batches(helper, n, bs):
    """n image batches [bs, ...] of the net's training set, each drawn when it is consumed, from the dataset's own source
    (the generator behind its iterator): the iterator hands out rotating pinned buffers, rewritten after POOL_SIZE draws
    (real data) or cycled (synthetic), so its batches must not be held; these are n distinct batches."""
    import torch
    it = helper.DATASET(is_train=True).build()
    for _ in range(n):
        yield torch.from_numpy(np.ascontiguousarray(it.generator(bs)[0]))


def calibration_ranges(args, cfg, state):
    """int8.calibrate over --int8_calibrate batches of the net's training set at --batch_size_calib"""
    from pocketflow_b200 import compact, int8
    from pocketflow_b200.flags import FLAGS
    net = importlib.import_module('pocketflow_b200.nets.' + args.net)
    bs = args.batch_size_calib or args.batch_size_eval
    FLAGS.batch_size = bs
    if args.data_dir_local:
        FLAGS.data_dir_local = args.data_dir_local
    helper = net.ModelHelper()
    graph, images, logits = compact.build_eval_graph(helper, bs)
    return int8.calibrate(graph, images, logits, state, cfg, calibration_batches(helper, args.int8_calibrate, bs),
                          args.int8_calib_stat)


def gpu_name(torch):
    try:
        return subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                                        '--format=csv,noheader'], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name(0)


def main(argv=None):
    args = parse(argv)
    import torch
    from export_chn_pruned import _capture, _replay_ms
    from pocketflow_b200 import compact, int8
    graph, images, logits, cfg = setup(args)
    state = load_state(args, graph, logits)
    for line in int8.report_lines(int8.select(graph, logits, cfg)):
        print(line)
    if not torch.cuda.is_available():
        raise RuntimeError('the integer model runs on the GPU: no CUDA device found')
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    im = int8.IntModel.from_checkpoint(graph, images, logits, state, cfg, dev)
    ranges, imc = None, None
    if args.int8_calibrate:
        ranges = calibration_ranges(args, cfg, state)
        print('calibrated activation ranges (%s of %d batches):' % (args.int8_calib_stat, args.int8_calibrate))
        for name, (lo, hi) in ranges.items():
            print('  %s: [%.9g, %.9g]' % (name, lo, hi))
        imc = int8.IntModel.from_checkpoint(graph, images, logits, state, cfg, dev, act_ranges=ranges)
        for line in int8.report_lines(imc.sel):
            print('calibrated ' + line)
    out = imc or im
    print('integer model written to ' + out.export(args.out) + ' (+ %s.int8.json)' % args.out)
    if args.no_time:
        return 0
    fq = int8.fake_quant_executor(graph, images, logits, compact.map_state(graph, compact.reachable_ops(graph, logits),
                                                                           state), cfg, dev)
    x = torch.randn(images.shape, generator=torch.Generator().manual_seed(0)).to(dev)
    fq.buf[images].copy_(x)
    im.ex.buf[images].copy_(x)
    arms = {'fake_quant': fq}
    for opt, arm in (('int8_narrow', 'integer_no_narrow'), ('int8_depthwise', 'integer_no_depthwise')):
        if cfg.get(opt):                      # the same integer model without the option's layers
            im_without = int8.IntModel.from_checkpoint(graph, images, logits, state,
                                                       {k: v for k, v in cfg.items() if k != opt}, dev)
            im_without.ex.buf[images].copy_(x)
            arms[arm] = im_without.ex
    arms['integer'] = im.ex
    if imc is not None:
        imc.ex.buf[images].copy_(x)
        arms['integer_calibrated'] = imc.ex
    graphs = {arm: _capture(lambda ex=ex: ex.forward(training=False), torch) for arm, ex in arms.items()}
    for gr in graphs.values():
        gr.replay()
    torch.cuda.synchronize()
    lf, li = fq.T(fq.logits_t).float(), im.ex.T(im.logits).float()
    diff = float((lf - li).abs().max() / lf.abs().max().clamp_min(1e-30))
    agree = float((lf.argmax(1) == li.argmax(1)).float().mean())
    for _ in range(args.nb_repts_warmup):
        for gr in graphs.values():
            gr.replay()
    ms = {arm: [] for arm in graphs}
    for _ in range(args.nb_rounds):
        for arm, gr in graphs.items():
            ms[arm].append(_replay_ms(gr, args.nb_repts, torch))
    bs = args.batch_size_eval
    res = dict(net=args.net, resnet_size=args.resnet_size, batch=bs, config=cfg,
               int_layers=sum(1 for _, w in im.sel if w is None), layers=len(im.sel), logits_max_rel_diff=diff,
               top1_agreement=agree, calibrated=bool(imc))
    for arm, v in ms.items():
        ips = sorted(bs / (t / 1e3) for t in v)
        res[arm] = dict(ms_per_batch=sorted(v), images_per_s_min=ips[0], images_per_s_median=float(np.median(ips)),
                        images_per_s_max=ips[-1])
        print('%-20s inference forward: %.3f ms / batch of %d | images/s min %.0f median %.0f max %.0f'
              % (arm, float(np.median(v)), bs, ips[0], float(np.median(ips)), ips[-1]))
    print('logits: max |fake-quant - integer| / max |fake-quant| = %.3e, top-1 agreement %.4f' % (diff, agree))
    res['gpu'] = gpu_name(torch)
    print('gpu: ' + res['gpu'])
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as f:
            json.dump(res, f, indent=1)
    return 0


if __name__ == '__main__':
    sys.exit(main())
