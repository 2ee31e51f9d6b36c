#!/usr/bin/env python
"""Time the fine-tune step of a channel-pruned model at its pruned width against the masked full-width step.

One process builds the `chn-pruned-gpu` learner of one net on synthetic data, zeroes int(cin * ratio) random input
channels of every conv (compact.fake_prune, the reference export tool's --enbl_fake_prune; no trained model needed), sets
the learner's masks from the result, and builds the compact step from that state (compact.CompactTrainer, what
--enbl_compact_ft runs).  Both steps are captured into CUDA graphs and replayed in alternating windows on the same batch.

    python tools/bench_compact_ft.py --net mobilenet_at_ilsvrc12 --enbl_fake_prune --fake_prune_ratio 0.5 --batch_size 256
    python tools/bench_compact_ft.py --net resnet_at_ilsvrc12 --resnet_size 50 --enbl_fake_prune --batch_size 128

Reported: images/s min / median / max over the windows, peak device memory while each step was built and run, the bytes
of the flat gradient buffer (what a data-parallel step all-reduces), and for every standalone channel scatter and every
BN apply with a fused gather its time and GB/s from the algorithmic bytes — scatter: 4 B read per compact element + 4 B
written per full-width element (+ 4 B read per full-width element when accumulating, + 4 B of hi + lo planes where the
step emits them); BN + gather: 4 B read per kept
element + 4 B (fp32) and / or 4 B (hi + lo planes) written per compact element.  Each of those kernels is timed alone
with an L2-sized buffer overwritten between launches.  The card's name, power limit and SM clock are read (never set)
and printed."""
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
    p.add_argument('--net', default='mobilenet_at_ilsvrc12', choices=('mobilenet_at_ilsvrc12', 'resnet_at_ilsvrc12'))
    p.add_argument('--resnet_size', type=int, default=50)
    p.add_argument('--batch_size', type=int, default=256)
    p.add_argument('--enbl_fake_prune', action='store_true', help='fake pruning (the only source of a pruned model here)')
    p.add_argument('--fake_prune_ratio', type=float, default=0.5)
    p.add_argument('--seed', type=int, default=0, help='np.random.seed of the fake pruning')
    p.add_argument('--nb_repts_warmup', type=int, default=10, help='graph replays of each step before timing')
    p.add_argument('--nb_repts', type=int, default=50, help='graph replays per timed window')
    p.add_argument('--nb_rounds', type=int, default=5, help='alternating (masked, compact) timed windows')
    p.add_argument('--json', default=None, help='write the measurements here')
    return p.parse_args(argv)


def _replay_ms(ex, lr, n, torch):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        ex.run_step(lr)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def _time_alone(fn, n, flush, torch):
    """mean ms of `fn` over n launches, each after the L2 has been overwritten"""
    for _ in range(3):
        fn()
    tot = 0.0
    for _ in range(n):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        tot += a.elapsed_time(b)
    return tot / n


def gather_scatter_kernels(cex, lr, n, torch):
    """[(op, kind, ms, algorithmic bytes)] of every channel scatter and every BN apply with a fused gather, launched
    with the arguments one eager step of the executor gives them (accumulate, dy planes)"""
    from pocketflow_b200 import ops
    flush = torch.empty(64 << 20, dtype=torch.float32, device=cex.device)        # 256 MB > the 50 MB L2
    out = []
    fused = {gop: bn for bn, gop in cex.bn_gather.items()}
    calls, launch = [], ops.scatter_channels
    ops.scatter_channels = lambda *a: (calls.append(a), launch(*a))[1]
    try:
        graph, cex._graph = cex._graph, None
        cex.run_step(lr)
    finally:
        ops.scatter_channels, cex._graph = launch, graph
    gathers = [op for op in reversed(cex.ops) if op.type == 'GatherChannels']
    assert len(calls) == len(gathers)
    for op, args in zip(gathers, calls):
        dy, inv, dx, acc, planes = args
        idx, t = cex.gather_idx[op], op.inputs[0]
        m, kept = op.output.numel // op.output.shape[-1], int((idx >= 0).sum().item())
        nbytes = 4 * op.output.numel + 4 * t.numel * ((2 if acc else 1) if dx is not None else 0) + \
            (4 * t.numel if planes is not None else 0)
        ms = _time_alone(lambda: launch(*args), n, flush, torch)
        kind = 'scatter_channels' + ('(acc)' if acc else '') + ('+planes' if planes is not None and dx is not None else
                                                               '->planes' if planes is not None else '')
        out.append((op.name, kind, ms, nbytes))
        bn = fused.get(op)
        if bn is not None:
            lo = cex.batch_norm[bn]
            x = cex.T(bn.inputs[0])
            nbytes = 4 * m * kept + (4 if lo.y_out is not None else 0) * op.output.numel + \
                (4 if lo.pl is not None else 0) * op.output.numel
            ms = _time_alone(lambda: ops.bn_apply_gather(x, *lo.batch, lo.act, lo.idx, lo.y_out, lo.pl), n, flush, torch)
            out.append((op.name, 'bn_apply_gather', ms, nbytes))
    return out


def main(argv=None):
    args = parse(argv)
    if not args.enbl_fake_prune:
        raise ValueError('give --enbl_fake_prune: this tool times a seed-initialised, fake-pruned model')
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError('the training steps run on the GPU: no CUDA device found')
    from pocketflow_b200 import compact, ops
    from pocketflow_b200.flags import FLAGS
    FLAGS.reset()
    importlib.reload(importlib.import_module('pocketflow_b200.datasets.ilsvrc12_dataset'))
    net = importlib.reload(importlib.import_module('pocketflow_b200.nets.' + args.net))
    from pocketflow_b200.learners.channel_pruning_gpu.learner import ChannelPrunedGpuLearner
    FLAGS.learner, FLAGS.batch_size = 'chn-pruned-gpu', args.batch_size
    if args.net.startswith('resnet'):
        FLAGS.resnet_size = args.resnet_size
    torch.cuda.set_device(0)
    lrn = ChannelPrunedGpuLearner(None, net.ModelHelper())
    ex = lrn.sess_train
    lrn.init_from_full()
    ex.store.load_state_dict(compact.fake_prune(ex.g, ex.logits_t, ex.store.state_dict(), args.fake_prune_ratio, args.seed),
                             strict=True)
    for v in lrn.maskable_vars:
        ops.cpg_channel_mask(ex.store.view(v), ex.store.view(v, ex.MASK))
    lrn.iterator_train.prefill()
    lrn.feed(ex, lrn.iterator_train)
    mem0 = torch.cuda.max_memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    ct = compact.CompactTrainer(ex)
    cex = ct.ex
    print('\n'.join(ct.report()))
    lr = lrn.lrn_rate(0)
    ex.forward()
    cex.forward()
    torch.cuda.synchronize()
    lf, lc = ex.T(ex.logits_t), cex.T(cex.logits_t)
    diff = float((lf - lc).abs().max() / lf.abs().max().clamp_min(1e-30))
    cex.capture()
    for _ in range(args.nb_repts_warmup):
        cex.run_step(lr)
    torch.cuda.synchronize()
    mem_c = torch.cuda.max_memory_allocated()
    ex.capture()
    for _ in range(args.nb_repts_warmup):
        ex.run_step(lr)
    ms = {'masked': [], 'compact': []}
    for _ in range(args.nb_rounds):
        ms['masked'].append(_replay_ms(ex, lr, args.nb_repts, torch))
        ms['compact'].append(_replay_ms(cex, lr, args.nb_repts, torch))
    bs = args.batch_size
    res = dict(net=args.net, resnet_size=args.resnet_size if args.net.startswith('resnet') else None, batch=bs,
               fake_prune_ratio=args.fake_prune_ratio, logits_max_rel_diff=diff,
               params_full=sum(v.numel for v in ex.variables), params_compact=sum(v.numel for v in cex.variables),
               flat_grad_bytes=dict(masked=4 * ex.G.numel(), compact=4 * cex.G.numel()),
               peak_memory_bytes=dict(masked_step_built=mem0, both_steps_built=mem_c))
    print('logits of the two models from the same state: max |diff| / max |logit| = %.2e' % diff)
    print('flat gradient buffer: %.1f MB masked, %.1f MB compact' % (4e-6 * ex.G.numel(), 4e-6 * cex.G.numel()))
    print('peak memory: %.2f GB with the masked step built, %.2f GB with both' % (mem0 / 2 ** 30, mem_c / 2 ** 30))
    for arm, v in ms.items():
        ips = sorted(bs / (t / 1e3) for t in v)
        res[arm] = dict(ms_per_step=sorted(v), images_per_s_min=ips[0], images_per_s_median=float(np.median(ips)),
                        images_per_s_max=ips[-1])
        print('%-8s step: %.3f ms / batch of %d | images/s min %.0f median %.0f max %.0f'
              % (arm, float(np.median(v)), bs, ips[0], float(np.median(ips)), ips[-1]))
    gk = gather_scatter_kernels(cex, lr, 20, torch)
    res['kernels'] = [dict(op=n, kind=k, us=t * 1e3, bytes=b, gb_per_s=b / (t * 1e-3) / 1e9) for n, k, t, b in gk]
    for kind in sorted({k for _, k, _, _ in gk}):
        sel = [(t, b) for _, k, t, b in gk if k == kind]
        tt, tb = sum(t for t, _ in sel), sum(b for _, b in sel)
        print('%s: %d launches, %.1f us in all, %.1f MB, %.0f GB/s' % (kind, len(sel), tt * 1e3, tb / 1e6,
                                                                      tb / (tt * 1e-3) / 1e9))
    try:
        res['gpu'] = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                                              '--format=csv,noheader'], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        res['gpu'] = torch.cuda.get_device_name(0)
    print('gpu (name, power limit, SM clock, max SM clock): ' + res['gpu'])
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as f:
            json.dump(res, f, indent=1)
    return 0


if __name__ == '__main__':
    sys.exit(main())
