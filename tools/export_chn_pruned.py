#!/usr/bin/env python
"""Export a channel-pruned model at its pruned width, and time it against the masked full-width model.

The counterpart of the reference's tools/conversion/export_chn_pruned_tflite_model.py, without TFLite: the latest
checkpoint of a channel-pruning learner (`--learner chn-pruned-gpu` / `chn-pruned-rmt`, npz or TF bundle) is turned into
a compact model (pocketflow_b200/compact.py), written as a compact checkpoint plus a sidecar JSON of the kept channels,
and the eval forward of both models is timed as CUDA-graph replays at --batch_size_eval, alternating in one process.

    python tools/export_chn_pruned.py --net mobilenet_at_ilsvrc12 --ckpt_dir ./models_cpg --out ./models_cpg_compact/model
    python tools/export_chn_pruned.py --net resnet_at_ilsvrc12 --resnet_size 50 --enbl_fake_prune --fake_prune_ratio 0.5 \
        --batch_size_eval 256 --out /tmp/rn50_compact/model --json /tmp/rn50.json

--enbl_fake_prune zeroes int(cin * ratio) random input channels of every conv (the reference's apply_fake_pruning,
seeded with np.random.seed(--seed)), so that speed can be measured without a trained model; without a checkpoint the
model keeps its seed initialisation.
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
    p.add_argument('--net', default='mobilenet_at_ilsvrc12', help='pocketflow_b200.nets module with a ModelHelper')
    p.add_argument('--resnet_size', type=int, default=None)
    p.add_argument('--mobilenet_version', type=int, default=None)
    p.add_argument('--ckpt_dir', default=None, help='directory of the masked checkpoint (default: none = seed init)')
    p.add_argument('--out', default='./models_compact/model', help='compact checkpoint path prefix')
    p.add_argument('--ckpt_format', default='npz', choices=('npz', 'tf'))
    p.add_argument('--batch_size_eval', type=int, default=100)
    p.add_argument('--enbl_fake_prune', action='store_true', help='enable fake pruning (for speed test only)')
    p.add_argument('--fake_prune_ratio', type=float, default=0.5, help='fake pruning ratio')
    p.add_argument('--seed', type=int, default=0, help='np.random.seed of the fake pruning')
    p.add_argument('--nb_repts_warmup', type=int, default=20, help='graph replays before timing')
    p.add_argument('--nb_repts', type=int, default=50, help='graph replays per timed window')
    p.add_argument('--nb_rounds', type=int, default=5, help='alternating (full, compact) timed windows')
    p.add_argument('--no_time', action='store_true', help='export only')
    p.add_argument('--json', default=None, help='write the measurements here')
    return p.parse_args(argv)


def load_state(args, graph, logits):
    from pocketflow_b200 import compact
    from pocketflow_b200.learners.abstract_learner import latest_checkpoint, load_checkpoint
    if args.ckpt_dir:
        fn = latest_checkpoint(args.ckpt_dir) if os.path.isdir(args.ckpt_dir) else None
        if fn is None:
            raise ValueError('no checkpoint found in ' + args.ckpt_dir)
        print('masked model restored from ' + fn)
        state = compact.map_state(graph, compact.reachable_ops(graph, logits), load_checkpoint(fn))
    else:
        if not args.enbl_fake_prune:
            raise ValueError('give --ckpt_dir, or --enbl_fake_prune to time a seed-initialised model')
        rng = np.random.default_rng(1)
        state = {v.name: v.initializer(rng, v.shape) for op in compact.reachable_ops(graph, logits)
                 for v in op.vars.values()}
    if args.enbl_fake_prune:
        state = compact.fake_prune(graph, logits, state, args.fake_prune_ratio, args.seed)
    return state


def _replay_ms(g, n, torch):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        g.replay()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def _capture(fn, torch):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


def gather_kernels(cm, n, torch):
    """Each gather of the compact model launched alone n times: [(op, kind, ms per launch, algorithmic bytes)].
    Bytes: 4 per kept input element read + 4 per output element written (fp32, or hi + lo planes of 2 each; 8 when
    both are written)."""
    from pocketflow_b200 import ops
    ex = cm.ex
    out = []
    for op in ex.ops:
        if op.type != 'GatherChannels':
            continue
        idx = ex.gather_idx[op]
        y, pl = ex.outputs_of(op)
        m = op.output.numel // op.output.shape[-1]
        kept = int((idx >= 0).sum().item())
        nbytes = 4 * m * kept + (4 if y is not None else 0) * op.output.numel + (4 if pl is not None else 0) * op.output.numel
        bn = next((b for b, gop in ex.bn_gather.items() if gop is op), None)
        if bn is not None:
            st = ex.store
            x = ex.T(bn.inputs[0])
            c = x.shape[-1]
            v = bn.vars
            fn = lambda: ops.bn_apply_eval_gather(x, x.numel() // c, c, st.view(v['moving_mean']),  # noqa: E731
                                                  st.view(v['moving_variance']), bn.attrs['epsilon'],
                                                  st.view(v['gamma']), st.view(v['beta']), ex.fused_act.get(bn, 0),
                                                  idx, y, pl)
            kind = 'bn_apply_eval_gather'
        else:
            x = ex.T(op.inputs[0])
            fn = lambda: ops.gather_channels(x, idx, y, pl)  # noqa: E731
            kind = 'gather_channels'
        for _ in range(3):
            fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n):
            fn()
        b.record()
        b.synchronize()
        out.append((op.name, kind, a.elapsed_time(b) / n, nbytes))
    return out


def main(argv=None):
    args = parse(argv)
    import torch
    from pocketflow_b200 import compact
    from pocketflow_b200.engine import Executor
    from pocketflow_b200.flags import FLAGS
    net = importlib.import_module('pocketflow_b200.nets.' + args.net)           # defines the net's flags
    FLAGS.reset()
    if args.resnet_size is not None:
        FLAGS.resnet_size = args.resnet_size
    if args.mobilenet_version is not None:
        FLAGS.mobilenet_version = args.mobilenet_version
    FLAGS.batch_size_eval = args.batch_size_eval
    mh = net.ModelHelper()
    graph, images, logits = compact.build_eval_graph(mh, args.batch_size_eval)
    state = load_state(args, graph, logits)
    if not torch.cuda.is_available():
        raise RuntimeError('the compact model runs on the GPU: no CUDA device found')
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    cm = compact.CompactModel.from_masked(graph, images, logits, state, dev)
    for name, cin, kept in cm.conv_report():
        print('%s: reducing %d channels to %d' % (name, cin, kept))
    print('compact model written to ' + cm.export(args.out, args.ckpt_format) + ' (+ %s.channels.json)' % args.out)
    n_full = sum(a.size for a in state.values())
    n_comp = sum(a.size for a in cm.state.values())
    print('parameters: %d -> %d (%.1f %%)' % (n_full, n_comp, 100.0 * n_comp / n_full))
    if args.no_time:
        return 0
    full = Executor(graph, images, logits, dev, train=False)
    full.store.load_state_dict(state, strict=True)
    x = torch.randn(images.shape, generator=torch.Generator().manual_seed(0)).to(dev)
    full.buf[images].copy_(x)
    cm.ex.buf[cm.images].copy_(x)
    g_full = _capture(lambda: full.forward(training=False), torch)
    g_comp = _capture(lambda: cm.ex.forward(training=False), torch)
    g_full.replay()
    g_comp.replay()
    torch.cuda.synchronize()
    lf, lc = full.T(full.logits_t).float(), cm.ex.T(cm.logits).float()
    diff = float((lf - lc).abs().max() / lf.abs().max().clamp_min(1e-30))
    for _ in range(args.nb_repts_warmup):
        g_full.replay()
        g_comp.replay()
    ms = {'full': [], 'compact': []}
    for _ in range(args.nb_rounds):
        ms['full'].append(_replay_ms(g_full, args.nb_repts, torch))
        ms['compact'].append(_replay_ms(g_comp, args.nb_repts, torch))
    bs = args.batch_size_eval
    res = dict(net=args.net, resnet_size=args.resnet_size, mobilenet_version=args.mobilenet_version, batch=bs,
               fake_prune_ratio=args.fake_prune_ratio if args.enbl_fake_prune else None, params_full=n_full,
               params_compact=n_comp, logits_max_rel_diff=diff)
    for arm, v in ms.items():
        ips = sorted(bs / (t / 1e3) for t in v)
        res[arm] = dict(ms_per_batch=sorted(v), images_per_s_min=ips[0], images_per_s_median=float(np.median(ips)),
                        images_per_s_max=ips[-1])
        print('%-8s eval forward: %.3f ms / batch of %d | images/s min %.0f median %.0f max %.0f'
              % (arm, float(np.median(v)), bs, ips[0], float(np.median(ips)), ips[-1]))
    gk = gather_kernels(cm, 200, torch)
    res['gathers'] = [dict(op=n, kind=k, us=t * 1e3, bytes=b, gb_per_s=b / (t * 1e-3) / 1e9) for n, k, t, b in gk]
    tot_t, tot_b = sum(t for _, _, t, _ in gk), sum(b for _, _, _, b in gk)
    if gk:
        print('gathers: %d launches, %.1f us in all, %.1f MB, %.0f GB/s' % (len(gk), tot_t * 1e3, tot_b / 1e6,
                                                                            tot_b / (tot_t * 1e-3) / 1e9))
    try:
        res['gpu'] = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                                              '--format=csv,noheader'], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        res['gpu'] = torch.cuda.get_device_name(0)
    print('gpu: ' + res['gpu'])
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as f:
            json.dump(res, f, indent=1)
    return 0


if __name__ == '__main__':
    sys.exit(main())
