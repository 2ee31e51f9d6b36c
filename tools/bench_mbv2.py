"""Time the captured MobileNet-v2 training step (`--mobilenet_version 2`, 224x224 synthetic batches) on one GPU.

    python tools/bench_mbv2.py [--batches 128 256] [--repeats 5] [--steps 20] [--out FILE]

* images/s of the CUDA-graph replay of one step for full-prec, uniform W8A8 (per-channel buckets) and the
  chn-pruned-gpu masked step (masks from a short selection run), at each batch that fits, with the peak memory;
* the per-category eager breakdown of one full-prec step (Executor.profile_step);
* the saving of the fused linear-bottleneck pass (pf_bn_apply_add): the full-prec step with the fusion on and with
  PF_FUSE_BN_ADD=0 (BN apply, pf_add, split), timed alternately in the same process;
* the time of the 1x1 convs at 56x56 that stay on the exact-fp32 CUDA-core kernels (channel counts 24 / 96 / 144 are
  multiples of 8 but not of 16), fwd + dgrad + wgrad.

Warm-up replays first, then --repeats timed runs of --steps replays each (CUDA events); every figure is min / median /
max over the runs.  The device name and power limit are read in the same run (nvidia-smi query, read-only).  Prints one
JSON document (also written to --out)."""
import argparse
import importlib
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pocketflow_b200 import ops  # noqa: E402
from pocketflow_b200.flags import FLAGS  # noqa: E402

LEARNERS = {
    'full-prec': {},
    'uniform-w8a8': dict(learner='uniform', uql_weight_bits=8, uql_activation_bits=8, uql_use_buckets=True,
                         uql_bucket_type='channel'),
    'chn-pruned-gpu': dict(learner='chn-pruned-gpu', cpg_prune_ratio=0.5),
}


def spread(v):
    v = sorted(v)
    return dict(min=round(v[0], 4), median=round(v[len(v) // 2], 4), max=round(v[-1], 4))


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader',
                               '-i', '0'], capture_output=True, text=True, timeout=30).stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def make(name, batch):
    FLAGS.reset()
    import pocketflow_b200.datasets.ilsvrc12_dataset as D
    importlib.reload(D)
    from pocketflow_b200.nets import mobilenet_at_ilsvrc12 as M
    M = importlib.reload(M)
    from pocketflow_b200.learners.learner_utils import create_learner
    for mod in ('channel_pruning_gpu', 'uniform_quantization'):
        importlib.import_module('pocketflow_b200.learners.%s.learner' % mod)
    FLAGS.learner, FLAGS.batch_size, FLAGS.nb_classes, FLAGS.mobilenet_version = 'full-prec', batch, 1001, 2
    for k, v in LEARNERS[name].items():
        setattr(FLAGS, k, v)
    lrn = create_learner(None, M.ModelHelper())
    if hasattr(lrn, 'choose_channels'):
        lrn.init_from_full()
        lrn.choose_channels(nb_iters_layer=2)
    ex = lrn.sess_train
    images, labels = lrn.iterator_train.next_batch()
    ex.buf[lrn.images].copy_(images)
    ex.buf[lrn.labels].copy_(labels)
    ex.capture()
    return lrn


def replay_ms(ex, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        ex.run_step(1e-4)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def time_fp32_convs(ex, reps=20):
    """fwd + dgrad + wgrad of the Conv2D ops at 56x56 that run on the exact-fp32 kernels, on the step's own buffers"""
    out = []
    for op in ex.ops:
        if op.type != 'Conv2D' or op in ex.tc or op in ex.im2col or op.output.shape[1] != 56:
            continue
        d, x, y = ex.desc[op], ex.T(op.inputs[0]), ex.buf[op.output]
        gy, gx = torch.randn_like(y), torch.empty_like(x)
        dw = torch.empty(op.vars['kernel'].shape, device=y.device)
        w = ex.kernel_of(op)
        ms = []
        for _ in range(2):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                ops.conv2d_fwd(d, x, w, None, False, y)
                ops.conv2d_dgrad(d, gy, w, ex.wt_ws, False, gx)
                ops.conv2d_wgrad(d, x, gy, ex.wgrad_ws, dw)
            b.record()
            torch.cuda.synchronize()
            ms.append(a.elapsed_time(b) / reps)
        out.append(dict(op=op.name, cin=op.inputs[0].shape[-1], cout=op.output.shape[-1], ms_fwd_dgrad_wgrad=round(ms[-1], 4)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batches', type=int, nargs='+', default=[128, 256])
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'tools/bench_mbv2.py needs a GPU'
    res = dict(device=torch.cuda.get_device_name(0), nvidia_smi_name_power_limit_max_sm_clock=card(),
               steps_per_run=args.steps, repeats=args.repeats, runs={})
    for name in LEARNERS:
        for batch in args.batches:
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            try:
                lrn = make(name, batch)
                ex = lrn.sess_train
                replay_ms(ex, args.warmup)
                ms = [replay_ms(ex, args.steps) for _ in range(args.repeats)]
            except torch.cuda.OutOfMemoryError as e:
                res['runs']['%s_b%d' % (name, batch)] = dict(error='out of memory: %s' % str(e).split('\n')[0][:200])
                continue
            res['runs']['%s_b%d' % (name, batch)] = dict(
                batch=batch, step_ms=spread(ms), images_per_s=spread([batch * 1e3 / m for m in ms]),
                peak_mem_gb=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2))
            if name == 'full-prec' and batch == args.batches[0]:
                res['breakdown_ms_eager_full_prec_b%d' % batch] = {k: round(v, 4) for k, v in
                                                                   sorted(ex.profile_step(1e-4).items())}
                res['fp32_convs_56x56_b%d' % batch] = time_fp32_convs(ex)
            del lrn, ex
    # fused linear bottleneck against BN apply + add + split, alternating in this process
    batch = args.batches[0]
    torch.cuda.empty_cache()
    fused = make('full-prec', batch)
    os.environ['PF_FUSE_BN_ADD'] = '0'
    plain = make('full-prec', batch)
    del os.environ['PF_FUSE_BN_ADD']
    assert len(fused.sess_train.bn_add) == 10 and not plain.sess_train.bn_add
    replay_ms(fused.sess_train, args.warmup)
    replay_ms(plain.sess_train, args.warmup)
    on, off = [], []
    for _ in range(args.repeats):
        on.append(replay_ms(fused.sess_train, args.steps))
        off.append(replay_ms(plain.sess_train, args.steps))
    bn_f = fused.sess_train.profile_step(1e-4)
    bn_p = plain.sess_train.profile_step(1e-4)
    res['bn_add_fusion_b%d' % batch] = dict(
        step_ms_fused=spread(on), step_ms_unfused=spread(off),
        saving_ms=spread([b - a for a, b in zip(on, off)]),
        eager_bn_apply_plus_add_ms=dict(fused=round(bn_f.get('bn_apply', 0) + bn_f.get('add_fwd', 0), 4),
                                        unfused=round(bn_p.get('bn_apply', 0) + bn_p.get('add_fwd', 0), 4)))
    js = json.dumps(res, indent=1)
    print(js)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(js)


if __name__ == '__main__':
    main()
