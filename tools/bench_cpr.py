"""Time the channel selection of the remastered channel-pruning learner (chn-pruned-rmt) on one GPU, per layer and per
phase (sample, gram, search, refit), beside the numpy oracle's CPU time for the sparse regression of one layer.

    python tools/bench_cpr.py [--net mobilenet|resnet20] [--nb_smpls 5000] [--out FILE]

MobileNet-v1 on synthetic ImageNet-shaped batches at the learner's default flags (5000 samples x 10 crops, 100 ISTA
iterations per solve, 100 Adam iterations of the refit).  One untimed warm-up selection first (module loading, first
launches, allocator growth), then --repeats timed selections, each from the same full model and the same cached batches;
every time is reported as min / median / max over the repeats.  The device name and its power limit are read in the
same run (nvidia-smi query, read-only).  Prints one JSON document (also written to --out)."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
from timeit import default_timer as timer

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def spread(v):
    v = sorted(v)
    return dict(min=round(v[0], 6), median=round(v[len(v) // 2], 6), max=round(v[-1], 6))


def power_limit():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return None
    return out or None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--net', default='mobilenet', choices=['mobilenet', 'resnet20'])
    ap.add_argument('--nb_smpls', type=int, default=5000)
    ap.add_argument('--batch_size', type=int, default=64)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--oracle_layer', type=int, default=1, help='layer whose regression the CPU oracle times')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    from pocketflow_b200.flags import FLAGS
    from pocketflow_b200.learners.learner_utils import create_learner
    import pocketflow_b200.learners.channel_pruning_rmt.learner  # noqa: F401  (declares the learner's flags)
    FLAGS.reset()
    if args.net == 'mobilenet':
        from pocketflow_b200.nets import mobilenet_at_ilsvrc12 as M
    else:
        from pocketflow_b200.nets import resnet_at_cifar10 as M
        FLAGS.resnet_size = 20
    tmp = tempfile.mkdtemp(prefix='pf_cpr_bench_')
    try:
        FLAGS.learner, FLAGS.batch_size, FLAGS.cpr_nb_smpls = 'chn-pruned-rmt', args.batch_size, args.nb_smpls
        FLAGS.cpr_save_path_ws = os.path.join(tmp, 'ws', 'model.ckpt')
        lrn = create_learner(None, M.ModelHelper())
        t0 = timer()
        cached = lrn.cache_batches()
        torch.cuda.synchronize()
        t_cache = timer() - t0
        lrn.choose_channels(cached=cached)                                  # warm-up, not timed
        totals, logs = [], []
        for _ in range(args.repeats):
            torch.cuda.synchronize()
            t0 = timer()
            lrn.choose_channels(cached=cached)
            torch.cuda.synchronize()
            totals.append(timer() - t0)
            logs.append(lrn.selection_log)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    phases = ('sample', 'gram', 'search', 'refit')
    layers = []
    for i, v in enumerate(lrn.maskable_vars):
        recs = [log[i] for log in logs]
        layers.append(dict(layer=i, kernel=v.name, shape=list(v.shape), ratio=recs[0]['ratio'],
                           nnz_target=recs[0]['nnz_target'], nnz=[r['nnz'] for r in recs],
                           solves=[len(r['search']) for r in recs], tc_refit=recs[0]['tc'],
                           times={k: spread([r['times'][k] for r in recs]) for k in phases}))
    phase_tot = {k: spread([sum(r['times'][k] for r in log) for log in logs]) for k in phases}
    # the numpy oracle's sparse regression (secondary sample, Gram, γ search, refit) of one layer of the same shape,
    # on random patches: the reference's float64 / float32 host work for that layer
    from oracle import cpr_oracle as C
    kh, kw, cin, cout = lrn.maskable_vars[args.oracle_layer].shape
    n = FLAGS.cpr_nb_smpls * FLAGS.cpr_nb_crops_per_smpl
    rng = np.random.RandomState(0)
    X = rng.randn(n, kh * kw * cin).astype(np.float32)
    w = (rng.randn(kh, kw, cin, cout) * 0.1).astype(np.float32)
    Y = (X @ w.reshape(-1, cout)).astype(np.float32)
    t0 = timer()
    C.cpr_solve_sparse_regression(rng, X, Y, w, FLAGS.cpr_prune_ratio, FLAGS.cpr_ista_lrn_rate, FLAGS.cpr_ista_nb_iters,
                                  FLAGS.cpr_lstsq_lrn_rate, FLAGS.cpr_lstsq_nb_iters, FLAGS.loss_w_dcy)
    t_orc = timer() - t0
    gpu_layer = [sum(log[args.oracle_layer]['times'][k] for k in ('gram', 'search', 'refit')) for log in logs]
    res = dict(net=args.net, device=torch.cuda.get_device_name(0), nvidia_smi_name_power_limit=power_limit(),
               batch_size=args.batch_size, nb_smpls=FLAGS.cpr_nb_smpls, nb_crops=FLAGS.cpr_nb_crops_per_smpl,
               cached_batches=len(cached), repeats=args.repeats, cache_s=round(t_cache, 4),
               selection_s=spread(totals), phases_s=phase_tot, layers=layers,
               oracle_cpu_layer=dict(layer=args.oracle_layer, shape=[kh, kw, cin, cout], regression_s=round(t_orc, 4),
                                     gpu_same_layer_s=spread(gpu_layer)))
    js = json.dumps(res, indent=1)
    print(js)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(js)


if __name__ == '__main__':
    main()
