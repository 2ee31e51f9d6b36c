#!/usr/bin/env python
"""Time the u8 level producer with a per-batch range (pf_bn_eval_levels_u8: range reset, range pass, level pass) against
the one-pass static-range producer of calibrated models (pf_bn_eval_levels_u8_static) on the producer shapes of
ResNet-50 at batch 128 and MobileNet-v2 at batch 256, alternating, with CUDA events.  Each line gives both times and
their HBM byte bounds (per-batch: 4 B read per element and pass + 1 B written; static: 4 B + 1 B) at the H100 SXM's
3.35 TB/s.

    python tools/bench_calib_levels.py [--reps 100] [--rounds 5] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12
# (label, pixels, channels)
SHAPES = [('rn50 b128 56x56x64', 128 * 56 * 56, 64), ('rn50 b128 28x28x128', 128 * 28 * 28, 128),
          ('rn50 b128 14x14x256', 128 * 14 * 14, 256), ('rn50 b128 7x7x512', 128 * 7 * 7, 512),
          ('mbv2 b256 56x56x144', 256 * 56 * 56, 144), ('mbv2 b256 28x28x192', 256 * 28 * 28, 192),
          ('mbv2 b256 14x14x576', 256 * 14 * 14, 576), ('mbv2 b256 7x7x960', 256 * 7 * 7, 960)]


def main(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument('--reps', type=int, default=100)
    p.add_argument('--rounds', type=int, default=5)
    p.add_argument('--json', default=None)
    a = p.parse_args(argv)
    import torch
    from pocketflow_b200 import ops
    dev = torch.device('cuda', 0)
    g = torch.Generator(device=dev).manual_seed(0)
    res = []
    for label, m, c in SHAPES:
        x = torch.randn(m * c, device=dev, generator=g)
        mean, var = torch.zeros(c, device=dev), torch.ones(c, device=dev)
        gamma, beta = torch.ones(c, device=dev), torch.zeros(c, device=dev)
        bn = (m, c, mean, var, 1e-5, gamma, beta)
        nseg = (c + 127) // 128
        lv = torch.empty(m * c, dtype=torch.uint8, device=dev)
        hdr = torch.zeros(2, dtype=torch.int32, device=dev)
        csum = torch.empty(m * nseg, device=dev)
        slot = torch.zeros(2, dtype=torch.int32, device=dev)
        ops.bn_eval_levels_u8(x, *bn, 1, 8, slot, lv, hdr, csum)
        static = slot.clone()
        arms = {'per_batch': lambda: ops.bn_eval_levels_u8(x, *bn, 1, 8, slot, lv, hdr, csum),
                'static': lambda: ops.bn_eval_levels_u8_static(x, *bn, 1, 8, static, lv, hdr, csum)}
        for fn in arms.values():
            for _ in range(10):
                fn()
        us = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, fn in arms.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.reps):
                    fn()
                e1.record()
                e1.synchronize()
                us[k].append(e0.elapsed_time(e1) * 1e3 / a.reps)
        n = m * c
        bound = {'per_batch': 9 * n / HBM * 1e6, 'static': 5 * n / HBM * 1e6}
        row = dict(shape=label, elements=n)
        for k in arms:
            t = sorted(us[k])[len(us[k]) // 2]
            row[k] = dict(us_median=t, us_min=min(us[k]), bound_us=bound[k], share_of_bound=bound[k] / t)
        res.append(row)
        print('%-22s per-batch %8.1f us (bound %7.1f, %.2f)   static %8.1f us (bound %7.1f, %.2f)   saved %6.1f us'
              % (label, row['per_batch']['us_median'], bound['per_batch'], row['per_batch']['share_of_bound'],
                 row['static']['us_median'], bound['static'], row['static']['share_of_bound'],
                 row['per_batch']['us_median'] - row['static']['us_median']))
    try:
        gpu = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                                       '--format=csv,noheader'], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        gpu = torch.cuda.get_device_name(0)
    print('gpu: ' + gpu)
    if a.json:
        with open(a.json, 'w') as f:
            json.dump(dict(gpu=gpu, rows=res), f, indent=1)
    return 0


if __name__ == '__main__':
    sys.exit(main())
