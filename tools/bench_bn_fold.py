"""Per-layer cost of the inference batch norm folded into the forward conv epilogue (Executor._plan_bn_fold), at the
ResNet-50 teacher of resnet50_uq8_dst_b128 (batch 128): for every conv -> BN pair the planner folds, the fused call
(pf_conv2d_tc_fwd_planes_bn) against the conv followed by pf_bn_apply_eval, each timed with CUDA events as the median
of N launches with the L2 cache flushed before every launch.  Prints one line per pair, the totals, the HBM bytes the
fold saves (the fp32 re-read of the conv output) and the card's name and power limit.
usage: python tools/bench_bn_fold.py [N] [--json PATH]"""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from pocketflow_b200 import engine, ops  # noqa: E402
from pocketflow_b200 import graph as G  # noqa: E402


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0) + ', power limit unknown'


def median_ms(fn, flush, n):
    ts = []
    for _ in range(n + 2):
        flush.add_(1.0)                           # 256 MB write: nothing of the previous launch stays in L2
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts = sorted(ts[2:])
    return ts[len(ts) // 2]


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 and sys.argv[1].isdigit() else 20
    out_json = sys.argv[sys.argv.index('--json') + 1] if '--json' in sys.argv else None
    dev = torch.device('cuda:0')
    mod = bench.setup_flags('resnet50_uq8_dst_b128')
    mh = mod.ModelHelper()
    g = G.Graph()
    with g.as_default():
        with G.variable_scope('data'):
            im, _ = mh.build_dataset_train().get_next()
        with G.variable_scope('distilled_model'):
            logits = mh.forward_eval(im)
    ex = engine.Executor(g, im, logits, dev, train=False)
    ex.buf[im].normal_()
    ex.forward()                                  # prepares the weights; every buffer holds this step's values
    torch.cuda.synchronize()
    flush = torch.zeros(64 << 20, device=dev)
    rows, tot_u, tot_f, tot_b = [], 0.0, 0.0, 0
    for conv, bn in ex.bn_fold.items():
        lo, bl = ex.conv[conv], ex.batch_norm[bn]
        bias, relu, y = lo._epilogue()
        res = ex.T(lo.res) if lo.res is not None else None

        def conv_call(bn_out=None):
            if lo.xp is not None:
                ops.conv2d_tc_fwd_planes(lo.d, lo.xp, lo.tw, bias, relu, y, res, bn_out)
            else:
                ops.conv2d_tc_fwd(lo.d, ex.T(lo.x), lo.tw, bias, relu, y, res, bn_out)

        def unfused():
            conv_call()
            ops.bn_apply_eval(y, *bl.moving, bl.act, bl.y_out, None, bl.pl)

        t_u = median_ms(unfused, flush, n)
        t_f = median_ms(lambda: conv_call(bl.bn_out), flush, n)
        t_c = median_ms(conv_call, flush, n)
        saved = 4 * y.numel()                     # the BN pass's read of the conv output
        d = lo.d
        row = dict(conv=conv.name.split('/')[-2] if '/' in conv.name else conv.name,
                   shape='%dx%dx%d->%d %dx%d/%d' % (d.h, d.w, d.c, d.k, d.r, d.s, d.stride_h),
                   residual=res is not None, f32_out=bl.y_out is not None, conv_ms=t_c, conv_bn_ms=t_u, fused_ms=t_f,
                   saved_mb=saved / 1e6)
        rows.append(row)
        tot_u += t_u
        tot_f += t_f
        tot_b += saved
        print('%-28s %-24s res %d f32 %d  conv %.3f  conv+bn %.3f  fused %.3f ms  (%+.1f %%)  saves %.1f MB' % (
            row['conv'], row['shape'], row['residual'], row['f32_out'], t_c, t_u, t_f, 100 * (t_f / t_u - 1),
            saved / 1e6), flush=True)
    print('%d pairs: conv + bn_apply_eval %.3f ms, fused %.3f ms (%.3f ms saved), %.2f GB not re-read per teacher '
          'forward' % (len(rows), tot_u, tot_f, tot_u - tot_f, tot_b / 1e9))
    c = card()
    print('card:', c)
    if out_json:
        with open(out_json, 'w') as f:
            json.dump(dict(card=c, launches=n, rows=rows, total_unfused_ms=tot_u, total_fused_ms=tot_f,
                           saved_gb=tot_b / 1e9), f, indent=1)


if __name__ == '__main__':
    main()
