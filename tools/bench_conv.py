"""Per-layer conv timing: tensor-core path vs exact-fp32 path at ResNet-50 / batch-256 shapes."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pocketflow_b200 import ops  # noqa: E402

SHAPES = [  # (name, n, h, w, c, k, r, s, stride, pad)
    ('s1 1x1 64->256', 256, 56, 56, 64, 256, 1, 1, 1, 0),
    ('s1 1x1 256->64', 256, 56, 56, 256, 64, 1, 1, 1, 0),
    ('s1 3x3 64->64', 256, 56, 56, 64, 64, 3, 3, 1, 1),
    ('s2 3x3 128->128', 256, 28, 28, 128, 128, 3, 3, 1, 1),
    ('s2 1x1 512->128', 256, 28, 28, 512, 128, 1, 1, 1, 0),
    ('s3 3x3 256->256', 256, 14, 14, 256, 256, 3, 3, 1, 1),
    ('s3 1x1 1024->256', 256, 14, 14, 1024, 256, 1, 1, 1, 0),
    ('s4 3x3 512->512', 256, 7, 7, 512, 512, 3, 3, 1, 1),
    ('s4 1x1 512->2048', 256, 7, 7, 512, 2048, 1, 1, 1, 0),
    ('s2 3x3 s2 128->128', 256, 56, 56, 128, 128, 3, 3, 2, 1),
]


def timeit(fn, iters=5):
    for _ in range(2):
        fn()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def main():
    dev = torch.device('cuda:0')
    res = []
    for name, n, h, w, c, k, r, s, st, pd in SHAPES:
        p = (h + 2 * pd - r) // st + 1
        d = ops.conv_desc(n, h, w, c, k, r, s, p, p, st, st, pd, pd)
        x = torch.randn(n, h, w, c, device=dev)
        wt = torch.randn(r, s, c, k, device=dev) * 0.05
        y = torch.empty(n, p, p, k, device=dev)
        dy = torch.randn(n, p, p, k, device=dev)
        dx = torch.empty_like(x)
        tw = ops.TcWeights(d, dev)
        tw.prepare(wt)
        wt_ws = torch.empty(wt.numel(), device=dev)
        fl = 2.0 * n * p * p * k * r * s * c
        t_tc = timeit(lambda: ops.conv2d_tc_fwd(d, x, tw, None, False, y))
        t_32 = timeit(lambda: ops.conv2d_fwd(d, x, wt, None, False, y), 3)
        t_dg = timeit(lambda: ops.conv2d_tc_dgrad(d, dy, tw, False, dx))
        t_dg32 = timeit(lambda: ops.conv2d_dgrad(d, dy, wt, wt_ws, False, dx), 3)
        dw = torch.empty_like(wt)
        ws = torch.empty(max(ops.conv2d_tc_wgrad_workspace_floats(d), ops.conv2d_wgrad_workspace_floats(d), 4), device=dev)
        t_wg = timeit(lambda: ops.conv2d_tc_wgrad(d, x, dy, ws, dw))
        t_wg32 = timeit(lambda: ops.conv2d_wgrad(d, x, dy, ws, dw), 3)
        row = dict(wgrad_tc_ms=t_wg, wgrad_tc_tflops=fl / t_wg / 1e9, wgrad_fp32_ms=t_wg32, layer=name, gflop=fl / 1e9, fwd_tc_ms=t_tc, fwd_tc_tflops=fl / t_tc / 1e9, fwd_fp32_ms=t_32,
                   fwd_fp32_tflops=fl / t_32 / 1e9, dgrad_tc_ms=t_dg, dgrad_tc_tflops=fl / t_dg / 1e9,
                   dgrad_fp32_ms=t_dg32)
        res.append(row)
        print(json.dumps(row), flush=True)
    os.makedirs('gpurun_out', exist_ok=True)
    json.dump(res, open('gpurun_out/bench_conv.json', 'w'), indent=1)


if __name__ == '__main__':
    main()
