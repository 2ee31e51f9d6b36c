"""Per-layer timing of the tensor-core conv kernels (fwd / dgrad / wgrad) at ResNet-50 shapes (batch 256, or BATCH),
each next to two lower bounds computed from the shape and the launch plan:
  * MMA bound : FLOPs of the MMAs the kernel issues (2 M N K per plane product: 1 + [A split] + [B split]) over the
                dense bf16 tensor-core peak;
  * byte bound: operand planes read once, the fp32 output written once, residual read once, over the HBM peak.
usage: python tools/bench_conv_tc.py [tag]   (env PF_TC_IMPL / PF_TC_BN select kernel variants; the JSON result goes to
OUT_DIR, default bench_out/)"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pocketflow_b200 import ops  # noqa: E402

BATCH = int(os.environ.get('BATCH', '256'))
PEAK_BF16 = 989e12        # H100 SXM data sheet, dense bf16 FLOP/s (700 W)
PEAK_HBM = 3.35e12        # H100 SXM data sheet, HBM3 bytes/s
SHAPES = [  # (name, n, h, w, c, k, r, s, stride, pad, count in ResNet-50)
    ('s1 1x1 64->64', BATCH, 56, 56, 64, 64, 1, 1, 1, 0, 1),
    ('s1 1x1 64->256', BATCH, 56, 56, 64, 256, 1, 1, 1, 0, 4),
    ('s1 1x1 256->64', BATCH, 56, 56, 256, 64, 1, 1, 1, 0, 2),
    ('s1 3x3 64->64', BATCH, 56, 56, 64, 64, 3, 3, 1, 1, 3),
    ('s2 1x1 256->128', BATCH, 56, 56, 256, 128, 1, 1, 1, 0, 1),
    ('s2 3x3 s2 128->128', BATCH, 56, 56, 128, 128, 3, 3, 2, 1, 1),
    ('s2 1x1 s2 256->512', BATCH, 56, 56, 256, 512, 1, 1, 2, 0, 1),
    ('s2 3x3 128->128', BATCH, 28, 28, 128, 128, 3, 3, 1, 1, 3),
    ('s2 1x1 128->512', BATCH, 28, 28, 128, 512, 1, 1, 1, 0, 4),
    ('s2 1x1 512->128', BATCH, 28, 28, 512, 128, 1, 1, 1, 0, 3),
    ('s3 3x3 256->256', BATCH, 14, 14, 256, 256, 3, 3, 1, 1, 5),
    ('s3 1x1 256->1024', BATCH, 14, 14, 256, 1024, 1, 1, 1, 0, 6),
    ('s3 1x1 1024->256', BATCH, 14, 14, 1024, 256, 1, 1, 1, 0, 5),
    ('s4 3x3 512->512', BATCH, 7, 7, 512, 512, 3, 3, 1, 1, 2),
    ('s4 1x1 512->2048', BATCH, 7, 7, 512, 2048, 1, 1, 1, 0, 3),
    ('s4 1x1 2048->512', BATCH, 7, 7, 2048, 512, 1, 1, 1, 0, 2),
]


_FLUSH = None


def timeit(fn, iters=5):
    global _FLUSH
    for _ in range(2):
        fn()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        if os.environ.get('FLUSH', '1') == '1':          # evict the operands from the 126 MB L2 between iterations
            if _FLUSH is None:
                _FLUSH = torch.empty(64 << 20, dtype=torch.float32, device='cuda:0')
            _FLUSH.fill_(1.0)
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def bounds(ps, plan, levels, n, h, w, c, k, r, s, p, nseg, resid):
    """(MMA bound ms, byte bound ms) of one launch; `levels`: the activation operand is one plane of levels"""
    na = 1 if (levels and plan['aff'] >= 1) else plan['na']
    nb = plan['nb']
    fl = 2.0 * n * p * p * k * r * s * c * (1 + (na == 2) + (nb == 2))
    gathered = n * h * w * c if ps in ('fwd', 'wgrad') else n * p * p * k
    other = n * p * p * k if ps == 'wgrad' else k * r * s * c
    out = {'fwd': n * p * p * k, 'dgrad': n * h * w * c, 'wgrad': k * r * s * c}[ps]
    by = 2 * na * gathered + 2 * nb * other + 4 * out
    if ps == 'fwd' and resid:
        by += 4 * out
    if ps == 'fwd' and plan['aff'] == 2:
        by += 4 * n * h * w * nseg                     # per-pixel channel sums
    return fl / PEAK_BF16 * 1e3, by / PEAK_HBM * 1e3


def main():
    tag = sys.argv[1] if len(sys.argv) > 1 else 'run'
    passes = os.environ.get('PASSES', 'fwd,dgrad,wgrad').split(',')
    dev = torch.device('cuda:0')
    res, tot = [], {}
    bsum = {}                 # per pass: sums (count-weighted) of time and max(MMA bound, byte bound) over TMA launches
    resid_on = os.environ.get('RESIDUAL', '0') == '1'
    variant = os.environ.get('VARIANT', '')
    only = os.environ.get('ONLY', '')
    for name, n, h, w, c, k, r, s, st, pd, cnt in SHAPES:
        if only and only not in name:
            continue
        p = (h + 2 * pd - r) // st + 1
        d = ops.conv_desc(n, h, w, c, k, r, s, p, p, st, st, pd, pd)
        x = torch.randn(n, h, w, c, device=dev)
        wt = torch.randn(r, s, c, k, device=dev) * 0.05
        y = torch.empty(n, p, p, k, device=dev)
        dy = torch.randn(n, p, p, k, device=dev)
        dx = torch.empty_like(x)
        dw = torch.empty_like(wt)
        tw = ops.TcWeights(d, dev)
        tw.prepare(wt)
        ws = torch.empty(max(ops.conv2d_tc_wgrad_workspace_floats(d), 4), device=dev)
        fl = 2.0 * n * p * p * k * r * s * c
        row = dict(layer=name, gflop=fl / 1e9, count=cnt)
        fns = dict(fwd=lambda: ops.conv2d_tc_fwd(d, x, tw, None, False, y),
                   dgrad=lambda: ops.conv2d_tc_dgrad(d, dy, tw, False, dx),
                   wgrad=lambda: ops.conv2d_tc_wgrad(d, x, dy, ws, dw))
        if os.environ.get('PLANES', '0') == '1':      # operands already split (as inside the training step)
            xp, dyp = ops.Planes(x.numel(), dev), ops.Planes(dy.numel(), dev)
            ops.split_bf16(x, xp)
            ops.split_bf16(dy, dyp)
            resid = None
            if os.environ.get('RESIDUAL', '0') == '1':     # RES_OFFSET: shift the residual buffer by that many bytes
                off = int(os.environ.get('RES_OFFSET', '0')) // 4
                rbuf = torch.randn(y.numel() + off, device=dev)
                resid = rbuf[off:].view(y.shape)
            fns = dict(fwd=lambda: ops.conv2d_tc_fwd_planes(d, xp, tw, None, False, y, resid),
                       dgrad=lambda: ops.conv2d_tc_dgrad_planes(d, dyp, tw, False, dx),
                       wgrad=lambda: ops.conv2d_tc_wgrad_planes(d, xp, dyp, ws, dw))
        if variant:
            # lsu: cp.async-fed kernels on split planes; tma: TMA-fed, split planes (3 MMAs per k-slice);
            # levels: TMA-fed, x and the weights as integer quantizer levels (fwd 1 MMA, wgrad 2 MMAs, dgrad as tma)
            import numpy as np
            ops.conv2d_tc_set_feed(0 if variant == 'lsu' else 1)
            xp, dyp = ops.Planes(x.numel(), dev), ops.Planes(dy.numel(), dev)
            ops.split_bf16(x, xp)
            ops.split_bf16(dy, dyp)
            resid = torch.randn_like(y) if os.environ.get('RESIDUAL', '0') == '1' else None   # conv3 + shortcut layers
            fns = dict(fwd=lambda: ops.conv2d_tc_fwd_planes(d, xp, tw, None, False, y, resid),
                       dgrad=lambda: ops.conv2d_tc_dgrad_planes(d, dyp, tw, False, dx),
                       wgrad=lambda: ops.conv2d_tc_wgrad_planes(d, xp, dyp, ws, dw))
            if variant == 'levels' and ops.conv2d_tc_tma_supported(d, 0) and ops.conv2d_tc_tma_supported(d, 2):
                lv = torch.randint(0, 256, (n, h, w, c), device=dev).float() * (torch.rand(n, h, w, c, device=dev) > 0.4)
                lp = ops.Planes(x.numel(), dev)
                lp.hi.copy_(lv.reshape(-1).to(torch.bfloat16))
                nseg = (c + 127) // 128
                csum = lv.reshape(-1, nseg, c // nseg).sum(2).contiguous()
                hdr = torch.from_numpy(np.array([(0.02, 1)], dtype=ops.ACT_HDR).view(np.uint8)).to(dev)
                act = ops.tc_act(lp, hdr, csum, nseg)
                wl = torch.randint(-128, 128, (k, r * s * c), device=dev).to(torch.bfloat16)
                al, be = torch.rand(k, device=dev) + 0.1, -torch.rand(k, device=dev)
                wq = ops.tc_wt(wl, None, al, be, True, 8)
                dya = ops.tc_act(dyp)
                keep = (lv, lp, csum, hdr, wl, al, be)      # noqa: F841 — keep the device buffers alive
                fns['fwd'] = lambda: ops.conv2d_tc_fwd_ex(d, act, wq, None, False, y, resid)
                fns['wgrad'] = lambda: ops.conv2d_tc_wgrad_ex(d, act, dya, ws, dw)
        line = '%-22s' % name
        for ps in passes:
            t = timeit(fns[ps])
            plan = ops.conv2d_tc_last_plan()
            mma_ms, byte_ms = bounds(ps, plan, variant == 'levels', n, h, w, c, k, r, s, p, (c + 127) // 128,
                                     resid_on and ps == 'fwd' and variant != '')
            row[ps + '_ms'], row[ps + '_tflops'] = t, fl / t / 1e9
            row[ps + '_mma_bound_ms'], row[ps + '_byte_bound_ms'], row[ps + '_feed'] = mma_ms, byte_ms, plan['feed']
            tot[ps] = tot.get(ps, 0.0) + t * cnt
            if plan['feed'] == 1:
                b = bsum.setdefault(ps, [0.0, 0.0])
                b[0] += t * cnt
                b[1] += max(mma_ms, byte_ms) * cnt
            line += '  %s %.3f ms %6.1f TF (%s, mma %.3f byte %.3f)' % (ps, t, fl / t / 1e9, 'tma' if plan['feed'] else 'lsu',
                                                                      mma_ms, byte_ms)
        print(line, flush=True)
        res.append(row)
    print('weighted totals (ms per ResNet-50 pass):', {k: round(v, 2) for k, v in tot.items()})
    for ps, (t, b) in bsum.items():
        print('%s, TMA launches: %.2f ms against a bound of %.2f ms (%.2fx)' % (ps, t, b, t / b))
    out_dir = os.environ.get('OUT_DIR', 'bench_out')
    os.makedirs(out_dir, exist_ok=True)
    json.dump(dict(tag=tag, batch=BATCH, device=torch.cuda.get_device_name(0), layers=res, totals=tot,
                   tma_time_vs_bound=bsum),
              open(os.path.join(out_dir, 'bench_conv_tc_%s.json' % tag), 'w'), indent=1)


if __name__ == '__main__':
    main()
