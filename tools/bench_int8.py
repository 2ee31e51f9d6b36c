#!/usr/bin/env python
"""Per-layer times of the u8 x u8 convolutions of an integer model against the fake-quant convolutions they replace.

Every convolution that the integer model (pocketflow_b200/int8.py) runs on the u8 kernel is launched alone, n times
between CUDA events, as is the same layer of the fake-quantized model (split-bf16 operands, three MMAs per k-slice),
both on the inputs a forward of the seed-initialised model left in their buffers.  Each line gives both times and the
u8 kernel's lower bound: the larger of the FLOP bound (2 M N K at the u8 data-sheet rate, 1,979 dense TOPS) and the byte
bound (u8 operands read once, fp32 output written once, at 3.35 TB/s).

With --int8_narrow the integer model also runs the layers whose channel counts are multiples of 16 but not of 64 (the
cp.async-fed u8 kernel); each line names the kernel that ran.

The integer model is built with its depthwise layers on u8 levels too (cfg['int8_depthwise']): each is timed the same
way against pf_dwconv_fwd on the fake-quant model's fp32 input, with the byte bound of each (u8: 1 B read per input
element, 4 B written per output; fp32: 4 B and 4 B) and the u8 kernel's share of its own.

    python tools/bench_int8.py --net resnet_at_ilsvrc12 --resnet_size 50 --batch_size_eval 128 --json out.json
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

U8_OPS_PER_S = 1979e12
HBM_BYTES_PER_S = 3.35e12


def parse(argv=None):
    p = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    p.add_argument('--net', default='resnet_at_ilsvrc12')
    p.add_argument('--resnet_size', type=int, default=None)
    p.add_argument('--mobilenet_version', type=int, default=None)
    p.add_argument('--batch_size_eval', type=int, default=128)
    p.add_argument('--launches', type=int, default=50, help='launches per timed layer')
    p.add_argument('--int8_narrow', action='store_true', help='also the layers of the cp.async-fed u8 kernel')
    p.add_argument('--json', default=None)
    return p.parse_args(argv)


def _ms(fn, n, torch):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def main(argv=None):
    args = parse(argv)
    import torch
    from export_uq_int8 import gpu_name, load_state, setup
    from pocketflow_b200 import compact, int8, ops
    args.ckpt_dir = None
    for k, v in dict(uql_weight_bits=8, uql_activation_bits=8, uql_use_buckets=True, uql_bucket_type='channel',
                     uql_bucket_size=256, uql_quantize_all_layers=False).items():
        setattr(args, k, v)
    args.int8_depthwise = True
    graph, images, logits, cfg = setup(args)
    state = load_state(args, graph, logits)
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    im = int8.IntModel.from_checkpoint(graph, images, logits, state, cfg, dev)
    fq = int8.fake_quant_executor(graph, images, logits, compact.map_state(graph, compact.reachable_ops(graph, logits),
                                                                           state), cfg, dev)
    x = torch.randn(images.shape, generator=torch.Generator().manual_seed(0)).to(dev)
    im.forward(x)
    fq.buf[images].copy_(x)
    fq.forward(training=False)
    torch.cuda.synchronize()
    fq_conv = {op.name: lo for op, lo in fq.conv.items()}
    rows, tot = [], dict(u8=0.0, fq=0.0, bound=0.0)
    for op, lo in im.ex.conv.items():
        if op not in im.ex.int_layers:
            continue
        d = lo.d
        m, k, n = d.n * d.p * d.q, d.r * d.s * d.c, d.k
        flop_s = 2.0 * m * n * k / U8_OPS_PER_S
        byte_s = (d.n * d.h * d.w * d.c + n * k + 4 * m * n) / HBM_BYTES_PER_S
        t_u8 = _ms(lo.forward, args.launches, torch)
        t_fq = _ms(fq_conv[op.name].forward, args.launches, torch)
        bound = max(flop_s, byte_s) * 1e3
        kern = 'tma' if ops.conv2d_u8_supported(d) else 'cp.async'
        rows.append(dict(op=op.name, kernel=kern, m=m, n=n, k=k, u8_ms=t_u8, fake_quant_ms=t_fq, bound_ms=bound,
                         bound_by='flops' if flop_s >= byte_s else 'bytes', u8_share_of_bound=bound / t_u8))
        for key, v in (('u8', t_u8), ('fq', t_fq), ('bound', bound)):
            tot[key] += v
        print('%-48s %-8s M %7d N %5d K %5d | u8 %.4f ms  fake-quant %.4f ms | bound %.4f ms (%s) = %.0f %% of u8'
              % (op.name, kern, m, n, k, t_u8, t_fq, bound, rows[-1]['bound_by'], 100 * bound / t_u8))
    print('all %d u8 layers: u8 %.3f ms, fake-quant %.3f ms, bound %.3f ms' % (len(rows), tot['u8'], tot['fq'],
                                                                              tot['bound']))
    dw_rows, dw_tot = [], dict(u8=0.0, fp32=0.0, bound=0.0, fp32_bound=0.0)
    for op, lo in im.ex.depthwise.items():
        if op not in im.ex.int_layers:
            continue
        d = lo.d
        nin, nout = d.n * d.h * d.w * d.c, d.n * d.p * d.q * d.c
        bound = (nin + d.r * d.s * d.c + 4 * nout) / HBM_BYTES_PER_S * 1e3
        bound32 = (4 * nin + 4 * d.r * d.s * d.c + 4 * nout) / HBM_BYTES_PER_S * 1e3
        x32, w32, y32 = fq.T(op.inputs[0]), fq.kernel_of(op), fq.buf[op.output]
        t_u8 = _ms(lo.forward, args.launches, torch)
        t_32 = _ms(lambda: ops.dwconv_fwd(d, x32, w32, y32), args.launches, torch)
        dw_rows.append(dict(op=op.name, h=d.h, w=d.w, c=d.c, stride=d.stride_h, u8_ms=t_u8, fp32_ms=t_32,
                            bound_ms=bound, fp32_bound_ms=bound32, u8_share_of_bound=bound / t_u8,
                            fp32_share_of_bound=bound32 / t_32))
        for key, v in (('u8', t_u8), ('fp32', t_32), ('bound', bound), ('fp32_bound', bound32)):
            dw_tot[key] += v
        print('%-48s %4dx%-4d C %4d s%d | u8 %.4f ms (%.0f %% of its byte bound)  fp32 %.4f ms (%.0f %%)'
              % (op.name, d.h, d.w, d.c, d.stride_h, t_u8, 100 * bound / t_u8, t_32, 100 * bound32 / t_32))
    if dw_rows:
        print('all %d u8 depthwise layers: u8 %.3f ms (bound %.3f), pf_dwconv_fwd %.3f ms (bound %.3f)'
              % (len(dw_rows), dw_tot['u8'], dw_tot['bound'], dw_tot['fp32'], dw_tot['fp32_bound']))
    res = dict(net=args.net, resnet_size=args.resnet_size, batch=args.batch_size_eval, layers=rows, totals=tot,
               depthwise=dw_rows, depthwise_totals=dw_tot, gpu=gpu_name(torch))
    print('gpu: ' + res['gpu'])
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as f:
            json.dump(res, f, indent=1)
    return 0


if __name__ == '__main__':
    sys.exit(main())
