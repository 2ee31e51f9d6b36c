"""Time the bucketed codebook kernels and the bucketed non-uniform training step on one GPU.

    python tools/bench_nuq_buckets.py [--iters 50] [--repeats 5] [--steps 20] [--out FILE] [--no-step]

* CUDA-event times of the codebook quantizer on the 52 quantized ResNet-50 kernels (23.4 M elements), per layer and
  with channel and split (256) buckets, at 4 and 8 bits: the forward (per-bucket min/max + quantize, keeping the
  centroid index), the quantize launch alone, the quantile init and the codebook gradient.  GB/s from the algorithmic
  bytes (quantize: 8 B/element read + write, 9 with the kept index; gradient: 5 B/element; quantile init: 4 B/element
  of the padded buckets) and the share of 3.35 TB/s (H100 SXM HBM3, data sheet);
* images/s of the CUDA-graph replay of the ResNet-50 4-bit + distillation step at batch 128 (the
  resnet50_nuq4_dst_b128 workload of bench.py) per layer and with channel and split buckets, one configuration after another.

Every figure is min / median / max over --repeats runs.  The device name and power limit are read in the same run
(nvidia-smi query, read-only).  Prints one JSON document (also written to --out when given)."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pocketflow_b200 import ops  # noqa: E402

HBM_GBS = 3350.0
MODES = {'layer': {}, 'channel': dict(use_buckets=True, bucket_type='channel'),
         'split256': dict(use_buckets=True, bucket_type='split', bucket_size=256)}


def spread(v):
    v = sorted(v)
    return dict(min=round(v[0], 4), median=round(v[len(v) // 2], 4), max=round(v[-1], 4))


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader',
                               '-i', '0'], capture_output=True, text=True, timeout=30).stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def resnet50_kernel_shapes():
    """HWIO kernels of ResNet-50 v2 (utils/external/resnet_model.py), creation order."""
    shapes = [(7, 7, 3, 64)]
    cin = 64
    for filters, blocks in zip([64, 128, 256, 512], [3, 4, 6, 3]):
        for b in range(blocks):
            if b == 0:
                shapes.append((1, 1, cin, filters * 4))
            shapes += [(1, 1, cin, filters), (3, 3, filters, filters), (1, 1, filters, filters * 4)]
            cin = filters * 4
    shapes.append((2048, 1001))
    return shapes


def time_ms(fn, iters, repeats):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    out = []
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(repeats):
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b) / iters)
    return out


def kernels(args):
    shapes = resnet50_kernel_shapes()[1:-1]
    torch.manual_seed(0)
    src = [torch.randn(s, device='cuda') * (2.0 / np.prod(s[:-1])) ** 0.5 for s in shapes]
    dst = [torch.empty_like(w) for w in src]
    n = sum(w.numel() for w in src)
    rows = []
    for bits in (4, 8):
        for mode, kw in MODES.items():
            # codebooks among "trainable variables": one flat buffer, [2^bits, nb] (per layer: 2^bits) views
            nbs = [ops.uq_bucket_layout(tuple(s.shape), kw.get('use_buckets', False), kw.get('bucket_type', 'channel'),
                                        kw.get('bucket_size', 256))[0] for s in src]
            sizes = [((1 << bits) * nb + 3) // 4 * 4 for nb in nbs]
            base = torch.zeros(sum(sizes), device='cuda')
            offs = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(int)
            views = [base[o:o + (1 << bits) * nb] for o, nb in zip(offs, nbs)]
            q = ops.CodebookWeightQuantizer(src, dst, bits, keep_index=True, cluster_views=views, cluster_base=base,
                                            **kw)
            q.quantile_init()
            grads = [torch.randn_like(w) for w in src]
            gbase = torch.zeros_like(base)
            padded = sum(int(s['padded']) for s in q.uq.segs)
            if kw:
                quant_only = lambda q=q: ops._lib.check(q.L.pf_nuq_bucket_quant(  # noqa: E731
                    ops._p(q.uq.segs_dev), ops._p(q.work_b_dev), len(q.work_b), ops._p(q.uq.scales), q.uq.n_buckets,
                    ops._p(q.cluster_base), ops._p(q.cluster_off), ops._p(q.idx), ops._p(q.idx_base), ops._stream()),
                    'pf_nuq_bucket_quant')
            else:
                quant_only = lambda q=q: ops._lib.check(q.L.pf_nuq_weight_quant_ex(  # noqa: E731
                    ops._p(q.uq.segs_dev), ops._p(q.uq.work_q_dev), len(q.uq.work_q), ops._p(q.uq.scales),
                    q.uq.n_buckets, ops._p(q.cluster_base), ops._p(q.cluster_off), ops._p(q.idx), ops._p(q.idx_base),
                    ops._stream()), 'pf_nuq_weight_quant_ex')
            for what, fn, nbytes in (('forward(minmax+quant)', q.forward, 9 * n + 4 * padded),
                                     ('quant', quant_only, 9 * n),
                                     ('quantile_init', q.quantile_init, 4 * padded if kw else 4 * n),
                                     ('cluster_grad', lambda: q.cluster_grad(grads, gbase), 5 * n)):
                ms = time_ms(fn, args.iters if what != 'quantile_init' else max(3, args.iters // 10), args.repeats)
                med = sorted(ms)[len(ms) // 2]
                gbs = nbytes / (med * 1e-3) / 1e9
                rows.append(dict(bits=bits, mode=mode, what=what, ms=spread(ms), algorithmic_bytes=int(nbytes),
                                 gbs_median=round(gbs, 1), share_of_hbm_peak=round(gbs / HBM_GBS, 3),
                                 launches='per-layer' if not kw else 'bucketed'))
                print(json.dumps(rows[-1]), flush=True)
            del q, base, gbase, grads
            torch.cuda.empty_cache()
    return rows


def make_step(bucket_type):
    import bench                                       # the benchmark's own workload definition, read only
    from pocketflow_b200.flags import FLAGS
    from pocketflow_b200.learners.learner_utils import create_learner
    mod = bench.setup_flags('resnet50_nuq4_dst_b128')
    if bucket_type:
        FLAGS.nuql_use_buckets, FLAGS.nuql_bucket_type, FLAGS.nuql_bucket_size = True, bucket_type, 256
    lrn = create_learner(None, mod.ModelHelper())
    ex = lrn.sess_train
    images, labels = lrn.iterator_train.next_batch()
    ex.buf[lrn.images].copy_(images)
    ex.buf[lrn.labels].copy_(labels)
    ex.run_step(1e-4)
    ex.capture()
    return lrn


def steps(args):
    """One configuration at a time (three ResNet-50 students with teachers do not fit together), --repeats timed
    runs of --steps graph replays each."""
    import gc
    out = {}
    for k, bt in (('layer', None), ('channel', 'channel'), ('split256', 'split')):
        lrn = make_step(bt)
        ex = lrn.sess_train
        ms = time_ms(lambda ex=ex: ex.run_step(1e-4), args.steps, args.repeats)
        out[k] = dict(images_per_sec=spread([128 / (m * 1e-3) for m in ms]),
                      peak_mem_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 1))
        print(json.dumps({'step': k, **out[k]}), flush=True)
        del lrn, ex
        gc.collect()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--out', default=None, help='also write the JSON document here')
    ap.add_argument('--no-step', action='store_true')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_nuq_buckets needs a GPU')
    torch.cuda.set_device(0)
    res = dict(card=card(), kernels=kernels(args))
    res['step_resnet50_nuq4_dst_b128'] = None if args.no_step else steps(args)
    res['card_after'] = card()
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
