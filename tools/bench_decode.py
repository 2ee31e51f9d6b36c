#!/usr/bin/env python
"""Decode throughput of the ILSVRC-12 input pipeline, host against device, on JPEGs generated from seeds (500x375 and
375x500, 4:2:0, quality 90; gradients plus noise, so the scans are denser than a typical photograph's):
  (a) host decode + crop images/s through the input pipeline's thread pool at --nb_threads 8 and 16;
  (a') the host half of --enbl_device_decode: header parse + crop draw + descriptor images/s at 1, 8 and 16 threads,
      and the per-batch packing of 256 images;
  (b) pf_jpeg_decode images/s at batch 128 and 256 (CUDA events, warmed up) and each kernel's time (torch.profiler);
  (c) train_step() images/s of ResNet-50 at batch 128 and MobileNet-v1 at batch 256 over TFRecords packed by
      tools/make_tfrecords.py, with host decoding, --enbl_device_preprocess and --enbl_device_decode.
Prints the card's name and power limit with the results, one JSON line per measurement."""
import argparse
import io
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def emit(**kw):
    print(json.dumps(kw), flush=True)


def make_jpegs(n, seed=0):
    from PIL import Image
    out = []
    for i in range(n):
        h, w = (375, 500) if i % 3 else (500, 375)
        rng = np.random.RandomState(seed + i)
        yy, xx = np.mgrid[0:h, 0:w]
        base = np.stack([(yy * 3 + i) % 256, (xx * 5) % 256, ((xx + yy) * 2) % 256], -1)
        img = ((rng.randint(0, 256, (h, w, 3)) // 4) + base * 3 // 4).astype(np.uint8)
        b = io.BytesIO()
        Image.fromarray(img).save(b, format='JPEG', quality=90, subsampling=2)
        out.append(b.getvalue())
    return out


def host_rate(jpegs, threads, seconds=5.0):
    from pocketflow_b200.datasets import ilsvrc12_dataset as D
    box = np.zeros((0, 4), np.float32)
    pool = ThreadPoolExecutor(threads)
    fn = lambda a: D.crop_and_descriptor(a[1], box, True, np.random.default_rng(a[0]))  # noqa: E731
    list(pool.map(fn, enumerate(jpegs[:2 * threads])))
    done, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < seconds:
        list(pool.map(fn, enumerate(jpegs)))
        done += len(jpegs)
    rate = done / (time.perf_counter() - t0)
    pool.shutdown()
    return rate


def host_parse_rate(jpegs, threads, seconds=5.0):
    """The host half of device decoding, per image in the pool (header parse, crop draw, descriptor, scan slice),
    and DecodeBatch's per-batch packing of 256 such images, in ms."""
    from pocketflow_b200.datasets import ilsvrc12_dataset as D, jpeg as J
    box = np.zeros((0, 4), np.float32)

    def fn(a):
        rng = np.random.default_rng(a[0])
        h = J.parse_header(a[1])
        window, desc = D.crop_window(h.height, h.width, box, True, rng)
        return None, desc, np.zeros(1001, np.float32), (a[1], window, J.descriptor(h, window), J.scan(h, a[1]))
    pool = ThreadPoolExecutor(threads)
    out = list(pool.map(fn, enumerate(jpegs[:256])))
    done, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < seconds:
        list(pool.map(fn, enumerate(jpegs)))
        done += len(jpegs)
    rate = done / (time.perf_counter() - t0)
    pool.shutdown()
    t0 = time.perf_counter()
    for _ in range(5):
        D.DecodeBatch(out)
    return rate, (time.perf_counter() - t0) / 5 * 1000.0


def device_rate(jpegs, b, iters=20):
    import torch
    from pocketflow_b200 import ops
    from pocketflow_b200.datasets import ilsvrc12_dataset as D, jpeg as J
    box = np.zeros((0, 4), np.float32)
    descs, scans, off = [], [], 0
    for i, buf in enumerate(jpegs[:b]):
        h = J.parse_header(buf)
        window, _ = D.crop_window(h.height, h.width, box, True, np.random.default_rng(i))
        descs.append(J.descriptor(h, window, crop_offset=off))
        scans.append(J.scan(h, buf))
        off += window[2] * window[3] * 3
    descs, scans, ws = J.pack(descs, scans)
    dev = torch.device('cuda')
    data = torch.from_numpy(scans.copy()).to(dev)
    desc = torch.from_numpy(descs.view(np.uint8).reshape(-1).copy()).to(dev)
    wst = torch.empty(ws, dtype=torch.int16, device=dev)
    crops = torch.empty(off, dtype=torch.uint8, device=dev)
    status = torch.empty(b, dtype=torch.int32, device=dev)
    for _ in range(3):
        ops.jpeg_decode(data, desc, b, wst, crops, status)
    torch.cuda.synchronize()
    assert int((status != 0).sum()) == 0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        ops.jpeg_decode(data, desc, b, wst, crops, status)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    stages = {}
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            ops.jpeg_decode(data, desc, b, wst, crops, status)
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        for k in ('entropy', 'idct', 'color'):
            if 'jpeg_%s_kernel' % k in ev.key:
                stages[k + '_ms'] = round(ev.device_time_total / 1000.0 / 5, 3)
    return b / (ms / 1000.0), ms, stages, len(scans) / b


def train_rate(net, batch, mode, data_dir, steps, warmup):
    import importlib
    import torch
    from pocketflow_b200.flags import FLAGS
    FLAGS.reset()
    mod = importlib.import_module('pocketflow_b200.nets.' + net)
    importlib.import_module('pocketflow_b200.learners.full_precision.learner')
    importlib.import_module('pocketflow_b200.learners.distillation_helper')
    importlib.reload(importlib.import_module('pocketflow_b200.datasets.ilsvrc12_dataset'))
    mod = importlib.reload(mod)
    if net == 'resnet_at_ilsvrc12':
        FLAGS.resnet_size = 50
    FLAGS.learner, FLAGS.batch_size = 'full-prec', batch
    FLAGS.summ_step = FLAGS.save_step = 10 ** 9
    FLAGS.data_dir_local, FLAGS.nb_threads, FLAGS.buffer_size = data_dir, 16, 256
    FLAGS.enbl_device_preprocess = mode == 'device_preprocess'
    FLAGS.enbl_device_decode = mode == 'device_decode'
    from pocketflow_b200.learners.learner_utils import create_learner
    lrn = create_learner(None, mod.ModelHelper())
    for _ in range(warmup):
        lrn.train_step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        lrn.train_step()
    torch.cuda.synchronize()
    return steps * batch / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--images', type=int, default=512)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--skip_train', action='store_true')
    ap.add_argument('--skip_decode', action='store_true')
    ap.add_argument('--train_one', nargs=4, metavar=('NET', 'BATCH', 'MODE', 'RECORDS'), help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.train_one:
        net, batch, mode, rec = a.train_one
        r = train_rate(net, int(batch), mode, rec, a.steps, a.warmup)
        emit(stage='train_step', net=net, batch=int(batch), mode=mode, images_per_s=round(r, 1))
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_decode.py measures on a GPU; none is visible')
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip().splitlines()
    emit(card=card[0] if card else 'unknown', host_cpus=len(os.sched_getaffinity(0)))
    jpegs = make_jpegs(a.images)
    emit(images=len(jpegs), mean_bytes=int(np.mean([len(j) for j in jpegs])))
    for t in (8, 16) if not a.skip_decode else ():
        emit(stage='host_decode_crop', nb_threads=t, images_per_s=round(host_rate(jpegs, t), 1))
    for t in (1, 8, 16) if not a.skip_decode else ():
        rate, pack_ms = host_parse_rate(jpegs, t)
        emit(stage='host_parse_crop', nb_threads=t, images_per_s=round(rate, 1), pack_256_ms=round(pack_ms, 2))
    for b in (128, 256) if not a.skip_decode else ():
        rate, ms, stages, scan = device_rate(jpegs, b)
        emit(stage='pf_jpeg_decode', batch=b, images_per_s=round(rate, 1), ms_per_batch=round(ms, 3),
             mean_scan_bytes=int(scan), **stages)
    if a.skip_train:
        return
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, 'jpegs')
        for i, buf in enumerate(jpegs):
            os.makedirs(os.path.join(src, 'n%03d' % (i % 10)), exist_ok=True)
            with open(os.path.join(src, 'n%03d' % (i % 10), '%d.JPEG' % i), 'wb') as f:
                f.write(buf)
        rec = os.path.join(tmp, 'records')
        subprocess.check_call([sys.executable, os.path.join(ROOT, 'tools', 'make_tfrecords.py'), src, rec, 'train', '4'],
                              stdout=subprocess.DEVNULL)
        for net, batch in (('resnet_at_ilsvrc12', 128), ('mobilenet_at_ilsvrc12', 256)):
            for mode in ('host_decode', 'device_preprocess', 'device_decode'):
                # one process per configuration: a learner's device memory is only given back when its process ends
                out = subprocess.run([sys.executable, os.path.abspath(__file__), '--train_one', net, str(batch), mode, rec,
                                      '--steps', str(a.steps), '--warmup', str(a.warmup)], capture_output=True, text=True)
                lines = [l for l in out.stdout.splitlines() if l.startswith('{')]
                print(lines[-1] if lines else json.dumps(dict(stage='train_step', net=net, batch=batch, mode=mode,
                                                              error=out.stderr.strip()[-300:])), flush=True)


if __name__ == '__main__':
    main()
