"""Seeded JPEG fixtures for the device-decode tests (test_jpeg_cpu.py, test_jpeg_gpu.py), written by Pillow."""
import ctypes
import io
import os
import subprocess

import numpy as np

from pocketflow_b200.datasets import jpeg as J  # noqa: F401  (the parser the fixtures feed)
from pocketflow_b200.utils import tf_record as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [(1, 1), (2, 9), (7, 9), (8, 8), (16, 16), (17, 33), (255, 257), (500, 375)]
SUBSAMPLING = {'444': 0, '422': 1, '420': 2, 'L': None}


def decode_jpeg(buf, crop=None):
    """The host decoder (imported on use: importing the dataset module defines its flags)."""
    from pocketflow_b200.datasets.ilsvrc12_dataset import decode_jpeg as host
    return host(buf, crop)


def jpeg_shape(buf):
    from pocketflow_b200.datasets.ilsvrc12_dataset import jpeg_shape as host
    return host(buf)


def image(h, w, seed):
    """Gradients plus noise: smooth enough for realistic coefficients, noisy enough to use long codes."""
    rng = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([(yy * 3 + seed) % 256, (xx * 5) % 256, ((xx + yy) * 2) % 256], -1)
    return ((rng.randint(0, 256, (h, w, 3)) // 3) + base * 2 // 3).astype(np.uint8)


def jpeg(h, w, seed, sub='420', quality=90, **kw):
    from PIL import Image
    img = Image.fromarray(image(h, w, seed))
    if sub == 'L':
        img = img.convert('L')
    elif sub == 'CMYK':
        img = img.convert('CMYK')
    else:
        kw['subsampling'] = SUBSAMPLING[sub]
    b = io.BytesIO()
    img.save(b, format='JPEG', quality=quality, **kw)
    return b.getvalue()


def png(h, w, seed):
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(image(h, w, seed)).save(b, format='PNG')
    return b.getvalue()


def device_matrix():
    """(name, bytes) of every device-decodable fixture: all sizes x 4:4:4 / 4:2:2 / 4:2:0 / grey x quality 50 / 90 / 100,
    plus optimised Huffman tables and restart intervals in blocks and in rows."""
    out = []
    for h, w in SIZES:
        for sub in SUBSAMPLING:
            for q in (50, 90, 100):
                out.append(('%dx%d_%s_q%d' % (h, w, sub, q), jpeg(h, w, 7 * h + w + q, sub, q)))
        out.append(('%dx%d_420_opt' % (h, w), jpeg(h, w, h + 3, '420', 90, optimize=True)))
        out.append(('%dx%d_422_rst3blocks' % (h, w), jpeg(h, w, h + 4, '422', 90, restart_marker_blocks=3)))
        out.append(('%dx%d_L_rst1row' % (h, w), jpeg(h, w, h + 5, 'L', 90, restart_marker_rows=1)))
        out.append(('%dx%d_420_rst2rows' % (h, w), jpeg(h, w, h + 6, '420', 75, restart_marker_rows=2)))
    return out


def host_matrix():
    """(name, bytes) of files the parser must send to the host decoder."""
    return [('progressive', jpeg(64, 80, 1, '420', 90, progressive=True)),
            ('progressive_L', jpeg(33, 17, 2, 'L', 90, progressive=True)),
            ('cmyk', jpeg(40, 48, 3, 'CMYK', 90)),
            ('png', png(30, 20, 4)),
            ('truncated', jpeg(120, 160, 5, '420', 90)[:-900]),
            ('empty', b'')]


def crops(h, w):
    """Windows (y, x, h, w): the whole image, an interior one and one touching each edge."""
    out = [(0, 0, h, w)]
    if h > 2 and w > 2:
        out.append((h // 3, w // 4, max(1, h // 2), max(1, w // 2)))
    out += [(0, w // 3, max(1, h // 4), w - w // 3), (h // 2, 0, h - h // 2, max(1, w // 5)),
            (h - max(1, h // 3), w // 2, max(1, h // 3), w - w // 2), (h // 4, w - max(1, w // 6), h - h // 4, max(1, w // 6))]
    return out


def host_decoder(tmp_path):
    """csrc/pf_jpeg.cu compiled for the host with -DPF_JPEG_HOST_TEST: pf_test_jpeg_decode_host(data, desc, n, ws,
    crops, status), the three kernels' bodies as loops over the same functions."""
    lib = str(tmp_path / 'libjpeg_host.so')
    subprocess.check_call(['g++', '-O2', '-std=c++17', '-x', 'c++', '-D__host__=', '-D__device__=', '-DPF_JPEG_HOST_TEST',
                           '-fPIC', '-shared', '-I', os.path.join(ROOT, 'include'), '-o', lib,
                           os.path.join(ROOT, 'pocketflow_b200', 'csrc', 'pf_jpeg.cu')])
    L = ctypes.CDLL(lib)
    L.pf_test_jpeg_decode_host.restype = None
    L.pf_test_jpeg_decode_host.argtypes = [ctypes.c_void_p] * 2 + [ctypes.c_int] + [ctypes.c_void_p] * 3
    return L


def host_preprocessor(tmp_path):
    """csrc/pf_preproc.cu compiled for the host with -DPF_PREPROC_HOST_TEST: pf_test_preprocess_host."""
    lib = str(tmp_path / 'libpreproc_host.so')
    subprocess.check_call(['g++', '-O2', '-std=c++17', '-x', 'c++', '-D__host__=', '-D__device__=', '-DPF_PREPROC_HOST_TEST',
                           '-ffp-contract=off', '-fPIC', '-shared', '-I', os.path.join(ROOT, 'include'), '-o', lib,
                           os.path.join(ROOT, 'pocketflow_b200', 'csrc', 'pf_preproc.cu')])
    fn = ctypes.CDLL(lib).pf_test_preprocess_host
    fn.restype = None
    fn.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float,
                   ctypes.c_float, ctypes.c_float, ctypes.c_void_p]
    return fn


def batch(items):
    """items = [(bytes, crop or None)] of device-decodable files -> (descriptor table, scan bytes uint8, workspace
    int16 elements, crop bytes, [(offset, shape)]) with the crops laid out back to back."""
    from pocketflow_b200.datasets import jpeg as J
    descs, scans, layout, off = [], [], [], 0
    for buf, crop in items:
        h = J.parse_header(buf)
        assert h.device, h.reason
        c = crop if crop is not None else (0, 0, h.height, h.width)
        descs.append(J.descriptor(h, c, crop_offset=off))
        scans.append(J.scan(h, buf))
        layout.append((off, (c[2], c[3], 3)))
        off += c[2] * c[3] * 3
    table, data, ws = J.pack(descs, scans)
    return table, data, ws, off, layout


def corrupt_huffman(buf):
    """The same file with 6 stuffed 0xFF bytes (48 one-bits) in the middle of its scan: no Huffman code is 16 ones,
    so the decoder meets a code that is not in its table wherever it is in the bit stream."""
    from pocketflow_b200.datasets import jpeg as J
    h = J.parse_header(buf)
    p = h.scan_start + h.scan_bytes // 2
    while buf[p - 1] == 0xFF or buf[p] == 0xFF or buf[p + 12] == 0x00:
        p += 1
    return buf[:p] + b'\xff\x00' * 6 + buf[p + 12:]


def example(jpeg, label, boxes=()):
    boxes = np.asarray(boxes, np.float32).reshape(-1, 4)
    return R.encode_example({
        'image/encoded': jpeg, 'image/class/label': [label], 'image/class/text': b'n0000',
        'image/object/bbox/ymin': boxes[:, 0], 'image/object/bbox/xmin': boxes[:, 1],
        'image/object/bbox/ymax': boxes[:, 2], 'image/object/bbox/xmax': boxes[:, 3]})


def shard_images(i):
    """Mostly baseline files, with a progressive one, a CMYK one, a PNG and a corrupted scan among them."""
    kinds = [lambda s: jpeg(180 + 8 * (s % 5), 250 - 6 * (s % 7), s, '420'),
             lambda s: jpeg(170, 230, s, 'L'),
             lambda s: jpeg(190, 260, s, '422', 95, restart_marker_rows=2),
             lambda s: jpeg(200, 240, s, '420', 90, progressive=True),
             lambda s: jpeg(160, 220, s, 'CMYK'),
             lambda s: png(150, 200, s),
             lambda s: corrupt_huffman(jpeg(210, 250, s, '444')),
             lambda s: jpeg(176, 256, s, '444', 100)]
    return kinds[i % len(kinds)](i)


def write_shards(d):
    os.makedirs(d, exist_ok=True)
    for shard in range(2):
        R.write_records(os.path.join(d, 'train-%05d-of-00002' % shard),
                        [example(shard_images(8 * shard + i), 1 + 8 * shard + i, [[0.2, 0.2, 0.9, 0.8]] if i % 2 else [])
                         for i in range(8)])
    R.write_records(os.path.join(d, 'validation-00000-of-00001'), [example(shard_images(3 + i), 500 + i) for i in range(6)])


def pipeline_batches(d, mode, is_train, n, b=4):
    """n batches of the image / label placeholders through AbstractLearner.feed, mode in host | preprocess | decode."""
    import torch
    from types import SimpleNamespace
    from pocketflow_b200 import graph as G
    from pocketflow_b200.flags import FLAGS
    from pocketflow_b200.datasets import ilsvrc12_dataset as D
    from pocketflow_b200.learners.abstract_learner import AbstractLearner
    FLAGS.reset()
    FLAGS.data_dir_local, FLAGS.batch_size, FLAGS.batch_size_eval, FLAGS.nb_classes = d, b, b, 1001
    FLAGS.buffer_size, FLAGS.nb_threads, FLAGS.prefetch_size = 5, 2, 1
    FLAGS.enbl_device_preprocess = mode == 'preprocess'
    FLAGS.enbl_device_decode = mode == 'decode'
    with G.Graph().as_default():
        ds = D.Ilsvrc12Dataset(is_train)
        ds.batch_size, ds.nb_classes = b, 1001
        it = ds.build()
        images, labels = it.get_next()
    dev = torch.device('cuda') if torch.cuda.is_available() and mode != 'host' else torch.device('cpu')
    ex = SimpleNamespace(buf={images: torch.full(images.shape, float('nan'), device=dev),
                              labels: torch.zeros(labels.shape, device=dev)})
    learner = SimpleNamespace(_feed_packed=lambda *a: AbstractLearner._feed_packed(None, *a))
    out = []
    for _ in range(n):
        AbstractLearner.feed(learner, ex, it)
        out.append((ex.buf[images].cpu().numpy().copy(), ex.buf[labels].cpu().numpy().copy()))
    FLAGS.reset()
    return out, it
