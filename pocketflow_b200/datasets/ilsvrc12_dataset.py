"""ILSVRC-12 dataset (/root/reference/datasets/ilsvrc12_dataset.py:27-127).

Without --data_dir_local the configs run on synthetic ImageNet-shaped batches (224x224x3, 1001 classes).  With it, the
TFRecord shards the reference trains from (`train-*-of-*`, `validation-*-of-*`; tf.train.Example with
'image/encoded' JPEG bytes, 'image/class/label' and 'image/object/bbox/*', :39-76) are read without TensorFlow
(utils/tf_record.py) and preprocessed the way utils/external/imagenet_preprocessing.py:225-260 does:

* training: one random crop sampled like tf.image.sample_distorted_bounding_box (covering >= 0.1 of a ground-truth
  box, aspect ratio in [0.75, 1.33], area in [0.05, 1] of the image, 100 attempts, else the whole image), random
  left-right flip, bilinear resize to 224x224, per-channel mean subtraction;
* evaluation: aspect-preserving bilinear resize to a 256-pixel short side, central 224x224 crop, mean subtraction.

The resize is TF1's `resize_images(..., BILINEAR, align_corners=False)`: source coordinate = destination index x
(in / out) with no half-pixel offset, fp32 interpolation.  The pipeline mirrors abstract_dataset.py:78-111: shuffled
file list sharded by rank, `cycle_length` files interleaved record by record, a `buffer_size` shuffle buffer,
`nb_threads` decoding threads, `prefetch_size` mini-batches prepared ahead by a background thread so decoding
overlaps the GPU step.

Restated from the published TensorFlow behaviour, not checked against TensorFlow output (absent here).  Known
deviations: JPEG decoding is libjpeg through Pillow (TensorFlow's own build may differ by +-1 LSB on some pixels); the
random stream is numpy's, so crops agree in distribution only; the shuffle buffer holds undecoded records (the
reference shuffles decoded images — same distribution, 100x less memory); the file order is drawn once per stream
rather than once per epoch, which keeps the `take(nb_smpls_val)` / `skip` split disjoint; record payload CRCs are
not checked by default (VERIFY_RECORDS), only the framing CRC."""
import glob
import io
import os
import queue
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from ..flags import FLAGS, DEFINE_integer, DEFINE_boolean
from ..utils.multi_gpu_wrapper import MultiGpuWrapper as mgw
from ..utils.tf_record import parse_example, read_records
from . import jpeg
from .abstract_dataset import AbstractDataset

DEFINE_integer('nb_classes', 1001, '# of classes')
DEFINE_integer('nb_smpls_train', 1281167, '# of samples for training')
DEFINE_integer('nb_smpls_val', 10000, '# of samples for validation')
DEFINE_integer('nb_smpls_eval', 50000, '# of samples for evaluation')
DEFINE_integer('batch_size', 64, 'batch size per GPU for training')
DEFINE_integer('batch_size_eval', 100, 'batch size for evaluation')
DEFINE_boolean('enbl_device_preprocess', False, 'ILSVRC-12: decode + crop on the host, resize / flip / mean on the GPU '
               '(pf_preprocess_images; not validated on a GPU yet)')
DEFINE_boolean('enbl_device_decode', False, 'ILSVRC-12: decode baseline JPEGs on the GPU too (pf_jpeg_decode, bit for bit '
               'with the host decoder; other files are decoded on the host); implies --enbl_device_preprocess')

IMAGE_HEI, IMAGE_WID, IMAGE_CHN = 224, 224, 3
CHANNEL_MEANS = np.array([123.68, 116.78, 103.94], np.float32)       # imagenet_preprocessing.py:40-43
RESIZE_MIN = 256
F32 = np.float32
VERIFY_RECORDS = 'length'        # True: also check every payload CRC (pure Python, ~1 ms per 100 kB image)


def _open(image_buffer):
    from PIL import Image                      # imported on first use: synthetic runs never need Pillow
    return Image.open(io.BytesIO(image_buffer))


def jpeg_shape(image_buffer):
    """(height, width) from the header alone (tf.image.extract_jpeg_shape)."""
    w, h = _open(image_buffer).size
    return h, w


def decode_jpeg(image_buffer, crop=None):
    """uint8 [h, w, 3] RGB; grey-scale and CMYK files are converted like decode_jpeg(channels=3).
    crop = (y, x, h, w): tf.image.decode_and_crop_jpeg."""
    img = _open(image_buffer).convert('RGB')
    if crop is not None:
        y, x, h, w = crop
        img = img.crop((x, y, x + w, y + h))
    return np.asarray(img, np.uint8)


def resize_bilinear(image, out_h, out_w):
    """TF1 resize_bilinear, align_corners=False, no half-pixel centres: [in_h, in_w, c] (uint8 or fp32) -> fp32
    [out_h, out_w, c]; per output pixel top = tl + (tr - tl) * lx, bottom likewise, out = top + (bottom - top) * ly.
    Only the 2 x out_h source rows that are referenced get converted and interpolated."""
    image = np.asarray(image)
    in_h, in_w = image.shape[:2]

    def taps(n_in, n_out):
        src = np.arange(n_out, dtype=F32) * (F32(n_in) / F32(n_out))
        lo = np.floor(src).astype(np.int64)
        hi = np.minimum(np.ceil(src).astype(np.int64), n_in - 1)
        return lo, hi, (src - lo.astype(F32)).astype(F32)
    y0, y1, ly = taps(in_h, out_h)
    x0, x1, lx = taps(in_w, out_w)
    c = image.shape[2]
    rows = np.take(image, np.concatenate([y0, y1]), axis=0)                 # top rows, then bottom rows
    left = np.take(rows, x0, axis=1).astype(F32, copy=False).reshape(2 * out_h, out_w * c)
    right = np.take(rows, x1, axis=1).astype(F32, copy=False).reshape(2 * out_h, out_w * c)
    right -= left
    right *= np.repeat(lx, c)                                               # (tr - tl) * lx
    right += left                                                           # tl + ...  (same roundings, in place)
    top, bot = right[:out_h], right[out_h:]
    bot = bot - top
    bot *= ly[:, None]
    bot += top
    return bot.reshape(out_h, out_w, c)


def smallest_size_at_least(height, width, resize_min=RESIZE_MIN):
    """imagenet_preprocessing.py:167-190 in fp32, truncating casts."""
    scale = F32(resize_min) / F32(min(height, width))
    return int(F32(height) * scale), int(F32(width) * scale)


def central_crop(image, crop_h, crop_w):
    top, left = (image.shape[0] - crop_h) // 2, (image.shape[1] - crop_w) // 2
    return image[top:top + crop_h, left:left + crop_w]


def _rint(v):
    return int(np.rint(F32(v)))                 # lrintf: round half to even


def _random_crop(width, height, min_rel_area, max_rel_area, aspect, rng):
    """One attempt of the crop generator behind sample_distorted_bounding_box: a height drawn uniformly between the
    ones that give the minimum / maximum area at this aspect ratio, then a uniform position.  None: attempt failed."""
    if max_rel_area <= 0 or aspect <= 0 or width <= 0 or height <= 0 or min_rel_area > max_rel_area:
        return None
    min_area, max_area = F32(min_rel_area) * width * height, F32(max_rel_area) * width * height
    h = _rint(np.sqrt(min_area / aspect))
    max_h = _rint(np.sqrt(max_area / aspect))
    if _rint(max_h * aspect) > width:
        max_h = int((width + 0.5 - 1e-7) / aspect)
        if _rint(max_h * aspect) > width:
            max_h -= 1
    max_h = min(max_h, height)
    h = min(h, max_h)
    if h < max_h:
        h += int(rng.integers(0, max_h - h + 1))
    w = _rint(h * aspect)
    area = F32(w * h)
    if area < min_area:
        h += 1
        w = _rint(h * aspect)
        area = F32(w * h)
    if area > max_area:
        h -= 1
        w = _rint(h * aspect)
        area = F32(w * h)
    if area < min_area or area > max_area or w > width or h > height or w <= 0 or h <= 0:
        return None
    y = int(rng.integers(0, height - h)) if h < height else 0
    x = int(rng.integers(0, width - w)) if w < width else 0
    return y, x, h, w


def sample_distorted_bounding_box(height, width, boxes, rng, min_object_covered=0.1, aspect_ratio_range=(0.75, 1.33),
                                  area_range=(0.05, 1.0), max_attempts=100):
    """(y, x, h, w) of a random crop; `boxes` = [[ymin, xmin, ymax, xmax]] in [0, 1] (none: the whole image counts as
    the object, use_image_if_no_bounding_boxes=True).  Falls back to the whole image after max_attempts."""
    rects = []
    for ymin, xmin, ymax, xmax in np.asarray(boxes, F32).reshape(-1, 4):
        rects.append((int(xmin * width), int(ymin * height), int(xmax * width), int(ymax * height)))
    if not rects:
        rects = [(0, 0, width, height)]
    for _ in range(max_attempts):
        aspect = float(rng.uniform(aspect_ratio_range[0], aspect_ratio_range[1]))
        crop = _random_crop(width, height, area_range[0], area_range[1], aspect, rng)
        if crop is None:
            continue
        y, x, h, w = crop
        for bx0, by0, bx1, by1 in rects:
            box_area = max(bx1 - bx0, 0) * max(by1 - by0, 0)
            if box_area <= 0:
                continue
            iw = max(min(x + w, bx1) - max(x, bx0), 0)
            ih = max(min(y + h, by1) - max(y, by0), 0)
            if iw * ih / float(box_area) >= min_object_covered:
                return crop
    return 0, 0, height, width


def preprocess_image(image_buffer, bbox, is_training, rng=None):
    """imagenet_preprocessing.py:225-260 -> fp32 [224, 224, 3]."""
    if is_training:
        h, w = jpeg_shape(image_buffer)
        crop = sample_distorted_bounding_box(h, w, bbox, rng)
        image = decode_jpeg(image_buffer, crop)
        if rng.random() < 0.5:
            image = image[:, ::-1]
        image = resize_bilinear(image, IMAGE_HEI, IMAGE_WID)
    else:
        image = decode_jpeg(image_buffer)
        image = resize_bilinear(image, *smallest_size_at_least(image.shape[0], image.shape[1]))
        image = central_crop(image, IMAGE_HEI, IMAGE_WID)
    return image - CHANNEL_MEANS


IMG_DESC = np.dtype([('offset', '<i8'), ('h', '<i4'), ('w', '<i4'), ('rh', '<i4'), ('rw', '<i4'), ('top', '<i4'),
                     ('left', '<i4'), ('flip', '<i4'), ('reserved', '<i4')])        # pf_img_desc (include/pf_b200.h)


def crop_and_descriptor(image_buffer, bbox, is_training, rng=None):
    """The host half of device-side preprocessing: (uint8 crop [h, w, 3], one IMG_DESC record with offset 0) such
    that pf_preprocess_images — or `preprocess_from_descriptor`, its numpy statement — yields exactly
    `preprocess_image(...)`.  Training: the distorted-bounding-box crop, flip flag drawn here, resized straight to
    224x224.  Evaluation: the whole image, resized to a 256 short side, central 224x224 window."""
    if is_training:
        window, d = crop_window(*jpeg_shape(image_buffer), bbox, True, rng)
        crop = decode_jpeg(image_buffer, window)
    else:
        crop = decode_jpeg(image_buffer)
        window, d = crop_window(crop.shape[0], crop.shape[1], bbox, False)
    return np.ascontiguousarray(crop), d


def crop_window(height, width, bbox, is_training, rng=None):
    """The crop (y, x, h, w) of an image of this size and its IMG_DESC record (offset 0), with the same random draws
    as crop_and_descriptor: the distorted bounding box, then the flip (training); the whole image (evaluation)."""
    d = np.zeros((), IMG_DESC)
    if is_training:
        window = sample_distorted_bounding_box(height, width, bbox, rng)
        d['flip'] = int(rng.random() < 0.5)
        d['rh'], d['rw'] = IMAGE_HEI, IMAGE_WID
    else:
        window = (0, 0, height, width)
        d['rh'], d['rw'] = smallest_size_at_least(height, width)
        d['top'], d['left'] = (int(d['rh']) - IMAGE_HEI) // 2, (int(d['rw']) - IMAGE_WID) // 2
    d['h'], d['w'] = window[2], window[3]
    return window, d


def preprocess_from_descriptor(crop, d, out_h=IMAGE_HEI, out_w=IMAGE_WID):
    """What the device kernel computes for one image, in numpy (the parity reference of pf_preprocess_images)."""
    h, w = int(d['h']), int(d['w'])
    sy = (np.arange(out_h, dtype=F32) + F32(d['top'])) * (F32(h) / F32(d['rh']))
    sx = (np.arange(out_w, dtype=F32) + F32(d['left'])) * (F32(w) / F32(d['rw']))
    y0, x0 = np.floor(sy).astype(np.int64), np.floor(sx).astype(np.int64)
    y1, x1 = np.minimum(np.ceil(sy).astype(np.int64), h - 1), np.minimum(np.ceil(sx).astype(np.int64), w - 1)
    ly, lx = (sy - y0.astype(F32))[:, None, None], (sx - x0.astype(F32))[None, :, None]
    if d['flip']:
        x0, x1 = w - 1 - x0, w - 1 - x1
    img = np.asarray(crop, F32).reshape(h, w, 3)
    tl, tr, bl, br = img[y0][:, x0], img[y0][:, x1], img[y1][:, x0], img[y1][:, x1]
    top = tl + (tr - tl) * lx
    bot = bl + (br - bl) * lx
    return (top + (bot - top) * ly) - CHANNEL_MEANS


def parse_example_proto(example_serialized, nb_classes):
    """ilsvrc12_dataset.py:39-76: (JPEG bytes, one-hot label [nb_classes], bbox [m, 4] as ymin, xmin, ymax, xmax)."""
    f = parse_example(example_serialized)
    encoded = f.get('image/encoded') or [b'']
    label = int(np.asarray(f.get('image/class/label', [-1])).reshape(-1)[0])
    coords = [np.asarray(f.get('image/object/bbox/' + k, []), F32).reshape(-1) for k in ('ymin', 'xmin', 'ymax', 'xmax')]
    n = min(len(c) for c in coords)
    bbox = np.stack([c[:n] for c in coords], axis=1) if n else np.zeros((0, 4), F32)
    onehot = np.zeros(nb_classes, F32)
    if 0 <= label < nb_classes:                  # tf.one_hot: an out-of-range index gives an all-zero row
        onehot[label] = 1.0
    return encoded[0], onehot, bbox


def parse_fn(example_serialized, is_train, nb_classes, rng=None):
    """ilsvrc12_dataset.py:78-97: (image fp32 [224,224,3], one-hot label [nb_classes])."""
    encoded, onehot, bbox = parse_example_proto(example_serialized, nb_classes)
    return preprocess_image(encoded, bbox, is_train, rng), onehot


def parse_packed_fn(example_serialized, is_train, nb_classes, rng=None):
    """The host half only: (uint8 crop, descriptor, one-hot label) — resize / flip / mean happen on the device."""
    encoded, onehot, bbox = parse_example_proto(example_serialized, nb_classes)
    crop, desc = crop_and_descriptor(encoded, bbox, is_train, rng)
    return crop, desc, onehot


def parse_decode_fn(example_serialized, is_train, nb_classes, rng=None):
    """The host half of device decoding: the header is parsed and the crop drawn from its size.  Baseline files give
    (None, IMG_DESC, one-hot label, (JPEG bytes, crop window, pf_jpeg_desc record, scan bytes)) for pf_jpeg_decode;
    every other file is decoded here, as parse_packed_fn does: (uint8 crop, IMG_DESC, one-hot label, None)."""
    encoded, onehot, bbox = parse_example_proto(example_serialized, nb_classes)
    h = jpeg.parse_header(encoded)
    if not h.device:
        crop, desc = crop_and_descriptor(encoded, bbox, is_train, rng)
        return crop, desc, onehot, None
    window, desc = crop_window(h.height, h.width, bbox, is_train, rng)
    return None, desc, onehot, (encoded, window, jpeg.descriptor(h, window), jpeg.scan(h, encoded))


class DecodeBatch(object):
    """One mini-batch for device decoding.  crops: the host-decoded crops back to back (they come first in the crop
    buffer); desc: IMG_DESC [b] with every crop's offset; labels [b, k]; jdesc: pf_jpeg_desc [m] of the m device
    images, whose crops follow the host ones; scans: their entropy-coded segments back to back; ws: workspace int16
    elements; nbytes: the whole crop buffer; fallback: [(JPEG bytes, crop window, crop offset)] of the m device images,
    for the host to decode the ones whose data the kernel flags."""

    def __init__(self, out):
        b = len(out)
        self.desc = np.stack([o[1] for o in out])
        self.labels = np.stack([o[2] for o in out])
        host = [i for i in range(b) if out[i][3] is None]
        dev = [i for i in range(b) if out[i][3] is not None]
        sizes = np.array([out[i][0].size if out[i][3] is None else int(out[i][1]['h']) * int(out[i][1]['w']) * 3
                          for i in host + dev], np.int64)
        offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        self.desc['offset'][host + dev] = offsets[:-1]
        self.nbytes = int(offsets[-1])
        self.crops = (np.concatenate([out[i][0].reshape(-1) for i in host]) if host else np.zeros(0, np.uint8))
        self.fallback = []
        for i in dev:
            encoded, window, d, _ = out[i][3]
            d['crop_offset'] = self.desc['offset'][i]
            self.fallback.append((encoded, window, int(d['crop_offset'])))
        self.jdesc, self.scans, self.ws = jpeg.pack([out[i][3][2] for i in dev], [out[i][3][3] for i in dev])


class ExampleStream(object):
    """generator(b) for BatchIterator(stream=True): endless, shuffled, decoded in a thread pool, prepared ahead."""

    def __init__(self, files, nb_classes, is_train, seed, skip=0, take=None, augment=None, packed=False,
                 device_decode=False):
        self.files, self.k, self.is_train = list(files), nb_classes, is_train
        self.packed = packed or device_decode                 # True: yield (crops, descriptors, labels), see PackedBatchIterator
        self.device_decode = device_decode                    # True: yield DecodeBatch, see DecodeBatchIterator
        self.augment = is_train if augment is None else augment
        self.skip, self.take = skip, take
        self.rng = np.random.default_rng(seed)
        if is_train:
            self.rng.shuffle(self.files)                      # Dataset.list_files(shuffle=True)
        self.buffer_size = max(1, FLAGS.buffer_size)
        self.cycle_length = max(1, FLAGS.cycle_length)
        self.pool = ThreadPoolExecutor(max(1, FLAGS.nb_threads))
        self.ready = queue.Queue(max(1, FLAGS.prefetch_size))
        self.worker, self.batch = None, None
        self.error = None

    def _one_pass(self):
        """parallel_interleave(cycle_length): one record from each of `cycle_length` open files in turn."""
        pending = list(self.files)
        active = []
        n = 0
        while pending or active:
            while pending and len(active) < self.cycle_length:
                active.append(read_records(pending.pop(0), VERIFY_RECORDS))
            for it in list(active):
                try:
                    rec = next(it)
                except StopIteration:
                    active.remove(it)
                    continue
                n += 1
                if n <= self.skip:
                    continue
                if self.take is not None and n > self.skip + self.take:
                    return
                yield rec

    def _shuffled(self):
        """shuffle_and_repeat(buffer_size): a sliding reservoir over the endlessly repeated pass."""
        buf = []
        while True:
            empty = True
            for rec in self._one_pass():
                empty = False
                if len(buf) < self.buffer_size:
                    buf.append(rec)
                    continue
                j = int(self.rng.integers(0, self.buffer_size))
                buf[j], rec = rec, buf[j]
                yield rec
            if empty:
                raise ValueError('no records in ' + ', '.join(self.files[:3]))
            if len(buf) < self.buffer_size:                   # fewer records than the buffer: drain it every pass
                self.rng.shuffle(buf)
                for rec in buf:
                    yield rec
                buf = []

    def _produce(self, b):
        try:
            records = self._shuffled()
            while True:
                raw = [next(records) for _ in range(b)]
                seeds = self.rng.integers(0, 2 ** 62, size=b)
                fn = parse_decode_fn if self.device_decode else (parse_packed_fn if self.packed else parse_fn)
                out = list(self.pool.map(
                    lambda a: fn(a[0], self.augment, self.k, np.random.default_rng(int(a[1]))), zip(raw, seeds)))
                if self.device_decode:
                    self.ready.put(DecodeBatch(out))
                elif self.packed:
                    desc = np.stack([o[1] for o in out])
                    sizes = np.array([o[0].size for o in out], np.int64)
                    desc['offset'] = np.concatenate([[0], np.cumsum(sizes)[:-1]])
                    self.ready.put((np.concatenate([o[0].reshape(-1) for o in out]), desc, np.stack([o[2] for o in out])))
                else:
                    self.ready.put((np.stack([o[0] for o in out]).astype(F32, copy=False), np.stack([o[1] for o in out])))
        except BaseException as e:  # pylint: disable=broad-except
            self.error = e
            self.ready.put(None)

    def __call__(self, b):
        if self.worker is None:
            self.batch = b
            self.worker = threading.Thread(target=self._produce, args=(b,), daemon=True)
            self.worker.start()
        if b != self.batch:
            raise ValueError('the stream was started with batch size %d, asked for %d' % (self.batch, b))
        item = self.ready.get()
        if item is None:
            raise RuntimeError('ILSVRC-12 input pipeline failed') from self.error
        return item


class Ilsvrc12Dataset(AbstractDataset):
    def __init__(self, is_train):
        super().__init__(is_train)   # zero-arg form: survives importlib.reload of this module
        self.batch_size = FLAGS.batch_size if is_train else FLAGS.batch_size_eval
        self.image_shape = (IMAGE_HEI, IMAGE_WID, IMAGE_CHN)
        self.nb_classes = FLAGS.nb_classes

    def _file_generators(self, enbl_trn_val_split):
        if FLAGS.data_disk != 'local':
            raise ValueError('unrecognized data disk: ' + FLAGS.data_disk)     # (HDFS access is cluster glue: out of scope)
        pattern = os.path.join(FLAGS.data_dir_local, 'train-*-of-*' if self.is_train else 'validation-*-of-*')
        files = sorted(glob.glob(pattern))
        if not files:
            raise FileNotFoundError('no ILSVRC-12 TFRecord files match ' + pattern)
        rank, size = (mgw.rank(), mgw.size()) if self.enbl_shard else (0, 1)
        files = files[rank::size] or files                   # filenames.shard(size, rank) (abstract_dataset.py:80-81)
        seed = 8765 + 7919 * rank + (0 if self.is_train else 1)
        if self.is_train and enbl_trn_val_split:
            nv = FLAGS.nb_smpls_val
            return [ExampleStream(files, self.nb_classes, True, seed, skip=nv, packed=FLAGS.enbl_device_preprocess,
                                  device_decode=FLAGS.enbl_device_decode),
                    ExampleStream(files, self.nb_classes, True, seed, take=nv, packed=FLAGS.enbl_device_preprocess,
                                  device_decode=FLAGS.enbl_device_decode)]
        return [ExampleStream(files, self.nb_classes, self.is_train, seed, packed=FLAGS.enbl_device_preprocess,
                              device_decode=FLAGS.enbl_device_decode)]
