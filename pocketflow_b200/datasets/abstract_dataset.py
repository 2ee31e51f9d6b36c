"""Abstract class for datasets (/root/reference/datasets/abstract_dataset.py:34-111).

`build()` returns an iterator whose `get_next()` yields the symbolic (images, labels) placeholders
of the current graph — what tf.data's `iterator.get_next()` returns in the reference — and whose
`next_batch()` produces the host mini-batch (pinned memory) that the learner copies into them
every step.  Multi-GPU training shards the stream by rank (reference: file-level sharding, :80-81)."""
from abc import ABC

import numpy as np
import torch

from .. import graph as G
from ..flags import FLAGS, DEFINE_string, DEFINE_integer
from ..utils.multi_gpu_wrapper import MultiGpuWrapper as mgw

DEFINE_string('data_disk', 'local', 'data disk\'s location (\'local\' | \'hdfs\')')
DEFINE_string('data_hdfs_host', None, 'HDFS host for data files')
DEFINE_string('data_dir_local', None, 'data directory - local (None: synthetic batches)')
DEFINE_string('data_dir_hdfs', None, 'data directory - HDFS')
DEFINE_integer('cycle_length', 4, '# of datasets to interleave from in parallel')
DEFINE_integer('nb_threads', 8, '# of threads for preprocessing the dataset')
DEFINE_integer('buffer_size', 1024, '# of elements to be buffered when prefetching')
DEFINE_integer('prefetch_size', 8, '# of mini-batches to be buffered when prefetching')


POOL_SIZE = 8   # distinct synthetic mini-batches kept in pinned host memory


class BatchIterator(object):
    def __init__(self, batch_size, image_shape, nb_classes, generator, stream=False):
        """generator(b) -> (images [b,...] float32, one-hot labels [b,k] float32) as numpy arrays.
        stream=False: the synthetic case — POOL_SIZE batches are generated once and cycled.
        stream=True : a real dataset — every call draws a fresh batch from the generator into one of POOL_SIZE
                      rotating pinned buffers.  The consumer calls `copy_enqueued()` right after it has enqueued
                      the async host->device copy of the batch it was handed; a slot is rewritten only after THAT
                      copy has executed (the host can run many steps ahead of the GPU — steps are enqueued without a
                      per-step synchronisation — so "POOL_SIZE calls later" alone is not a guarantee)."""
        self.batch_size, self.image_shape, self.nb_classes = batch_size, tuple(image_shape), nb_classes
        self.generator = generator
        self.stream = stream
        self.images, self.labels = None, None
        self.pin = torch.cuda.is_available()
        self.pool, self.pool_size, self.cursor = [], POOL_SIZE, 0
        self.slot_copied, self.last_slot = {}, None        # slot -> CUDA event recorded after its H2D copy was enqueued

    def copy_enqueued(self):
        """To be called by the consumer on the stream it has just enqueued the H2D copy of the last batch on."""
        if self.stream and self.pin and self.last_slot is not None:
            ev = self.slot_copied.get(self.last_slot)
            if ev is None:
                ev = self.slot_copied[self.last_slot] = torch.cuda.Event()
            ev.record()

    def _wait_slot_free(self, slot):
        ev = self.slot_copied.get(slot)
        if ev is not None:
            ev.synchronize()

    def get_next(self):
        """Symbolic (images, labels) of the current default graph."""
        self.images = G.placeholder((self.batch_size,) + self.image_shape, 'images')
        self.labels = G.placeholder((self.batch_size, self.nb_classes), 'labels')
        self.images.iterator = self
        return self.images, self.labels

    def prefill(self):
        """Generate the whole pool now (keeps host-side synthesis out of timed regions)."""
        while len(self.pool) < self.pool_size:
            self.next_batch()

    def next_batch(self):
        """Next mini-batch as (images, labels) in pinned host memory.  The synthetic stream is a pool of
        POOL_SIZE distinct pre-generated batches cycled in order (what tf.data's prefetch buffer holds
        in the reference: decoding happens off the step's critical path, datasets/abstract_dataset.py:107)."""
        if len(self.pool) < self.pool_size:
            img, lab = self.generator(self.batch_size)
            hi = torch.empty((self.batch_size,) + self.image_shape, dtype=torch.float32, pin_memory=self.pin)
            hl = torch.empty((self.batch_size, self.nb_classes), dtype=torch.float32, pin_memory=self.pin)
            hi.copy_(torch.from_numpy(img))
            hl.copy_(torch.from_numpy(lab))
            self.pool.append((hi, hl))
            self.last_slot = len(self.pool) - 1
            return hi, hl
        self.last_slot = self.cursor % self.pool_size
        out = self.pool[self.last_slot]
        self.cursor += 1
        if self.stream:
            img, lab = self.generator(self.batch_size)
            self._wait_slot_free(self.last_slot)
            out[0].copy_(torch.from_numpy(img))
            out[1].copy_(torch.from_numpy(lab))
        return out


class PackedBatchIterator(BatchIterator):
    """Mini-batches for device-side preprocessing: generator(b) -> (uint8 array holding every decoded crop back to
    back, descriptor table [b] (one 40-byte pf_img_desc each), one-hot labels [b, k]).  `next_packed()` stages them in
    rotating pinned buffers (the crop buffer of a slot grows on demand); the learner copies the three pieces to the
    GPU and runs pf_preprocess_images into the step's image placeholder."""

    def __init__(self, batch_size, image_shape, nb_classes, generator):
        super().__init__(batch_size, image_shape, nb_classes, generator, stream=True)
        self.slots = [None] * POOL_SIZE

    def next_batch(self):
        raise TypeError('a packed iterator yields undecoded-size crops: use next_packed()')

    def next_packed(self):
        """(crops uint8 [capacity >= nbytes], nbytes, descriptors uint8 [b * 40], labels fp32 [b, k]) in pinned memory."""
        crops, desc, lab = self.generator(self.batch_size)
        desc_bytes = np.ascontiguousarray(desc).view(np.uint8).reshape(-1)
        i = self.last_slot = self.cursor % POOL_SIZE
        self.cursor += 1
        self._wait_slot_free(i)
        slot = self.slots[i]
        if slot is None or slot[0].numel() < crops.size:
            cap = int(crops.size * 1.25) + 4096
            slot = self.slots[i] = (torch.empty(cap, dtype=torch.uint8, pin_memory=self.pin),
                                    torch.empty(desc_bytes.size, dtype=torch.uint8, pin_memory=self.pin),
                                    torch.empty((self.batch_size, self.nb_classes), dtype=torch.float32, pin_memory=self.pin))
        slot[0][:crops.size].copy_(torch.from_numpy(crops))
        slot[1].copy_(torch.from_numpy(desc_bytes))
        slot[2].copy_(torch.from_numpy(lab))
        return slot[0], int(crops.size), slot[1], slot[2]


class DecodeBatchIterator(PackedBatchIterator):
    """Mini-batches for device decoding: generator(b) -> a DecodeBatch (datasets/ilsvrc12_dataset.py).  `next_decode()`
    stages its arrays in rotating pinned buffers; the learner decodes the device images with pf_jpeg_decode one
    batch ahead, then runs pf_preprocess_images."""

    FIELDS = ('crops', 'desc', 'labels', 'jdesc', 'scans')

    def next_packed(self):
        raise TypeError('a decode iterator yields undecoded JPEG scans: use next_decode()')

    def next_decode(self):
        """({field: (pinned uint8 buffer, nbytes)} for FIELDS, the DecodeBatch)."""
        batch = self.generator(self.batch_size)
        i = self.last_slot = self.cursor % POOL_SIZE
        self.cursor += 1
        self._wait_slot_free(i)
        slot = self.slots[i] = self.slots[i] or {}
        staged = {}
        for key in self.FIELDS:
            flat = np.ascontiguousarray(getattr(batch, key)).reshape(-1).view(np.uint8)
            buf = slot.get(key)
            if buf is None or buf.numel() < flat.size:
                buf = slot[key] = torch.empty(int(flat.size * 1.25) + 4096, dtype=torch.uint8, pin_memory=self.pin)
            buf[:flat.size].copy_(torch.from_numpy(flat))
            staged[key] = (buf, int(flat.size))
        return staged, batch


class AbstractDataset(ABC):
    def __init__(self, is_train):
        self.is_train = is_train
        self.batch_size = None
        self.image_shape = None
        self.nb_classes = None
        self.enbl_shard = (is_train and FLAGS.enbl_multi_gpu)

    def _generator(self):
        """Synthetic stream shaped like the real data (SURVEY §8d): standardised images
        ~ N(0,1), uniformly random one-hot labels.  Seeds: images 1234, labels 1235 (+rank when
        sharded, so every rank sees its own slice of the global batch)."""
        rank = mgw.rank() if self.enbl_shard else 0
        rng_i = np.random.default_rng(1234 + 7919 * rank + (0 if self.is_train else 1))
        rng_l = np.random.default_rng(1235 + 7919 * rank + (0 if self.is_train else 1))
        shape, k = self.image_shape, self.nb_classes

        def gen(b):
            img = rng_i.standard_normal(size=(b,) + tuple(shape), dtype=np.float32)
            lab = np.zeros((b, k), np.float32)
            lab[np.arange(b), rng_l.integers(0, k, size=b)] = 1.0
            return img, lab
        return gen

    def _file_generators(self, enbl_trn_val_split):
        """Real-data hook: subclasses that can read their files return generator(s) here (None: synthetic)."""
        return None

    def build(self, enbl_trn_val_split=False):
        gens = self._file_generators(enbl_trn_val_split) if FLAGS.data_dir_local else None
        if gens is not None:
            its = [DecodeBatchIterator(self.batch_size, self.image_shape, self.nb_classes, g_)
                   if getattr(g_, 'device_decode', False) else
                   PackedBatchIterator(self.batch_size, self.image_shape, self.nb_classes, g_)
                   if getattr(g_, 'packed', False) else
                   BatchIterator(self.batch_size, self.image_shape, self.nb_classes, g_, stream=True) for g_ in gens]
            return tuple(its) if len(its) > 1 else its[0]
        it = BatchIterator(self.batch_size, self.image_shape, self.nb_classes, self._generator())
        if self.is_train and enbl_trn_val_split:
            return it, BatchIterator(self.batch_size, self.image_shape, self.nb_classes, self._generator())
        return it
