"""Abstract class for learners — the plugin surface of the reference
(/root/reference/learners/abstract_learner.py:32-158), without TensorFlow."""
from abc import ABC
from abc import abstractmethod
import contextlib
import glob
import os
import shutil
import subprocess

import numpy as np
import torch

from .. import ops
from ..flags import FLAGS, DEFINE_string, DEFINE_integer, DEFINE_boolean
from ..utils.misc_utils import auto_barrier as auto_barrier_impl
from ..utils.misc_utils import is_primary_worker as is_primary_worker_impl
from ..utils.multi_gpu_wrapper import MultiGpuWrapper as mgw
from ..utils import tf_bundle

DEFINE_string('model_http_url', None, 'HTTP/HTTPS url for remote model files')
DEFINE_integer('summ_step', 100, 'summarizaton step size')
DEFINE_integer('save_step', 10000, 'model saving step size')
DEFINE_string('save_path', './models/model.ckpt', 'model\'s save path')
DEFINE_string('save_path_eval', './models_eval/model.ckpt', 'model\'s save path for evaluation')
DEFINE_string('ckpt_format', 'npz', 'checkpoint format to write: npz | tf (TensorFlow V2 bundle)')
DEFINE_boolean('enbl_dst', False, 'enable the distillation loss for training')
DEFINE_boolean('enbl_warm_start', False, 'enable warm start for training')
DEFINE_boolean('enbl_compact_ft', False, 'fine-tune the channel-pruned model at its pruned width (chn-pruned-gpu / chn-pruned-rmt)')


def latest_checkpoint(ckpt_dir):
    """tf.train.latest_checkpoint over both formats this build reads: its own .npz files and TensorFlow V2 bundles
    named by the directory's `checkpoint` state file (what the reference's savers and model archives contain);
    the newer of the two wins."""
    files = sorted(glob.glob(os.path.join(ckpt_dir, '*.npz')), key=os.path.getmtime)
    native = files[-1] if files else None
    bundle = tf_bundle.latest_checkpoint(ckpt_dir)
    if bundle is not None and (native is None or os.path.getmtime(bundle + '.index') >= os.path.getmtime(native)):
        return bundle
    return native


def save_checkpoint(path, state, step=None):
    """tf.train.Saver.save(sess, path, global_step): `--ckpt_format npz` (default) or `tf`, the V2 bundle the
    reference's own tools restore (variable names without the ':0' output suffix, plus `global_step`)."""
    os.makedirs(os.path.dirname(path) or '.', exist_ok=True)
    if FLAGS.ckpt_format == 'tf':
        tensors = {(k[:-2] if k.endswith(':0') else k): v for k, v in state.items()}
        if step is not None:
            tensors.setdefault('global_step', np.asarray(step, np.int64))
        return tf_bundle.save(path, tensors, step)
    if FLAGS.ckpt_format != 'npz':
        raise ValueError('unknown --ckpt_format %r (npz | tf)' % FLAGS.ckpt_format)
    fn = path + ('-%d' % step if step is not None else '') + '.npz'
    np.savez(fn, **{k.replace('/', '|'): v for k, v in state.items()})
    return fn


def load_checkpoint(fn):
    """{variable name (with ':0'): array} from either format; `fn` is what latest_checkpoint returned."""
    if fn.endswith('.npz'):
        d = np.load(fn)
        return {k.replace('|', '/'): d[k] for k in d.files}
    return {k + ':0': v for k, v in tf_bundle.load(fn).items()}


def calc_prune_ratio(tensors):
    """Overall pruning ratio 1 - nnz/size (weight_sparsification/learner.py:51-65)."""
    nnz = sum(int(torch.count_nonzero(t).item()) for t in tensors)
    tot = sum(t.numel() for t in tensors)
    return np.float32(np.float32(1.0) - np.float32(nnz) / np.float32(tot))


class AbstractLearner(ABC):  # pylint: disable=too-many-instance-attributes
    """A learner takes a ModelHelper (data pipeline + model definition) and performs training or
    evaluation with its specific algorithm (abstract_learner.py:41-54)."""

    def __init__(self, sm_writer, model_helper):
        self.sm_writer = sm_writer
        self.data_scope = 'data'
        self.model_scope = 'model'

        # one process per GPU; torch.distributed replaces Horovod + mpi4py (abstract_learner.py:68-74)
        if FLAGS.enbl_multi_gpu:
            mgw.init()
            self.mpi_comm = mgw
        else:
            self.mpi_comm = None
        if torch.cuda.is_available():
            self.device = torch.device('cuda', mgw.local_rank() if FLAGS.enbl_multi_gpu else 0)
            torch.cuda.set_device(self.device)
        else:
            self.device = torch.device('cpu')

        self.build_dataset_train = model_helper.build_dataset_train
        self.build_dataset_eval = model_helper.build_dataset_eval
        self.forward_train = model_helper.forward_train
        self.forward_eval = model_helper.forward_eval
        self.calc_loss = model_helper.calc_loss
        self.setup_lrn_rate = model_helper.setup_lrn_rate
        self.warm_start = model_helper.warm_start
        self.dump_n_eval = model_helper.dump_n_eval
        self.model_name = model_helper.model_name
        self.dataset_name = model_helper.dataset_name
        self.forward_w_labels = model_helper.forward_w_labels

        self.ckpt_file = 'models_%s_at_%s.tar.gz' % (self.model_name, self.dataset_name)
        self.graph_train = None
        self._iterator_eval = None

    @abstractmethod
    def train(self):
        """Train a model and periodically produce checkpoint files."""

    @abstractmethod
    def evaluate(self):
        """Restore a model from the latest checkpoint files and then evaluate it."""

    def download_model(self):
        """Download remote model files and then uncompress (abstract_learner.py:105-125)."""
        if latest_checkpoint(os.path.dirname(FLAGS.save_path)) is not None:
            return
        if FLAGS.model_http_url is None:
            raise ValueError('local model files do not exist and <model_http_url> is not set')
        subprocess.call(['wget', os.path.join(FLAGS.model_http_url, self.ckpt_file)])
        if os.path.exists(self.ckpt_file):
            if os.path.isdir(os.path.dirname(FLAGS.save_path)):
                shutil.rmtree(os.path.dirname(FLAGS.save_path))
            subprocess.call(['tar', '-xvf', self.ckpt_file])
        else:
            raise FileNotFoundError(
                'pre-trained model not avaialable: {} / {}'.format(self.model_name, self.dataset_name))

    def auto_barrier(self):
        auto_barrier_impl(self.mpi_comm)

    # ------------------------------------------------------------------ checkpoints
    def restore_model(self, path, store=None, require='all', optional=()):
        """saver.restore(sess, tf.train.latest_checkpoint(dirname(path))) — every learner's __restore_model (e.g.
        learners/full_precision/learner.py:193-205).  A checkpoint that does not hold the model's trainable variables
        (wrong net, wrong scope) raises instead of 'restoring' nothing."""
        ckpt_dir = os.path.dirname(path)
        fn = latest_checkpoint(ckpt_dir) if os.path.isdir(ckpt_dir) else None
        if fn is None:
            raise ValueError('no checkpoint found in ' + ckpt_dir)
        store = self.sess_train.store if store is None else store
        found, total = store.load_state_dict(load_checkpoint(fn), strict=False, require=require, optional=optional)
        print('model restored from %s (%d of %d trainable variables)' % (fn, found, total))
        return fn

    def restore_for_eval(self, path):
        """The reference's evaluate() first restores the latest checkpoint into its separate evaluation graph.  Here the
        evaluation pass runs on the training executor's own parameters: while training they ARE what was just saved
        (nothing to do); under --exec_mode eval nothing has been trained, so the checkpoint must be loaded."""
        if FLAGS.exec_mode == 'eval':
            self.restore_model(path)

    def eval_nb_iters(self, nb_iters=None):
        """ceil(nb_smpls_eval / batch_size_eval) (e.g. learners/full_precision/learner.py:95).  Real data is read at
        the step's batch size (eval_iterator), so the count follows that size; the synthetic pool keeps the
        reference's count."""
        if nb_iters:
            return int(nb_iters)
        bs = self.iterator_train.batch_size if FLAGS.data_dir_local else FLAGS.batch_size_eval
        return int(np.ceil(float(FLAGS.nb_smpls_eval) / bs))

    def eval_losses(self, nb_iters=None):
        """fetch_losses() of each of eval_nb_iters(nb_iters) evaluation batches, run through sess_train's forward pass"""
        ex = self.sess_train
        out = []
        for _ in range(self.eval_nb_iters(nb_iters)):
            self.feed(ex, self.eval_iterator())
            ex.forward_eval_loss()
            out.append(ex.fetch_losses())
        return out

    @classmethod
    def is_primary_worker(cls, scope='global'):
        return is_primary_worker_impl(scope)

    @property
    def vars(self):
        """List of all global variables of the model scope."""
        return [v for v in self.graph_train.variables.values() if v.name.startswith(self.model_scope + '/')]

    @property
    def trainable_vars(self):
        return [v for v in self.vars if v.trainable]

    @property
    def update_ops(self):
        """BN moving-statistic updates: fused into the BN statistics kernel here."""
        return []

    def eval_iterator(self):
        """The stream `evaluate()` draws from.  The reference evaluates on `build_dataset_eval()` in a separate graph
        (e.g. learners/full_precision/learner.py:140-160); here the evaluation pass reuses the step's buffers, so the
        evaluation split is read at the TRAINING batch size and copied into the same input placeholders.  Synthetic
        runs (no --data_dir_local) have no split and keep cycling the training pool."""
        if not FLAGS.data_dir_local:
            return self.iterator_train
        if self._iterator_eval is None:
            it = self.build_dataset_eval()
            it.batch_size = self.iterator_train.batch_size          # buffers are allocated lazily, at the first batch
            it.images, it.labels = self.iterator_train.images, self.iterator_train.labels
            self._iterator_eval = it
        return self._iterator_eval

    # ------------------------------------------------------------------ shared step plumbing
    def feed(self, executor, iterator):
        """Host -> device copy of the next mini-batch from pinned memory (the only per-step H2D).

        Input pipelining (what tf.data's prefetch_to_device does for the reference,
        datasets/abstract_dataset.py:107): the copy of batch i+1 runs on a copy stream into a staging buffer while
        step i computes; at the start of step i+1 the staged batch is moved into the graph's input buffers with a
        device-to-device copy (155 MB: ~0.05 ms).  Every step still copies exactly one batch host -> device."""
        dev_images, dev_labels = executor.buf[iterator.images], executor.buf[iterator.labels]
        if hasattr(iterator, 'next_packed'):
            return self._feed_packed(iterator, dev_images, dev_labels)
        if dev_images.device.type != 'cuda' or os.environ.get('PF_INPUT_PREFETCH', '1') == '0':
            images, labels = iterator.next_batch()
            dev_images.copy_(images, non_blocking=True)
            dev_labels.copy_(labels, non_blocking=True)
            iterator.copy_enqueued()
            return images.numel() * 4 + labels.numel() * 4
        st = getattr(iterator, '_staging', None)
        main = torch.cuda.current_stream()
        if st is None:
            st = iterator._staging = dict(images=torch.empty_like(dev_images), labels=torch.empty_like(dev_labels),
                                          stream=torch.cuda.Stream(), ready=torch.cuda.Event(), free=torch.cuda.Event(),
                                          primed=False)
            st['free'].record(main)

        def stage_next():
            images, labels = iterator.next_batch()
            st['stream'].wait_event(st['free'])                # the previous staged batch has been consumed
            with torch.cuda.stream(st['stream']):
                st['images'].copy_(images, non_blocking=True)
                st['labels'].copy_(labels, non_blocking=True)
                st['ready'].record()
                iterator.copy_enqueued()
            return images.numel() * 4 + labels.numel() * 4
        if not st['primed']:
            stage_next()
            st['primed'] = True
        main.wait_event(st['ready'])
        dev_images.copy_(st['images'], non_blocking=True)
        dev_labels.copy_(st['labels'], non_blocking=True)
        st['free'].record(main)
        return stage_next()                                    # overlaps with the step that is about to run

    def _feed_packed(self, iterator, dev_images, dev_labels):
        """Device-side input preprocessing (--enbl_device_preprocess): the host decodes and crops, the uint8 crops
        (about a third of the fp32 batch's bytes), their descriptor table and the labels are copied, and ONE kernel
        (pf_preprocess_images) resizes / flips / centres them straight into the step's image placeholder."""
        if hasattr(iterator, 'next_decode'):
            return AbstractLearner._feed_decoded(iterator, dev_images, dev_labels)
        crops, nbytes, desc, labels = iterator.next_packed()
        dev = getattr(iterator, '_packed_dev', None)
        if dev is None or dev[0].numel() < nbytes:
            dev = iterator._packed_dev = (torch.empty(int(nbytes * 1.25) + 4096, dtype=torch.uint8, device=dev_images.device),
                                          torch.empty(desc.numel(), dtype=torch.uint8, device=dev_images.device))
        dev[0][:nbytes].copy_(crops[:nbytes], non_blocking=True)
        dev[1].copy_(desc, non_blocking=True)
        dev_labels.copy_(labels, non_blocking=True)
        iterator.copy_enqueued()
        ops.preprocess_images(dev[0], dev[1], dev_images)
        return nbytes + desc.numel() + labels.numel() * 4

    @staticmethod
    def _feed_decoded(iterator, dev_images, dev_labels):
        """Device-side JPEG decoding (--enbl_device_decode).  Batch i+1's scans are copied and decoded by
        pf_jpeg_decode on a side stream while step i runs, into one of two device slots (so a decode never overwrites
        crops that pf_preprocess_images still reads); its per-image status comes back to pinned memory.  When batch
        i+1 is fed, the host decodes the images the kernel flagged and copies their crops into place, then
        pf_preprocess_images runs on the main stream.  Returns the bytes copied host -> device for the staged batch."""
        cuda = dev_images.device.type == 'cuda'
        st = getattr(iterator, '_decode_state', None)
        if st is None:
            st = iterator._decode_state = dict(slots=[{}, {}], next=0, primed=False,
                                               stream=torch.cuda.Stream() if cuda else None)
            if cuda:
                for s in st['slots']:
                    s['ready'], s['free'] = torch.cuda.Event(), torch.cuda.Event()
                    s['free'].record(torch.cuda.current_stream())

        def grown(s, key, n, dtype, pin=False):
            t = s.get(key)
            if t is None or t.numel() < n:
                cap = max(int(n * 1.25) + 64, 64)
                t = s[key] = (torch.empty(cap, dtype=dtype, pin_memory=True) if pin else
                              torch.empty(cap, dtype=dtype, device=dev_images.device))
            return t

        def stage(s):
            staged, batch = iterator.next_decode()
            if cuda:
                st['stream'].wait_event(s['free'])                     # preprocessing of the slot's last batch is done
            with torch.cuda.stream(st['stream']) if cuda else contextlib.nullcontext():
                crops = grown(s, 'crops', max(batch.nbytes, 1), torch.uint8)
                desc = grown(s, 'desc', staged['desc'][1], torch.uint8)
                labels = grown(s, 'labels', staged['labels'][1], torch.uint8)
                m = len(batch.jdesc)
                for key, dst in (('crops', crops), ('desc', desc), ('labels', labels)):
                    buf, n = staged[key]
                    dst[:n].copy_(buf[:n], non_blocking=True)
                status = grown(s, 'status', max(m, 1), torch.int32)
                status_host = grown(s, 'status_host', max(m, 1), torch.int32, pin=cuda)
                if m:
                    jdesc = grown(s, 'jdesc', staged['jdesc'][1], torch.uint8)
                    scans = grown(s, 'scans', max(staged['scans'][1], 1), torch.uint8)
                    ws = grown(s, 'ws', max(batch.ws, 64), torch.int16)
                    for key, dst in (('jdesc', jdesc), ('scans', scans)):
                        buf, n = staged[key]
                        dst[:n].copy_(buf[:n], non_blocking=True)
                    ops.jpeg_decode(scans, jdesc, m, ws, crops, status)
                    status_host[:m].copy_(status[:m], non_blocking=True)
                iterator.copy_enqueued()
                if cuda:
                    s['ready'].record()
            s['batch'] = batch
            return sum(n for _, n in staged.values())

        if not st['primed']:
            stage(st['slots'][st['next']])
            st['primed'] = True
        cur = st['slots'][st['next']]
        batch = cur['batch']
        if cuda:
            cur['ready'].synchronize()
        flagged = np.flatnonzero(cur['status_host'][:len(batch.jdesc)].numpy()) if len(batch.jdesc) else []
        if len(flagged):
            from ..datasets.ilsvrc12_dataset import decode_jpeg
        for j in flagged:                                  # data the kernel does not vouch for: the host decoder's result
            encoded, window, offset = batch.fallback[j]
            crop = decode_jpeg(encoded, window).reshape(-1).copy()
            cur['crops'][offset:offset + crop.size].copy_(torch.from_numpy(crop))
        main = torch.cuda.current_stream() if cuda else None
        if cuda:
            main.wait_event(cur['ready'])
        n, k = dev_labels.shape
        dev_labels.copy_(cur['labels'][:n * k * 4].view(torch.float32).view(n, k), non_blocking=True)
        ops.preprocess_images(cur['crops'], cur['desc'][:n * 40], dev_images)
        if cuda:
            cur['free'].record(main)
        st['next'] ^= 1
        return stage(st['slots'][st['next']])             # decodes under the step that is about to run

    def grad_allreduce(self):
        """The one collective of the data-parallel step (replaces DistributedOptimizer,
        utils/multi_gpu_wrapper.py:82-89)."""
        if FLAGS.enbl_multi_gpu and mgw.size() > 1:
            return mgw.allreduce_flat_
        return None
