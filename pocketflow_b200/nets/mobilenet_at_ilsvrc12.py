"""MobileNet-v1 / v2 on ILSVRC-12 behind the ModelHelper plugin surface
(/root/reference/nets/mobilenet_at_ilsvrc12.py:29-160)."""
from .. import graph as G
from ..flags import FLAGS, DEFINE_integer, DEFINE_float
from ..datasets.ilsvrc12_dataset import Ilsvrc12Dataset
from ..utils.lrn_rate_utils import setup_lrn_rate_exponential_decay
from ..utils.multi_gpu_wrapper import MultiGpuWrapper as mgw
from .classification_helper import ClassificationModelHelper
from . import mobilenet_v1 as MobileNetV1
from . import mobilenet_v2 as MobileNetV2

DEFINE_integer('mobilenet_version', 1, 'MobileNet version (1 or 2)')
DEFINE_float('mobilenet_depth_mult', 1.0, 'channel multiplier of every layer')
DEFINE_float('nb_epochs_rat', 1.0, 'scales the number of training epochs')
DEFINE_float('lrn_rate_init', 0.045, 'learning rate at batch size batch_size_norm')
DEFINE_float('batch_size_norm', 96, 'batch size the initial learning rate is quoted for')
DEFINE_float('momentum', 0.9, 'momentum of the SGD optimizer')
DEFINE_float('loss_w_dcy', 4e-5, 'weight of the L2 term')


def forward_fn(inputs, is_train):
    if FLAGS.mobilenet_version == 1:
        return MobileNetV1.mobilenet_v1(inputs, num_classes=FLAGS.nb_classes, is_training=is_train,
                                        depth_multiplier=FLAGS.mobilenet_depth_mult)
    if FLAGS.mobilenet_version == 2:
        return MobileNetV2.mobilenet_v2(inputs, num_classes=FLAGS.nb_classes, is_training=is_train,
                                        depth_multiplier=FLAGS.mobilenet_depth_mult)
    raise ValueError('invalid MobileNet version: {}'.format(FLAGS.mobilenet_version))


class ModelHelper(ClassificationModelHelper):
    DATASET, DATASET_NAME = Ilsvrc12Dataset, 'ilsvrc_12'
    NB_EPOCHS, IDXS_EPOCH, DECAY_RATES = 100, [30, 60, 80, 90], [1.0, 0.1, 0.01, 0.001, 0.0001]
    # v2: 412 epochs, the rate decays by 0.98 ** 2.5 every 2.5 epochs (mobilenet_at_ilsvrc12.py:127-132)
    V2_NB_EPOCHS, V2_EPOCH_STEP = 412, 2.5
    # the filter names TF-layers' scope; slim calls its batch-norm scope 'BatchNorm', so gamma / beta ARE regularised
    # here — what the reference does (mobilenet_at_ilsvrc12.py:107-109, SURVEY A.6-9)
    L2_SKIPS = 'batch_normalization'

    def __init__(self, data_format='channels_last'):
        assert data_format == 'channels_last', 'MobileNet only supports \'channels_last\' data format'
        super(ModelHelper, self).__init__(data_format)

    def network(self, inputs, is_train):
        return forward_fn(inputs, is_train=is_train)

    def metrics(self, labels, outputs):
        """'accuracy' is the top-5 figure here (mobilenet_at_ilsvrc12.py:110-113)."""
        top1, top5 = G.accuracy(labels, outputs), G.in_top_k_accuracy(labels, outputs, 5)
        return {'accuracy': top5, 'acc_top1': top1, 'acc_top5': top5}

    def setup_lrn_rate(self, global_step):
        if FLAGS.mobilenet_version == 1:
            return super(ModelHelper, self).setup_lrn_rate(global_step)
        if FLAGS.mobilenet_version != 2:
            raise ValueError('invalid MobileNet version: {}'.format(FLAGS.mobilenet_version))
        batch_size = FLAGS.batch_size * (mgw.size() if FLAGS.enbl_multi_gpu else 1)
        lrn_rate = setup_lrn_rate_exponential_decay(global_step, batch_size, self.V2_EPOCH_STEP,
                                                    0.98 ** self.V2_EPOCH_STEP)
        nb_iters = int(FLAGS.nb_smpls_train * self.V2_NB_EPOCHS * FLAGS.nb_epochs_rat / batch_size)
        return lrn_rate, nb_iters

    @property
    def model_name(self):
        return 'mobilenet_v%d' % FLAGS.mobilenet_version
