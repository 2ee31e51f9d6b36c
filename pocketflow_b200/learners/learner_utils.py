"""Utility function for creating the specified learner (/root/reference/learners/learner_utils.py:33-66)."""
from ..flags import FLAGS


def create_learner(sm_writer, model_helper):
    """Create the learner as specified by FLAGS.learner."""
    learner = None
    if FLAGS.enbl_compact_ft and FLAGS.learner not in ('chn-pruned-gpu', 'chn-pruned-rmt'):
        raise ValueError('--enbl_compact_ft applies to the channel-pruning learners (chn-pruned-gpu, chn-pruned-rmt), '
                         'not to ' + FLAGS.learner)
    if FLAGS.learner == 'full-prec':
        from .full_precision.learner import FullPrecLearner
        learner = FullPrecLearner(sm_writer, model_helper)
    elif FLAGS.learner == 'weight-sparse':
        from .weight_sparsification.learner import WeightSparseLearner
        learner = WeightSparseLearner(sm_writer, model_helper)
    elif FLAGS.learner == 'chn-pruned-gpu':
        from .channel_pruning_gpu.learner import ChannelPrunedGpuLearner
        learner = ChannelPrunedGpuLearner(sm_writer, model_helper)
    elif FLAGS.learner == 'chn-pruned-rmt':
        from .channel_pruning_rmt.learner import ChannelPrunedRmtLearner
        learner = ChannelPrunedRmtLearner(sm_writer, model_helper)
    elif FLAGS.learner == 'uniform':
        from .uniform_quantization.learner import UniformQuantLearner
        learner = UniformQuantLearner(sm_writer, model_helper)
    elif FLAGS.learner == 'non-uniform':
        from .nonuniform_quantization.learner import NonUniformQuantLearner
        learner = NonUniformQuantLearner(sm_writer, model_helper)
    elif FLAGS.learner == 'channel':
        from .channel_pruning.learner import ChannelPrunedLearner
        learner = ChannelPrunedLearner(sm_writer, model_helper)
    elif FLAGS.learner in ('dis-chn-pruned', 'uniform-tf'):
        raise ValueError('learner %s is outside the hot-path scope of this build (SURVEY.md §8)' % FLAGS.learner)
    else:
        raise ValueError('unrecognized learner\'s name: ' + FLAGS.learner)
    return learner
