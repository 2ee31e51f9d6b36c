"""The body shared by the per-net execution scripts (/root/reference/nets/*_run.py:36-72): parse the flags, build the
ModelHelper and the learner `--learner` names, train or evaluate; a ValueError ends the run with exit status 1, as in
the reference.  Launch one process per GPU with torchrun and pass --enbl_multi_gpu for data-parallel training
(scripts/run_local.sh:44-47 uses mpirun)."""
import sys
import traceback

from ..flags import FLAGS
from ..learners.learner_utils import create_learner
# every learner declares its flags at import time; they must exist before the command line is parsed
from ..learners.full_precision import learner as _fp  # noqa: F401
from ..learners.weight_sparsification import learner as _ws  # noqa: F401
from ..learners.channel_pruning_gpu import learner as _cpg  # noqa: F401
from ..learners.channel_pruning_rmt import learner as _cpr  # noqa: F401
from ..learners.uniform_quantization import learner as _uq  # noqa: F401
from ..learners.nonuniform_quantization import learner as _nuq  # noqa: F401


def run(model_helper_cls, argv=None):
    try:
        FLAGS.parse(sys.argv[1:] if argv is None else argv)
        if FLAGS.debug:
            print('FLAGS:')
            for key in sorted(FLAGS._defaults):  # pylint: disable=protected-access
                print('{}: {}'.format(key, getattr(FLAGS, key)))
        if FLAGS.exec_mode not in ('train', 'eval'):            # (checked before the learner is built: fail fast)
            raise ValueError('unrecognized execution mode: ' + FLAGS.exec_mode)
        model_helper = model_helper_cls()
        learner = create_learner(None, model_helper)          # no TensorBoard summary writer in this build
        if FLAGS.exec_mode == 'train':
            learner.train()
        else:
            learner.download_model()
            learner.evaluate()
        return 0
    except ValueError:
        traceback.print_exc()
        return 1
