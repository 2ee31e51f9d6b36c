"""Full-precision learner (no model compression applied)
(/root/reference/learners/full_precision/learner.py:30-228): plain Momentum training."""
from timeit import default_timer as timer

import numpy as np

from ... import graph as G
from ...engine import Executor
from ...flags import FLAGS
from ...utils.multi_gpu_wrapper import MultiGpuWrapper as mgw
from ..abstract_learner import AbstractLearner, save_checkpoint
from ..distillation_helper import DistillationHelper


class FullPrecLearner(AbstractLearner):  # pylint: disable=too-many-instance-attributes
    def __init__(self, sm_writer, model_helper, model_scope=None, enbl_dst=None):
        super(FullPrecLearner, self).__init__(sm_writer, model_helper)
        if model_scope is not None:
            self.model_scope = model_scope
        self.enbl_dst = enbl_dst if enbl_dst is not None else FLAGS.enbl_dst
        if self.enbl_dst:
            self.helper_dst = DistillationHelper(sm_writer, model_helper, self.mpi_comm)
        self.__build()

    def train(self, nb_iters=None):
        ex = self.sess_train
        self.warm_start(ex)
        if FLAGS.enbl_multi_gpu:
            mgw.broadcast_global_variables([ex.store.P, ex.store.O])
        time_prev = timer()
        total = self.nb_iters_train if nb_iters is None else nb_iters
        for idx_iter in range(total):
            self.train_step()
            if (idx_iter + 1) % FLAGS.summ_step == 0 and self.is_primary_worker('global'):
                r = ex.fetch_losses()
                speed = FLAGS.batch_size * FLAGS.summ_step / (timer() - time_prev) * (mgw.size() if FLAGS.enbl_multi_gpu else 1)
                print('iter #%d: lr = %.4e | loss = %.4e | speed = %.2f pics / sec'
                      % (idx_iter + 1, self.lrn_rate(idx_iter), r['loss'], speed))
                time_prev = timer()
            # save & evaluate the model at certain steps (learner.py:79-82)
            if self.is_primary_worker('global') and (idx_iter + 1) % FLAGS.save_step == 0:
                self.__save_model()
                self.evaluate()
        if self.is_primary_worker('global'):
            self.__save_model()
            self.evaluate()

    def __save_model(self):
        ex = self.sess_train
        print('model saved to ' + save_checkpoint(FLAGS.save_path, ex.store.state_dict(), ex.step_count))

    def train_step(self):
        ex = self.sess_train
        self.h2d_bytes = self.feed(ex, self.iterator_train)
        ex.run_step(self.lrn_rate(ex.step_count), self.grad_allreduce())

    def evaluate(self, nb_iters=None):
        self.restore_for_eval(FLAGS.save_path)
        out = [r['loss'] for r in self.eval_losses(nb_iters)]
        print('loss = %.4e' % np.mean(out))
        return float(np.mean(out))

    def __build(self):
        self.graph_train = G.Graph()
        with self.graph_train.as_default():
            with G.variable_scope(self.data_scope):
                self.iterator_train = self.build_dataset_train()
                images, labels = self.iterator_train.get_next()
            self.images, self.labels = images, labels
            logits_dst = self.helper_dst.calc_logits(None, images) if self.enbl_dst else None
            with G.variable_scope(self.model_scope):
                logits = self.forward_train(images)
                loss, metrics = self.calc_loss(labels, logits, self.trainable_vars)
                if self.enbl_dst:
                    loss += self.helper_dst.calc_loss(logits, logits_dst)
                self.lrn_rate, self.nb_iters_train = self.setup_lrn_rate(None)
        world = mgw.size() if FLAGS.enbl_multi_gpu else 1
        teacher = None
        if self.enbl_dst:
            teacher = Executor(self.graph_train, images, logits_dst, self.device, train=False, seed=2)
            self.helper_dst.restore(teacher.store)
        self.sess_train = Executor(self.graph_train, images, logits, self.device, train=True, loss=loss, labels=labels,
                                   optimizer=dict(kind='momentum', momentum=FLAGS.momentum), teacher=teacher,
                                   seed=1, grad_scale=1.0 / world)
        if teacher is not None:
            teacher.buf[images] = self.sess_train.buf[images]
            self.sess_train.share_im2col_from(teacher)
