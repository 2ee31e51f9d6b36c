"""What the channel-pruning learners (chn-pruned-gpu, chn-pruned-rmt, channel) share: the full model under scope
'model' and the pruned model under 'pruned_model' in one graph, the restore of the full model into the pruned one, the
selection executors, and the masked fine-tuning with its save and evaluate cadence."""
import os
from abc import abstractmethod
from timeit import default_timer as timer

import numpy as np

from .. import graph as G
from ..engine import Executor, ParamStore
from ..flags import FLAGS
from ..utils.multi_gpu_wrapper import MultiGpuWrapper as mgw
from .abstract_learner import AbstractLearner, calc_prune_ratio, latest_checkpoint, save_checkpoint
from .distillation_helper import DistillationHelper


class ChannelPrunedBase(AbstractLearner):  # pylint: disable=too-many-instance-attributes
    FUSE_ADD = True             # whether sess_train fuses residual Adds into the producing conv's epilogue
    SAVE_PATH_FLAG = None       # the flag naming the fine-tuned model's save path

    def __init__(self, sm_writer, model_helper):
        super(ChannelPrunedBase, self).__init__(sm_writer, model_helper)
        # scopes of the full & channel-pruned models (channel_pruning_gpu/learner.py:126-128); `vars` /
        # `trainable_vars` are the pruned model's
        self.model_scope_full = 'model'
        self.model_scope_prnd = 'pruned_model'
        self.model_scope = self.model_scope_prnd
        self.compact = None             # compact.CompactTrainer under --enbl_compact_ft
        if FLAGS.enbl_dst:
            self.helper_dst = DistillationHelper(sm_writer, model_helper, self.mpi_comm)
        self.__build()

    @abstractmethod
    def layer_ratios(self):
        """each layer's pruning (or preserve) ratio; called before any executor is built, so it may refuse flags"""

    # ------------------------------------------------------------------ graph
    def __build(self):
        self.graph_train = G.Graph()
        with self.graph_train.as_default():
            with G.variable_scope(self.data_scope):
                self.iterator_train = self.build_dataset_train()
                images, labels = self.iterator_train.get_next()
            self.images, self.labels = images, labels
            logits_dst = self.helper_dst.calc_logits(None, images) if FLAGS.enbl_dst else None
            with G.variable_scope(self.model_scope_full):
                logits_full = self.forward_train(images)
            with G.variable_scope(self.model_scope_prnd):
                logits = self.forward_train(images)
                loss, metrics = self.calc_loss(labels, logits, self.trainable_vars)
                if FLAGS.enbl_dst:
                    loss += self.helper_dst.calc_loss(logits, logits_dst)
                self.lrn_rate, self.nb_iters_train = self.setup_lrn_rate(None)
        # maskable = trainable variables read by ops named .../Conv2D, depthwise excluded (channel_pruning_gpu/
        # learner.py:52-66); the i-th Conv2D of the full model is regressed onto by the i-th of the pruned (:347-352)
        conv_of = lambda scope: [op for op in self.graph_train.ops
                                 if op.name.endswith('/Conv2D') and op.name.startswith(scope + '/')]
        self.conv_ops_full, self.conv_ops_prnd = conv_of(self.model_scope_full), conv_of(self.model_scope_prnd)
        assert len(self.conv_ops_full) == len(self.conv_ops_prnd)
        self.maskable_vars = [op.vars['kernel'] for op in self.conv_ops_prnd]
        self.maskable_var_names = [v.name for v in self.maskable_vars]
        self.nb_layers = len(self.conv_ops_prnd)
        self.prune_ratios = self.layer_ratios()
        world = mgw.size() if FLAGS.enbl_multi_gpu else 1
        teacher = None
        if FLAGS.enbl_dst:
            teacher = Executor(self.graph_train, images, logits_dst, self.device, train=False, seed=2)
            self.helper_dst.restore(teacher.store)
        # both models start from the same seed: the pruned model IS the full model until channels are chosen
        self.sess_train = Executor(self.graph_train, images, logits, self.device, train=True, loss=loss, labels=labels,
                                   optimizer=dict(kind='momentum', momentum=FLAGS.momentum),
                                   maskable=self.maskable_vars, teacher=teacher, seed=1, grad_scale=1.0 / world,
                                   fuse_add=self.FUSE_ADD)
        if teacher is not None:
            teacher.buf[images] = self.sess_train.buf[images]
            self.sess_train.share_im2col_from(teacher)
        self.logits_full, self.logits_prnd = logits_full, logits
        self.store_full = ParamStore([v for v in self.graph_train.variables.values()
                                      if v.name.startswith(self.model_scope_full + '/')], self.device, seed=1)

    def restore_full(self):
        """Restore the full model from the pre-trained checkpoint and copy it into the pruned model
        (channel_pruning_gpu/learner.py:141-149, :283-289; channel_pruning_rmt/learner.py:355-379)."""
        ckpt_dir = os.path.dirname(FLAGS.save_path)
        if os.path.isdir(ckpt_dir) and latest_checkpoint(ckpt_dir) is not None:
            self.restore_model(FLAGS.save_path, store=self.store_full)
        elif FLAGS.data_dir_local:
            raise ValueError('channel pruning of a real model needs its pre-trained checkpoint in ' + ckpt_dir)
        else:
            print('no pre-trained checkpoint in %s: the full model keeps its seed initialisation (synthetic run)' % ckpt_dir)
        full = self.store_full.state_dict()
        renamed = {self.model_scope_prnd + k[len(self.model_scope_full):]: v for k, v in full.items()}
        self.sess_train.store.load_state_dict(renamed, strict=True)

    init_from_full = restore_full          # chn-pruned-gpu also resets its masks and optimizer on top of it

    # ------------------------------------------------------------------ channel selection
    def full_executor(self, images_buf):
        """the full model for selection: forward only, training-mode BN without moving-average updates (only the pruned
        scope's update ops are ever run, channel_pruning_gpu/learner.py:283-286), every conv and Add output
        materialised, fed from images_buf"""
        ex = Executor(self.graph_train, self.images, self.logits_full, self.device, store=self.store_full,
                      train=False, fuse_add=False, update_moving_stats=False)
        ex.buf[self.images] = images_buf
        return ex

    def selection_executors(self):
        """(full, pruned) executors for sampling, both as full_executor() builds them; one image buffer feeds both"""
        ex_p = Executor(self.graph_train, self.images, self.logits_prnd, self.device, store=self.sess_train.store,
                        train=False, fuse_add=False, update_moving_stats=False)
        return self.full_executor(ex_p.buf[self.images]), ex_p

    def cache_batches(self, nb_batches):
        """nb_batches training mini-batches, drawn once, kept on the device"""
        ex = self.sess_train
        cached = []
        for _ in range(nb_batches):
            self.feed(ex, self.iterator_train)
            cached.append(ex.buf[self.images].clone())
        return cached

    @staticmethod
    def check_regressable(ex, op):
        if op in ex.fused_act:
            raise ValueError('%s: a conv with a fused activation has no materialised output to regress onto' % op.name)

    # ------------------------------------------------------------------ fine-tuning
    def select_on_primary(self, path, select=True):
        """choose_channels() on the primary worker alone, which saves the selected model to `path` (skipped if not
        `select`); then every worker restores that file, builds its masks and starts from the same state"""
        if select:
            if self.is_primary_worker('global'):
                time_prev = timer()
                self.choose_channels()
                print('time (channel selection): %.2f (s)' % (timer() - time_prev))
            self.auto_barrier()
        self.restore_model(path)
        self.init_masks()
        if FLAGS.enbl_multi_gpu:
            mgw.broadcast_global_variables([self.sess_train.store.P, self.sess_train.store.O])

    def fine_tune(self, nb_iters=None, save_first=True, label='pr_krn', path_eval=None):
        """nb_iters (default nb_iters_train) masked steps, with a progress line every summ_step steps and a save and
        evaluation every save_step steps and at the end.  save_first: start the fine-tuning at the pruned width
        (--enbl_compact_ft), save and evaluate before the first step.  label: the progress line's name for the pruning
        ratio.  path_eval: a further checkpoint written at the end."""
        if save_first:
            if FLAGS.enbl_compact_ft:
                # the steps run on a compact executor planned from the selected masks; sess_train evaluates and saves
                from ..compact import CompactTrainer
                self.compact = CompactTrainer(self.sess_train)
                if self.is_primary_worker('global'):
                    print('\n'.join(self.compact.report()))
            if self.is_primary_worker('global'):
                self.__save_model()
                self.evaluate()
            self.auto_barrier()
        ex = self.sess_step
        time_prev = timer()
        total = self.nb_iters_train if nb_iters is None else nb_iters
        for idx_iter in range(total):
            self.train_step()
            if (idx_iter + 1) % FLAGS.summ_step == 0 and self.is_primary_worker('global'):
                r = ex.fetch_losses()
                speed = FLAGS.batch_size * FLAGS.summ_step / (timer() - time_prev) * (mgw.size() if FLAGS.enbl_multi_gpu else 1)
                print('iter #%d: lr = %.4e | loss = %.4e | %s = %.4e | speed = %.2f pics / sec'
                      % (idx_iter + 1, self.lrn_rate(idx_iter), r['loss'], label, self.pr_maskable(), speed))
                time_prev = timer()
            # save the model at certain steps (channel_pruning_gpu/learner.py:171-175).  The reference barriers after
            # EVERY iteration; the gradient all-reduce already keeps the ranks in step, so only the iterations where the
            # primary worker does extra work need one (a per-step NCCL barrier would drain the device queue every step).
            if (idx_iter + 1) % FLAGS.save_step == 0:
                if self.is_primary_worker('global'):
                    self.__save_model()
                    self.evaluate()
                self.auto_barrier()
        if self.is_primary_worker('global'):
            self.__save_model()
            if path_eval is not None:
                print('model saved to ' + save_checkpoint(path_eval, self.sess_train.store.state_dict()))
            self.evaluate()

    @property
    def sess_step(self):
        """the executor whose run_step is one fine-tune step"""
        return self.sess_train if self.compact is None else self.compact.ex

    def __save_model(self):
        if self.compact is not None:
            self.compact.push()                   # the compact state expanded into sess_train
        ex = self.sess_train
        print('model saved to ' + save_checkpoint(getattr(FLAGS, self.SAVE_PATH_FLAG), ex.store.state_dict(),
                                                  ex.step_count))

    def train_step(self):
        ex = self.sess_step
        self.h2d_bytes = self.feed(self.sess_train, self.iterator_train)
        ex.run_step(self.lrn_rate(ex.step_count), self.grad_allreduce())

    def evaluate(self, nb_iters=None):
        """restore the latest checkpoint beside the save path under --exec_mode eval, then (mean loss, pruning ratio)"""
        self.restore_for_eval(getattr(FLAGS, self.SAVE_PATH_FLAG))
        losses = [r['loss'] for r in self.eval_losses(nb_iters)]
        return float(np.mean(losses)), float(self.pr_maskable())

    def pr_maskable(self):
        return calc_prune_ratio([self.sess_train.store.view(v) for v in self.maskable_vars])
