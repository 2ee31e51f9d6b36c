"""Weight sparsification learner (/root/reference/learners/weight_sparsification/learner.py:32-383):
Zhu & Gupta gradual magnitude pruning.  Masks are rebuilt every ws_mask_update_step steps by an
exact radix select (pf_ws_mask_build); every step the gradient is masked inside the fused
Momentum kernel (pf_momentum_step)."""
import os
import re
from timeit import default_timer as timer

import numpy as np
import torch

from ... import graph as G
from ... import ops
from ...engine import Executor, ParamStore
from ...flags import FLAGS, DEFINE_string, DEFINE_float, DEFINE_integer
from ...utils.multi_gpu_wrapper import MultiGpuWrapper as mgw
from ..abstract_learner import AbstractLearner, calc_prune_ratio, latest_checkpoint, load_checkpoint, save_checkpoint
from ..distillation_helper import DistillationHelper
from .pr_optimizer import PROptimizer
from .utils import get_maskable_vars

DEFINE_string('ws_save_path', './models_ws/model.ckpt', 'WS: model\'s save path')
DEFINE_float('ws_prune_ratio', 0.75, 'WS: target pruning ratio')
DEFINE_string('ws_prune_ratio_prtl', 'optimal', 'WS: pruning ratio protocol (\'uniform\' | \'heurist\' | \'optimal\')')
DEFINE_integer('ws_nb_rlouts', 200, 'WS: # of roll-outs for the RL agent')
DEFINE_integer('ws_nb_rlouts_min', 50, 'WS: minimal # of roll-outs for the RL agent to start training')
DEFINE_string('ws_reward_type', 'single-obj', 'WS: reward type (\'single-obj\' OR \'multi-obj\')')
DEFINE_float('ws_lrn_rate_rg', 3e-2, 'WS: learning rate for layerwise regression')
DEFINE_integer('ws_nb_iters_rg', 20, 'WS: # of iterations for layerwise regression')
DEFINE_float('ws_lrn_rate_ft', 3e-4, 'WS: learning rate for global fine-tuning')
DEFINE_integer('ws_nb_iters_ft', 400, 'WS: # of iterations for global fine-tuning')
DEFINE_integer('ws_nb_iters_feval', 25, 'WS: # of iterations for fast evaluation')
DEFINE_float('ws_prune_ratio_exp', 3.0, 'WS: pruning ratio\'s exponent term')
DEFINE_float('ws_iter_ratio_beg', 0.1, 'WS: iteration ratio (at starting time)')
DEFINE_float('ws_iter_ratio_end', 0.5, 'WS: iteration ratio (at ending time)')
DEFINE_float('ws_mask_update_step', 500, 'WS: step size for updating the pruning mask')


class WeightSparseLearner(AbstractLearner):  # pylint: disable=too-many-instance-attributes
    def __init__(self, sm_writer, model_helper):
        super(WeightSparseLearner, self).__init__(sm_writer, model_helper)
        self.mask_scope = 'mask'
        self._pr_full_state = None
        if FLAGS.enbl_dst:
            self.helper_dst = DistillationHelper(sm_writer, model_helper, self.mpi_comm)
        self.__build_train()

    def train(self, nb_iters=None):
        ex = self.sess_train
        if FLAGS.enbl_multi_gpu:
            mgw.broadcast_global_variables([ex.store.P, ex.store.O])
        last_mask_applied = False
        time_prev = timer()
        total = self.nb_iters_train if nb_iters is None else nb_iters
        for idx_iter in range(total):
            self.train_step()
            if (idx_iter + 1) % FLAGS.summ_step == 0 and self.is_primary_worker('global'):
                self.__monitor_progress(idx_iter, timer() - time_prev)
                time_prev = timer()
            if (idx_iter + 1) % FLAGS.ws_mask_update_step == 0:
                iter_ratio = float(idx_iter + 1) / self.nb_iters_train
                if iter_ratio >= FLAGS.ws_iter_ratio_beg:
                    if iter_ratio <= FLAGS.ws_iter_ratio_end:
                        self.prune()
                    elif not last_mask_applied:
                        last_mask_applied = True
                        self.prune()
            # save & evaluate the model at certain steps (learner.py:131-134)
            if self.is_primary_worker('global') and (idx_iter + 1) % FLAGS.save_step == 0:
                self.__save_model()
                self.evaluate()
        if self.is_primary_worker('global'):
            self.__save_model()
            self.evaluate()

    def train_step(self):
        ex = self.sess_train
        self.h2d_bytes = self.feed(ex, self.iterator_train)
        ex.run_step(self.lrn_rate(ex.step_count), self.grad_allreduce())

    def prune(self):
        """sess.run([prune_op, init_opt_op]) (learner.py:128): rebuild every mask at the current
        dynamic ratio, zero the pruned weights, re-initialise the momentum slots."""
        ex = self.sess_train
        step = ex.step_count      # global_step after the increment of this iteration
        ratios = [self.__calc_prune_ratio_dyn(r, step) for (_, r) in self.var_names_n_prune_ratios]
        ex.mask_builder.build(ratios)
        ex.reset_optimizer_slots()
        return ratios

    def evaluate(self, nb_iters=None):
        self.restore_for_eval(FLAGS.ws_save_path)
        ex = self.sess_train
        losses = [r['loss'] for r in self.eval_losses(nb_iters)]
        pr = calc_prune_ratio([ex.store.view(v) for v in self.maskable_vars])
        print('loss = %.4e | pr_msk = %.4e' % (np.mean(losses), pr))
        return float(np.mean(losses)), float(pr)

    # ------------------------------------------------------------------ what the 'optimal' ratio search drives
    # (pr_optimizer.py:495-548 runs these on a second pair of graphs; here they compose calls of the training step's own
    # executor plus a forward-only executor holding the full model.  Deviations, flagged: the short global fine-tuning
    # uses this learner's momentum optimizer at --ws_lrn_rate_ft instead of Adam, with BN in training mode; the
    # layer-wise regression stage follows the reference: inference-mode BN, Adam at --ws_lrn_rate_rg, masked gradients.)
    def pr_reset(self):
        """The full (pre-trained) model with every weight alive and a fresh optimizer."""
        ex = self.sess_train
        if self._pr_full_state is None:
            ckpt_dir = os.path.dirname(FLAGS.save_path)
            fn = latest_checkpoint(ckpt_dir) if os.path.isdir(ckpt_dir) else None
            self._pr_full_state = load_checkpoint(fn) if fn is not None else ex.store.state_dict()
        ex.store.load_state_dict(self._pr_full_state, strict=False)
        ex.MASK.fill_(1.0)
        ex.reset_optimizer_state()
        if FLAGS.enbl_multi_gpu:
            mgw.broadcast_global_variables([ex.store.P, ex.store.O])

    def pr_prune(self, prune_ratios):
        """init_op of the search (pr_optimizer.py:192-199): pruned = full * (|full| > percentile(|full|, ratio))."""
        self.pr_reset()
        self.sess_train.mask_builder.build([float(r) for r in prune_ratios])

    def pr_core_ops(self):
        """core_ops of __build_layer_rg_ops (pr_optimizer.py:291-296): the ops whose outputs are regressed, paired by
        index with the maskable variables."""
        if self.model_name.startswith('mobilenet'):
            patterns = ['pointwise/Conv2D', 'Conv2d_1c_1x1/Conv2D']
        else:
            patterns = ['Conv2D', 'MatMul']
        return [op for op in self.sess_train.ops if op.name.startswith(self.model_scope)
                and any(re.search(pt, op.name) is not None for pt in patterns)]

    def pr_regress_layers(self, nb_iters_rg):
        """Layer-wise regression (pr_optimizer.py:283-314, :542-548): for every core op in turn, nb_iters_rg Adam steps
        (--ws_lrn_rate_rg) on its kernel, with masked gradients, of l2_loss(out_pruned - out_full) — both networks in
        inference mode (forward_eval), the full one holding the pre-trained weights.  Returns the losses, [layer][iteration]."""
        ex = self.sess_train
        core_ops = self.pr_core_ops()
        if len(core_ops) != len(self.maskable_vars):
            raise ValueError('%d core ops for %d maskable variables' % (len(core_ops), len(self.maskable_vars)))
        if getattr(self, '_pr_full', None) is None:
            variables = [v for v in self.graph_train.variables.values() if v.name.startswith(self.model_scope + '/')]
            store = ParamStore(variables, self.device, seed=1)
            full = Executor(self.graph_train, self.images, ex.logits_t, self.device, store=store, train=False,
                            update_moving_stats=False)
            full.buf[self.images] = ex.buf[self.images]
            nmax = max(op.output.numel for op in core_ops)
            self._pr_full = dict(ex=full, store=store, diff=torch.empty(nmax, dtype=torch.float32, device=self.device),
                                 sc=torch.empty(nmax, dtype=torch.float32, device=self.device),
                                 diff2=torch.empty(nmax, dtype=torch.float32, device=self.device),
                                 loss=torch.zeros(1, dtype=torch.float32, device=self.device),
                                 ws=torch.empty(ops.L2_PARTIALS, dtype=torch.float32, device=self.device),
                                 hp=torch.zeros(4, dtype=torch.float32, device=self.device))
        st = self._pr_full
        st['store'].load_state_dict(self._pr_full_state, strict=False)
        full, world = st['ex'], (mgw.size() if FLAGS.enbl_multi_gpu else 1)
        losses = []
        with ex.standalone_forward():
            for op, var in zip(core_ops, self.maskable_vars):
                assert op.vars['kernel'] is var, 'core ops and maskable variables are paired by index'
                w, mask = ex.store.view(var), ex.store.view(var, ex.MASK)
                grad = ex.store.view(var, ex.G)
                m_slot, v_slot = torch.zeros_like(w), torch.zeros_like(w)
                b1p, b2p = np.float32(0.9), np.float32(0.999)
                n = op.output.numel
                losses.append([])
                for _ in range(nb_iters_rg):
                    self.feed(ex, self.iterator_train)
                    full.forward(training=False, upto=op)
                    ex.forward(training=False, upto=op)
                    diff = st['diff'][:n]
                    ops.cpg_diff_l2(ex.buf[op.output].reshape(-1), full.buf[op.output].reshape(-1), diff, st['loss'], st['ws'])
                    if op in ex.fused_add:
                        # the conv's epilogue added the block's shortcut — out = conv + shortcut in BOTH networks — so the
                        # difference of the conv outputs is the difference of the sums minus that of the shortcuts
                        other, sc = ex.fused_add[op][1], st['sc'][:n]
                        ops.cpg_diff_l2(ex.T(other).reshape(-1), full.T(other).reshape(-1), sc, st['loss'], st['ws'])
                        ops.cpg_diff_l2(diff, sc, st['diff2'][:n], st['loss'], st['ws'])
                        diff = st['diff2'][:n]
                    ex.layer_wgrad(op, diff.view(op.output.shape), grad)
                    if world > 1:
                        mgw.allreduce_flat_(grad)
                        grad.mul_(1.0 / world)
                    ops.mul(grad, mask, grad)
                    st['hp'].copy_(torch.tensor([FLAGS.ws_lrn_rate_rg, b1p, b2p, 0.0], dtype=torch.float32))
                    ops.adam_step(w.reshape(-1), m_slot.reshape(-1), v_slot.reshape(-1), grad.reshape(-1), st['hp'])
                    b1p, b2p = np.float32(b1p * np.float32(0.9)), np.float32(b2p * np.float32(0.999))
                    losses[-1].append(float(st['loss'].item()))
        return losses

    def pr_retrain(self, nb_iters_rg, nb_iters_ft):
        ex = self.sess_train
        if nb_iters_rg > 0:
            self.pr_regress_layers(nb_iters_rg)
        for _ in range(nb_iters_ft):
            self.feed(ex, self.iterator_train)
            ex.run_step(FLAGS.ws_lrn_rate_ft, self.grad_allreduce())

    def pr_evaluate(self):
        """(loss, metrics) over ws_nb_iters_feval mini-batches (pr_optimizer.py:566-590)."""
        ex = self.sess_train
        nb_iters = FLAGS.ws_nb_iters_feval if FLAGS.ws_nb_iters_feval > 0 else \
            max(1, FLAGS.nb_smpls_eval // FLAGS.batch_size_eval)
        rows = []
        for _ in range(nb_iters):
            self.feed(ex, self.eval_iterator())
            ex.forward_eval_loss()
            r = ex.fetch_losses()
            rows.append((r['loss'], r['acc_top1'], r['acc_top5']))
        loss, top1, top5 = [float(v) for v in np.mean(np.array(rows, np.float64), axis=0)]
        metrics = {'accuracy': top1} if self.dataset_name == 'cifar_10' else {'acc_top1': top1, 'acc_top5': top5}
        return loss, metrics

    def __build_train(self):
        self.graph_train = G.Graph()
        with self.graph_train.as_default():
            with G.variable_scope(self.data_scope):
                self.iterator_train = self.build_dataset_train()
                images, labels = self.iterator_train.get_next()
            self.images, self.labels = images, labels
            logits_dst = self.helper_dst.calc_logits(None, images) if FLAGS.enbl_dst else None
            with G.variable_scope(self.model_scope):
                logits = self.forward_train(images)
                self.maskable_var_names = [var.name for var in self.maskable_vars]
                loss, metrics = self.calc_loss(labels, logits, self.trainable_vars)
                if FLAGS.enbl_dst:
                    loss += self.helper_dst.calc_loss(logits, logits_dst)
                self.lrn_rate, self.nb_iters_train = self.setup_lrn_rate(None)
        world = mgw.size() if FLAGS.enbl_multi_gpu else 1
        teacher = None
        if FLAGS.enbl_dst:
            teacher = Executor(self.graph_train, images, logits_dst, self.device, train=False, seed=2)
            self.helper_dst.restore(teacher.store)
        self.sess_train = Executor(self.graph_train, images, logits, self.device, train=True, loss=loss,
                                   labels=labels, optimizer=dict(kind='momentum', momentum=FLAGS.momentum),
                                   maskable=self.maskable_vars, teacher=teacher, seed=1, grad_scale=1.0 / world)
        if teacher is not None:
            teacher.buf[images] = self.sess_train.buf[images]
            self.sess_train.share_im2col_from(teacher)
        self.masks = [self.sess_train.store.view(v, self.sess_train.MASK) for v in self.maskable_vars]
        # pruning ratios: host formulas, or ('optimal') the RL search driving this very step (pr_* methods below)
        if FLAGS.exec_mode == 'train':
            self.var_names_n_prune_ratios = PROptimizer(self.maskable_vars, self.dataset_name, tuner=self).run()
            if FLAGS.ws_prune_ratio_prtl == 'optimal':
                self.pr_reset()
            for var, (name, _) in zip(self.maskable_vars, self.var_names_n_prune_ratios):
                assert var.name == name, 'unmatched variable names: %s vs. %s' % (var.name, name)

    def __calc_prune_ratio_dyn(self, prune_ratio_fnl, global_step):
        """float32 graph arithmetic of learner.py:296-312, evaluated on the host."""
        idx_iter_beg = int(self.nb_iters_train * FLAGS.ws_iter_ratio_beg)
        idx_iter_end = int(self.nb_iters_train * FLAGS.ws_iter_ratio_end)
        f = np.float32
        base = f(f(int(global_step) - idx_iter_beg) / f(idx_iter_end - idx_iter_beg))
        base = f(min(f(1.0), max(f(0.0), base)))
        return f(f(prune_ratio_fnl) * f(f(1.0) - f(np.power(f(f(1.0) - base), f(FLAGS.ws_prune_ratio_exp)))))

    def __save_model(self):
        fn = save_checkpoint(FLAGS.ws_save_path, self.sess_train.store.state_dict(), self.sess_train.step_count)
        print('model saved to ' + fn)

    def __monitor_progress(self, idx_iter, time_step):
        ex = self.sess_train
        r = ex.fetch_losses()
        speed = FLAGS.batch_size * FLAGS.summ_step / time_step
        if FLAGS.enbl_multi_gpu:
            speed *= mgw.size()
        pr_msk = calc_prune_ratio([ex.store.view(v) for v in self.maskable_vars])
        print('iter #%d: lr = %.4e | loss = %.4e | pr_msk = %.4e | speed = %.2f pics / sec'
              % (idx_iter + 1, self.lrn_rate(idx_iter), r['loss'], pr_msk, speed))

    @property
    def maskable_vars(self):
        """List of all maskable variables."""
        return get_maskable_vars(self.trainable_vars)
