"""Channel pruning learner, GPU variant (/root/reference/learners/channel_pruning_gpu/learner.py:30-568).

Two copies of the network live in one graph, as in the reference (:207-223): the FULL model under scope 'model'
(restored from the pre-trained checkpoint, never trained) and the channel-pruned model under 'pruned_model'
(initialised from the full one, :283-289).  train() = channel selection, layer by layer (:445-518), then whole-network
fine-tuning with masked gradients (:404-443):
  * selection of layer i: reg_loss_i = l2_loss(conv_i(full) - conv_i(pruned)) on the same mini-batch (:339-354);
    proximal gradient descent on the kernel of conv_i — W <- prox(W - lr dreg/dW), prox = group soft-threshold over
    INPUT channels at the `prune_perctl`-th percentile of the group norms, the percentile ramping up to the layer's
    target ratio, lr adapted by the sign of the loss change (:375-383, :476-497); then the mask of the surviving
    channels (:250-260) and a layer-wise Adam fine-tuning of the same regression loss with masked gradients
    (:385-396, :499-507).  Device side: two forward passes (tensor-core convs), pf_cpg_diff_l2, ONE conv wgrad,
    pf_cpg_group_norms -> exact percentile (pf_select_desc) -> pf_cpg_prox_apply / pf_adam_step.
  * steady state: the masked Momentum step of the weight-sparse learner with input-channel masks (pf_momentum_step).
Flagged deviations: with several workers the reference adapts lr_pgd from each worker's LOCAL loss (the workers'
python loops can then disagree); here the loss is averaged over the workers first.  A channel whose norm is exactly 0
while the threshold is 0 gives 0/0 = NaN in the reference's shrink factor; here it stays 0.  Without a pre-trained
checkpoint (synthetic runs) the full model keeps its seed initialisation.
--enbl_compact_ft (off by default) runs the fine-tune steps at the pruned width (compact.CompactTrainer) and expands the
state back before every save, so the masked full-width checkpoint, evaluate() and the export tool are unchanged.  Its
deviations: (a) producer channels that no consumer reads are frozen at their post-selection values instead of decaying
under weight decay, and the reported loss omits their L2 term; they cannot influence the logits either way; (b) the
fp32 accumulation order of a narrowed K dimension differs from the masked one, so logits agree to rounding."""
from timeit import default_timer as timer

import numpy as np
import torch

from ... import ops
from ...flags import FLAGS, DEFINE_string, DEFINE_float, DEFINE_boolean, DEFINE_integer
from ...utils.multi_gpu_wrapper import MultiGpuWrapper as mgw
from ..channel_pruning_base import ChannelPrunedBase

DEFINE_string('cpg_save_path', './models_cpg/model.ckpt', 'CPG: model\'s save path')
DEFINE_string('cpg_save_path_eval', './models_cpg_eval/model.ckpt', 'CPG: model\'s save path for evaluation')
DEFINE_string('cpg_prune_ratio_type', 'uniform', 'CPG: pruning ratio type (\'uniform\' OR \'list\')')
DEFINE_float('cpg_prune_ratio', 0.5, 'CPG: uniform pruning ratio')
DEFINE_boolean('cpg_skip_ht_layers', True, 'CPG: skip head & tail layers for pruning')
DEFINE_string('cpg_prune_ratio_file', None, 'CPG: file path to the list of pruning ratios')
DEFINE_float('cpg_lrn_rate_pgd_init', 1e-10, 'CPG: proximal gradient descent\'s initial learning rate')
DEFINE_float('cpg_lrn_rate_pgd_incr', 1.4, 'CPG: proximal gradient descent\'s learning rate\'s increase ratio')
DEFINE_float('cpg_lrn_rate_pgd_decr', 0.7, 'CPG: proximal gradient descent\'s learning rate\'s decrease ratio')
DEFINE_float('cpg_lrn_rate_adam', 1e-2, 'CPG: Adam\'s initial learning rate')
DEFINE_integer('cpg_nb_iters_layer', 1000, 'CPG: # of iterations for layer-wise FT')


class ChannelPrunedGpuLearner(ChannelPrunedBase):  # pylint: disable=too-many-instance-attributes
    # the selection regresses on the step executor's own conv outputs, so no residual Add is fused into them
    FUSE_ADD = False
    SAVE_PATH_FLAG = 'cpg_save_path'

    def __init__(self, sm_writer, model_helper):
        super(ChannelPrunedGpuLearner, self).__init__(sm_writer, model_helper)
        self.channels_chosen = False
        # the full model's executor, built lazily: it is only needed while channels are being chosen
        self.sess_full = None

    # ------------------------------------------------------------------ training
    def train(self, nb_iters=None):
        self.init_from_full()
        # choose channels and evaluate the model before re-training (:152-157)
        self.choose_channels()
        self.fine_tune(nb_iters, label='pr_msk')

    def init_from_full(self):
        """restore_full(), then masks = 1, fresh optimizers, broadcast (:141-149, :283-289)"""
        self.restore_full()
        ex = self.sess_train
        ex.MASK.fill_(1.0)
        ex.reset_optimizer_state()
        ex.step_count = 0
        self.channels_chosen = False
        if FLAGS.enbl_multi_gpu:
            mgw.broadcast_global_variables([ex.store.P, ex.store.O, self.store_full.P, self.store_full.O])

    def layer_ratios(self):
        """each layer's pruning ratio (:448-459)"""
        if FLAGS.cpg_prune_ratio_type == 'uniform':
            ratios = [FLAGS.cpg_prune_ratio] * self.nb_layers
            if FLAGS.cpg_skip_ht_layers:
                ratios[0] = ratios[-1] = 0.0
        elif FLAGS.cpg_prune_ratio_type == 'list':
            with open(FLAGS.cpg_prune_ratio_file, 'r') as i_file:
                ratios = [float(sub_str) for sub_str in i_file.readline().strip().split(',')]
            assert len(ratios) == self.nb_layers
        else:
            raise ValueError('unrecognized pruning ratio type: ' + FLAGS.cpg_prune_ratio_type)
        return ratios

    # ------------------------------------------------------------------ channel selection (:445-518)
    def __selection_state(self):
        if self.sess_full is None:
            self.sess_full = self.full_executor(self.sess_train.buf[self.images])    # one mini-batch feeds both models
            dev = self.device
            nmax = max(op.output.numel for op in self.conv_ops_prnd)
            self._sel = dict(diff=torch.empty(nmax, dtype=torch.float32, device=dev),
                             loss=torch.zeros(1, dtype=torch.float32, device=dev),
                             ws=torch.empty(ops.L2_PARTIALS, dtype=torch.float32, device=dev),
                             hp=torch.zeros(4, dtype=torch.float32, device=dev))
        return self._sel

    def layer_regression(self, idx_layer):
        """One mini-batch through both models: reg_loss of layer idx (device scalar) and its gradient w.r.t. the
        pruned model's kernel of that layer, written into the step's gradient buffer.  The pruned model runs its WHOLE
        forward pass (the reference's layer ops depend on every BN update op of the pruned scope, :376, :393)."""
        ex, sel = self.sess_train, self.__selection_state()
        op_f, op_p = self.conv_ops_full[idx_layer], self.conv_ops_prnd[idx_layer]
        self.feed(ex, self.iterator_train)
        self.sess_full.forward(training=True, upto=op_f)
        with ex.standalone_forward():
            ex.forward(training=True)
        n = op_p.output.numel
        diff = sel['diff'][:n]
        ops.cpg_diff_l2(ex.buf[op_p.output].reshape(-1), self.sess_full.buf[op_f.output].reshape(-1), diff,
                        sel['loss'], sel['ws'])
        grad = ex.store.view(op_p.vars['kernel'], ex.G)
        ex.layer_wgrad(op_p, diff.view(op_p.output.shape), grad)
        if FLAGS.enbl_multi_gpu and mgw.size() > 1:                        # DistributedOptimizer: average (:368-370)
            mgw.allreduce_flat_(grad)
            mgw.allreduce_flat_(sel['loss'])
            grad.mul_(1.0 / mgw.size())
            sel['loss'].mul_(1.0 / mgw.size())
        return sel['loss'], grad

    def choose_channels(self, nb_iters_layer=None):
        """Choose channels for all convolutional layers (:445-518): the host loop; the device work is in sel_* below."""
        nb_workers = mgw.size() if FLAGS.enbl_multi_gpu else 1
        if nb_iters_layer is None:
            nb_iters_layer = int(FLAGS.cpg_nb_iters_layer / nb_workers)
        ratio_list = self.prune_ratios
        self.selection_log = []
        for idx_layer in range(self.nb_layers):
            if ratio_list[idx_layer] == 0.0:                               # skip if no pruning is required
                continue
            if self.is_primary_worker('global'):
                print('layer #%d: pr = %.2f (target)' % (idx_layer, ratio_list[idx_layer]))
            time_prev = timer()
            # ---- stochastic proximal gradient descent with an increasing percentile (:476-497)
            reg_loss_prev = 0.0
            lrn_rate_pgd = FLAGS.cpg_lrn_rate_pgd_init
            for idx_iter in range(nb_iters_layer):
                prune_perctl = ratio_list[idx_layer] * 100.0 * (idx_iter + 1) / nb_iters_layer
                reg_loss = self.sel_prune(idx_layer, lrn_rate_pgd, prune_perctl)
                self.selection_log.append(('prune', idx_layer, idx_iter, reg_loss, lrn_rate_pgd, prune_perctl))
                if reg_loss < reg_loss_prev:
                    lrn_rate_pgd *= FLAGS.cpg_lrn_rate_pgd_incr
                else:
                    lrn_rate_pgd *= FLAGS.cpg_lrn_rate_pgd_decr
                reg_loss_prev = reg_loss
            # ---- fine-tune with selected channels only (:499-507): masked Adam on the same regression loss
            self.sel_update_mask(idx_layer)
            for idx_iter in range(nb_iters_layer):
                reg_loss = self.sel_finetune(idx_layer, idx_iter)
                self.selection_log.append(('finetune', idx_layer, idx_iter, reg_loss))
            # ---- re-compute the pruning ratio (:509-514)
            if self.is_primary_worker('global'):
                print('layer #%d: pr = %.2f (actual) | time = %.2f'
                      % (idx_layer, self.sel_prune_ratio(idx_layer), timer() - time_prev))
        self.channels_chosen = True

    # device side of one selection iteration
    def __layer_tensors(self, idx_layer):
        ex, var = self.sess_train, self.maskable_vars[idx_layer]
        cin = var.shape[2] if len(var.shape) == 4 else var.shape[0]
        sel = self.__selection_state()
        if sel.get('layer') != idx_layer:                                  # per-layer scratch: norms, Adam slots
            sel.update(layer=idx_layer, norms=torch.empty(cin, dtype=torch.float32, device=self.device),
                       m=None, v=None)
        return ex.store.view(var), ex.store.view(var, ex.MASK), cin, sel

    def sel_prune(self, idx_layer, lrn_rate_pgd, prune_perctl):
        """sess.run([layer_ops[i]['prune'], reg_losses[i]], feed_dict={lr, percentile}) (:481-484)"""
        w, _, _, sel = self.__layer_tensors(idx_layer)
        loss_dev, grad = self.layer_regression(idx_layer)
        ops.cpg_prox_step(w, grad, lrn_rate_pgd, prune_perctl, sel['norms'])
        return float(loss_dev.item())

    def sel_update_mask(self, idx_layer):
        """sess.run(mask_updt_ops[i]) (:500)"""
        w, mask, _, sel = self.__layer_tensors(idx_layer)
        ops.cpg_channel_mask(w, mask, sel['norms'])
        sel['m'], sel['v'] = torch.zeros_like(w), torch.zeros_like(w)      # this layer's Adam slots (init_opt, :397)
        sel['b1p'], sel['b2p'] = np.float32(0.9), np.float32(0.999)        # beta powers: float32 running products

    def sel_finetune(self, idx_layer, idx_iter):
        """sess.run([layer_ops[i]['finetune'], reg_losses[i]]) (:502-503): Adam at cpg_lrn_rate_adam, gradient * mask"""
        w, mask, _, sel = self.__layer_tensors(idx_layer)
        loss_dev, grad = self.layer_regression(idx_layer)
        ops.mul(grad, mask, grad)
        sel['hp'].copy_(torch.tensor([FLAGS.cpg_lrn_rate_adam, sel['b1p'], sel['b2p'], 0.0], dtype=torch.float32))
        ops.adam_step(w.reshape(-1), sel['m'].reshape(-1), sel['v'].reshape(-1), grad.reshape(-1), sel['hp'])
        sel['b1p'], sel['b2p'] = np.float32(sel['b1p'] * np.float32(0.9)), np.float32(sel['b2p'] * np.float32(0.999))
        return float(loss_dev.item())

    def sel_prune_ratio(self, idx_layer):
        _, mask, cin, _ = self.__layer_tensors(idx_layer)
        nnz = int(torch.count_nonzero(mask.reshape(-1, cin, mask.shape[-1]).sum(dim=(0, 2))).item())
        return 1.0 - float(nnz) / cin
