"""Channel pruning learner, remastered (/root/reference/learners/channel_pruning_rmt/learner.py:113-892).

Two copies of the network live in one graph, as in the reference (:332-379): the FULL model under scope 'model'
(restored from the pre-trained checkpoint, never trained) and the channel-pruned model under 'pruned_model'
(initialised from the full one, :375-379).  train() = channel selection, layer by layer (:546-649), then whole-network
fine-tuning with masked gradients (:146-193); evaluate() reads cpr_save_path's latest checkpoint (:195-209, :857-869).
The layers are the kernels read by ops named .../Conv2D (depthwise convs excluded, MobileNet's logits conv and ResNet's
projection convs included, :54-77); the i-th Conv2D of the full model is paired with the i-th of the pruned model
(:396-430).

Selection of layer i (no gradient descent on the network):
  * sampling (:608-631, :651-725): ceil(cpr_nb_smpls / batch_size) training mini-batches are drawn once and reused
    for every layer (:579-582).  Per batch both models run forward_train up to conv i (training-mode BN, no
    moving-average updates); cpr_nb_crops_per_smpl output positions are drawn, each shared by the whole batch; the
    pruned model's R x S x Cin input patches and the FULL model's Cout outputs there are gathered on the device
    (pf_cpr_sample) straight into their rows of the regression problem.  patch * W == output is checked for both
    models (mean squared error < 1e-6, :715-723): an error raises.
  * sparse regression (:727-812): G = F^T F and b = F^T y in float64 over a secondary sample of the rows
    (pf_cpr_gram), then a γ search whose every LASSO solve is one cooperative ISTA launch (pf_cpr_ista).
  * refit (:814-842): Adam on ||X W - Y||^2 over the kept channels (ops.CprLstsq: 1x1 conv fwd / wgrad +
    pf_adam_step), then W * [|m| > 0] (pf_cpr_mask_channels).
A layer whose ratio is 0 (the first layer under cpr_skip_frst_layer, the last under cpr_skip_last_layer, a name
matched by cpr_skip_op_names) is NOT skipped: as in the reference it is sampled, searched with target nnz = Cin and
refit, so its weights change.
Steady state: the masked Momentum step of the weight-sparse learner with input-channel masks mask = sum W^2 > 0
(:255-263; pf_cpg_group_norms + pf_cpg_channel_mask).

All host randomness comes from one np.random.RandomState(seed), drawn in the reference's order: per cached batch
randint(oh), randint(ow) per crop; then choice (the kept instances); per layer choice (the secondary sample), uniform
(the initial mask).  Multi-GPU: every reference worker runs its own selection but only rank 0's result survives the
save to cpr_save_path_ws and the restore every rank does (:146-156, :645-649); here rank 0 alone selects, saves, and
every rank restores that file — the same result.  The other ranks wait at a barrier for the whole selection (the
reference's ranks select side by side); a selection longer than the collective backend's timeout (torch.distributed's
default: 10 min for NCCL) needs a larger one at process-group creation.
Flagged deviations: the refit's Adam moment update is TF's m += (g - m)(1 - beta1) (pf_adam_step) instead of the
reference's beta1 m + (1 - beta1) g (:499-500), and its GEMMs run on the conv kernels (split-bf16 tensor cores where
the shape allows) — the refit is held to a tolerance.  A conv whose bias is fused into its epilogue (MobileNet's
logits) has the bias subtracted from the gathered outputs (fp32 rounding of y - b).  A conv with a fused activation
(conv -> Relu with nothing between, LeNet) has no materialised pre-activation output and is refused.  Without a
pre-trained checkpoint (synthetic runs) the full model keeps its seed initialisation.
--enbl_compact_ft (off by default) runs the fine-tune steps at the pruned width (compact.CompactTrainer), after the
selection or after --cpr_warm_start, and expands the
state back before every save, so the masked full-width checkpoint, evaluate() and the export tool are unchanged.  Its
deviations: (a) producer channels that no consumer reads are frozen at their post-selection values instead of decaying
under weight decay, and the reported loss omits their L2 term; they cannot influence the logits either way; (b) the
fp32 accumulation order of a narrowed K dimension differs from the masked one, so logits agree to rounding."""
import math
from timeit import default_timer as timer

import numpy as np
import torch

from ... import ops
from ...flags import FLAGS, DEFINE_string, DEFINE_float, DEFINE_boolean, DEFINE_integer
from ..abstract_learner import save_checkpoint
from ..channel_pruning_base import ChannelPrunedBase

DEFINE_string('cpr_save_path', './models_cpr/model.ckpt', 'CPR: model\'s save path')
DEFINE_string('cpr_save_path_eval', './models_cpr_eval/model.ckpt', 'CPR: model\'s save path for evaluation')
DEFINE_string('cpr_save_path_ws', './models_cpr_ws/model.ckpt', 'CPR: model\'s save path for warm start')
DEFINE_float('cpr_prune_ratio', 0.5, 'CPR: pruning ratio')
DEFINE_boolean('cpr_skip_frst_layer', True, 'CPR: skip the first layer for pruning')
DEFINE_boolean('cpr_skip_last_layer', False, 'CPR: skip the last layer for pruning')
DEFINE_string('cpr_skip_op_names', None, 'CPR: comma-separated Conv2D operations names to be skipped')
DEFINE_integer('cpr_nb_smpls', 5000, 'CPR: # of cached training samples for channel pruning')
DEFINE_integer('cpr_nb_crops_per_smpl', 10, 'CPR: # of random crops per sample')
DEFINE_float('cpr_ista_lrn_rate', 1e-2, 'CPR: ISTA\'s learning rate')
DEFINE_integer('cpr_ista_nb_iters', 100, 'CPR: # of iterations in ISTA')
DEFINE_float('cpr_lstsq_lrn_rate', 1e-3, 'CPR: least-sqaure regression\'s learning rate')
DEFINE_integer('cpr_lstsq_nb_iters', 100, 'CPR: # of iterations in least-square regression')
DEFINE_boolean('cpr_warm_start', False, 'CPR: use a channel-pruned model for warm start '
                                        '(the channel selection process will be skipped)')

ERR_MAX = 1e-6          # bound on mean((patch * W - output)^2) of the sampling check (:722-723)


def prune_ratio_list(kernel_names, prune_ratio, skip_frst_layer, skip_last_layer, skip_op_names):
    """each layer's pruning ratio (:549-567); 0 does not skip the layer"""
    ratios = [prune_ratio] * len(kernel_names)
    if skip_frst_layer:
        ratios[0] = 0.0
    if skip_last_layer:
        ratios[-1] = 0.0
    skip_names = skip_op_names.split(',') if skip_op_names is not None else []
    for idx, name in enumerate(kernel_names):
        for skip_name in skip_names:
            if skip_name in name:
                ratios[idx] = 0.0
                print('skip %s since no pruning is required' % name)
                break
    return ratios


def draw_samples(rng, nb_mbtcs, bs, oh, ow, nb_crops, nb_insts_min):
    """The host draws of one layer's sampling loop (:611-628): per cached batch, (randint(oh), randint(ow)) per crop,
    until more than nb_insts_min instances are collected; then the kept instances.  Returns
    ([per batch: [(oh, ow)] * nb_crops], dst) where dst[g] = row of instance g in the regression problem (-1: dropped);
    instance g = offset of its batch + crop * bs + n, the order of the reference's vstack."""
    draws, nb_insts = [], 0
    for _ in range(nb_mbtcs):
        pos = []
        for _ in range(nb_crops):
            idx_oh = rng.randint(oh)
            idx_ow = rng.randint(ow)
            pos.append((idx_oh, idx_ow))
        draws.append(pos)
        nb_insts += bs * nb_crops
        if nb_insts > nb_insts_min:
            break
    idxs_inst = rng.choice(nb_insts, size=(nb_insts_min), replace=False)
    dst = np.full(nb_insts, -1, dtype=np.int64)
    dst[idxs_inst] = np.arange(nb_insts_min)
    return draws, dst


def sample_rows(pos, bs, dst):
    """int32 [bs * len(pos), 4] rows (n, oh, ow, dst) of one batch, crop-major (pf_cpr_sample)"""
    rows = np.zeros((len(pos) * bs, 4), dtype=np.int32)
    for k, (idx_oh, idx_ow) in enumerate(pos):
        rows[k * bs:(k + 1) * bs, 0] = np.arange(bs)
        rows[k * bs:(k + 1) * bs, 1] = idx_oh
        rows[k * bs:(k + 1) * bs, 2] = idx_ow
    rows[:, 3] = dst
    return rows


def draw_regression(rng, nb_insts, cin, cout):
    """the host draws of one layer's sparse regression (:751-770): the secondary sample of
    N' = ceil(min(N, N / Cout * 10)) instances, then the initial mask (float64 [Cin, 1])"""
    bs_rdc = int(math.ceil(min(nb_insts, nb_insts / cout * 10.0)))
    idxs = rng.choice(nb_insts, size=(bs_rdc), replace=False)
    return idxs, rng.uniform(size=(cin, 1))


def gamma_search(solve, nnz_target):
    """<gamma>'s upper bound by doubling from 0.1, then bisection (:787-812).  solve(gamma) -> nnz; the mask of the
    last solve is the result.  Returns [(gamma, nnz)] of every solve."""
    log = []
    ubnd = 0.1
    while True:
        nb_chns_nnz = solve(ubnd)
        log.append((ubnd, nb_chns_nnz))
        if nb_chns_nnz <= nnz_target:
            break
        ubnd *= 2.0
    lbnd = 0.0
    while nb_chns_nnz != nnz_target and ubnd - lbnd > 1e-8:
        val = (lbnd + ubnd) / 2.0
        nb_chns_nnz = solve(val)
        log.append((val, nb_chns_nnz))
        if nb_chns_nnz < nnz_target:
            ubnd = val
        elif nb_chns_nnz > nnz_target:
            lbnd = val
        else:
            break
    return log


class ChannelPrunedRmtLearner(ChannelPrunedBase):  # pylint: disable=too-many-instance-attributes
    SAVE_PATH_FLAG = 'cpr_save_path'

    def __init__(self, sm_writer, model_helper, seed=1):
        super(ChannelPrunedRmtLearner, self).__init__(sm_writer, model_helper)
        self.seed = seed                                                   # of the host RandomState

    # ------------------------------------------------------------------ training (:146-193)
    def train(self, nb_iters=None):
        self.select_on_primary(FLAGS.cpr_save_path_ws, select=not FLAGS.cpr_warm_start)
        self.fine_tune(nb_iters, path_eval=FLAGS.cpr_save_path_eval)

    def init_masks(self):
        """masks = reduce_sum(W^2, [0, 1, 3]) > 0 per input channel (:255-263), fresh optimizer state (:159)"""
        ex = self.sess_train
        for v in self.maskable_vars:
            ops.cpg_channel_mask(ex.store.view(v), ex.store.view(v, ex.MASK))
        ex.reset_optimizer_state()
        ex.step_count = 0

    def layer_ratios(self):
        return prune_ratio_list([v.name for v in self.maskable_vars], FLAGS.cpr_prune_ratio, FLAGS.cpr_skip_frst_layer,
                                FLAGS.cpr_skip_last_layer, FLAGS.cpr_skip_op_names)

    # ------------------------------------------------------------------ channel selection (:546-649)
    def cache_batches(self, nb_batches=None):
        """ceil(cpr_nb_smpls / batch_size) training mini-batches by default, drawn once (:579-582)"""
        if nb_batches is None:
            nb_batches = int(math.ceil(FLAGS.cpr_nb_smpls / FLAGS.batch_size))
        return super(ChannelPrunedRmtLearner, self).cache_batches(nb_batches)

    def choose_channels(self, cached=None):
        """Choose channels for all convolutional layers (:546-649), save the result to cpr_save_path_ws."""
        self.init_from_full()
        rng = np.random.RandomState(self.seed)
        if cached is None:
            cached = self.cache_batches()
        ex_f, ex_p = self.selection_executors()
        self.selection_log = []
        for idx_layer in range(self.nb_layers):
            if self.is_primary_worker('global'):
                print('layer #%d: pr = %.2f (target)' % (idx_layer, self.prune_ratios[idx_layer]))
                print('kernel name = %s, shape = %s' % (self.maskable_vars[idx_layer].name,
                                                       self.maskable_vars[idx_layer].shape))
            self.select_layer(idx_layer, rng, cached, ex_f, ex_p)
            print('pruning ratio: %e (krn)' % self.pr_maskable())
        del ex_f, ex_p
        torch.cuda.empty_cache()
        print('model saved to ' + save_checkpoint(FLAGS.cpr_save_path_ws, self.sess_train.store.state_dict()))

    def select_layer(self, idx_layer, rng, cached, ex_f, ex_p):
        """sampling, sparse regression and refit of one layer; returns its log record"""
        op_f, op_p = self.conv_ops_full[idx_layer], self.conv_ops_prnd[idx_layer]
        for ex_, op in ((ex_f, op_f), (ex_p, op_p)):
            self.check_regressable(ex_, op)
        ratio = self.prune_ratios[idx_layer]
        dev = self.device
        w_p = self.sess_train.store.view(op_p.vars['kernel'])
        w_f = self.store_full.view(op_f.vars['kernel'])
        kh, kw, cin, cout = w_p.shape
        kdim = kh * kw * cin
        d = ex_p.desc[op_p]
        bs = d.n
        times = {}
        sync = torch.cuda.synchronize

        # ---- sampling (:608-631)
        t0 = timer()
        nb_insts_min = FLAGS.cpr_nb_crops_per_smpl * FLAGS.cpr_nb_smpls
        draws, dst = draw_samples(rng, len(cached), bs, d.p, d.q, FLAGS.cpr_nb_crops_per_smpl, nb_insts_min)
        X = torch.empty(nb_insts_min, kdim, dtype=torch.float32, device=dev)
        Y = torch.empty(nb_insts_min, cout, dtype=torch.float32, device=dev)
        nloc = bs * FLAGS.cpr_nb_crops_per_smpl
        Xs = torch.empty(nloc, kdim, dtype=torch.float32, device=dev)
        Ys, P, R = (torch.empty(nloc, cout, dtype=torch.float32, device=dev) for _ in range(3))
        l2ws = torch.empty(ops.L2_PARTIALS, dtype=torch.float32, device=dev)
        errs = torch.zeros(len(draws), 2, 4, dtype=torch.float32, device=dev)
        dchk = ops.conv_desc(nloc, 1, 1, kdim, cout, 1, 1, 1, 1, 1, 1, 0, 0)
        local = np.arange(nloc)
        bias_f = self.store_full.view(op_f.vars['bias']) if 'bias' in op_f.vars else None
        bias_p = self.sess_train.store.view(op_p.vars['bias']) if 'bias' in op_p.vars else None

        def conv_input(ex_, op):
            xp = ex_.planes_of(op.inputs[0])
            return (None, xp) if xp is not None else (ex_.T(op.inputs[0]).contiguous(), None)

        for b, pos in enumerate(draws):
            ex_p.buf[self.images].copy_(cached[b])
            ex_f.forward(training=True, upto=op_f)
            ex_p.forward(training=True, upto=op_p)
            x_p, xp_p = conv_input(ex_p, op_p)
            x_f, xp_f = conv_input(ex_f, op_f)
            y_f, y_p = ex_f.buf[op_f.output], ex_p.buf[op_p.output]
            rows = torch.from_numpy(sample_rows(pos, bs, dst[b * nloc:(b + 1) * nloc])).to(dev)
            ops.cpr_sample(d, x_p, y_f, rows, X, Y, planes=xp_p, bias=bias_f)
            # patch * W == output for both models (:715-723), mean squared error on the device
            rows_loc = torch.from_numpy(sample_rows(pos, bs, local)).to(dev)
            for j, (x_, xp_, y_, w_, bias_) in enumerate(((x_f, xp_f, y_f, w_f, bias_f), (x_p, xp_p, y_p, w_p, bias_p))):
                ops.cpr_sample(d, x_, y_, rows_loc, Xs, Ys, planes=xp_, bias=bias_)
                ops.conv2d_fwd(dchk, Xs, w_, None, False, P)
                ops.cpg_diff_l2(P, Ys, R, errs[b, j, :1], l2ws)
        err = errs[:, :, 0].cpu().numpy().astype(np.float64) * 2.0 / (nloc * cout)
        if not np.all(err < ERR_MAX):
            raise RuntimeError('layer #%d: unable to recover output feature maps - full / prnd (%e / %e)'
                               % (idx_layer, err[:, 0].max(), err[:, 1].max()))
        del Xs, Ys, P, R
        sync()
        times['sample'] = timer() - t0

        # ---- sparse regression (:740-812)
        t0 = timer()
        nnz_target = int(cin * (1.0 - ratio))
        idxs, m0_np = draw_regression(rng, nb_insts_min, cin, cout)
        idx_dev = torch.from_numpy(idxs.astype(np.int32)).to(dev)
        g = torch.empty((cin + 1) ** 2 + 1, dtype=torch.float64, device=dev)
        gf = torch.empty(cin * cin, dtype=torch.float32, device=dev)
        bf = torch.empty(cin, dtype=torch.float32, device=dev)
        ops.cpr_gram(X, Y, idx_dev, w_p, g, gf, bf)
        m0 = torch.from_numpy(m0_np.astype(np.float32).reshape(-1)).to(dev)   # (a float32 placeholder, :440)
        sync()
        times['gram'] = timer() - t0
        t0 = timer()
        m = torch.empty(cin, dtype=torch.float32, device=dev)
        ws = torch.empty(2 * cin, dtype=torch.float32, device=dev)
        nnz = torch.zeros(1, dtype=torch.int32, device=dev)

        def solve(gamma):
            ops.cpr_ista(gf, bf, m0, FLAGS.cpr_ista_lrn_rate, gamma, FLAGS.cpr_ista_nb_iters, m, ws, nnz)
            nb = int(nnz.item())
            print('x = %e -> nb_chns_nnz = %d' % (gamma, nb))
            return nb
        search = gamma_search(solve, nnz_target)
        times['search'] = timer() - t0

        # ---- least-square refit (:814-842)
        t0 = timer()
        ops.cpr_mask_channels(X, m, kh * kw, cin, 1)
        del g, gf, bf
        lst = ops.CprLstsq(X, Y, self.sess_train.conv_path)
        loss_beg, loss_end = lst.run(w_p, FLAGS.cpr_lstsq_nb_iters, FLAGS.cpr_lstsq_lrn_rate, FLAGS.loss_w_dcy)
        ops.cpr_mask_channels(w_p, m, kh * kw, cin, cout)
        print('losses: %e -> %e (reg)' % (loss_beg, loss_end))
        sync()
        times['refit'] = timer() - t0
        rec = dict(layer=idx_layer, ratio=ratio, nnz_target=nnz_target, search=search, nnz=search[-1][1],
                   loss=(loss_beg, loss_end), mask=m.cpu().numpy(), idxs=idxs, m0=m0.cpu().numpy(),
                   err=err, times=times, tc=(lst.tc_fwd, lst.tc_wgrad))
        self.selection_log.append(rec)
        return rec
