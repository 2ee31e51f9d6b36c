"""LASSO channel-pruning learner (/root/reference/learners/channel_pruning/learner.py, channel_pruner.py).

He, Zhang & Sun, "Channel Pruning for Accelerating Very Deep Neural Networks" (ICCV 2017).  Two copies of the network
live in one graph, as in the other channel-pruning learners: the FULL model under scope 'model' (restored from the
pre-trained checkpoint, never changed) and the model being pruned under 'pruned_model'.  The reference prunes one model
in place and keeps the full model's sampled features from before the first layer was pruned (extract_features,
channel_pruner.py:263-341); the full model's outputs here are those same values, recomputed per layer on the same cached
batches.

train() = channel selection (compress, :727-800), layer by layer in `thisconvs` order (the ops named .../Conv2D,
depthwise convs excluded), then fine-tuning with masked gradients.  Layer i:
  * preserve ratio: 1 for the first and the last layer; otherwise cp_uniform_preserve_ratio (--cp_prune_option uniform)
    or the i-th entry of cp_prune_list_file (list; 1 past its end).  A ratio of exactly 1 leaves the layer untouched.
    The kept count is max(int(np.around(Cin * ratio)), 1) (:607).
  * sampling (:263-341, :391-412): cp_nb_batches training batches are drawn once.  Per batch and per sampled tensor
    (every conv output, and after a conv that is the last of a residual block its Add output) cp_nb_points_per_layer
    positions are drawn, each shared by the whole batch.  X = the current model's R x S x Cin input patches there, Y =
    the FULL model's conv outputs (pf_cp_sample).  After the last conv of a residual block Y += the Add's output of the
    full model minus that of the current model, at the Add's own positions (residual_branch_diff, :579-586).
  * selection: with cp_lasso, min(400, N // 20) rows are drawn with randint, the design matrix
    product[(s, o), c] = sum_hw X[s, hw, c] W2[hw, c, o] and its Gram [P | y]^T [P | y] are formed in float64 on the
    device (pf_cp_gram), and the LARS-Lasso path (lars.py) is bisected on alpha as the reference does (:496-565).
    Without cp_lasso: the kept channels are those of largest L1 norm of W2 (:623-626).
  * refit (:569-573, :627-630): the kept input channels' weights are the least-squares fit of Y on X's kept columns.
    The normal equations [X_k | Y]^T [X_k | Y] are formed in float64 on the device (pf_cp_normal_eq) and solved in
    float64 by Cholesky, falling back to numpy.linalg.lstsq where they are singular to working precision.  sklearn's LinearRegression
    solves X_k W = Y by lstsq directly: on a full-rank X_k the two agree to float64 eps times cond(X_k)^2, and on a
    rank-deficient X_k both return the minimum-norm solution.
  * prune_W2 / prune_W1 (:665-725, :757-768): W2's dropped input channels are zeroed; if the conv is W1-prunable
    (producer_conv below), its producer's output channels and bias are zeroed, walking through depthwise producers to
    their own producer.
Fine-tuning: the masked Momentum step of the other channel-pruning learners (Executor.run_step with the maskable
kernels), where every conv kernel's mask is its kept input channels times its kept output channels (the reference's
fake_pruning_dict, learner.py:381-421), for nb_iters_train steps.  The selected model is saved to
cp_channel_pruned_path, the fine-tuned one to save_path (the reference's __save_model), both as masked full-width
checkpoints, so --exec_mode eval and tools/export_chn_pruned.py read them as they read the other learners'.

All host randomness comes from one np.random.RandomState(seed), drawn in the reference's order: per batch and per sampled
tensor randint(H, size=cp_nb_points_per_layer) then randint(W, ...); then per selected layer (with cp_lasso) the
design-matrix rows.
Not supported: --cp_prune_option auto (the reference's default, a DDPG search over the preserve ratios) raises, and
list groups are refused: --cp_prune_option list with cp_list_group below the number of convs (the reference re-samples,
saves and fine-tunes at every group boundary) and cp_finetune / cp_retrain (which only act between groups) raise.
--enbl_compact_ft is refused for this learner.  Flagged deviations: a conv with a fused activation (LeNet) has no
materialised output to regress onto and is refused; a depthwise producer that is not itself W1-prunable (the
reference would loop forever) has its own channels zeroed instead."""
from timeit import default_timer as timer

import numpy as np
import torch

from ... import ops
from ...flags import FLAGS, DEFINE_string, DEFINE_float, DEFINE_boolean, DEFINE_integer
from ..abstract_learner import save_checkpoint
from ..channel_pruning_base import ChannelPrunedBase
from . import lars

# learner.py:38-80
DEFINE_string('cp_prune_option', 'auto', 'the action we want to prune the channel you can select one of the following '
              'option: uniform: prune with a uniform compression ratio; list: prune with a list of compression ratio')
DEFINE_string('cp_prune_list_file', 'ratio.list',
              'the prune list file which contains the compression ratio of each convolution layers')
DEFINE_string('cp_channel_pruned_path', './models/pruned_model.ckpt', 'channel pruned model\'s save path')
DEFINE_string('cp_best_path', './models/best_model.ckpt', 'channel pruned model\'s temporary save path')
DEFINE_string('cp_original_path', './models/original_model.ckpt', 'channel pruned model\'s temporary save path')
DEFINE_float('cp_preserve_ratio', 0.5, 'How much computation cost desired to be preserved after pruning')
DEFINE_float('cp_uniform_preserve_ratio', 0.6, 'How much computation cost desired to be preserved each layer')
DEFINE_float('cp_noise_tolerance', 0.15,
             'the noise tolerance which is used to restrict the maximum reward to avoid an unexpected speedup')
DEFINE_float('cp_lrn_rate_ft', 1e-4, 'CP: learning rate for global fine-tuning')
DEFINE_float('cp_nb_iters_ft_ratio', 0.2, 'CP: the ratio of total iterations for global fine-tuning')
DEFINE_boolean('cp_finetune', False, 'CP: whether finetuning between each list group')
DEFINE_boolean('cp_retrain', False, 'CP: whether retraining between each list group')
DEFINE_integer('cp_list_group', 1000, 'CP: # of iterations for fast evaluation')
DEFINE_integer('cp_nb_rlouts', 200, 'CP: # of roll-outs for the RL agent')
DEFINE_integer('cp_nb_rlouts_min', 50, 'CP: # of roll-outs for the RL agent')
# channel_pruner.py:35-49
DEFINE_boolean('cp_lasso', True, 'If True use lasso and reconstruction otherwise prune according to weight magnitude')
DEFINE_boolean('cp_quadruple', False, 'Restric the channels after pruning is a mutiple of 4')
DEFINE_string('cp_reward_policy', 'accuracy', 'If reward_policy equals accuracy, it means learning to achieve high '
              'accuracy with guaranteed low flops, else if reward_policy equals flops, it means learning to achieve low '
              'flops with guaranted accuracy.')
DEFINE_integer('cp_nb_points_per_layer', 10, 'Sample how many point for each layer')
DEFINE_integer('cp_nb_batches', 30, 'Input how many bathes data into a model')

PASS_W1 = ('Relu', 'FusedBatchNorm', 'MaxPool', 'Identity', 'Relu6')          # model_wrapper.py:351-356 (BiasAdd is
PASS_ADD = ('Relu', 'FusedBatchNorm', 'DepthwiseConv2dNative', 'MaxPool', 'Relu6')   # part of Conv2D here) / :322-327


def producer_conv(op):
    """is_W1_prunable (model_wrapper.py:343-369) over graph.py's ops: the Conv2D / depthwise op reached from op's input
    through Relu, Relu6, batch norm, max pooling and Identity only, or None.  A conv with explicit (pad_beg, pad_end)
    padding is ResNet's strided fixed-padding conv, which the reference builds as tf.pad + VALID conv: the Pad op ends
    the walk there, so it is not W1-prunable."""
    if not isinstance(op.attrs.get('padding', 'same'), str):
        return None
    o = op
    while True:
        o = o.inputs[0].op if o.inputs else None
        if o is None or o.type == 'Placeholder':
            return None
        if o.type in PASS_W1:
            continue
        if o.type in ('Conv2D', 'DepthwiseConv2dNative'):
            return o
        return None


def add_after(op):
    """get_Add_if_is_last_in_resblock (model_wrapper.py:303-341): follow the FIRST consumer that is a Relu, Relu6, batch
    norm, depthwise conv or max pooling; the Add op if the walk ends at one, else None"""
    cur = op
    while True:
        go_on = False
        for c in cur.output.consumers:
            cur = c
            if c.type in PASS_ADD:
                go_on = True
                break
        if go_on:
            continue
        return cur if cur.type == 'Add' and cur is not op else None


def w1_target(op):
    """the op whose output channels prune_W1 zeroes for conv `op` (:757-766), or None"""
    father = producer_conv(op)
    while father is not None and father.type == 'DepthwiseConv2dNative':
        grand = producer_conv(father)
        if grand is None:
            break
        father = grand
    return father


def sampled_tensors(convs):
    """extract_features' names (:215-227, :291-292): every conv's output, and after a conv that is the last of a residual
    block its Add's output, duplicates removed (first occurrence kept).  Returns the ops whose outputs are sampled."""
    out = []
    for op in convs:
        for o in (op, add_after(op)):
            if o is not None and o not in out:
                out.append(o)
    return out


def preserve_ratios(nb_layers, option, uniform_ratio, list_file):
    """each layer's preserve ratio as compress() receives it (:727-747, learner.py:513-566)"""
    if option == 'auto':
        raise ValueError('--cp_prune_option auto (the DDPG search over preserve ratios) is not supported by this build; '
                         'pass --cp_prune_option uniform or --cp_prune_option list')
    if option == 'uniform':
        ratios = [float(uniform_ratio)] * nb_layers
    elif option == 'list':
        lst = [float(r) for r in np.loadtxt(list_file, delimiter=',', ndmin=1)]
        ratios = [lst[i] if i < len(lst) else 1.0 for i in range(nb_layers)]
    else:
        raise ValueError('unrecognized --cp_prune_option: ' + option)
    ratios[0] = 1.0
    ratios[-1] = 1.0
    return ratios


def refuse_list_groups(nb_layers, option, list_group, finetune, retrain):
    """The reference's list mode prunes cp_list_group layers at a time; between groups it re-extracts the features
    from the partly pruned model, saves, and fine-tunes (learner.py:531-579), with cp_finetune / cp_retrain choosing
    how.  Only the single group (every conv in one group) is built here: the rest raises rather than silently running
    a different algorithm."""
    if finetune or retrain:
        raise ValueError('--cp_finetune / --cp_retrain (fine-tuning between list groups) are not supported by this '
                         'build: leave them False')
    if option == 'list' and list_group < nb_layers:
        raise ValueError('--cp_prune_option list with --cp_list_group %d below the number of convs (%d) prunes in '
                         'several groups, which this build does not support: pass --cp_list_group %d or more'
                         % (list_group, nb_layers, nb_layers))


def kept_count(c, ratio):
    return max(int(np.around(c * ratio)), 1)


def draw_positions(rng, nb_batches, shapes, nb_points):
    """[batch][tensor] = (x_samples, y_samples) (:317-330); shapes: (H, W) of every sampled tensor"""
    return [[(rng.randint(0, h, nb_points), rng.randint(0, w, nb_points)) for h, w in shapes] for _ in range(nb_batches)]


def sample_rows(pos, pos_add, bs, base):
    """int32 [bs * nb_points, 8] rows (n, oh, ow, dst, rh, rw, 0, 0) of one batch; row order n-major, then the point
    (feat[:, x_samples, y_samples, :].reshape(-1, C))"""
    xs, ys = pos
    k = len(xs)
    rows = np.zeros((bs * k, 8), dtype=np.int32)
    rows[:, 0] = np.repeat(np.arange(bs), k)
    rows[:, 1] = np.tile(xs, bs)
    rows[:, 2] = np.tile(ys, bs)
    rows[:, 3] = base + np.arange(bs * k)
    if pos_add is not None:
        rows[:, 4] = np.tile(pos_add[0], bs)
        rows[:, 5] = np.tile(pos_add[1], bs)
    return rows


class ChannelPrunedLearner(ChannelPrunedBase):  # pylint: disable=too-many-instance-attributes
    SAVE_PATH_FLAG = 'save_path'

    def __init__(self, sm_writer, model_helper, seed=1):
        super(ChannelPrunedLearner, self).__init__(sm_writer, model_helper)
        self.seed = seed                                                   # of the host RandomState
        self.sampled_prnd = sampled_tensors(self.conv_ops_prnd)
        self.sampled_full = sampled_tensors(self.conv_ops_full)

    # ------------------------------------------------------------------ training
    def train(self, nb_iters=None):
        self.select_on_primary(FLAGS.cp_channel_pruned_path)
        self.fine_tune(nb_iters, save_first=False)

    def init_masks(self):
        """mask = kept input channels x kept output channels of every conv kernel (learner.py:406-419), read from the
        zeros the selection left: an input channel is kept if any of its weights is non-zero, an output channel if
        any of its weights is; fresh optimizer state (:426)"""
        ex = self.sess_train
        for v in self.maskable_vars:
            w = ex.store.view(v)
            nz = w != 0
            keep_in = nz.any(dim=3).any(dim=1).any(dim=0)
            keep_out = nz.any(dim=2).any(dim=1).any(dim=0)
            m = keep_in.view(1, 1, -1, 1) & keep_out.view(1, 1, 1, -1)
            ex.store.view(v, ex.MASK).copy_(m.expand_as(w).to(torch.float32))
        ex.reset_optimizer_state()
        ex.step_count = 0

    def layer_ratios(self):
        """each layer's preserve ratio; list groups are refused first, before any executor is built"""
        refuse_list_groups(self.nb_layers, FLAGS.cp_prune_option, FLAGS.cp_list_group, FLAGS.cp_finetune,
                           FLAGS.cp_retrain)
        return preserve_ratios(self.nb_layers, FLAGS.cp_prune_option, FLAGS.cp_uniform_preserve_ratio,
                               FLAGS.cp_prune_list_file)

    # ------------------------------------------------------------------ channel selection
    def cache_batches(self, nb_batches=None):
        """cp_nb_batches training mini-batches by default, drawn once (:310-314)"""
        if nb_batches is None:
            nb_batches = FLAGS.cp_nb_batches
        return super(ChannelPrunedLearner, self).cache_batches(nb_batches)

    def choose_channels(self, cached=None):
        """compress() over every layer (learner.py:513-529), then save to cp_channel_pruned_path"""
        self.init_from_full()
        rng = np.random.RandomState(self.seed)
        if cached is None:
            cached = self.cache_batches()
        shapes = [(op.output.shape[1], op.output.shape[2]) for op in self.sampled_prnd]
        self.positions = draw_positions(rng, len(cached), shapes, FLAGS.cp_nb_points_per_layer)
        ex_f, ex_p = self.selection_executors()
        self.selection_log = []
        for idx_layer in range(self.nb_layers):
            ratio = self.prune_ratios[idx_layer]
            if ratio == 1:
                continue
            if self.is_primary_worker('global'):
                print('layer #%d: preserve ratio = %.2f, kernel = %s %s'
                      % (idx_layer, ratio, self.maskable_vars[idx_layer].name, self.maskable_vars[idx_layer].shape))
            self.select_layer(idx_layer, rng, cached, ex_f, ex_p)
        del ex_f, ex_p
        torch.cuda.empty_cache()
        print('pruning ratio: %e (krn)' % self.pr_maskable())
        print('model saved to ' + save_checkpoint(FLAGS.cp_channel_pruned_path, self.sess_train.store.state_dict()))

    def sample_layer(self, idx_layer, cached, ex_f, ex_p):
        """X [N, R*S*Cin] (fp32) and Y [N, Cout] (float64) of one layer on the device, N = batches x batch x points"""
        op_f, op_p = self.conv_ops_full[idx_layer], self.conv_ops_prnd[idx_layer]
        for ex_, op in ((ex_f, op_f), (ex_p, op_p)):
            self.check_regressable(ex_, op)
        add_f, add_p = add_after(op_f), add_after(op_p)
        t_conv = self.sampled_prnd.index(op_p)
        t_add = self.sampled_prnd.index(add_p) if add_p is not None else None
        d = ex_p.desc[op_p]
        bs, nb_pts = d.n, FLAGS.cp_nb_points_per_layer
        kh, kw, cin, cout = self.sess_train.store.view(op_p.vars['kernel']).shape
        nloc = bs * nb_pts
        X = torch.empty(nloc * len(cached), kh * kw * cin, dtype=torch.float32, device=self.device)
        Y = torch.empty(nloc * len(cached), cout, dtype=torch.float64, device=self.device)
        bias_f = self.store_full.view(op_f.vars['bias']) if 'bias' in op_f.vars else None
        for b, images in enumerate(cached):
            ex_p.buf[self.images].copy_(images)
            ex_f.forward(training=True, upto=add_f if add_f is not None else op_f)
            ex_p.forward(training=True, upto=add_p if add_p is not None else op_p)
            xp = ex_p.planes_of(op_p.inputs[0])
            x = None if xp is not None else ex_p.T(op_p.inputs[0]).contiguous()
            pos = self.positions[b]
            rows = sample_rows(pos[t_conv], pos[t_add] if t_add is not None else None, bs, b * nloc)
            rf = rc = None
            if add_f is not None:
                rf, rc = ex_f.T(add_f.output).contiguous(), ex_p.T(add_p.output).contiguous()
            ops.cp_sample(d, x, ex_f.buf[op_f.output], torch.from_numpy(rows).to(self.device), X, Y, planes=xp,
                          bias=bias_f, res_full=rf, res_cur=rc)
        return X, Y

    def select_layer(self, idx_layer, rng, cached, ex_f, ex_p):
        """prune_kernel + prune_W1 + prune_W2 of one layer (:588-640, :665-725, :756-768); returns its log record"""
        op_p = self.conv_ops_prnd[idx_layer]
        sync = torch.cuda.synchronize
        times = {}
        store = self.sess_train.store
        w_p = store.view(op_p.vars['kernel'])
        kh, kw, cin, cout = w_p.shape
        c_new = kept_count(cin, self.prune_ratios[idx_layer])

        t0 = timer()
        X, Y = self.sample_layer(idx_layer, cached, ex_f, ex_p)
        sync()
        times['sample'] = timer() - t0
        nb_samples = X.shape[0]
        search, samples = [], None
        if FLAGS.cp_lasso:
            t0 = timer()
            samples = rng.randint(0, nb_samples, min(400, nb_samples // 20))
            g = torch.empty((cin + 1) ** 2 + 1, dtype=torch.float64, device=self.device)
            ops.cp_gram(X, Y, torch.from_numpy(samples.astype(np.int32)).to(self.device), w_p, g)
            g_aug = g[:(cin + 1) ** 2].view(cin + 1, cin + 1).cpu().numpy()
            times['gram'] = timer() - t0
            t0 = timer()
            idxs, search = lars.lasso_select(g_aug[:cin, :cin], g_aug[:cin, cin], len(samples) * cout, c_new,
                                             quadruple=FLAGS.cp_quadruple)
            times['solve'] = timer() - t0
        else:
            idxs = lars.l1_select(w_p.cpu().numpy(), c_new)

        # ---- refit of the kept channels (:569-573)
        t0 = timer()
        kept = np.where(idxs)[0]
        cols = (np.arange(kh * kw)[:, None] * cin + kept[None, :]).reshape(-1)
        k = cols.size
        g = torch.empty((k + cout) ** 2 + 1, dtype=torch.float64, device=self.device)
        ops.cp_normal_eq(X, Y, torch.from_numpy(cols.astype(np.int32)).to(self.device), g)
        g_aug = g[:(k + cout) ** 2].view(k + cout, k + cout).cpu().numpy()
        coef, how = lars.solve_normal_equations(g_aug[:k, :k], g_aug[:k, k:])
        w_new = np.zeros((kh, kw, cin, cout), dtype=np.float32)
        w_new[:, :, kept, :] = coef.reshape(kh, kw, len(kept), cout)
        w_p.copy_(torch.from_numpy(w_new))
        times['refit'] = timer() - t0
        del X, Y

        # ---- prune_W1 (:665-699)
        father = w1_target(op_p)
        if father is not None:
            drop = torch.from_numpy(~idxs).to(self.device)
            wf = store.view(father.vars['kernel'])
            if father.type == 'DepthwiseConv2dNative':
                wf[:, :, drop, :] = 0
            else:
                wf[:, :, :, drop] = 0
            if 'bias' in father.vars:
                store.view(father.vars['bias'])[drop] = 0
        sync()
        rec = dict(layer=idx_layer, c_new=c_new, kept=idxs.copy(), search=search, samples=samples, refit=how,
                   father=father.name if father is not None else None, times=times)
        print('layer #%d: Cin %d -> %d (%s), father = %s, times = %s'
              % (idx_layer, cin, int(idxs.sum()), how, rec['father'], ', '.join('%s %.3f s' % kv for kv in times.items())))
        self.selection_log.append(rec)
        return rec
