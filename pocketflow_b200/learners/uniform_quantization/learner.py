"""Uniform Quantization Learner (/root/reference/learners/uniform_quantization/learner.py:34-428).
Without buckets, min/max is calculated per layer, otherwise per bucket."""
import os
from timeit import default_timer as timer

import numpy as np

from ... import graph as G
from ...engine import Executor
from ...flags import FLAGS, DEFINE_integer, DEFINE_boolean, DEFINE_string
from ...utils.multi_gpu_wrapper import MultiGpuWrapper as mgw
from ...utils.lrn_rate_utils import piecewise_constant
from ..abstract_learner import AbstractLearner, latest_checkpoint, load_checkpoint, save_checkpoint
from ..distillation_helper import DistillationHelper
from .utils import UniformQuantization
from .bit_optimizer import BitOptimizer

DEFINE_integer('uql_weight_bits', 4, 'Number of bits to use for quantizing weights')
DEFINE_integer('uql_activation_bits', 32, 'Number of bits to use for quantizing activations')
DEFINE_boolean('uql_use_buckets', False, 'Use bucketing or not')
DEFINE_integer('uql_bucket_size', 256, 'Number of bucket size')
DEFINE_integer('uql_quant_epochs', 60, 'To be determined by datasets')
DEFINE_string('uql_save_quant_model_path', './uql_quant_models/uql_quant_model.ckpt',
              'dir to save quantization model')
DEFINE_boolean('uql_quantize_all_layers', False, 'If False, leaving first and last layers unquantized')
DEFINE_string('uql_bucket_type', 'channel', 'Two types for now: [channel, split]')


def setup_bnds_decay_rates(model_name, dataset_name):
    """ NOTE: The bnd_decay_rates here is mgw_size invariant (learner.py:50-70).
    lenet@cifar_10 leaves bnds unbound in the reference (UnboundLocalError, SURVEY A.6-1): the
    ResNet/CIFAR schedule is used for it here, a flagged deviation."""
    batch_size = FLAGS.batch_size if not FLAGS.enbl_multi_gpu else FLAGS.batch_size * mgw.size()
    nb_batches_per_epoch = int(FLAGS.nb_smpls_train / batch_size)
    mgw_size = int(mgw.size()) if FLAGS.enbl_multi_gpu else 1
    init_lr = FLAGS.lrn_rate_init * FLAGS.batch_size * mgw_size / FLAGS.batch_size_norm \
        if FLAGS.enbl_multi_gpu else FLAGS.lrn_rate_init
    if dataset_name == 'cifar_10':
        bnds = [nb_batches_per_epoch * 15, nb_batches_per_epoch * 40]
        decay_rates = [1e-3, 1e-4, 1e-5]
    elif dataset_name == 'ilsvrc_12':
        if model_name.startswith('resnet'):
            bnds = [nb_batches_per_epoch * 5, nb_batches_per_epoch * 20]
            decay_rates = [1e-4, 1e-5, 1e-6]
        elif model_name.startswith('mobilenet'):
            bnds = [nb_batches_per_epoch * 5, nb_batches_per_epoch * 30]
            decay_rates = [1e-4, 1e-5, 1e-6]
        else:
            raise ValueError('no fine-tuning schedule for model: ' + model_name)
    else:
        raise ValueError('Unrecognized dataset name')
    finetune_steps = nb_batches_per_epoch * FLAGS.uql_quant_epochs
    init_lr = init_lr if FLAGS.enbl_warm_start else FLAGS.lrn_rate_init
    return init_lr, bnds, decay_rates, finetune_steps


class UniformQuantLearner(AbstractLearner):
    # pylint: disable=too-many-instance-attributes
    '''Uniform quantization for weights and activations'''

    def __init__(self, sm_writer, model_helper):
        super(UniformQuantLearner, self).__init__(sm_writer, model_helper)
        if FLAGS.enbl_dst:
            self.helper_dst = DistillationHelper(sm_writer, model_helper, self.mpi_comm)
        self.ops = {}
        self.bit_placeholders = {}
        self.statistics = {}
        self._rl_initial_state = None
        self.__build_train()
        # The reference requires a pre-trained checkpoint here (download_model, learner.py:95-97);
        # the synthetic benchmark path starts from the seeded initialisation instead (SURVEY A.6-10).
        self.auto_barrier()
        bit_optimizer = BitOptimizer(self.dataset_name, self.weights, self.statistics, tuner=self,
                                     barrier_fn=self.auto_barrier)
        # the step is compiled with the flag bit-widths; the RL search (if enabled) then drives that step with
        # per-roll-out bit-widths and leaves the best allocation in place (learner.py:108-111)
        self.optimal_w_bit_list = [FLAGS.uql_weight_bits] * self.statistics['nb_matmuls']
        self.optimal_a_bit_list = [FLAGS.uql_activation_bits] * self.statistics['nb_activations']
        self.__compile()
        self.auto_barrier()
        if FLAGS.uql_enbl_rl_agent:
            self.optimal_w_bit_list, self.optimal_a_bit_list = bit_optimizer.run()
            self.rl_restore()
            self.rl_set_bits(self.optimal_w_bit_list, self.optimal_a_bit_list)
            self.auto_barrier()

    # ------------------------------------------------------------------ training
    def train(self, nb_iters=None):
        total_iters = self.finetune_steps if nb_iters is None else nb_iters
        if FLAGS.enbl_warm_start:
            self.__restore_model(is_train=True)
        self.auto_barrier()
        if FLAGS.enbl_multi_gpu:
            mgw.broadcast_global_variables([self.sess_train.store.P, self.sess_train.store.O])
        time_prev = timer()
        for idx_iter in range(total_iters):
            self.train_step()
            if (idx_iter + 1) % FLAGS.summ_step == 0:
                time_prev = self.__monitor_progress(self.sess_train.fetch_losses(), time_prev, idx_iter)
            if (idx_iter + 1) % FLAGS.save_step == 0:
                self.__save_model()
                self.evaluate()
                self.auto_barrier()
        self.__save_model()
        self.evaluate()

    def train_step(self):
        """One `sess.run(ops['train'])`: H2D of the batch, then the captured device step."""
        ex = self.sess_train
        self.h2d_bytes = self.feed(ex, self.iterator_train)
        ex.run_step(self.lrn_rate(ex.step_count), self.grad_allreduce())

    def evaluate(self, nb_iters=None):
        if not self.is_primary_worker():
            return None
        self.restore_for_eval(FLAGS.uql_save_quant_model_path)
        rows = self.eval_losses(nb_iters)
        losses, accuracies = [r['loss'] for r in rows], [r['acc_top1'] for r in rows]
        print('loss: {}'.format(np.mean(np.array(losses))))
        print('accuracy: {}'.format(np.mean(np.array(accuracies))))
        if FLAGS.uql_use_buckets:
            self.__show_bucket_storage(self.ops['bucket_storage'])
        return float(np.mean(losses)), float(np.mean(accuracies))

    def __eval_batch_size(self):
        """Real data is evaluated at the step's batch size (AbstractLearner.eval_iterator); the synthetic pool keeps
        the reference's nb_smpls_eval / batch_size_eval iteration count."""
        return self.iterator_train.batch_size if FLAGS.data_dir_local else FLAGS.batch_size_eval

    # ------------------------------------------------------------------ what the RL bit search drives
    def rl_restore(self):
        """Back to the pre-trained weights with a fresh optimizer (bit_optimizer.py:196-201): the latest checkpoint
        under --save_path if there is one, else the state this learner was built with."""
        ex = self.sess_train
        if self._rl_initial_state is None:
            fn = latest_checkpoint(os.path.dirname(FLAGS.save_path)) if os.path.isdir(os.path.dirname(FLAGS.save_path)) \
                else None
            self._rl_initial_state = load_checkpoint(fn) if fn is not None else ex.store.state_dict()
        ex.store.load_state_dict(self._rl_initial_state, strict=False)
        ex.reset_optimizer_state()
        if FLAGS.enbl_multi_gpu:
            mgw.broadcast_global_variables([ex.store.P, ex.store.O])

    def rl_set_bits(self, w_bits, a_bits):
        self.sess_train.set_quant_bits(w_bits, a_bits)

    def rl_finetune(self, nb_steps, disp_steps):
        """`nb_steps` training steps at the current bit-widths, then the fine-tuning step counter back to zero
        (bit_optimizer.py:243-252)."""
        time_prev = timer()
        for t_step in range(nb_steps):
            self.train_step()
            if disp_steps and (t_step + 1) % disp_steps == 0:
                time_prev = self.__monitor_progress(self.sess_train.fetch_losses(), time_prev, t_step)
        self.sess_train.step_count = 0

    def rl_evaluate(self):
        """(loss, top-1, top-5) averaged over nb_smpls_eval // batch_size_eval mini-batches (bit_optimizer.py:278-289)."""
        ex = self.sess_train
        losses, top1, top5 = [], [], []
        for _ in range(max(1, FLAGS.nb_smpls_eval // self.__eval_batch_size())):
            self.feed(ex, self.eval_iterator())
            ex.forward_eval_loss()
            r = ex.fetch_losses()
            losses.append(r['loss'])
            top1.append(r['acc_top1'])
            top5.append(r['acc_top5'])
        return float(np.mean(losses)), float(np.mean(top1)), float(np.mean(top5))

    # ------------------------------------------------------------------ graph
    def __build_train(self):
        self.graph_train = G.Graph()
        with self.graph_train.as_default():
            with G.variable_scope(self.data_scope):
                self.iterator_train = self.build_dataset_train()
                images, labels = self.iterator_train.get_next()
            self.images, self.labels = images, labels
            self.logits_dst = self.helper_dst.calc_logits(None, images) if FLAGS.enbl_dst else None
            with G.variable_scope(self.model_scope):
                logits = self.forward_train(images)
                self.logits = logits
                self.weights = [v for v in self.trainable_vars if 'kernel' in v.name or 'weight' in v.name]
                if not FLAGS.uql_quantize_all_layers:
                    self.weights = self.weights[1:-1]
                self.statistics['num_weights'] = [v.numel for v in self.weights]
                self.__quantize_train_graph()
                loss, metrics = self.calc_loss(labels, logits, self.trainable_vars)
                if self.dataset_name not in ('cifar_10', 'ilsvrc_12'):
                    raise ValueError("Unrecognized dataset name")
                if FLAGS.enbl_dst:
                    loss += self.helper_dst.calc_loss(logits, self.logits_dst)
                self.loss_spec, self.metrics = loss, metrics
        init_lr, bnds, decay_rates, self.finetune_steps = setup_bnds_decay_rates(self.model_name, self.dataset_name)
        self.lrn_rate = piecewise_constant([i for i in bnds], [init_lr * decay_rate for decay_rate in decay_rates])

    def __quantize_train_graph(self):
        """ Insert quantization nodes to the training graph. """
        uni_quant = UniformQuantization(self.graph_train, FLAGS.uql_bucket_size, FLAGS.uql_use_buckets,
                                        FLAGS.uql_bucket_type)
        matmul_ops = uni_quant.search_matmul_op(FLAGS.uql_quantize_all_layers)
        act_ops = uni_quant.search_activation_op()
        self.statistics['nb_matmuls'] = len(matmul_ops)
        self.statistics['nb_activations'] = len(act_ops)
        self.matmul_op_names = [op.name for op in matmul_ops]
        self.act_op_names = [op.name for op in act_ops]
        self.uni_quant = uni_quant

    def __compile(self):
        """Bind the bit lists (the reference feeds them through placeholders every sess.run) and lower
        the edited graph to kernels."""
        uq = self.uni_quant
        uq.insert_quant_op_for_weights(self.__build_quant_dict(self.matmul_op_names, self.optimal_w_bit_list))
        uq.insert_quant_op_for_activations(self.__build_quant_dict(self.act_op_names, self.optimal_a_bit_list))
        self.ops['bucket_storage'] = uq.bucket_storage
        world = mgw.size() if FLAGS.enbl_multi_gpu else 1
        teacher = None
        if FLAGS.enbl_dst:
            teacher = Executor(self.graph_train, self.images, self.logits_dst, self.device, train=False, seed=2)
            self.helper_dst.restore(teacher.store)
        self.sess_train = Executor(self.graph_train, self.images, self.logits, self.device, train=True,
                                   loss=self.loss_spec, labels=self.labels, optimizer=dict(kind='adam'),
                                   weight_quant=uq.weight_quant_spec(), act_quant=uq.act_quant_spec(),
                                   teacher=teacher, seed=1, grad_scale=1.0 / world)
        if teacher is not None:
            teacher.buf[self.images] = self.sess_train.buf[self.images]
            self.sess_train.share_im2col_from(teacher)
        self.sess_eval = self.sess_train

    @staticmethod
    def __build_quant_dict(names, bits):
        assert len(names) == len(bits), 'the length of op names and bit lists does not match'
        return dict(zip(names, bits))

    # ------------------------------------------------------------------ checkpoints / logging
    def __save_model(self):
        if not self.is_primary_worker():
            return
        fn = save_checkpoint(FLAGS.uql_save_quant_model_path, self.sess_train.store.state_dict(),
                             self.sess_train.step_count)
        print('quantized model saved to ' + fn)

    def __restore_model(self, is_train):
        self.restore_model(FLAGS.save_path if is_train else FLAGS.uql_save_quant_model_path)

    def __monitor_progress(self, r, time_prev, idx_iter):
        if not self.is_primary_worker():
            return None
        speed = FLAGS.batch_size * FLAGS.summ_step / (timer() - time_prev)
        if FLAGS.enbl_multi_gpu:
            speed *= mgw.size()
        lrn_rate = self.lrn_rate(idx_iter)
        if FLAGS.enbl_dst:
            print('iter #%d: lr = %e | dst_loss = %.4f | model_loss = %.4f | loss = %.4f | acc_top1 = %.4f | '
                  'acc_top5 = %.4f | speed = %.2f pics / sec'
                  % (idx_iter + 1, lrn_rate, r['dst_loss'], r['model_loss'], r['loss'], r['acc_top1'],
                     r['acc_top5'], speed))
        else:
            print('iter #%d: lr = %e | model_loss = %.4f | loss = %.4f | acc_top1 = %.4f | acc_top5 = %.4f | '
                  'speed = %.2f pics / sec'
                  % (idx_iter + 1, lrn_rate, r['model_loss'], r['loss'], r['acc_top1'], r['acc_top5'], speed))
        return timer()

    def __show_bucket_storage(self, bucket_storage):
        weight_storage = sum(self.statistics['num_weights']) * FLAGS.uql_weight_bits
        print('bucket storage: %d bit / %.3f kb | weight storage: %d bit / %.3f kb | ratio: %.3f'
              % (bucket_storage, bucket_storage / (8. * 1024.), weight_storage, weight_storage / (8. * 1024.),
                 bucket_storage * 1. / weight_storage))
