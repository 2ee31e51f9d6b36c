"""GPU checks of the searches and the device preprocessing:
* the RL bit search (reference: learners/uniform_quantization/bit_optimizer.py:137-327) and the pruning-ratio search
  (learners/weight_sparsification/pr_optimizer.py:411-611) through the REAL learners' compiled step;
* --enbl_device_preprocess end to end (utils/external/imagenet_preprocessing.py:225-260 on the device): the image
  placeholder equals the host pipeline's batch bit for bit.
The tool scripts hold the checks (they are also runnable stand-alone); a failed assert fails the test."""
import importlib.util
import os

import pytest
from support import make

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _tool(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, 'tools', name + '.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_rl_bit_search_through_the_real_learner():
    _tool('rl_smoke').main()


def test_pruning_ratio_search_through_the_real_learner():
    _tool('rl_smoke').ws_main()


def test_device_preprocess_feeds_the_same_batches_as_the_host_pipeline():
    pytest.importorskip('PIL')
    _tool('preproc_e2e_check').main()


def test_nuq_rl_bit_search_through_the_real_learner():
    """--nuql_enbl_rl_agent: the uniform learner's roll-out loop on the nuql_* flags through the REAL non-uniform learner
    (restore, per-layer bit-widths, codebooks re-fitted by the quantile initialisation, fine-tune, evaluate)."""
    import numpy as np
    from pocketflow_b200.flags import FLAGS
    lrn = make('resnet_at_cifar10', 'non-uniform', 16, reload=None, resnet_size=8, nuql_enbl_rl_agent=True,
               nuql_nb_rlouts=4, nuql_tune_global_steps=2, nuql_equivalent_bits=4, nuql_w_bit_min=2, nuql_w_bit_max=6,
               nb_smpls_eval=64, batch_size_eval=16, enbl_dst=False)
    ex = lrn.sess_train
    bits = lrn.optimal_w_bit_list
    assert len(bits) == len(ex.wq_ops) and all(2 <= b <= 6 for b in bits)
    used = sum(b * n for b, n in zip(bits, lrn.statistics['num_weights']))
    assert used <= 4 * sum(lrn.statistics['num_weights'])                          # the budget holds
    assert ex.wq.uq.bits == [int(b) for b in bits]
    state = ex.store.state_dict()
    for op, b in zip(ex.wq_ops, bits):
        c = state[op.vars['clusters'].name]
        assert c.shape == (64,)                                                    # sized for nuql_w_bit_max
        assert np.all(np.diff(c[:1 << b]) >= 0) and np.all(c[1 << b:] == 0)        # quantiles, then unused entries
    lrn.train_step()
    assert np.isfinite(ex.fetch_losses()['loss'])
    FLAGS.reset()
