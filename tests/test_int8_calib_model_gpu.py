"""Calibrated integer models end to end, on ResNet-20 with `int8_narrow`, MobileNet-v1 and -v2 with `int8_depthwise`
(v2 also `int8_narrow`) at batch 128 and ResNet-50 at batch 16, from a --learner uniform checkpoint:
(a) calibrated on exactly the batch then evaluated, the integer model's logits are bit-identical to the per-batch integer
    model's, and the calibrated fake-quant executor's to the per-batch fake-quant executor's;
(b) a calibrated model's logits of each image are the same bits at batch 1, 7 and the full batch;
(c) calibrated integer against calibrated fake-quant logits, within 1.5x the largest distance measured, and top-1
    agreement (layer by layer against float64 with static ranges: tests/test_int8_calib_tap_gpu.py);
(e) export -> load reproduces the calibrated model's logits bit for bit."""
import gc
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from support import INT8_MODELS, QUIET, free, int8_graph, make  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
BATCH = {'resnet20_narrow': 128, 'resnet50': 16, 'mobilenet_v1_depthwise': 128, 'mobilenet_v2_depthwise_narrow': 128}


@pytest.fixture(autouse=True)
def _release():
    yield
    from pocketflow_b200.flags import FLAGS
    FLAGS.reset()
    gc.collect()
    free()


def _state(key):
    """a --learner uniform checkpoint state (8-bit per-channel weights, 8-bit activations) after two training steps"""
    net, flags, _ = INT8_MODELS[key]
    reload = 'cifar10_dataset' if 'cifar' in net else 'ilsvrc12_dataset'
    lrn = make(net, 'uniform', 16, reload=reload, **dict(QUIET, uql_weight_bits=8, uql_activation_bits=8, **flags))
    for _ in range(2):
        lrn.train_step()
    state = lrn.sess_train.store.state_dict()
    del lrn
    free()
    return state


def _images(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)).to(DEV)


@pytest.mark.parametrize('key', sorted(BATCH))
def test_calibrated_model(key, tmp_path):
    from pocketflow_b200 import compact, int8
    B = BATCH[key]
    state = _state(key)
    g, images, logits, cfg = int8_graph(key, B)
    full = compact.map_state(g, compact.reachable_ops(g, logits), state)
    x = _images(images.shape, 1)

    # (a) calibration on the evaluated batch reproduces the per-batch models bit for bit
    im = int8.IntModel.from_checkpoint(g, images, logits, state, cfg, DEV)
    li = im.forward(x).clone()
    r_int = im.calibrate([x])
    assert all(lo == 0 for lo, _ in r_int.values()), key
    imc = int8.IntModel.from_checkpoint(g, images, logits, state, cfg, DEV, act_ranges=r_int)
    assert imc.sel == im.sel and imc.ex.aq_static
    lc = imc.forward(x).clone()
    assert torch.equal(lc.view(torch.int32), li.view(torch.int32)), float((lc - li).abs().max())
    del im
    fq = int8.fake_quant_executor(g, images, logits, full, cfg, DEV)
    fq.buf[images].copy_(x)
    lf = fq.forward(training=False).clone()
    del fq
    r_fq = int8.calibrate(g, images, logits, state, cfg, [x], device=DEV)
    assert sorted(r_fq) == sorted(r_int)
    fqc = int8.fake_quant_executor(g, images, logits, full, cfg, DEV, act_ranges=r_fq)
    fqc.buf[images].copy_(x)
    lfc = fqc.forward(training=False).clone()
    assert torch.equal(lfc.view(torch.int32), lf.view(torch.int32)), float((lfc - lf).abs().max())
    del fqc

    # (c) calibrated integer vs calibrated fake-quant, both with the fake-quant model's ranges
    imf = int8.IntModel.from_checkpoint(g, images, logits, state, cfg, DEV, act_ranges=r_fq)
    lif = imf.forward(x).clone()
    fqf = int8.fake_quant_executor(g, images, logits, full, cfg, DEV, act_ranges=r_fq)
    fqf.buf[images].copy_(x)
    lff = fqf.forward(training=False).clone()
    d = float((lif - lff).abs().max() / lff.abs().max())
    agree = float((lif.argmax(1) == lff.argmax(1)).float().mean())
    print('%s: calibrated int vs calibrated fake-quant: max rel %.3e, top-1 agreement %.4f' % (key, d, agree))
    # measured on an H100 80GB HBM3 at 700 W: 7.1e-4 (MobileNet-v1) .. 4.0e-3 (ResNet-20), all top-1 agreeing; the
    # float64 comparison with static ranges is tests/test_int8_calib_tap_gpu.py
    assert torch.isfinite(lif).all() and d < 6e-3 and agree >= 0.99
    del fqf, imf

    # (e) export -> load
    path = str(tmp_path / 'm')
    imc.export(path)
    assert json.load(open(path + '.int8.json'))['version'] == 3
    im2 = int8.IntModel.load(g, images, logits, path, DEV)
    assert torch.equal(im2.forward(x).view(torch.int32), lc.view(torch.int32))
    del im2

    # (b) batch independence: batch 1 and 7 models with the same ranges against rows of the full batch
    for b, row0 in ((1, 0), (1, B - 1), (7, B // 2 - 3)):
        gb, ib, lb, cb = int8_graph(key, b)
        mb = int8.IntModel.from_checkpoint(gb, ib, lb, state, cb, DEV, act_ranges=r_int)
        got = mb.forward(x[row0:row0 + b]).clone()
        want = lc[row0:row0 + b]
        assert torch.equal(got.view(torch.int32), want.view(torch.int32)), \
            (b, row0, float((got - want).abs().max() / want.abs().max()))
        del mb
    # a second full batch whose other rows differ: the same rows keep their bits
    x2 = _images(images.shape, 2)
    x2[:5] = x[:5]
    l2 = imc.forward(x2).clone()
    assert torch.equal(l2[:5].view(torch.int32), lc[:5].view(torch.int32))
