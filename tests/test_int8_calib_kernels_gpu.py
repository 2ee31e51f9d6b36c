"""The static-range quantizers of calibrated models: pf_bn_eval_levels_u8_static (power-of-two C and C % 16 == 0,
ReLU and ReLU6, 2 - 8 bits), pf_bn_apply_eval_quant_static (fp32 and split-bf16 planes) and pf_uq_act_quant_static,
against the clamped static-range quantizer in float32 on the exact BN output (pf_bn_apply_eval's), with a range whose
hi lies well inside the data so that clamping runs; and, with the static range equal to the batch's, byte-identical
to their per-batch counterparts."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import pf_oracle as O  # noqa: E402
from pocketflow_b200 import ops  # noqa: E402

pytestmark = pytest.mark.gpu
F32 = np.float32
DEV = torch.device('cuda', 0)


def static_quantize(x, bits, lo, hi):
    """(levels, values) of the activation quantizer with min / max replaced by [lo, hi] and x clamped to it first"""
    y = np.clip(np.asarray(x, F32), F32(lo), F32(hi)).astype(F32)
    alpha, beta, k = (F32(hi) - F32(lo)).astype(F32) + F32(1e-10), F32(lo), O.uq_k(bits)
    lv = np.rint((((y - beta) / alpha).astype(F32) * k).astype(F32)).astype(F32)
    return lv, O.uq_inv_scale((lv / k).astype(F32), alpha, beta)


def _bn(m, c, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(m, c, generator=g) * 2 + 0.5).to(DEV)
    mean = (torch.randn(c, generator=g) * 0.3).to(DEV)
    var = (torch.rand(c, generator=g) + 0.5).to(DEV)
    gamma = (torch.rand(c, generator=g) + 0.5).to(DEV)
    beta = (torch.randn(c, generator=g) * 0.2).to(DEV)
    return x, (m, c, mean, var, 1e-5, gamma, beta)


def _y(x, bn, act):
    """act(bn(x)) as pf_bn_apply_eval computes it (the op chain every producer shares)"""
    y = torch.empty_like(x)
    ops.bn_apply_eval(x, *bn, act, y)
    return y


def _dec(slots):
    """(lo, hi) rows of range slots"""
    return ops.decode_ordered(slots.cpu().numpy().view(np.uint32)).reshape(-1, 2)


def _split(v):
    """the split-bf16 planes (hi = bf16(v), lo = bf16(v - hi)) of an fp32 tensor, as one bf16 buffer hi | lo"""
    hi = v.reshape(-1).to(torch.bfloat16)
    return torch.cat([hi, (v.reshape(-1) - hi.float()).to(torch.bfloat16)])


CASES = [(m, c) for c in (64, 128, 256, 512) for m in (1000,)] + [(m, c) for c in (48, 96, 144, 960) for m in (777,)]


@pytest.mark.parametrize('m,c', CASES)
@pytest.mark.parametrize('act', [1, 2])
@pytest.mark.parametrize('bits', [2, 5, 8])
def test_static_levels_against_oracle(m, c, act, bits):
    x, bn = _bn(m, c, seed=c * 10 + act + bits)
    y = _y(x, bn, act).cpu().numpy()
    hi = F32(np.quantile(y[y > 0], 0.6))            # 40 % of the positive values lie above hi
    rng = ops.range_slots([(0.0, hi)], DEV)[0]
    levels = torch.full((m * c,), 0xAB, dtype=torch.uint8, device=DEV)
    hdr = torch.zeros(2, dtype=torch.int32, device=DEV)
    nseg = (c + 127) // 128
    csum = torch.full((m * nseg,), float('nan'), device=DEV)
    ops.bn_eval_levels_u8_static(x, *bn, act, bits, rng, levels, hdr, csum)
    torch.cuda.synchronize()
    want, _ = static_quantize(y, bits, 0.0, hi)
    got = levels.cpu().numpy().reshape(m, c)
    assert (y > hi).sum() > 0.2 * y.size and want.max() == 2 ** bits - 1
    assert np.array_equal(got, want.astype(np.uint8))
    ws = np.stack([want[:, s * 128:(s + 1) * 128].sum(1, dtype=np.float64) for s in range(nseg)], 1)
    assert np.array_equal(csum.cpu().numpy().reshape(m, nseg).astype(np.float64), ws)
    h = hdr.cpu().numpy()
    alpha = (hi - F32(0)).astype(F32) + F32(1e-10)
    assert h[0] == np.array([alpha / O.uq_k(bits)], F32).view(np.int32)[0] and h[1] == 1
    assert _dec(rng)[0].tolist() == [0.0, float(hi)]              # read only


@pytest.mark.parametrize('m,c', CASES)
@pytest.mark.parametrize('act', [1, 2])
@pytest.mark.parametrize('bits', [2, 8])
def test_static_levels_equal_per_batch(m, c, act, bits):
    """static range = this batch's range: levels, csum and header byte-identical to pf_bn_eval_levels_u8"""
    x, bn = _bn(m, c, seed=c + act + 7 * bits)
    nseg = (c + 127) // 128
    out = []
    slot = torch.zeros(2, dtype=torch.int32, device=DEV)
    for static in (False, True):
        levels = torch.zeros(m * c, dtype=torch.uint8, device=DEV)
        hdr = torch.zeros(2, dtype=torch.int32, device=DEV)
        csum = torch.zeros(m * nseg, device=DEV)
        if static:
            ops.bn_eval_levels_u8_static(x, *bn, act, bits, slot.clone(), levels, hdr, csum)
        else:
            ops.bn_eval_levels_u8(x, *bn, act, bits, slot, levels, hdr, csum)
        out.append((levels, hdr, csum.view(torch.int32)))
    torch.cuda.synchronize()
    lo, hi = _dec(slot)[0]
    assert lo == 0 and hi > 0
    for a, b in zip(*out):
        assert torch.equal(a, b)


@pytest.mark.parametrize('m,c', [(1000, 64), (777, 96), (500, 20)])
@pytest.mark.parametrize('act', [1, 2])
@pytest.mark.parametrize('bits', [2, 5, 8, 16])
def test_static_bn_quant(m, c, act, bits):
    """pf_bn_apply_eval_quant_static: fp32 and planes against the oracle with clamping, and bit-identical to
    pf_bn_apply_eval (+ range) followed by pf_uq_act_quant(_planes) when the range is the batch's"""
    x, bn = _bn(m, c, seed=3 * c + act + bits)
    y = _y(x, bn, act)
    yn = y.cpu().numpy()
    hi = F32(np.quantile(yn[yn > 0], 0.7))
    rng = ops.range_slots([(0.0, hi)], DEV)[0]
    planes = ops.Planes(m * c, DEV) if (m * c) % 8 == 0 else None
    got = torch.full_like(x, float('nan'))
    ops.bn_apply_eval_quant_static(x, *bn, act, rng, bits, got, planes)
    _, want = static_quantize(yn, bits, 0.0, hi)
    assert np.array_equal(got.cpu().numpy().view(np.uint32), want.view(np.uint32))
    if planes is not None:
        assert torch.equal(planes.buf.view(torch.int16), _split(got).view(torch.int16))
    # the batch's own range: the two-pass fake-quant lowering, byte for byte
    slot = torch.zeros(2, dtype=torch.int32, device=DEV)
    ops.minmax_reset(slot.view(1, 2))
    y2 = torch.empty_like(x)
    ops.bn_apply_eval(x, *bn, act, y2, slot)
    p2 = ops.Planes(m * c, DEV) if planes is not None else None
    ref = torch.empty_like(x)
    ops.act_quant(y2, ref, slot, bits, p2)
    got2 = torch.empty_like(x)
    p3 = ops.Planes(m * c, DEV) if planes is not None else None
    ops.bn_apply_eval_quant_static(x, *bn, act, slot.clone(), bits, got2, p3)
    assert torch.equal(got2.view(torch.int32), ref.view(torch.int32))
    if planes is not None:
        assert torch.equal(p2.buf.view(torch.int16), p3.buf.view(torch.int16))


@pytest.mark.parametrize('n', [4096, 1001, 3])
@pytest.mark.parametrize('bits', [2, 8])
def test_static_act_quant(n, bits):
    """pf_uq_act_quant_static against the oracle with clamping on both sides, and identical to pf_uq_act_minmax +
    pf_uq_act_quant with the batch's range"""
    g = torch.Generator().manual_seed(n + bits)
    x = (torch.randn(n, generator=g) * 3).to(DEV)
    lo, hi = F32(-1.0), F32(1.5)
    y = torch.full_like(x, float('nan'))
    ops.act_quant_static(x, y, ops.range_slots([(lo, hi)], DEV)[0], bits)
    _, want = static_quantize(x.cpu().numpy(), bits, lo, hi)
    assert np.array_equal(y.cpu().numpy().view(np.uint32), want.view(np.uint32))
    slot = torch.zeros(2, dtype=torch.int32, device=DEV)
    ops.minmax_reset(slot.view(1, 2))
    ops.act_minmax(x, slot)
    ref = torch.empty_like(x)
    ops.act_quant(x, ref, slot, bits)
    ops.act_quant_static(x, y, slot.clone(), bits)
    assert torch.equal(y.view(torch.int32), ref.view(torch.int32))
