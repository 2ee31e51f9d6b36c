"""The chunked epilogue of the ping-pong TMA convolution (conv_tma_kernel).

A split-bf16 tile at BN = 128 without a residual / accumulate operand or a folded batch norm goes through a staging
tile of one 32-column chunk instead of the whole 128 x 128 tile, which gives its pipeline a third 64 KB stage (forward
and unit-stride dgrad).  The outputs keep their bits: at ResNet-50 layers (batch 128) the TMA kernel gives the bits of
the cp.async kernel at the same BN, both on the chunked path and on the whole-tile path that tiles with a residual,
accumulation or a folded batch norm keep."""
import numpy as np
import pytest
import torch

from pocketflow_b200 import ops

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
SPLIT_STAGE_BN128 = 2 * 128 * 128 + 2 * 128 * 128      # two activation planes + two weight planes, bytes


@pytest.fixture(autouse=True)
def _knobs(monkeypatch):
    for name in ('PF_TC_BN', 'PF_TC_RING'):
        monkeypatch.delenv(name, raising=False)
    yield
    ops.conv2d_tc_set_feed(-1)


def planes(t):
    pl = ops.Planes(t.numel(), DEV)
    ops.split_bf16(t, pl)
    return pl


def layer(n, hw, c, k, r):
    d = ops.conv_desc(n, hw, hw, c, k, r, r, hw, hw, 1, 1, r // 2, r // 2)
    g = torch.Generator().manual_seed(n + hw + c + k + r)
    tw = ops.TcWeights(d, DEV)
    tw.prepare((torch.randn(r, r, c, k, generator=g) / np.sqrt(r * r * c)).to(DEV))
    return d, g, tw


def stages(plan):
    assert plan['feed'] == 1 and plan['bn'] == 128 and plan['na'] == 2 and plan['nb'] == 2, plan
    return plan['stages'] // SPLIT_STAGE_BN128


@pytest.mark.parametrize('pass_', ['fwd', 'dgrad'])
def test_split_tiles_without_extra_operand_get_three_stages(pass_):
    n, hw, c, k = 2, 14, 256, 256
    d, g, tw = layer(n, hw, c, k, 3)
    ops.conv2d_tc_set_feed(1)
    if pass_ == 'dgrad':
        dy = planes(torch.randn(n, hw, hw, k, generator=g).to(DEV))
        ops.conv2d_tc_dgrad_planes(d, dy, tw, False, torch.empty(n, hw, hw, c, device=DEV))
        assert stages(ops.conv2d_tc_last_plan()) >= 3
        ops.conv2d_tc_dgrad_planes(d, dy, tw, True, torch.zeros(n, hw, hw, c, device=DEV))
    else:
        x = planes(torch.randn(n, hw, hw, c, generator=g).to(DEV))
        ops.conv2d_tc_fwd_planes(d, x, tw, None, False, torch.empty(n, hw, hw, k, device=DEV))
        assert stages(ops.conv2d_tc_last_plan()) >= 3
        ops.conv2d_tc_fwd_planes(d, x, tw, None, False, torch.empty(n, hw, hw, k, device=DEV),
                                 torch.randn(n, hw, hw, k, device=DEV))
    torch.cuda.synchronize()
    assert stages(ops.conv2d_tc_last_plan()) == 2          # the whole-tile epilogue keeps its plan


# ResNet-50 layers at batch 128 (name, h = w, c, k, r): nk >= 3 on every one, so the chunked path runs where allowed
RESNET = [('s2 3x3 128->128', 28, 128, 128, 3), ('s3 1x1 1024->256', 14, 1024, 256, 1),
          ('s3 1x1 256->1024', 14, 256, 1024, 1), ('s4 3x3 512->512', 7, 512, 512, 3)]


@pytest.mark.parametrize('extra', [False, True], ids=['chunked', 'whole-tile'])
@pytest.mark.parametrize('spec', RESNET, ids=[s[0] for s in RESNET])
def test_resnet50_shapes_tma_is_bitwise_cp_async(spec, extra):
    name, hw, c, k, r = spec
    n = 128
    d, g, tw = layer(n, hw, c, k, r)
    x = planes(torch.randn(n, hw, hw, c, generator=g).to(DEV))
    bias = torch.randn(k, generator=g).to(DEV)
    res = torch.randn(n, hw, hw, k, generator=g).to(DEV) if extra else None
    dy = planes(torch.randn(n, hw, hw, k, generator=g).to(DEV))
    prior = torch.randn(n, hw, hw, c, generator=g).to(DEV)
    fwd, dgrad = [], []
    for feed in (1, 0):
        ops.conv2d_tc_set_feed(feed)
        y = torch.full((n, hw, hw, k), float('nan'), device=DEV)
        ops.conv2d_tc_fwd_planes(d, x, tw, bias, True, y, res)
        plan = ops.conv2d_tc_last_plan()
        assert plan['feed'] == feed and (feed == 0 or stages(plan) == (2 if extra else 3)), plan
        dx = prior.clone() if extra else torch.full((n, hw, hw, c), float('nan'), device=DEV)
        ops.conv2d_tc_dgrad_planes(d, dy, tw, extra, dx)
        assert ops.conv2d_tc_last_plan()['feed'] == feed
        torch.cuda.synchronize()
        fwd.append(y)
        dgrad.append(dx)
    assert torch.isfinite(fwd[0]).all() and torch.isfinite(dgrad[0]).all()
    assert torch.equal(fwd[0], fwd[1]), '%s: fwd differs from the cp.async kernel' % name
    assert torch.equal(dgrad[0], dgrad[1]), '%s: dgrad differs from the cp.async kernel' % name
