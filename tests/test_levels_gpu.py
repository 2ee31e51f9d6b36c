"""Integer-level operands of the TMA-fed tensor-core kernels (include/pf_b200.h: pf_tc_act / pf_tc_wt):
* the producer pf_bn_apply_quant_levels against pf_bn_apply_quant (the value every level stands for, the device header,
  the per-pixel channel sums) — bit-level agreement of the represented values;
* the level preparation of the weights against the oracle's quantizer (oracle/pf_oracle.py, itself pinned to
  learners/uniform_quantization/utils.py:163-245);
* forward / weight-gradient kernels on level operands against float64 (1e-5 for level x level: exact integer products,
  fp32 accumulation; 2e-5 where one operand is split-bf16)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import pf_oracle as O
from pocketflow_b200 import ops

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')


def bn_setup(m, c, seed, act):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(m, c, generator=g) * 1.7 + 0.3).to(DEV)
    mean, rstd = torch.randn(c, generator=g).to(DEV) * 0.2, (torch.rand(c, generator=g) + 0.5).to(DEV)
    gamma, beta = (torch.rand(c, generator=g) + 0.5).to(DEV), (torch.randn(c, generator=g) * 0.3).to(DEV)
    if act == 0:
        beta = beta + 4.0          # tensor minimum > 0 is impossible without an activation; keep it generic instead
    return x, mean, rstd, gamma, beta


@pytest.mark.parametrize('m,c', [(37, 16), (64, 64), (1000, 64), (129, 128), (77, 256), (50, 1024), (33, 2048), (6272, 64)])
@pytest.mark.parametrize('bits,act', [(8, 1), (4, 1), (8, 2), (32, 1), (8, 0)])
def test_bn_apply_quant_levels_matches_planes_kernel(m, c, bits, act):
    x, mean, rstd, gamma, beta = bn_setup(m, c, m + c + bits + act, act)
    # range of act(bn(x)) the reference way: a min/max pass over the activation
    y = torch.empty_like(x)
    slot = torch.zeros(2, dtype=torch.int32, device=DEV)
    ops.act_range_reset(slot)
    ops.bn_apply(x, m, c, mean, rstd, gamma, beta, act, y, slot)
    # reference: the existing fused kernel (fp32 + split planes), bit-exact against the oracle elsewhere
    yq = torch.empty_like(x)
    ref_pl = ops.Planes(x.numel(), DEV)
    ops.bn_apply_quant(x, m, c, mean, rstd, gamma, beta, act, slot, bits, yq, ref_pl)
    # levels producer
    yq2 = torch.empty_like(x)
    pl = ops.Planes(x.numel(), DEV)
    pl.hi.fill_(float('nan'))
    pl.lo.fill_(float('nan'))
    hdr = torch.zeros(2, dtype=torch.int32, device=DEV)
    nseg = (c + 127) // 128
    csum = torch.full((m * nseg,), float('nan'), device=DEV)
    ops.bn_apply_quant_levels(x, m, c, mean, rstd, gamma, beta, act, slot, bits, yq2, pl, hdr, csum)
    torch.cuda.synchronize()
    assert torch.equal(yq, yq2), 'the fp32 copy must be the same fake-quantized tensor'
    h = hdr.cpu().numpy().view(ops.ACT_HDR)[0]
    mn = float(ops.decode_ordered(slot.cpu().numpy().view(np.uint32))[0])
    want_levels = bits <= 8 and mn == 0.0
    assert int(h['nplanes']) == (1 if want_levels else 2)
    seg = min(c, 128)
    if want_levels:
        lv = pl.hi.float().view(m, c)
        assert float(lv.min()) >= 0 and float(lv.max()) <= 2 ** bits - 1 and torch.equal(lv, lv.round())
        val = lv * float(h['scale'])
        # one level = alpha / k; the reference value is fl(alpha * fl(level / k)): equal to ~1 ulp
        assert (val - yq.view(m, c)).abs().max().item() <= 3e-7 * yq.abs().max().item()
        stored = lv
    else:
        assert float(h['scale']) == 1.0
        assert torch.equal(pl.hi, ref_pl.hi) and torch.equal(pl.lo, ref_pl.lo)
        stored = (pl.hi.float() + pl.lo.float()).view(m, c)
    want = stored.double().view(m, nseg, seg).sum(2)
    got = csum.view(m, nseg).double()
    tol = 0.0 if want_levels else 1e-5 * float(want.abs().max())     # fp32 butterfly sum of <= 128 values
    assert (got - want).abs().max().item() <= tol


@pytest.mark.parametrize('shape', [(3, 3, 64, 64), (1, 1, 256, 64), (1, 1, 64, 192), (3, 3, 128, 128)])
@pytest.mark.parametrize('bits,per_channel', [(8, True), (8, False), (4, True), (2, False)])
def test_weight_level_preparation_matches_oracle_quantizer(shape, bits, per_channel):
    r, s, c, k = shape
    g = torch.Generator().manual_seed(r + c + k + bits)
    ws = [torch.randn(r, s, c, k, generator=g) * 0.1, torch.randn(1, 1, 64, 64, generator=g)]
    src = [w.to(DEV).contiguous() for w in ws]
    dst = [torch.empty_like(t) for t in src]
    q = ops.UniformWeightQuantizer(src, dst, bits, use_buckets=per_channel, bucket_type='channel')
    q.forward()
    items, levels = [], {}
    for i, w in enumerate(src):
        rr, ss, cc, kk = w.shape
        d = ops.conv_desc(2, 8, 8, cc, kk, rr, ss, 8, 8, 1, 1, rr // 2, ss // 2)
        tw = ops.TcWeights(d, DEV)
        tw.f_lo.fill_(7.0)                                   # must stay untouched in level mode
        items.append((tw, dst[i]))
        b0, ncols, n = int(q.segs[i]['bucket0']), int(q.segs[i]['ncols']), q.n_buckets
        levels[i] = (w, q.scales[b0:b0 + ncols], q.scales[n + b0:n + b0 + ncols], q.scales[2 * n + b0:2 * n + b0 + ncols],
                     ncols, bits)
    batch = ops.TcWeightsBatch(items, DEV, levels)
    batch.prepare(levels=True)
    torch.cuda.synchronize()
    kq = float(2 ** bits - 1)
    for i, w in enumerate(ws):
        rr, ss, cc, kk = w.shape
        tw = items[i][0]
        qref = O.uniform_quantize(w.numpy(), bits, use_buckets=per_channel, bucket_type='channel')
        assert np.array_equal(dst[i].cpu().numpy(), qref)
        w2 = w.numpy().reshape(-1, kk)
        mn, mx = (w2.min(0), w2.max(0)) if per_channel else (w2.min(), w2.max())
        alpha = (mx - mn).astype(np.float32) + np.float32(1e-10)
        lev = np.rint(((w2 - mn).astype(np.float32) / alpha).astype(np.float32) * np.float32(kq))     # [k_rows, cout]
        got = tw.f_hi.float().cpu().numpy().reshape(kk, -1)[:, :w2.shape[0]].T + float(2 ** (bits - 1))
        assert np.array_equal(got, lev), 'levels differ from the quantizer\'s'
        assert float(tw.f_lo.min()) == 7.0 and float(tw.f_lo.max()) == 7.0
        # dgrad copies: split planes of the QUANTIZED values
        dq = (tw.d_hi.float() + tw.d_lo.float()).cpu().numpy().reshape(cc, -1)        # [cin][(r,s,cout)]
        want = qref.reshape(rr * ss, cc, kk).transpose(1, 0, 2).reshape(cc, -1)
        assert np.abs(dq[:, :want.shape[1]] - want).max() <= 2.0 ** -16 * np.abs(want).max()
    # plain preparation of the same batch object: split planes of the tensors handed in (the quantized weights)
    batch.prepare(levels=False)
    torch.cuda.synchronize()
    for i in range(len(ws)):
        tw = items[i][0]
        single = ops.TcWeights(tw.d, DEV)
        single.prepare(dst[i])
        assert torch.equal(tw.f_hi, single.f_hi) and torch.equal(tw.f_lo, single.f_lo)


CASES = [(2, 9, 7, 64, 64, 3, 3, 1, 1, 1), (2, 12, 12, 128, 128, 3, 3, 2, 0, 1), (2, 14, 14, 256, 512, 1, 1, 2, 0, 0),
         (2, 7, 7, 512, 2048, 1, 1, 1, 0, 0), (2, 56, 56, 64, 64, 3, 3, 1, 1, 1), (2, 14, 14, 64, 192, 3, 3, 1, 1, 1),
         # 3x3 over 2 and 4 channel segments of the window sum J (nseg = C / 128), stride 1 and 2
         (2, 14, 14, 256, 256, 3, 3, 1, 1, 1), (2, 13, 13, 512, 512, 3, 3, 2, 1, 1), (2, 14, 14, 512, 128, 3, 3, 2, 0, 1),
         # 123 x 5 = 615 tiles: every CTA of a 132-SM H100 walks 4-5 tiles, and as 5 does not divide 132 its n0 (and
         # the per-CTA column table of the epilogue) changes from one tile to the next
         (20, 28, 28, 128, 640, 1, 1, 1, 0, 0)]


def _ref_conv(x, wt, case):
    n, h, w, c, k, r, s, st, p0, p1 = case
    return F.conv2d(F.pad(x.double().permute(0, 3, 1, 2), (p0, p1, p0, p1)), wt.double().permute(3, 2, 0, 1),
                    stride=st).permute(0, 2, 3, 1)


def weight_scales(nb, wrange, g):
    """per-bucket alpha, beta of the weight quantizer.  'sym': a range around zero; 'pos': all weights >= 0; 'offset': a
    range far from zero, where the rank-1 term o_c * J is most of the result and the level product a small correction"""
    alpha = torch.rand(nb, generator=g) * 0.5 + 0.05
    if wrange == 'sym':
        beta = -alpha * (0.3 + 0.4 * torch.rand(nb, generator=g))
    elif wrange == 'pos':
        beta = alpha * 0.2 * torch.rand(nb, generator=g)
    else:
        beta = alpha * (20.0 + 10.0 * torch.rand(nb, generator=g))
    return alpha, beta


@pytest.mark.parametrize('case', CASES)
@pytest.mark.parametrize('bits,per_channel', [(8, True), (4, False)])
def test_level_operand_kernels_match_float64(case, bits, per_channel):
    check_level_operand_kernels(case, bits, per_channel, 'sym')


@pytest.mark.parametrize('case', CASES)
@pytest.mark.parametrize('bits,per_channel,wrange', [(8, True, 'pos'), (8, False, 'offset')])
def test_level_operand_kernels_with_offset_weight_ranges(case, bits, per_channel, wrange):
    """all-positive weights, and a range far from zero where the rank-1 term o_c * J dominates the result"""
    check_level_operand_kernels(case, bits, per_channel, wrange)


def check_level_operand_kernels(case, bits, per_channel, wrange):
    n, h, w, c, k, r, s, st, p0, p1 = case
    p, q = (h + p0 + p1 - r) // st + 1, (w + p0 + p1 - s) // st + 1
    d = ops.conv_desc(n, h, w, c, k, r, s, p, q, st, st, p0, p0)
    assert ops.conv2d_tc_tma_supported(d, 0) and ops.conv2d_tc_tma_supported(d, 2)
    g = torch.Generator().manual_seed(sum(case) + bits)
    kq, centre = (1 << bits) - 1, float(1 << (bits - 1))
    j = torch.randint(0, 256, (n, h, w, c), generator=g).float() * (torch.rand(n, h, w, c, generator=g) > 0.4)
    s_a = 0.0173
    lv = torch.randint(0, kq + 1, (r, s, c, k), generator=g).float()
    nb = k if per_channel else 1
    alpha, beta = weight_scales(nb, wrange, g)
    rk = float(np.float32(1.0) / np.float32(kq))
    qw = (alpha.double() * rk) * lv.double() + beta.double()
    qa = j.double() * s_a
    bias, res = torch.randn(k, generator=g), torch.randn(n, p, q, k, generator=g)
    ref = torch.relu(_ref_conv(qa, qw, case) + bias.double()) + res.double()
    hdr = torch.from_numpy(np.array([(s_a, 1)], dtype=ops.ACT_HDR).view(np.uint8)).to(DEV)
    nseg = (c + 127) // 128
    csum = j.reshape(-1, nseg, c // nseg).sum(2).contiguous().to(DEV)
    apl = ops.Planes(j.numel(), DEV)
    apl.hi.copy_(j.reshape(-1).to(torch.bfloat16))
    apl.lo.fill_(float('nan'))
    act = ops.tc_act(apl, hdr, csum, nseg)
    wl = (lv - centre).permute(3, 0, 1, 2).reshape(k, r * s * c).to(torch.bfloat16).contiguous().to(DEV)
    pad = (-nb) % 4
    A = torch.cat([alpha, torch.zeros(pad)]).to(DEV)
    B = torch.cat([beta, torch.zeros(pad)]).to(DEV)
    Y = torch.full((n, p, q, k), float('nan'), device=DEV)
    ops.conv2d_tc_fwd_ex(d, act, ops.tc_wt(wl, None, A, B, per_channel, bits), bias.to(DEV), True, Y, res.to(DEV))
    torch.cuda.synchronize()
    assert (Y.double().cpu() - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()
    # levels x split-bf16 weights (2 MMAs) and the weight gradient levels (x) split dy (2 MMAs)
    wt = torch.randn(r, s, c, k, generator=g) * (2.0 / (r * s * c)) ** 0.5
    tw = ops.TcWeights(d, DEV)
    tw.prepare(wt.to(DEV).contiguous())
    wv = (tw.f_hi.double() + tw.f_lo.double()).cpu().view(k, -1)[:, :r * s * c].reshape(k, r, s, c).permute(1, 2, 3, 0)
    ref2 = torch.relu(_ref_conv(qa, wv, case) + bias.double()) + res.double()
    Y.fill_(float('nan'))
    ops.conv2d_tc_fwd_ex(d, act, ops.tc_wt(tw.f_hi, tw.f_lo), bias.to(DEV), True, Y, res.to(DEV))
    torch.cuda.synchronize()
    assert (Y.double().cpu() - ref2).abs().max().item() <= 2e-5 * ref2.abs().max().item()
    dy = torch.randn(n, p, q, k, generator=g)
    wd = torch.zeros(k, c, r, s, dtype=torch.float64, requires_grad=True)
    F.conv2d(F.pad(qa.permute(0, 3, 1, 2), (p0, p1, p0, p1)), wd, stride=st).backward(dy.double().permute(0, 3, 1, 2))
    refw = wd.grad.permute(2, 3, 1, 0)
    dyp = ops.Planes(dy.numel(), DEV)
    ops.split_bf16(dy.to(DEV), dyp)
    ws = torch.empty(max(ops.conv2d_tc_wgrad_planes_workspace_floats(d), 4), device=DEV)
    DW = torch.full((r, s, c, k), 5.0, device=DEV)
    ops.conv2d_tc_wgrad_ex(d, act, ops.tc_act(dyp), ws, DW)
    torch.cuda.synchronize()
    assert (DW.double().cpu() - refw).abs().max().item() <= 2e-5 * refw.abs().max().item()


W8A32_CASES = [(2, 9, 7, 64, 64, 3, 3, 1, 1, 1), (2, 14, 14, 256, 256, 3, 3, 1, 1, 1), (2, 13, 13, 512, 512, 3, 3, 2, 1, 1),
               (20, 28, 28, 128, 640, 1, 1, 1, 0, 0)]


@pytest.mark.parametrize('case', W8A32_CASES)
@pytest.mark.parametrize('wrange', ['sym', 'offset'])
def test_w8a32_operands_match_float64(case, wrange):
    """W8A32: the activation is not quantized, so pf_bn_apply_quant_levels writes split planes, a header that says
    2 planes (scale 1) and the fp32 channel sums; the weights are levels.  The kernel learns na = 2 from the device
    header; the rank-1 correction uses the producer's own channel sums."""
    n, h, w, c, k, r, s, st, p0, p1 = case
    p, q = (h + p0 + p1 - r) // st + 1, (w + p0 + p1 - s) // st + 1
    d = ops.conv_desc(n, h, w, c, k, r, s, p, q, st, st, p0, p0)
    m = n * h * w
    x, mean, rstd, gamma, beta_bn = bn_setup(m, c, sum(case), 1)
    y = torch.empty_like(x)
    slot = torch.zeros(2, dtype=torch.int32, device=DEV)
    ops.act_range_reset(slot)
    ops.bn_apply(x, m, c, mean, rstd, gamma, beta_bn, 1, y, slot)
    apl = ops.Planes(x.numel(), DEV)
    hdr = torch.zeros(2, dtype=torch.int32, device=DEV)
    nseg = (c + 127) // 128
    csum = torch.full((m * nseg,), float('nan'), device=DEV)
    ops.bn_apply_quant_levels(x, m, c, mean, rstd, gamma, beta_bn, 1, slot, 32, None, apl, hdr, csum)
    torch.cuda.synchronize()
    assert int(hdr.cpu().numpy().view(ops.ACT_HDR)[0]['nplanes']) == 2
    xa = (apl.hi.double() + apl.lo.double()).cpu().view(n, h, w, c)
    act = ops.tc_act(apl, hdr, csum, nseg)
    g = torch.Generator().manual_seed(sum(case) + 5)
    lv = torch.randint(0, 256, (r, s, c, k), generator=g).float()
    alpha, beta = weight_scales(k, wrange, g)
    qw = (alpha.double() * float(np.float32(1.0) / np.float32(255.0))) * lv.double() + beta.double()
    wl = (lv - 128.0).permute(3, 0, 1, 2).reshape(k, r * s * c).to(torch.bfloat16).contiguous().to(DEV)
    bias, res = torch.randn(k, generator=g), torch.randn(n, p, q, k, generator=g)
    ref = torch.relu(_ref_conv(xa, qw, case) + bias.double()) + res.double()
    A, B = alpha.to(DEV), beta.to(DEV)             # tc_wt holds raw pointers: keep the tensors alive
    Y = torch.full((n, p, q, k), float('nan'), device=DEV)
    ops.conv2d_tc_fwd_ex(d, act, ops.tc_wt(wl, None, A, B, True, 8), bias.to(DEV), True, Y, res.to(DEV))
    torch.cuda.synchronize()
    plan = ops.conv2d_tc_last_plan()
    assert plan['feed'] == 1 and plan['aff'] == 2 and plan['na'] == 2 and plan['nb'] == 1, plan
    assert (Y.double().cpu() - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()
    # weight gradient: x (split, under the 2-plane header) (x) split dy
    dy = torch.randn(n, p, q, k, generator=g)
    wd = torch.zeros(k, c, r, s, dtype=torch.float64, requires_grad=True)
    F.conv2d(F.pad(xa.permute(0, 3, 1, 2), (p0, p1, p0, p1)), wd, stride=st).backward(dy.double().permute(0, 3, 1, 2))
    refw = wd.grad.permute(2, 3, 1, 0)
    dyp = ops.Planes(dy.numel(), DEV)
    ops.split_bf16(dy.to(DEV), dyp)
    ws = torch.empty(max(ops.conv2d_tc_wgrad_planes_workspace_floats(d), 4), device=DEV)
    DW = torch.full((r, s, c, k), float('nan'), device=DEV)
    ops.conv2d_tc_wgrad_ex(d, act, ops.tc_act(dyp), ws, DW)
    torch.cuda.synchronize()
    assert ops.conv2d_tc_last_plan()['aff'] == 1
    assert (DW.double().cpu() - refw).abs().max().item() <= 2e-5 * refw.abs().max().item()


def test_level_operands_are_refused_where_tma_cannot_feed_them():
    d = ops.conv_desc(2, 8, 8, 16, 32, 3, 3, 8, 8, 1, 1, 1, 1)              # Cin = 16: cp.async kernels only
    assert ops.conv2d_tc_supported(d) and not ops.conv2d_tc_tma_supported(d, 0)
    pl = ops.Planes(2 * 8 * 8 * 16, DEV)
    hdr = torch.zeros(2, dtype=torch.int32, device=DEV)
    tw = ops.TcWeights(d, DEV)
    y = torch.empty(2, 8, 8, 32, device=DEV)
    with pytest.raises(ValueError):
        ops.conv2d_tc_fwd_ex(d, ops.tc_act(pl, hdr), ops.tc_wt(tw.f_hi, tw.f_lo), None, False, y)
