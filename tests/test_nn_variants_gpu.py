"""Kernel-variant sweep of the depthwise convolution, batch-norm and max-pool kernels against float64.

Which kernel runs is decided on the host from the shape and two knobs read on every launch: PF_DW_ROWS (0: no
row-blocked depthwise kernels) and PF_BN_GRIDCAP (grid cap of the BN apply / backward kernels in multiples of the SM
count).  Each case forces one variant and checks it:
  * depthwise: pf_dwconv_last_variant names the dispatch target the case expects; fwd / dgrad within 1e-5 and wgrad
    within 1e-5 of max|float64 grouped conv|, outputs starting as NaN and accumulate targets as a known tensor;
  * batch-norm: statistics against float64, rstd within one ulp of fp32(1 / sqrt(fl(var + eps))), apply bit-exact
    against the fp32 op chain ((x - mean) * rstd) * gamma + beta, the range slot bit-exact, and backward against a
    float64 reference whose activation mask comes from that same fp32 chain (no mask can flip);
  * max-pool: y bit-exact, argmax equal to the FIRST maximum in row-major window order on inputs full of ties, dx
    against a float64 gather of dy over that argmax.
The last test fails if a depthwise dispatch target was never reached."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import pf_oracle as O
from pocketflow_b200 import ops
from support import bn_chain, fq_chain, pool_dx_ref, pool_ref, rel_err, sms, split_planes

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
NT = 256

SEEN = {}                         # depthwise variant -> first case id that ran it
RAN = set()
WORST = {}                        # (family, form) -> worst error relative to its bar's scale


def note(family, form, err):
    WORST[(family, form)] = max(WORST.get((family, form), 0.0), err)


# ------------------------------------------------------------------------------------------ depthwise
def dw_expected(case, rows):
    """(fwd, dgrad, wgrad) dispatch targets of pf_dwconv.cu for a case"""
    n, h, w, c, k, st, p0, p1 = case
    p = (h + p0 + p1 - k) // st + 1
    is3 = k == 3 and (c // 4) > 0 and NT % (c // 4) == 0
    if not is3:
        return 'fwd generic', 'dgrad generic', 'wgrad generic'
    if st == 1:
        if rows and p >= 4 and h >= 4:
            return 'fwd rows', 'dgrad rows', 'wgrad rows'
        return 'fwd 3x3 s1', 'dgrad 3x3 s1', 'wgrad 3x3 s1'
    dg = ('dgrad block p%d' % p0) if (rows and p0 <= 1) else 'dgrad 3x3 s2'
    return 'fwd 3x3 s2', dg, 'wgrad 3x3 s2'


def dw_items(case, variant):
    """work items of a grid-stride depthwise launch (one thread each)"""
    n, h, w, c, k, st, p0, p1 = case
    p = (h + p0 + p1 - k) // st + 1
    q = (w + p0 + p1 - k) // st + 1
    c4 = c // 4
    if variant == 'fwd rows':
        return n * -(-p // 4) * q * c4
    if variant == 'dgrad rows':
        return n * -(-h // 4) * w * c4
    if variant.startswith('dgrad block'):
        return n * -(-h // 2) * -(-w // 2) * c4
    return n * (p * q if variant.startswith('fwd') else h * w) * c4


# (id, (n, h, w, c, k, stride, pad_t/l, pad_b/r), PF_DW_ROWS)
DW_CASES = [
    # row-blocked stride 1: ragged last row block, P % 4 = 1, 2, 3 and 0; SAME (1, 1) and VALID
    ('rows_p13', (2, 13, 13, 32, 3, 1, 1, 1), 1),
    ('rows_p14', (2, 14, 14, 64, 3, 1, 1, 1), 1),
    ('rows_p7', (3, 7, 7, 128, 3, 1, 1, 1), 1),
    ('rows_valid_p9', (2, 11, 10, 32, 3, 1, 0, 0), 1),
    ('rows_p12_c1024', (1, 12, 12, 1024, 3, 1, 1, 1), 1),
    ('s1_p3', (4, 3, 3, 64, 3, 1, 1, 1), 1),                        # P < 4: the one-output kernel even with rows on
    # the same shapes with PF_DW_ROWS=0
    ('s1_norows_p13', (2, 13, 13, 32, 3, 1, 1, 1), 0),
    ('s1_norows_p7', (3, 7, 7, 128, 3, 1, 1, 1), 0),
    # stride 2: SAME (0, 1) on even sizes, (1, 1) on odd and even, VALID
    ('s2_even_same01', (2, 14, 14, 64, 3, 2, 0, 1), 1),
    ('s2_odd_same11', (2, 13, 13, 32, 3, 2, 1, 1), 1),
    ('s2_even_pad11', (2, 16, 12, 32, 3, 2, 1, 1), 1),
    ('s2_odd_valid', (3, 15, 15, 16, 3, 2, 0, 0), 1),
    ('s2_norows_even_same01', (2, 14, 14, 64, 3, 2, 0, 1), 0),
    ('s2_norows_odd_same11', (2, 13, 13, 32, 3, 2, 1, 1), 0),
    # generic kernels: a 2x2 window, and C = 12 (256 % (C / 4) != 0); windows above 9 taps are refused
    ('generic_2x2', (2, 11, 9, 16, 2, 1, 0, 1), 1),
    ('generic_2x2_s2', (2, 12, 12, 32, 2, 2, 0, 0), 1),
    ('generic_c12', (3, 10, 10, 12, 3, 1, 1, 1), 1),
    ('generic_c12_s2', (2, 9, 9, 12, 3, 2, 1, 1), 1),
    # several grid-stride iterations per thread (more than SMs x 8 x 256 items), several ragged wgrad splits
    ('big_rows', (16, 57, 57, 128, 3, 1, 1, 1), 1),
    ('big_s1_norows', (8, 57, 57, 128, 3, 1, 1, 1), 0),
    ('big_s2_block_p0', (15, 56, 56, 128, 3, 2, 0, 1), 1),
    ('big_s2_block_p1', (16, 57, 57, 128, 3, 2, 1, 1), 1),
    ('big_s2_norows', (15, 56, 56, 128, 3, 2, 0, 1), 0),
    ('big_generic', (8, 57, 57, 128, 2, 1, 0, 1), 1),
]


def dw_ref(x, w, case):
    """float64 grouped conv, NHWC x [k, k, C, 1] -> NHWC, implicit bottom / right padding p1"""
    n, h, wd, c, k, st, p0, p1 = case
    return F.conv2d(F.pad(x.permute(0, 3, 1, 2), (p0, p1, p0, p1)), w.permute(2, 3, 0, 1), stride=st,
                    groups=c).permute(0, 2, 3, 1)


@pytest.mark.parametrize('cid,case,rows', DW_CASES, ids=[c[0] for c in DW_CASES])
def test_depthwise_variant(cid, case, rows, monkeypatch):
    monkeypatch.setenv('PF_DW_ROWS', str(rows))
    n, h, w, c, k, st, p0, p1 = case
    p = (h + p0 + p1 - k) // st + 1
    q = (w + p0 + p1 - k) // st + 1
    g = torch.Generator().manual_seed(sum(case) + rows)
    x = torch.randn(n, h, w, c, generator=g).to(DEV)
    wt = (torch.randn(k, k, c, 1, generator=g) * 0.3).to(DEV)
    dy = torch.randn(n, p, q, c, generator=g).to(DEV)
    d = ops.conv_desc(n, h, w, c, c, k, k, p, q, st, st, p0, p0)
    exp_f, exp_d, exp_w = dw_expected(case, rows)
    xd = x.double().requires_grad_(True)
    wd = wt.double().requires_grad_(True)
    yd = dw_ref(xd, wd, case)
    yd.backward(dy.double())

    y = torch.full((n, p, q, c), float('nan'), device=DEV)
    ops.dwconv_fwd(d, x, wt, y)
    assert ops.dwconv_last_variant() == exp_f
    dx = torch.full((n, h, w, c), float('nan'), device=DEV)
    ops.dwconv_dgrad(d, dy, wt, False, dx)
    assert ops.dwconv_last_variant() == exp_d
    prior = torch.randn(n, h, w, c, generator=g).to(DEV)
    dx2 = prior.clone()
    ops.dwconv_dgrad(d, dy, wt, True, dx2)
    assert ops.dwconv_last_variant() == exp_d
    nws = ops.dwconv_wgrad_workspace_floats(d)
    ws = torch.full((max(nws, 4),), float('nan'), device=DEV)
    dw = torch.full_like(wt, float('nan'))
    ops.dwconv_wgrad(d, x, dy, ws, dw)
    assert ops.dwconv_last_variant() == exp_w
    torch.cuda.synchronize()

    errs = (rel_err(y, yd.detach()), rel_err(dx, xd.grad), rel_err(dx2, xd.grad + prior.double()),
            rel_err(dw, wd.grad))
    for (form, e) in zip(('fwd', 'dgrad', 'dgrad acc', 'wgrad'), errs):
        note('dwconv', form, e)
    assert max(errs) <= 1e-5, (cid, errs)

    if cid.startswith('big'):
        cap = sms() * 8 * NT
        for v in (exp_f, exp_d):
            assert dw_items(case, v) > cap, (cid, v, dw_items(case, v), cap)
        # several pixel (or row-block item) splits, the last one ragged
        splits = nws // (k * k * c)
        items = n * (-(-p // 4) if exp_w == 'wgrad rows' else p) * q
        per = -(-items // splits)
        assert splits > 1 and items % per != 0, (cid, splits, items, per)
    for v in (exp_f, exp_d, exp_w):
        SEEN.setdefault(v, cid)
    RAN.add(cid)


def test_rows_and_one_output_kernels_agree_bit_for_bit(monkeypatch):
    """The row-blocked stride-1 forward keeps the one-output kernel's accumulation order: the same bits."""
    case = (3, 13, 11, 64, 3, 1, 1, 1)
    n, h, w, c, k, st, p0, p1 = case
    g = torch.Generator().manual_seed(7)
    x = torch.randn(n, h, w, c, generator=g).to(DEV)
    wt = torch.randn(3, 3, c, 1, generator=g).to(DEV)
    d = ops.conv_desc(n, h, w, c, c, 3, 3, h, w, 1, 1, 1, 1)
    ys = []
    for rows in ('1', '0'):
        monkeypatch.setenv('PF_DW_ROWS', rows)
        y = torch.full((n, h, w, c), float('nan'), device=DEV)
        ops.dwconv_fwd(d, x, wt, y)
        ys.append((ops.dwconv_last_variant(), y))
    assert [v for v, _ in ys] == ['fwd rows', 'fwd 3x3 s1']
    assert torch.equal(ys[0][1], ys[1][1])


# ------------------------------------------------------------------------------------------ batch-norm


def bn_splits(m, c):
    col_tiles = -(-c // 256)
    splits = min(-(-8 * sms() // col_tiles), -(-m // 64), ops.BN_MAX_SPLITS)
    splits = max(splits, 1)
    rps = -(-m // splits)
    return -(-m // rps), rps


def chan_stationary(m, c, gridcap):
    """whether bn_apply / bn_bwd run the channel-stationary loop (grid stride a multiple of C) — pf_nn.cu chan_grid"""
    nvec = m * c // 4
    want = max(1, min(-(-nvec // NT), sms() * gridcap))
    c4 = c // 4
    mult = 1
    while (mult * NT) % c4 and mult < 64:
        mult *= 2
    if (mult * NT) % c4 == 0:
        want = -(-want // mult) * mult
    return (want * NT * 4) % c == 0, want


# (id, m, c, mean, std, PF_BN_GRIDCAP or None, constant channel)
BN_CASES = [
    ('single_split', 48, 64, 0.5, 2.0, None, False),
    ('ragged_splits', 100003, 64, 3.0, 2.0, None, False),
    ('c260_partial_tile', 4200, 260, -1.0, 1.5, None, False),
    ('rotating_c12', 5002, 12, 0.3, 1.0, None, False),
    ('rotating_c36', 40000, 36, 0.3, 1.0, None, False),
    ('rotating_c20', 60000, 20, 0.3, 1.0, None, False),
    ('gridcap1_stationary', 20011, 64, 0.2, 1.0, 1, False),
    ('gridcap1_rotating', 20012, 20, 0.2, 1.0, 1, False),
    ('mean50_std0.1', 100003, 64, 50.0, 0.1, None, False),
    ('constant_channel', 9001, 32, 1.0, 1.0, None, True),
]


@pytest.mark.parametrize('act', [0, 1, 2])
@pytest.mark.parametrize('cid,m,c,mu,sd,cap,const', BN_CASES, ids=[b[0] for b in BN_CASES])
def test_batch_norm_variant(cid, m, c, mu, sd, cap, const, act, monkeypatch):
    if cap is not None:
        monkeypatch.setenv('PF_BN_GRIDCAP', str(cap))
    g = torch.Generator().manual_seed(m + c + act)
    x = torch.randn(m, c, generator=g) * sd + mu
    if const:
        x[:, 3] = 2.5
    x = x.to(DEV)
    gamma = (torch.rand(c, generator=g) + 0.5).to(DEV)
    beta = (torch.randn(c, generator=g) * (2.0 if act == 2 else 0.3)).to(DEV)
    dy = torch.randn(m, c, generator=g).to(DEV)
    eps, mom = 1e-5, 0.997
    splits, rps = bn_splits(m, c)
    if cid == 'single_split':
        assert splits == 1
    if cid in ('ragged_splits', 'mean50_std0.1'):
        assert splits > 100 and m % rps != 0
    stationary, grid = chan_stationary(m, c, cap or 8)
    assert stationary == ('rotating' not in cid and c != 260), (cid, stationary)
    if cap == 1:      # grid-stride loops: the 4-way unrolled body and the tail (stationary), several turns (rotating)
        assert m * c // 4 > (4 if stationary else 2) * grid * NT
    if not stationary and c != 12:
        # the rotating loop wraps its channel (c += step; c -= C): more than one turn per thread.  C = 12 turns once: on
        # 132 SMs every grid large enough for a second turn is a multiple of 3, which makes the stride a multiple of C
        assert m * c // 4 > grid * NT, (cid, m * c // 4, grid * NT)

    # statistics
    mean, var, rstd = (torch.full((c,), float('nan'), device=DEV) for _ in range(3))
    mm0, mv0 = torch.randn(c, generator=g).to(DEV), (torch.rand(c, generator=g) + 0.5).to(DEV)
    mm, mv = mm0.clone(), mv0.clone()
    ws = torch.full((5 * c * ops.BN_MAX_SPLITS,), float('nan'), device=DEV)
    slot = torch.zeros(2, dtype=torch.int32, device=DEV)
    ops.minmax_reset(slot.view(1, 2))
    ops.bn_train_stats_range(x, m, c, eps, mom, mean, var, rstd, mm, mv, gamma, beta, act, slot, ws)
    xd = x.double()
    m64, v64 = xd.mean(0), xd.var(0, unbiased=False)
    e_mean = ((mean.double() - m64).abs() / (m64.abs() + v64.sqrt())).max().item()
    e_var = ((var.double() - v64).abs() / v64.clamp_min(1e-30)).max().item() if not const else \
        ((var.double() - v64).abs() / v64.max()).max().item()
    note('bn', 'mean', e_mean)
    note('bn', 'var', e_var)
    assert e_mean <= 1e-6 and e_var <= 1e-5, (cid, e_mean, e_var)
    if const:
        assert var[3].item() == 0.0 and mean[3].item() == 2.5
    r64 = 1.0 / torch.sqrt((var + eps).double())          # fl(var + eps) in fp32, then rsqrt in fp64
    r32 = r64.float()
    ulp = (torch.nextafter(r32, torch.full_like(r32, float('inf'))) - r32).double()
    assert ((rstd.double() - r64).abs() <= ulp).all(), cid
    om = 1.0 - mom
    e_mm = rel_err(mm, mm0.double() * mom + m64 * om)
    e_mv = rel_err(mv, mv0.double() * mom + xd.var(0, unbiased=True) * om)
    note('bn', 'moving', max(e_mm, e_mv))
    assert max(e_mm, e_mv) <= 1e-6, (cid, e_mm, e_mv)
    y_ref = bn_chain(x, mean, rstd, gamma, beta, act)
    rng = ops.decode_ordered(slot.cpu().numpy().view(np.uint32))
    assert rng[0] == y_ref.min().item() and rng[1] == y_ref.max().item(), (cid, rng)
    # the plain-statistics entry point gives the same bits
    mean2, var2, rstd2 = (torch.full((c,), float('nan'), device=DEV) for _ in range(3))
    ops.bn_train_stats(x, m, c, eps, mom, mean2, var2, rstd2, None, None, ws)
    assert torch.equal(mean, mean2) and torch.equal(var, var2) and torch.equal(rstd, rstd2)

    # apply: fp32, planes, range slot
    y = torch.full_like(x, float('nan'))
    pl = ops.Planes(x.numel(), DEV)
    slot2 = torch.zeros(2, dtype=torch.int32, device=DEV)
    ops.minmax_reset(slot2.view(1, 2))
    ops.bn_apply(x, m, c, mean, rstd, gamma, beta, act, y, slot2, pl)
    h, l = split_planes(y_ref)
    assert torch.equal(y, y_ref) and torch.equal(pl.hi, h) and torch.equal(pl.lo, l), cid
    assert torch.equal(slot, slot2)
    # fused fake-quant with the range of y
    q_ref, lv_ref = fq_chain(y_ref, torch.tensor(rng[0], device=DEV), torch.tensor(rng[1], device=DEV), 8)
    q = torch.full_like(x, float('nan'))
    ops.bn_apply_quant(x, m, c, mean, rstd, gamma, beta, act, slot, 8, q)
    assert torch.equal(q, q_ref), cid
    if c >= 16 and c & (c - 1) == 0:
        # levels form; act 0 has a negative range minimum: the general path inside LEVELS_ONLY (hi / lo planes)
        nseg = -(-c // 128)
        hdr = torch.zeros(2, dtype=torch.int32, device=DEV)
        csum = torch.full((m * nseg,), float('nan'), device=DEV)
        pl3 = ops.Planes(x.numel(), DEV)
        ops.bn_apply_quant_levels(x, m, c, mean, rstd, gamma, beta, act, slot, 8, None, pl3, hdr, csum)
        torch.cuda.synchronize()
        hd = hdr.cpu().numpy().view(ops.ACT_HDR)[0]
        if rng[0] == 0.0:
            assert int(hd['nplanes']) == 1
            assert torch.equal(pl3.hi.float(), lv_ref.reshape(-1))
            assert ((lv_ref >= 0) & (lv_ref <= 255)).all()
            scale = float(hd['scale'])
            e_lv = ((lv_ref.double() * scale - q_ref.double()).abs().max()).item()
            assert e_lv <= 3e-7 * max(1.0, q_ref.abs().max().item()), (cid, e_lv)
            # integer levels: the segment sums are exact
            seg_ref = lv_ref.double().view(m, nseg, min(c, 128)).sum(-1).reshape(-1)
            assert torch.equal(csum.double(), seg_ref), cid
        else:
            assert act == 0 and int(hd['nplanes']) == 2 and float(hd['scale']) == 1.0
            assert rng[0] < 0.0        # the fallback really ran
            h, l = split_planes(q_ref)
            assert torch.equal(pl3.hi, h) and torch.equal(pl3.lo, l), cid
            # fp32 sums of the fake-quantized values over each segment
            qs = q_ref.double().view(m, nseg, min(c, 128))
            e_cs = ((csum.double() - qs.sum(-1).reshape(-1)).abs() / qs.abs().sum(-1).reshape(-1).clamp_min(1e-30))
            note('bn', 'csum / sum|terms|', e_cs.max().item())
            assert e_cs.max().item() <= 1e-6, cid

    # backward: mask from the fp32 chain; float64 sums on the fed fp32 statistics
    z = ((x - mean) * rstd) * gamma + beta
    mask = torch.ones_like(z, dtype=torch.bool) if act == 0 else (z > 0)
    if act == 2:
        mask &= z < 6
    xh = (xd - mean.double()) * rstd.double()
    dz = dy.double() * mask
    db_ref, dg_ref = dz.sum(0), (dz * xh).sum(0)
    db_mag, dg_mag = dz.abs().sum(0), (dz * xh).abs().sum(0)
    dx_ref = gamma.double() * rstd.double() * (dz - db_ref / m - xh * dg_ref / m)
    dga, dbe = torch.full((c,), float('nan'), device=DEV), torch.full((c,), float('nan'), device=DEV)
    dx = torch.full_like(x, float('nan'))
    ops.bn_bwd(dy, x, m, c, mean, rstd, gamma, beta, act, dga, dbe, dx, False, ws)
    torch.cuda.synchronize()
    e_db = ((dbe.double() - db_ref).abs() / db_mag.clamp_min(1e-30)).max().item()
    e_dg = ((dga.double() - dg_ref).abs() / dg_mag.clamp_min(1e-30)).max().item()
    e_dx = rel_err(dx, dx_ref)
    note('bn', 'dbeta / sum|terms|', e_db)
    note('bn', 'dgamma / sum|terms|', e_dg)
    note('bn', 'dx', e_dx)
    assert e_db <= 1e-6 and e_dg <= 1e-6 and e_dx <= 1e-5, (cid, e_db, e_dg, e_dx)
    prior = torch.randn(m, c, generator=g).to(DEV)
    dx2 = prior.clone()
    pl4 = ops.Planes(x.numel(), DEV)
    ops.bn_bwd(dy, x, m, c, mean, rstd, gamma, beta, act, dga, dbe, dx2, True, ws, pl4)
    torch.cuda.synchronize()
    e_acc = rel_err(dx2, dx_ref + prior.double())
    note('bn', 'dx accumulate', e_acc)
    assert e_acc <= 1e-5, (cid, e_acc)
    h, l = split_planes(dx2)
    assert torch.equal(pl4.hi, h) and torch.equal(pl4.lo, l)
    dx3 = torch.full_like(x, float('nan'))
    ops.bn_bwd(dy, x, m, c, mean, rstd, gamma, beta, act, dga, dbe, dx3, False, ws)
    assert torch.equal(dx3, dx)                       # deterministic


def test_bn_apply_quant_matches_the_numpy_oracle():
    """One tensor through oracle/pf_oracle.uniform_quantize itself: the fp32 torch chain above is that op order."""
    g = torch.Generator().manual_seed(5)
    m, c = 777, 96
    x = (torch.randn(m, c, generator=g) * 2 - 0.3).to(DEV)
    gamma, beta = (torch.rand(c, generator=g) + 0.5).to(DEV), (torch.randn(c, generator=g) * 0.3).to(DEV)
    mean, var, rstd = (torch.empty(c, device=DEV) for _ in range(3))
    ws = torch.empty(5 * c * ops.BN_MAX_SPLITS, device=DEV)
    slot = torch.zeros(2, dtype=torch.int32, device=DEV)
    ops.minmax_reset(slot.view(1, 2))
    ops.bn_train_stats_range(x, m, c, 1e-5, 0.9, mean, var, rstd, None, None, gamma, beta, 0, slot, ws)
    y = bn_chain(x, mean, rstd, gamma, beta, 0)
    q = torch.empty_like(x)
    ops.bn_apply_quant(x, m, c, mean, rstd, gamma, beta, 0, slot, 8, q)
    assert np.array_equal(q.cpu().numpy(), O.uniform_quantize(y.cpu().numpy(), 8, mode='activation'))


# ------------------------------------------------------------------------------------------ max-pool


# (id, n, h, w, c, k, stride, pad_t, pad_b, input)
POOL_CASES = [
    ('3x3s2_even_pad01_relu', 4, 112, 112, 64, 3, 2, 0, 1, 'relu'),
    ('3x3s2_odd_pad11_relu', 4, 113, 113, 64, 3, 2, 1, 1, 'relu'),
    ('3x3s2_even_pad11_levels', 3, 20, 20, 32, 3, 2, 1, 1, 'levels'),
    ('3x3s2_odd_pad01_levels', 3, 21, 21, 32, 3, 2, 0, 1, 'levels'),
    ('generic_2x2s2_valid_relu', 8, 28, 28, 64, 2, 2, 0, 0, 'relu'),
    ('generic_2x2s2_valid_levels', 8, 24, 24, 32, 2, 2, 0, 0, 'levels'),
    ('generic_3x3s1_same_levels', 2, 15, 15, 16, 3, 1, 1, 1, 'levels'),
]


@pytest.mark.parametrize('cid,n,h,w,c,k,st,pt,pb,kind', POOL_CASES, ids=[p[0] for p in POOL_CASES])
def test_maxpool_variant(cid, n, h, w, c, k, st, pt, pb, kind):
    g = torch.Generator().manual_seed(n + h + c + k)
    x = torch.randn(n, h, w, c, generator=g)
    x = torch.relu(torch.round(x * 2)) / 4 if kind == 'relu' else torch.round(x * 1.5) / 8    # a few levels: ties
    x = x.to(DEV)
    P = (h + pt + pb - k) // st + 1
    Q = P if h == w else (w + pt + pb - k) // st + 1
    y_ref, am_ref, (_, _, hp, wp), ties = pool_ref(x, k, st, pt, pb, P, Q)
    assert ties > 0.05, (cid, ties)          # windows whose maximum appears more than once pin the first-max rule
    d = ops.conv_desc(n, h, w, c, c, k, k, P, Q, st, st, pt, pt)
    y = torch.full((n, P, Q, c), float('nan'), device=DEV)
    am = torch.full((n, P, Q, c), 77, dtype=torch.uint8, device=DEV)
    ops.maxpool_fwd(d, x, y, am)
    torch.cuda.synchronize()
    assert torch.equal(y, y_ref), cid
    assert torch.equal(am.long(), am_ref.long()), cid
    dy = torch.randn(n, P, Q, c, generator=g).to(DEV)
    dx_ref = pool_dx_ref(dy, am_ref.long(), k, st, pt, P, Q, n, h, w, c, hp, wp)
    dx = torch.full((n, h, w, c), float('nan'), device=DEV)
    ops.maxpool_bwd(d, dy, am, dx)
    prior = torch.randn(n, h, w, c, generator=g).to(DEV)
    dx2 = prior.clone()
    ops.maxpool_bwd(d, dy, am, dx2, True)
    torch.cuda.synchronize()
    e, e2 = rel_err(dx, dx_ref), rel_err(dx2, dx_ref + prior.double())
    note('maxpool', 'dx', max(e, e2))
    assert e <= 1e-6 and e2 <= 1e-6, (cid, e, e2)


# ------------------------------------------------------------------------------------------ coverage
def test_every_depthwise_variant_was_reached():
    """Runs last: the depthwise cases above reach all 14 dispatch targets of pf_dwconv.cu."""
    if not {c[0] for c in DW_CASES} <= RAN:
        pytest.skip('only part of the sweep ran')
    print('depthwise targets reached: ' + ', '.join('%s=%s' % kv for kv in sorted(SEEN.items())))
    print('worst errors: ' + ', '.join('%s %s %.2e' % (f, k, e) for (f, k), e in sorted(WORST.items())))
    missing = set(ops.DW_VARIANTS) - set(SEEN)
    assert not missing, 'depthwise targets never reached: %s' % sorted(missing)
