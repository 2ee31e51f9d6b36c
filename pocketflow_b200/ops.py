"""Host-side operator layer over the C ABI (include/pf_b200.h).

Holds PyTorch CUDA tensors (device memory, streams) and calls libpf_b200.so through ctypes.  Each
class/function names the reference op chain it replaces.  Pure host logic (bucket layouts, work
tables, percentile ranks) lives in functions that need no GPU, so it is unit-tested on CPU.
"""
import ctypes
import os

import numpy as np
import torch

from . import lib as _lib

UQ_SEG = np.dtype([('src', 'u8'), ('dst', 'u8'), ('numel', 'i8'), ('padded', 'i8'),
                   ('ncols', 'i4'), ('bucket0', 'i4'), ('bits', 'i4'), ('reserved', 'i4')])
WORK = np.dtype([('seg', 'i4'), ('kind', 'i4'), ('start', 'i8'), ('count', 'i4'),
                 ('c0', 'i4'), ('ncol_tile', 'i4'), ('reserved', 'i4')])
WS_SEG = np.dtype([('w', 'u8'), ('bkup', 'u8'), ('mask', 'u8'), ('numel', 'i8')])
assert UQ_SEG.itemsize == 48 and WORK.itemsize == 32 and WS_SEG.itemsize == 32

CHUNK = 8192            # elements per CTA work item of the elementwise multi-tensor kernels
WS_WORKSPACE_U32 = 264  # PF_WS_WORKSPACE_U32_PER_SEG
L2_PARTIALS = 1024      # PF_L2_PARTIALS


# ----------------------------------------------------------------------------- host-only helpers
def uq_bucket_layout(shape, use_buckets, bucket_type, bucket_size):
    """(ncols, padded) of a weight tensor: bucket id of flat element i is i % ncols.

    Mirrors __channel_bucket / __split_bucket (learners/uniform_quantization/utils.py:247-289)."""
    numel = int(np.prod(shape))
    if not use_buckets:
        return 1, numel
    if bucket_type == 'channel':
        return int(shape[-1]), numel
    if bucket_type == 'split':
        if bucket_size <= 0:
            raise ValueError('Bucket size must be a postive integer')
        multiple, rest = divmod(numel, bucket_size)
        if rest:
            multiple += 1
        return multiple, multiple * bucket_size
    raise ValueError("Unrecognized bucket type, must be 'weight' or 'channel'.")


def flat_works(numels, chunk=CHUNK):
    """kind-0 work items: chunks [start, start+count) of each tensor (start % 4 == 0)."""
    rows = []
    for s, n in enumerate(numels):
        for start in range(0, int(n), chunk):
            rows.append((s, 0, start, min(chunk, int(n) - start), 0, 0, 0))
    return np.array(rows, dtype=WORK) if rows else np.zeros(0, dtype=WORK)


def minmax_works(segs):
    """Work table of pf_uq_weight_minmax: flat chunks for per-layer ranges, column tiles x row
    ranges of the [padded/ncols, ncols] view for bucketed ranges."""
    rows = []
    for s, seg in enumerate(segs):
        ncols, numel, padded = int(seg['ncols']), int(seg['numel']), int(seg['padded'])
        if ncols == 1:
            for start in range(0, numel, CHUNK):
                rows.append((s, 0, start, min(CHUNK, numel - start), 0, 0, 0))
            continue
        tile = min(ncols, 1024 if ncols % 4 == 0 else 256)
        nrows = padded // ncols
        rows_per = max(64, (2 * CHUNK) // tile)
        for c0 in range(0, ncols, tile):
            tc = min(tile, ncols - c0)
            for r0 in range(0, nrows, rows_per):
                rows.append((s, 1, r0, min(rows_per, nrows - r0), c0, tc, 0))
    return np.array(rows, dtype=WORK) if rows else np.zeros(0, dtype=WORK)


NUQ_BUCKET_SMEM_FLOATS = 8192   # codebook floats of one bucketed-quantize tile (pf_nuq.cu kBucketSmemFloats)
NUQ_BUCKET_MAX_ROWS = 16384     # PF_NUQ_BUCKET_MAX_ROWS: largest bucket the quantile init sorts in shared memory


def nuq_bucket_tile_width(bits):
    """Columns (buckets) per tile of the bucketed codebook kernels: the tile's [2^bits, width] codebooks fit in
    NUQ_BUCKET_SMEM_FLOATS, and one thread per column fits in a 256-thread CTA."""
    return min(256, NUQ_BUCKET_SMEM_FLOATS >> int(bits))


def nuq_bucket_works(segs):
    """Work tables of the bucketed codebook kernels over the [padded/nb, nb] views: (tiles, finals, partial floats).
    tiles: kind-1 items, columns [c0, c0+ncol_tile) x a row range, reserved = float offset of the tile's 2^bits x
    ncol_tile gradient partials; finals: one item per column tile, start/count = its range of `tiles`."""
    rows, finals, poff = [], [], 0
    for s, seg in enumerate(segs):
        nb, padded, bits = int(seg['ncols']), int(seg['padded']), int(seg['bits'])
        k, tw = 1 << bits, nuq_bucket_tile_width(bits)
        nrows = padded // nb
        rows_per = max(2 * CHUNK // tw, 4 * k)
        for c0 in range(0, nb, tw):
            tc = min(tw, nb - c0)
            first = len(rows)
            for r0 in range(0, nrows, rows_per):
                rows.append((s, 1, r0, min(rows_per, nrows - r0), c0, tc, poff))
                poff += k * tc
            finals.append((s, 1, first, len(rows) - first, c0, tc, 0))
    if poff >= 2 ** 31:
        raise ValueError('too many codebook-gradient partials for one launch')
    mk = lambda r: np.array(r, dtype=WORK) if r else np.zeros(0, dtype=WORK)
    return mk(rows), mk(finals), poff


def nuq_bucket_quantile_positions(rows, bits):
    """Ascending sort positions of centroids j < 2^bits of a bucket of `rows` elements: percentile(x_n,
    (j+1)*100/(k+1), axis=0) with the 'nearest' rule (utils.py:349-366), padded to 256 entries."""
    k = 1 << int(bits)
    pos = np.zeros(256, np.int32)
    for j in range(k):
        pos[j] = rows - 1 - percentile_rank_desc(rows, (j + 1) * 100 / (k + 1))
    return pos


def percentile_rank_desc(n, q):
    """Index into the descending sort gathered by tf.contrib.distributions.percentile
    (interpolation='nearest'): clip(int32(rint((n-1)*(1-q/100))), 0, n-1) in float64."""
    idx = int(np.rint((float(n) - 1.0) * (1.0 - float(q) / 100.0)))
    return min(max(idx, 0), n - 1)


def ws_rank_desc(n, prune_ratio):
    """Rank used by WeightSparseLearner.__build_masks: q = float32(ratio)*100 in float32
    (learners/weight_sparsification/learner.py:284)."""
    return percentile_rank_desc(n, np.float32(np.float32(prune_ratio) * np.float32(100.0)))


def decode_ordered(u):
    """numpy inverse of the ordered-uint float encoding used by the min/max slots."""
    u = np.asarray(u).astype(np.uint32)
    bits = np.where(u & 0x80000000, u & 0x7FFFFFFF, ~u).astype(np.uint32)
    return bits.view(np.float32)


def encode_ordered(f):
    """the ordered-uint encoding (pf_enc) of fp32 values, as uint32: the inverse of decode_ordered"""
    u = np.asarray(f, np.float32).view(np.uint32)
    return np.where(u & np.uint32(0x80000000), ~u, u | np.uint32(0x80000000)).astype(np.uint32)


# ----------------------------------------------------------------------------- device plumbing
def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _upload(arr, device):
    return torch.from_numpy(np.ascontiguousarray(arr).view(np.uint8).copy()).to(device)


def _check_f32(*ts):
    for t in ts:
        if t is None:
            continue
        if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
            raise ValueError('expected a contiguous float32 CUDA tensor')
        if t.data_ptr() % 16:
            raise ValueError('tensor storage must be 16-byte aligned')


def launch_count():
    return int(_lib.load().pf_launch_count())


def launch_count_reset():
    _lib.load().pf_launch_count_reset()


# ----------------------------------------------------------------------------- a1/a3 weights
class UniformWeightQuantizer:
    """Multi-tensor weight fake-quantizer: ONE min/max launch + ONE quantize launch for all layers.

    Stands in for UniformQuantization.insert_quant_op_for_weights' per-layer
    __uniform_quantize(mode='weight') (learners/uniform_quantization/utils.py:81-113, 163-199)."""

    def __init__(self, srcs, dsts, bits, use_buckets=False, bucket_type='channel', bucket_size=256):
        self.L = _lib.load()
        if len(srcs) != len(dsts):
            raise ValueError('srcs/dsts length mismatch')
        _check_f32(*srcs)
        _check_f32(*dsts)
        if bucket_size < 0:
            raise ValueError('Bucket size must be a postive integer')
        if bucket_type not in ('split', 'channel'):
            raise ValueError("Unrecognized bucket type, must be 'weight' or 'channel'.")
        self.srcs, self.dsts = list(srcs), list(dsts)
        self.device = srcs[0].device if srcs else torch.device('cuda')
        segs = np.zeros(len(srcs), dtype=UQ_SEG)
        b0 = 0
        for i, (s, d) in enumerate(zip(srcs, dsts)):
            ncols, padded = uq_bucket_layout(tuple(s.shape), use_buckets, bucket_type, bucket_size)
            segs[i] = (s.data_ptr(), d.data_ptr(), s.numel(), padded, ncols, b0, 8, 0)
            b0 += (ncols + 3) // 4 * 4
        self.segs = segs
        self.n_buckets = max(b0, 4)
        self.bucket_counts = [int(s['ncols']) for s in segs]
        self.mn = torch.empty(self.n_buckets, dtype=torch.int32, device=self.device)
        self.mx = torch.empty(self.n_buckets, dtype=torch.int32, device=self.device)
        self.scales = torch.empty(3 * self.n_buckets, dtype=torch.float32, device=self.device)
        self.work_mm = minmax_works(segs)
        self.work_q = flat_works([int(s['numel']) for s in segs])
        self.work_mm_dev = _upload(self.work_mm, self.device)
        self.work_q_dev = _upload(self.work_q, self.device)
        self.grad_segs_dev = None
        self.set_bits(bits)

    def set_bits(self, bits):
        bits = [int(b) for b in (bits if hasattr(bits, '__len__') else [bits] * len(self.srcs))]
        if len(bits) != len(self.srcs):
            raise ValueError('one bit-width per tensor expected')
        if any(b < 1 or b > 32 for b in bits):
            raise ValueError('bit-widths must be in [1, 32]')
        self.bits = bits
        self.segs['bits'] = bits
        self.segs_dev = _upload(self.segs, self.device)
        self.grad_segs_dev = None
        self.__dict__.pop('_grad_subsets', None)

    def reset_ranges(self):
        st = _stream()
        _lib.check(self.L.pf_fill_u32(_p(self.mn), self.n_buckets, 0xFFFFFFFF, st), 'pf_fill_u32')
        _lib.check(self.L.pf_fill_u32(_p(self.mx), self.n_buckets, 0, st), 'pf_fill_u32')

    def minmax(self):
        self.reset_ranges()
        _lib.check(self.L.pf_uq_weight_minmax(_p(self.segs_dev), _p(self.work_mm_dev), len(self.work_mm),
                                              _p(self.mn), _p(self.mx), _stream()), 'pf_uq_weight_minmax')
        _lib.check(self.L.pf_uq_weight_scales(_p(self.mn), _p(self.mx), self.n_buckets, _p(self.scales), _stream()),
                   'pf_uq_weight_scales')

    def quantize(self):
        _lib.check(self.L.pf_uq_weight_quant(_p(self.segs_dev), _p(self.work_q_dev), len(self.work_q),
                                             _p(self.scales), self.n_buckets, _stream()), 'pf_uq_weight_quant')

    def forward(self):
        if not self.srcs:
            return
        self.minmax()
        self.quantize()

    def ste_backward_(self, grads, indices=None):
        """In-place STE chain on the gradients w.r.t. the quantized weights (a3).  indices: only these tensors (the
        gradient buckets of the data-parallel step finish at different times)."""
        _check_f32(*grads)
        if indices is not None:
            key = tuple(indices)
            cache = self.__dict__.setdefault('_grad_subsets', {})
            ent = cache.get(key)
            if ent is None or ent[0] != [grads[i].data_ptr() for i in indices]:
                gs = self.segs[list(indices)].copy()
                gs['src'] = [grads[i].data_ptr() for i in indices]
                gs['dst'] = gs['src']
                work = flat_works([int(s['numel']) for s in gs])
                ent = cache[key] = ([grads[i].data_ptr() for i in indices], _upload(gs, self.device),
                                    _upload(work, self.device), len(work))
            _lib.check(self.L.pf_uq_weight_ste_bwd(_p(ent[1]), _p(ent[2]), ent[3], _p(self.scales), self.n_buckets,
                                                   _stream()), 'pf_uq_weight_ste_bwd')
            return
        if self.grad_segs_dev is None or self._grad_ptrs != [g.data_ptr() for g in grads]:
            gs = self.segs.copy()
            gs['src'] = [g.data_ptr() for g in grads]
            gs['dst'] = gs['src']
            self.grad_segs_dev = _upload(gs, self.device)
            self._grad_ptrs = [g.data_ptr() for g in grads]
        _lib.check(self.L.pf_uq_weight_ste_bwd(_p(self.grad_segs_dev), _p(self.work_q_dev), len(self.work_q),
                                               _p(self.scales), self.n_buckets, _stream()), 'pf_uq_weight_ste_bwd')

    def ranges(self):
        """Per tensor (min, max) arrays decoded from the slots (host copy; tests/diagnostics)."""
        mn = decode_ordered(self.mn.cpu().numpy().view(np.uint32))
        mx = decode_ordered(self.mx.cpu().numpy().view(np.uint32))
        out = []
        for s in self.segs:
            b0, nc = int(s['bucket0']), int(s['ncols'])
            out.append((mn[b0:b0 + nc].copy(), mx[b0:b0 + nc].copy()))
        return out

    def bucket_storage_bits(self):
        """2*32 bits per bucket (utils.py:299-306)."""
        return sum(self.bucket_counts) * 32 * 2


# ----------------------------------------------------------------------------- a2 activations
def act_range_reset(minmax):
    L = _lib.load()
    st = _stream()
    _lib.check(L.pf_fill_u32(_p(minmax), 1, 0xFFFFFFFF, st), 'pf_fill_u32')
    _lib.check(L.pf_fill_u32(ctypes.c_void_p(minmax.data_ptr() + 4), 1, 0, st), 'pf_fill_u32')


def act_minmax(x, minmax):
    """Accumulate the per-tensor range of x into minmax (int32[2], ordered-uint)."""
    _check_f32(x)
    _lib.check(_lib.load().pf_uq_act_minmax(_p(x), x.numel(), _p(minmax), _stream()), 'pf_uq_act_minmax')


def act_quant(x, y, minmax, bits, planes=None):
    """y = Q(x); `planes` = Planes to (also) receive y in the tensor-core operand format (y may then be None)."""
    _check_f32(x, y)
    if not 1 <= int(bits) <= 32:
        raise ValueError('bit-widths must be in [1, 32]')
    if planes is None:
        _lib.check(_lib.load().pf_uq_act_quant(_p(x), _p(y), x.numel(), _p(minmax), int(bits), _stream()),
                   'pf_uq_act_quant')
    else:
        _lib.check(_lib.load().pf_uq_act_quant_planes(_p(x), _p(y), _p(planes.hi), _p(planes.lo), x.numel(), _p(minmax),
                                                      int(bits), _stream()), 'pf_uq_act_quant_planes')


def act_quant_static(x, y, rng, bits):
    """y = Q(clamp(x, lo, hi)) with a static range rng (int32[2], ordered-uint lo / hi: range_slots) in one pass"""
    _check_f32(x, y)
    _lib.check(_lib.load().pf_uq_act_quant_static(_p(x), _p(y), x.numel(), _p(rng), int(bits), _stream()),
               'pf_uq_act_quant_static')


def range_slots(ranges, device):
    """int32 [n, 2]: the fp32 ranges [(lo, hi), ...] in the range slots' ordered-uint encoding (encode_ordered)"""
    enc = encode_ordered(np.asarray(ranges, np.float32).reshape(-1, 2))
    return torch.from_numpy(enc.view(np.int32)).to(device)


def act_fake_quant(x, bits, out=None, minmax=None):
    """Q(x) with per-tensor range — __uniform_quantize(mode='activation') (utils.py:51-79)."""
    if out is None:
        out = torch.empty_like(x)
    if minmax is None:
        minmax = torch.empty(2, dtype=torch.int32, device=x.device)
    act_range_reset(minmax)
    act_minmax(x, minmax)
    act_quant(x, out, minmax, bits)
    return out


# ----------------------------------------------------------------------------- a5 masks
class MaskBuilder:
    """Multi-tensor magnitude-mask build — WeightSparseLearner.__build_masks
    (learners/weight_sparsification/learner.py:260-294)."""

    def __init__(self, ws, bkups, masks):
        self.L = _lib.load()
        _check_f32(*ws)
        _check_f32(*bkups)
        _check_f32(*masks)
        self.ws, self.bkups, self.masks = list(ws), list(bkups), list(masks)
        self.device = ws[0].device
        segs = np.zeros(len(ws), dtype=WS_SEG)
        for i, (w, b, m) in enumerate(zip(ws, bkups, masks)):
            if not (w.numel() == b.numel() == m.numel()):
                raise ValueError('w/bkup/mask size mismatch')
            segs[i] = (w.data_ptr(), b.data_ptr(), m.data_ptr(), w.numel())
        self.segs = segs
        self.segs_dev = _upload(segs, self.device)
        self.work = flat_works([w.numel() for w in ws])
        self.work_dev = _upload(self.work, self.device)
        self.workspace = torch.zeros(len(ws) * WS_WORKSPACE_U32, dtype=torch.int32, device=self.device)
        self.thr = torch.zeros(len(ws), dtype=torch.float32, device=self.device)
        self.ranks = torch.zeros(len(ws), dtype=torch.int64, device=self.device)

    def build(self, prune_ratios):
        """prune_ratios: one (dynamic) float32 ratio per tensor."""
        ranks = [ws_rank_desc(w.numel(), r) for w, r in zip(self.ws, prune_ratios)]
        self.ranks.copy_(torch.tensor(ranks, dtype=torch.int64), non_blocking=False)
        _lib.check(self.L.pf_ws_mask_build(_p(self.segs_dev), len(self.ws), _p(self.work_dev), len(self.work),
                                           _p(self.ranks), _p(self.workspace), _p(self.thr), _stream()),
                   'pf_ws_mask_build')
        return ranks


def select_desc(tensors, queries):
    """Exact order statistics: queries = [(tensor_index, rank_desc)], returns a float32 CUDA tensor.
    Used by the codebook quantile init (learners/nonuniform_quantization/utils.py:349-366)."""
    L = _lib.load()
    _check_f32(*tensors)
    dev = tensors[0].device
    segs = np.zeros(len(tensors), dtype=WS_SEG)
    for i, t in enumerate(tensors):
        segs[i] = (0, t.data_ptr(), 0, t.numel())
    qseg = np.array([q[0] for q in queries], dtype=np.int32)
    ranks = torch.tensor([int(q[1]) for q in queries], dtype=torch.int64, device=dev)
    work = flat_works([tensors[q[0]].numel() for q in queries])
    ws = torch.zeros(len(queries) * WS_WORKSPACE_U32, dtype=torch.int32, device=dev)
    out = torch.empty(len(queries), dtype=torch.float32, device=dev)
    segs_dev, qseg_dev, work_dev = _upload(segs, dev), _upload(qseg, dev), _upload(work, dev)
    _lib.check(L.pf_select_desc(_p(segs_dev), _p(qseg_dev), len(queries), _p(work_dev), len(work),
                                _p(ranks), _p(ws), _p(out), _stream()), 'pf_select_desc')
    torch.cuda.current_stream().synchronize()   # tables above go out of scope
    return out


# ----------------------------------------------------------------------------- a6/a9 optimizers
def momentum_step(w, acc, g, mask, hp, momentum, wd=0.0, grad_scale=1.0):
    """g*mask + MomentumOptimizer.apply_gradients on a flat range
    (learners/weight_sparsification/learner.py:201-212, 314-332).  hp[0] = lr (device)."""
    _check_f32(w, acc, g, mask, hp)
    _lib.check(_lib.load().pf_momentum_step(_p(w), _p(acc), _p(g), _p(mask), w.numel(), _p(hp),
                                            float(momentum), float(wd), float(grad_scale), _stream()),
               'pf_momentum_step')


def adam_step(w, m, v, g, hp, beta1=0.9, beta2=0.999, eps=1e-8, wd=0.0, grad_scale=1.0):
    """tf.train.AdamOptimizer step on a flat range (uniform_quantization/learner.py:244).
    hp = [lr, beta1_power, beta2_power] (device)."""
    _check_f32(w, m, v, g, hp)
    _lib.check(_lib.load().pf_adam_step(_p(w), _p(m), _p(v), _p(g), w.numel(), _p(hp), float(beta1),
                                        float(beta2), float(eps), float(wd), float(grad_scale), _stream()),
               'pf_adam_step')


# ----------------------------------------------------------------------------- a7/a8 losses
def softmax_ce(logits, labels, teacher=None, tempr=4.0, w_dst=4.0, dlogits=None, out=None, row_ws=None):
    """hard CE (+ distillation CE) forward and d/dlogits.  Returns (out[4], dlogits):
    out = [hard, dst, top-1 accuracy, top-5 accuracy]."""
    _check_f32(logits, labels, teacher)
    n, k = logits.shape
    if labels.shape != logits.shape or (teacher is not None and teacher.shape != logits.shape):
        raise ValueError('labels/teacher must match logits shape')
    if dlogits is None:
        dlogits = torch.empty_like(logits)
    if out is None:
        out = torch.empty(4, dtype=torch.float32, device=logits.device)
    if row_ws is None:
        row_ws = torch.empty(4 * n, dtype=torch.float32, device=logits.device)
    _lib.check(_lib.load().pf_softmax_ce_fwd_bwd(_p(logits), _p(labels), _p(teacher), n, k, float(tempr),
                                                 float(w_dst), _p(dlogits), _p(out), _p(row_ws), _stream()),
               'pf_softmax_ce_fwd_bwd')
    return out, dlogits


def l2_loss(v, scale, out, partial_ws, accumulate=False):
    """out[0] (+)= scale * sum(v^2)/2 — tf.nn.l2_loss terms (nets/resnet_at_cifar10.py:105-107)."""
    _check_f32(v, out, partial_ws)
    _lib.check(_lib.load().pf_l2_loss(_p(v), v.numel(), float(scale), int(bool(accumulate)), _p(out),
                                      _p(partial_ws), _stream()), 'pf_l2_loss')


# ----------------------------------------------------------------------------- a11 codebooks
class CodebookWeightQuantizer:
    """Multi-tensor codebook quantizer, per-layer range —
    NonUniformQuantization.__nonuni_quantize (learners/nonuniform_quantization/utils.py:168-194).

    The codebooks are either a private [tensors, 256] table (`clusters`), or — `cluster_views` — 1-D views of ONE flat
    buffer `cluster_base` that the caller owns: the reference's trainable `clusters` variables (utils.py:297), which then
    sit among the model's parameters (optimizer, weight decay, checkpoints, broadcast all apply to them).

    use_buckets: one range and one codebook per bucket — NonUniformQuantization.__bucket_quantize (utils.py:196-243),
    the 'channel' / 'split' layouts of uq_bucket_layout.  The codebooks of a tensor with nb buckets are then a [K, nb]
    matrix (column b = bucket b, K >= 2^bits rows): cluster_views of K * nb floats, or a private [256, nb] table per
    tensor (codebooks())."""

    def __init__(self, srcs, dsts, bits, keep_index=False, cluster_views=None, cluster_base=None,
                 use_buckets=False, bucket_type='split', bucket_size=256):
        self.L = _lib.load()
        _check_f32(*srcs)
        _check_f32(*dsts)
        self.use_buckets = bool(use_buckets)
        if self.use_buckets:
            self._init_buckets(srcs, dsts, bits, keep_index, cluster_views, cluster_base, bucket_type, bucket_size)
            return
        self.uq = UniformWeightQuantizer(srcs, dsts, bits)       # per-layer ranges + tables
        if any(b > 8 for b in self.uq.bits):
            raise ValueError('codebook bit-widths must be <= 8')
        self.srcs, self.dsts = list(srcs), list(dsts)
        self.device = self.uq.device
        self.cluster_views, self.cluster_base, self.cluster_off = None, None, None
        if cluster_views is not None:
            _check_f32(cluster_base, *cluster_views)
            offs = []
            for v, b in zip(cluster_views, self.uq.bits):
                off = (v.data_ptr() - cluster_base.data_ptr()) // 4
                if v.numel() < (1 << b) or off < 0 or off + v.numel() > cluster_base.numel():
                    raise ValueError('codebook views must hold at least 2^bits floats inside cluster_base')
                offs.append(off)
            self.cluster_views, self.cluster_base = list(cluster_views), cluster_base
            self.cluster_off = torch.tensor(offs, dtype=torch.int64, device=self.device)
            self.clusters = None
        else:
            self.clusters = torch.zeros(len(srcs), 256, dtype=torch.float32, device=self.device)
        self.idx = None
        if keep_index:
            offs, tot = [], 0
            for s in srcs:
                offs.append(tot)
                tot += (s.numel() + 15) // 16 * 16
            self.idx = torch.zeros(tot, dtype=torch.uint8, device=self.device)
            self.idx_base = torch.tensor(offs, dtype=torch.int64, device=self.device)
            self.idx_offsets = offs
        self._grad_tables = None

    def _init_buckets(self, srcs, dsts, bits, keep_index, cluster_views, cluster_base, bucket_type, bucket_size):
        if bucket_type == 'split' and int(bucket_size) <= 0:
            raise ValueError('split buckets need a positive bucket size (got %d)' % int(bucket_size))
        self.uq = UniformWeightQuantizer(srcs, dsts, bits, True, bucket_type, bucket_size)   # per-bucket ranges
        if any(b > 8 for b in self.uq.bits):
            raise ValueError('codebook bit-widths must be <= 8')
        self.srcs, self.dsts = list(srcs), list(dsts)
        self.device = self.uq.device
        self.nb = [int(s['ncols']) for s in self.uq.segs]
        self.rows = [int(s['padded']) // int(s['ncols']) for s in self.uq.segs]
        if any(r > NUQ_BUCKET_MAX_ROWS for r in self.rows):
            raise ValueError('a bucket holds %d elements; the bucketed quantile init supports up to %d'
                             % (max(self.rows), NUQ_BUCKET_MAX_ROWS))
        self.cluster_views = None
        if cluster_views is not None:
            _check_f32(cluster_base, *cluster_views)
            offs, krows = [], []
            for v, b, nb in zip(cluster_views, self.uq.bits, self.nb):
                off = (v.data_ptr() - cluster_base.data_ptr()) // 4
                if v.numel() % nb or v.numel() < (1 << b) * nb or off < 0 or off + v.numel() > cluster_base.numel():
                    raise ValueError('bucketed codebook views must hold [K >= 2^bits, nb] floats inside cluster_base')
                offs.append(off)
                krows.append(v.numel() // nb)
            self.cluster_views, self.cluster_base = list(cluster_views), cluster_base
            self.clusters = None
        else:
            offs, krows, tot = [], [], 0
            for nb in self.nb:
                offs.append(tot)
                krows.append(256)
                tot += (256 * nb + 3) // 4 * 4
            self.clusters = torch.zeros(max(tot, 4), dtype=torch.float32, device=self.device)
            self.cluster_base = self.clusters
        self.cluster_krows, self.cluster_offsets = krows, offs
        self.cluster_off = torch.tensor(offs, dtype=torch.int64, device=self.device)
        self.idx = None
        if keep_index:
            ioffs, tot = [], 0
            for s in srcs:
                ioffs.append(tot)
                tot += (s.numel() + 15) // 16 * 16
            self.idx = torch.zeros(tot, dtype=torch.uint8, device=self.device)
            self.idx_base = torch.tensor(ioffs, dtype=torch.int64, device=self.device)
            self.idx_offsets = ioffs
        qi = [(s, 2, 0, r, b, k, 0) for s, (nb, r, k) in enumerate(zip(self.nb, self.rows, krows)) for b in range(nb)]
        self.work_qi = np.array(qi, dtype=WORK) if qi else np.zeros(0, dtype=WORK)
        self.work_qi_dev = _upload(self.work_qi, self.device)
        self._bucket_tables()

    def _bucket_tables(self):
        """Tables that depend on the bit-widths: the tiles (their width is 8192 / 2^bits at most) and the quantile
        positions."""
        self.work_b, self.work_fin, n_partial = nuq_bucket_works(self.uq.segs)
        self.work_b_dev = _upload(self.work_b, self.device)
        self.work_fin_dev = _upload(self.work_fin, self.device)
        self.partial = torch.empty(max(n_partial, 1), dtype=torch.float32, device=self.device)
        pos = np.stack([nuq_bucket_quantile_positions(r, b) for r, b in zip(self.rows, self.uq.bits)]) \
            if self.rows else np.zeros((1, 256), np.int32)
        self.qpos_dev = torch.from_numpy(pos.reshape(-1).astype(np.int32)).to(self.device)
        self._grad_tables = None

    def codebooks(self):
        """[K, nb] views of the codebooks (column b = bucket b's 2^bits centroids in its first rows)."""
        if self.cluster_views is not None:
            return [v.view(-1, nb) for v, nb in zip(self.cluster_views, self.nb)]
        return [self.clusters[o:o + k * nb].view(k, nb)
                for o, k, nb in zip(self.cluster_offsets, self.cluster_krows, self.nb)]

    def bucket_storage_bits(self):
        """alpha and beta of every bucket, 32 bits each (utils.py:487-494)."""
        return self.uq.bucket_storage_bits()

    def quantile_values(self):
        """clusters_j = percentile(x_n, (j+1)*100/(k+1)) (utils.py:349-366), [tensors][k] as numpy.  x -> x_n is
        monotone non-decreasing in fp32, so the order statistic is selected on the raw weights (exact radix select)
        and normalised afterwards with the same fp32 ops.  With buckets: [tensors] of [2^bits, nb] arrays."""
        if self.use_buckets:
            self.quantile_init()
            return [c[:1 << b].cpu().numpy() for c, b in zip(self.codebooks(), self.uq.bits)]
        self.uq.minmax()
        queries = []
        for i, s in enumerate(self.srcs):
            k = 1 << self.uq.bits[i]
            for j in range(k):
                queries.append((i, percentile_rank_desc(s.numel(), (j + 1) * 100 / (k + 1))))
        vals = select_desc(self.srcs, queries).cpu().numpy()
        rng = self.uq.ranges()
        out, pos = [], 0
        for i in range(len(self.srcs)):
            k = 1 << self.uq.bits[i]
            mn, mx = rng[i][0][0], rng[i][1][0]
            alpha = np.float32(np.float32(mx - mn) + np.float32(1e-10))
            out.append(((vals[pos:pos + k] - mn).astype(np.float32) / alpha).astype(np.float32))
            pos += k
        return out

    def set_bits(self, bits):
        """New bit-widths (the RL bit search): a codebook keeps its place and uses its first 2^bits entries; call
        quantile_init() afterwards."""
        bits = [int(b) for b in (bits if hasattr(bits, '__len__') else [bits] * len(self.srcs))]
        if any(b < 1 or b > 8 for b in bits):
            raise ValueError('codebook bit-widths must be in [1, 8]')
        if self.use_buckets:
            if any(k < (1 << b) for k, b in zip(self.cluster_krows, bits)):
                raise ValueError('a codebook variable has fewer than 2^bits rows')
            self.uq.set_bits(bits)
            self._bucket_tables()
            return
        if self.cluster_views is not None and any(v.numel() < (1 << b) for v, b in zip(self.cluster_views, bits)):
            raise ValueError('a codebook variable is smaller than 2^bits')
        self.uq.set_bits(bits)
        self._grad_tables = None

    def quantile_init(self):
        if self.use_buckets:
            # per-bucket ranges, then every bucket's order statistics in one launch
            self.uq.minmax()
            if len(self.work_qi):
                _lib.check(self.L.pf_nuq_bucket_quantile_init(
                    _p(self.uq.segs_dev), _p(self.work_qi_dev), len(self.work_qi), max(self.rows), _p(self.qpos_dev),
                    _p(self.uq.scales), self.uq.n_buckets, _p(self.cluster_base), _p(self.cluster_off), _stream()),
                    'pf_nuq_bucket_quantile_init')
            return
        vals = self.quantile_values()
        if self.cluster_views is not None:
            for v, c in zip(self.cluster_views, vals):
                v.zero_()                                   # entries past 2^bits stay 0 (no weight-decay term)
                v[:c.size].copy_(torch.from_numpy(c))
            return
        c = np.zeros((len(self.srcs), 256), np.float32)
        for i, v in enumerate(vals):
            c[i, :v.size] = v
        self.clusters.copy_(torch.from_numpy(c))

    def forward(self):
        self.uq.minmax()
        idx_base = _p(self.idx_base) if self.idx is not None else None
        if self.use_buckets:
            _lib.check(self.L.pf_nuq_bucket_quant(_p(self.uq.segs_dev), _p(self.work_b_dev), len(self.work_b),
                                                  _p(self.uq.scales), self.uq.n_buckets, _p(self.cluster_base),
                                                  _p(self.cluster_off), _p(self.idx), idx_base, _stream()),
                       'pf_nuq_bucket_quant')
            return
        if self.cluster_views is not None:
            _lib.check(self.L.pf_nuq_weight_quant_ex(_p(self.uq.segs_dev), _p(self.uq.work_q_dev), len(self.uq.work_q),
                                                     _p(self.uq.scales), self.uq.n_buckets, _p(self.cluster_base),
                                                     _p(self.cluster_off), _p(self.idx), idx_base, _stream()),
                       'pf_nuq_weight_quant_ex')
        else:
            _lib.check(self.L.pf_nuq_weight_quant(_p(self.uq.segs_dev), _p(self.uq.work_q_dev), len(self.uq.work_q),
                                                  _p(self.uq.scales), self.uq.n_buckets, _p(self.clusters),
                                                  _p(self.idx), idx_base, _stream()), 'pf_nuq_weight_quant')

    def cluster_grad(self, grads, grad_base):
        """dL/dc_j = alpha * sum_{idx = j} g (learner.py:252-261 through utils.py:303-306, :433): `grads` = the gradients
        w.r.t. the QUANTIZED tensors (one per src), results written to grad_base + the codebooks' offsets (grad_base has
        the layout of cluster_base).  Needs keep_index and store-resident codebooks."""
        if self.idx is None or self.cluster_off is None:
            raise ValueError('cluster_grad needs keep_index=True and cluster_views')
        _check_f32(grad_base, *grads)
        ptrs = [g.data_ptr() for g in grads]
        if self.use_buckets:
            # dL/dc[j, b] = alpha_b * sum over bucket b's real elements with idx = j
            if self._grad_tables is None or self._grad_tables[0] != ptrs:
                gs = self.uq.segs.copy()
                gs['src'] = ptrs
                gs['dst'] = ptrs
                self._grad_tables = (ptrs, _upload(gs, self.device))
            _lib.check(self.L.pf_nuq_bucket_cluster_grad(
                _p(self._grad_tables[1]), _p(self.work_b_dev), len(self.work_b), _p(self.work_fin_dev),
                len(self.work_fin), _p(self.idx), _p(self.idx_base), _p(self.uq.scales), _p(self.partial),
                _p(grad_base), _p(self.cluster_off), _stream()), 'pf_nuq_bucket_cluster_grad')
            return
        if self._grad_tables is None or self._grad_tables[0] != ptrs:
            gs = self.uq.segs.copy()
            gs['src'] = ptrs
            gs['dst'] = ptrs
            first = np.zeros(len(self.srcs) + 1, np.int32)
            for w in self.uq.work_q:
                first[int(w['seg']) + 1] += 1
            first = np.cumsum(first).astype(np.int32)
            self._grad_tables = (ptrs, _upload(gs, self.device), _upload(first, self.device),
                                 torch.empty(max(len(self.uq.work_q), 1) * 256, dtype=torch.float32, device=self.device))
        _, gsegs, first_dev, partial = self._grad_tables
        _lib.check(self.L.pf_nuq_cluster_grad(_p(gsegs), len(self.srcs), _p(self.uq.work_q_dev), len(self.uq.work_q),
                                              _p(first_dev), _p(self.idx), _p(self.idx_base), _p(self.uq.scales),
                                              _p(partial), _p(grad_base), _p(self.cluster_off), _stream()),
                   'pf_nuq_cluster_grad')


# ----------------------------------------------------------------------------- a4 conv / a13 layers
BN_MAX_SPLITS = 1024


def conv_desc(n, h, w, c, k, r, s, p, q, sh, sw, pt, pl):
    return _lib.ConvDesc(n, h, w, c, k, r, s, p, q, sh, sw, pt, pl)


def im2col(d, x, kpad, cols):
    _lib.check(_lib.load().pf_im2col(ctypes.byref(d), _p(x), int(kpad), _p(cols), _stream()), 'pf_im2col')


def conv2d_fwd(d, x, w, bias, relu, y):
    _lib.check(_lib.load().pf_conv2d_fwd(ctypes.byref(d), _p(x), _p(w), _p(bias), int(bool(relu)), _p(y), _stream()),
               'pf_conv2d_fwd')


def conv2d_dgrad(d, dy, w, wt_ws, accumulate, dx):
    _lib.check(_lib.load().pf_conv2d_dgrad(ctypes.byref(d), _p(dy), _p(w), _p(wt_ws), int(bool(accumulate)), _p(dx),
                                           _stream()), 'pf_conv2d_dgrad')


def conv2d_wgrad_workspace_floats(d):
    return int(_lib.load().pf_conv2d_wgrad_workspace_bytes(ctypes.byref(d))) // 4


def conv2d_wgrad(d, x, dy, ws, dw):
    _lib.check(_lib.load().pf_conv2d_wgrad(ctypes.byref(d), _p(x), _p(dy), _p(ws), _p(dw), _stream()),
               'pf_conv2d_wgrad')


def bn_train_stats(x, m, c, eps, momentum, mean, var, rstd, mov_mean, mov_var, ws):
    _lib.check(_lib.load().pf_bn_train_stats(_p(x), m, c, float(eps), float(momentum), _p(mean), _p(var), _p(rstd),
                                             _p(mov_mean), _p(mov_var), _p(ws), _stream()), 'pf_bn_train_stats')


def bn_train_stats_range(x, m, c, eps, momentum, mean, var, rstd, mov_mean, mov_var, gamma, beta, act, minmax, ws):
    """batch statistics + range of act(bn(x)) (for the activation quantizer) in the same pass over x"""
    _lib.check(_lib.load().pf_bn_train_stats_range(_p(x), m, c, float(eps), float(momentum), _p(mean), _p(var), _p(rstd),
                                                   _p(mov_mean), _p(mov_var), _p(gamma), _p(beta), int(act), _p(minmax),
                                                   _p(ws), _stream()), 'pf_bn_train_stats_range')


def bn_apply_eval(x, m, c, mov_mean, mov_var, eps, gamma, beta, act, y, minmax=None, planes=None):
    """inference-mode BN (+act) in one launch, to fp32 and/or operand planes"""
    _lib.check(_lib.load().pf_bn_apply_eval(_p(x), m, c, _p(mov_mean), _p(mov_var), float(eps), _p(gamma), _p(beta), int(act),
                                            _p(y), _p(planes.hi if planes is not None else None),
                                            _p(planes.lo if planes is not None else None), _p(minmax), _stream()),
               'pf_bn_apply_eval')


def bn_apply_eval_quant_static(x, m, c, mov_mean, mov_var, eps, gamma, beta, act, rng, bits, y=None, planes=None):
    """Q(clamp(act(bn(x)), lo, hi)) with the moving statistics and a static range rng (range_slots) in one launch, to
    fp32 and/or operand planes"""
    _lib.check(_lib.load().pf_bn_apply_eval_quant_static(
        _p(x), m, c, _p(mov_mean), _p(mov_var), float(eps), _p(gamma), _p(beta), int(act), _p(rng), int(bits), _p(y),
        _p(planes.hi if planes is not None else None), _p(planes.lo if planes is not None else None), _stream()),
        'pf_bn_apply_eval_quant_static')


def bn_apply_quant(x, m, c, mean, rstd, gamma, beta, act, rng, bits, y=None, planes=None):
    """Q(act(bn(x))) with a known range, to fp32 and/or operand planes"""
    _lib.check(_lib.load().pf_bn_apply_quant(_p(x), m, c, _p(mean), _p(rstd), _p(gamma), _p(beta), int(act), _p(rng),
                                             int(bits), _p(y), _p(planes.hi if planes is not None else None),
                                             _p(planes.lo if planes is not None else None), _stream()), 'pf_bn_apply_quant')


def bn_apply_quant_levels(x, m, c, mean, rstd, gamma, beta, act, rng, bits, y, planes, hdr, csum):
    """Q(act(bn(x))) as a pf_tc_act: integer levels (or hi / lo planes) + device header + channel sums"""
    _lib.check(_lib.load().pf_bn_apply_quant_levels(_p(x), m, c, _p(mean), _p(rstd), _p(gamma), _p(beta), int(act), _p(rng),
                                                    int(bits), _p(y), _p(planes.hi), _p(planes.lo), _p(hdr), _p(csum), _stream()),
               'pf_bn_apply_quant_levels')


def bn_eval_prepare(mov_var, c, eps, rstd):
    _lib.check(_lib.load().pf_bn_eval_prepare(_p(mov_var), c, float(eps), _p(rstd), _stream()), 'pf_bn_eval_prepare')


def bn_apply(x, m, c, mean, rstd, gamma, beta, act, y, minmax=None, planes=None):
    if planes is None:
        _lib.check(_lib.load().pf_bn_apply(_p(x), m, c, _p(mean), _p(rstd), _p(gamma), _p(beta), int(act), _p(y),
                                           _p(minmax), _stream()), 'pf_bn_apply')
    else:
        _lib.check(_lib.load().pf_bn_apply_planes(_p(x), m, c, _p(mean), _p(rstd), _p(gamma), _p(beta), int(act), _p(y),
                                                  _p(planes.hi), _p(planes.lo), _p(minmax), _stream()),
                   'pf_bn_apply_planes')


def bn_bwd(dy, x, m, c, mean, rstd, gamma, beta, act, dgamma, dbeta, dx, accumulate, ws, planes=None):
    if planes is None:
        _lib.check(_lib.load().pf_bn_bwd(_p(dy), _p(x), m, c, _p(mean), _p(rstd), _p(gamma), _p(beta), int(act),
                                         _p(dgamma), _p(dbeta), _p(dx), int(bool(accumulate)), _p(ws), _stream()),
                   'pf_bn_bwd')
    else:
        _lib.check(_lib.load().pf_bn_bwd_planes(_p(dy), _p(x), m, c, _p(mean), _p(rstd), _p(gamma), _p(beta), int(act),
                                                _p(dgamma), _p(dbeta), _p(dx), int(bool(accumulate)), _p(planes.hi),
                                                _p(planes.lo), _p(ws), _stream()), 'pf_bn_bwd_planes')


def bn_apply_add(x, m, c, mean, rstd, gamma, beta, res, y=None, planes=None):
    """y = bn(x) + res (linear bottleneck + residual, training-mode statistics), to fp32 and / or operand planes"""
    _lib.check(_lib.load().pf_bn_apply_add(_p(x), m, c, _p(mean), _p(rstd), _p(gamma), _p(beta), _p(res), _p(y),
                                           _p(planes.hi if planes is not None else None),
                                           _p(planes.lo if planes is not None else None), _stream()), 'pf_bn_apply_add')


def bn_apply_add_eval(x, m, c, mov_mean, mov_var, eps, gamma, beta, res, y=None, planes=None):
    """y = bn(x) + res with the moving statistics (inference mode), to fp32 and / or operand planes"""
    _lib.check(_lib.load().pf_bn_apply_add_eval(_p(x), m, c, _p(mov_mean), _p(mov_var), float(eps), _p(gamma), _p(beta),
                                                _p(res), _p(y), _p(planes.hi if planes is not None else None),
                                                _p(planes.lo if planes is not None else None), _stream()),
               'pf_bn_apply_add_eval')


def gather_channels(x, idx, y=None, planes=None, x_planes=None):
    """y[..., j] = x[..., idx[j]] (0 where idx[j] < 0) over the last (channel) axis, to fp32 `y` and / or operand
    `planes`.  The input is `x` (fp32) or, when x is None, `x_planes` = (Planes, rows m, channels cin)."""
    cout = idx.numel()
    if x is not None:
        cin = x.shape[-1]
        m = x.numel() // cin
        xh = xl = None
    else:
        (xp, m, cin) = x_planes
        xh, xl = xp.hi, xp.lo
    _lib.check(_lib.load().pf_gather_channels(_p(x), _p(xh), _p(xl), m, cin, cout, _p(idx), _p(y),
                                              _p(planes.hi if planes is not None else None),
                                              _p(planes.lo if planes is not None else None), _stream()),
               'pf_gather_channels')


def bn_apply_eval_gather(x, m, c, mov_mean, mov_var, eps, gamma, beta, act, idx, y=None, planes=None):
    """gather(act(bn(x))) with the moving statistics in one launch: x is [m, c], the result [m, idx.numel()] goes to
    fp32 `y` and / or operand `planes`"""
    _lib.check(_lib.load().pf_bn_apply_eval_gather(_p(x), m, c, _p(mov_mean), _p(mov_var), float(eps), _p(gamma),
                                                   _p(beta), int(act), idx.numel(), _p(idx), _p(y),
                                                   _p(planes.hi if planes is not None else None),
                                                   _p(planes.lo if planes is not None else None), _stream()),
               'pf_bn_apply_eval_gather')


def bn_apply_gather(x, m, c, mean, rstd, gamma, beta, act, idx, y=None, planes=None):
    """gather(act(bn(x))) with the batch statistics (training mode) in one launch: x is [m, c], the result
    [m, idx.numel()] goes to fp32 `y` and / or operand `planes`"""
    _lib.check(_lib.load().pf_bn_apply_gather(_p(x), m, c, _p(mean), _p(rstd), _p(gamma), _p(beta), int(act),
                                              idx.numel(), _p(idx), _p(y),
                                              _p(planes.hi if planes is not None else None),
                                              _p(planes.lo if planes is not None else None), _stream()),
               'pf_bn_apply_gather')


def scatter_table(index, cin):
    """inverse of a gather's index table (numpy int32 [cin]): the compact position of every full-width channel, -1 for
    a channel the gather dropped — what scatter_channels takes"""
    index = np.asarray(index, np.int64)
    kept = index[index >= 0]
    if len(np.unique(kept)) != len(kept) or (len(kept) and kept.max() >= cin):
        raise ValueError('a gather index table holds every channel of its input at most once')
    inv = np.full(cin, -1, np.int32)
    inv[kept] = np.nonzero(index >= 0)[0]
    return inv


def scatter_channels(dy, inv, dx=None, accumulate=False, planes=None):
    """backward of gather_channels: dx[..., c] (+)= dy[..., inv[c]] (0 where inv[c] < 0; with `accumulate` those
    channels are left as they are), to fp32 `dx` and / or the `planes` of the final value"""
    cout, cin = dy.shape[-1], inv.numel()
    _lib.check(_lib.load().pf_scatter_channels(_p(dy), dy.numel() // cout, cin, cout, _p(inv), int(bool(accumulate)),
                                               _p(dx), _p(planes.hi if planes is not None else None),
                                               _p(planes.lo if planes is not None else None), _stream()),
               'pf_scatter_channels')


def dropout_fwd(x, keep_prob, seed, rank, state, y, mask, stream_id=0, layout=None, full_width=None):
    """slim.dropout in a training pass: y = (x / keep) * mask, mask = floor(keep + u) (uint8), u from Philox4x32-10 keyed
    by (seed, rank) at the step held in `state` (int64 [2] on the device, advanced by the launch) of stream `stream_id`
    (one per Dropout op of a graph).  layout (int32 [C] on the device, C = x.shape[-1], -1 for padding) and full_width:
    x is the channel-pruned view of a [..., full_width] tensor, and draws the full-width mask gathered by the layout
    (pf_dropout_fwd_mapped)"""
    assert state.dtype == torch.int64 and state.numel() >= 2 and mask.dtype == torch.uint8 and mask.numel() >= x.numel()
    args = (_p(x), x.numel(), float(keep_prob), int(seed) & 0xffffffff, int(rank) & 0xffffffff,
            int(stream_id) & 0xffffffff)
    if layout is None:
        _lib.check(_lib.load().pf_dropout_fwd(*args, _p(state), _p(y), _p(mask), _stream()), 'pf_dropout_fwd')
        return
    assert layout.dtype == torch.int32 and layout.numel() == x.shape[-1]
    _lib.check(_lib.load().pf_dropout_fwd_mapped(*args, _p(layout), layout.numel(), int(full_width), _p(state), _p(y),
                                                 _p(mask), _stream()), 'pf_dropout_fwd_mapped')


def dropout_bwd(dy, mask, keep_prob, dx, accumulate=False):
    """dx (+)= (dy * mask) / keep"""
    _lib.check(_lib.load().pf_dropout_bwd(_p(dy), _p(mask), dy.numel(), float(keep_prob), int(bool(accumulate)), _p(dx),
                                          _stream()), 'pf_dropout_bwd')


def add(a, b, out, accumulate=False):
    _lib.check(_lib.load().pf_add(_p(a), _p(b), a.numel(), int(bool(accumulate)), _p(out), _stream()), 'pf_add')


def fold_diag_blocks(src, g, m, n, dst):
    _lib.check(_lib.load().pf_fold_diag_blocks(_p(src), int(g), int(m), int(n), _p(dst), _stream()), 'pf_fold_diag_blocks')


def relu_bwd(dy, y, dx, act=1, accumulate=False):
    _lib.check(_lib.load().pf_relu_bwd(_p(dy), _p(y), y.numel(), int(act), int(bool(accumulate)), _p(dx), _stream()),
               'pf_relu_bwd')


def colsum(a, m, c, out):
    _lib.check(_lib.load().pf_colsum(_p(a), m, c, _p(out), _stream()), 'pf_colsum')


def maxpool_fwd(d, x, y, argmax=None):
    _lib.check(_lib.load().pf_maxpool_fwd(ctypes.byref(d), _p(x), _p(y), _p(argmax), _stream()), 'pf_maxpool_fwd')


def maxpool_bwd(d, dy, argmax, dx, accumulate=False):
    _lib.check(_lib.load().pf_maxpool_bwd(ctypes.byref(d), _p(dy), _p(argmax), int(bool(accumulate)), _p(dx),
                                          _stream()), 'pf_maxpool_bwd')


def global_avgpool_fwd(x, n, hw, c, y):
    _lib.check(_lib.load().pf_global_avgpool_fwd(_p(x), n, hw, c, _p(y), _stream()), 'pf_global_avgpool_fwd')


def global_avgpool_bwd(dy, n, hw, c, dx, accumulate=False):
    _lib.check(_lib.load().pf_global_avgpool_bwd(_p(dy), n, hw, c, int(bool(accumulate)), _p(dx), _stream()),
               'pf_global_avgpool_bwd')


def softmax_fwd(x, y):
    _lib.check(_lib.load().pf_softmax_fwd(_p(x), x.shape[0], x.shape[1], _p(y), _stream()), 'pf_softmax_fwd')


def softmax_bwd(dy, y, dx):
    _lib.check(_lib.load().pf_softmax_bwd(_p(dy), _p(y), y.shape[0], y.shape[1], _p(dx), _stream()), 'pf_softmax_bwd')


def minmax_reset(slots):
    """slots: int32 [n, 2] -> every pair = (0xFFFFFFFF, 0)."""
    _lib.check(_lib.load().pf_minmax_reset(_p(slots), slots.numel() // 2, _stream()), 'pf_minmax_reset')


# ----------------------------------------------------------------------------- a4 on tensor cores
def conv2d_tc_supported(d):
    return bool(_lib.load().pf_conv2d_tc_supported(ctypes.byref(d)))


class TcWeights:
    """Split-bf16, K-major copies of one conv kernel for the tensor-core path (fwd and dgrad operands)."""

    def __init__(self, d, device, need_dgrad=True):
        L = _lib.load()
        self.d = d
        nf = int(L.pf_conv2d_tc_weight_elems(ctypes.byref(d), 0))
        self.f_hi = torch.zeros(nf, dtype=torch.bfloat16, device=device)
        self.f_lo = torch.zeros(nf, dtype=torch.bfloat16, device=device)
        self.d_hi = self.d_lo = None
        if need_dgrad:
            nd = int(L.pf_conv2d_tc_weight_elems(ctypes.byref(d), 1))
            self.d_hi = torch.zeros(nd, dtype=torch.bfloat16, device=device)
            self.d_lo = torch.zeros(nd, dtype=torch.bfloat16, device=device)

    def prepare(self, w):
        _lib.check(_lib.load().pf_conv2d_tc_prep_weight(ctypes.byref(self.d), _p(w), _p(self.f_hi), _p(self.f_lo),
                                                        _p(self.d_hi), _p(self.d_lo), _stream()),
                   'pf_conv2d_tc_prep_weight')


TC_PREP_SEG = np.dtype([('w', np.uint64), ('fwd_hi', np.uint64), ('fwd_lo', np.uint64), ('dgrad_hi', np.uint64),
                        ('dgrad_lo', np.uint64), ('rs', np.int32), ('c', np.int32), ('k', np.int32),
                        ('kpad_f', np.int32), ('kpad_d', np.int32), ('q_bits', np.int32), ('q_alpha', np.uint64),
                        ('q_beta', np.uint64), ('q_ralpha', np.uint64), ('q_ncols', np.int32), ('reserved', np.int32)],
                       align=True)
assert TC_PREP_SEG.itemsize == 96


class TcWeightsBatch:
    """One launch that refreshes the split-bf16 copies of MANY conv kernels (pf_conv2d_tc_prep_weights_multi)."""

    def __init__(self, items, device, levels=None):
        """items: list of (TcWeights, fp32 HWIO weight tensor [R,S,C,K]).
        levels: {item index: (unquantized weight tensor, alpha, beta, ralpha device views at the tensor's first bucket,
        ncols, bits)} — those kernels are prepared as integer levels from the UNQUANTIZED weights (pf_tc_prep_seg)."""
        segs = np.zeros(len(items), dtype=TC_PREP_SEG)
        rows = []
        self.levels = dict(levels or {})
        for i, (tw, w) in enumerate(items):
            r, s_, c, k = w.shape if w.dim() == 4 else (1, 1) + tuple(w.shape)
            segs[i] = (w.data_ptr(), tw.f_hi.data_ptr(), tw.f_lo.data_ptr(),
                       tw.d_hi.data_ptr() if tw.d_hi is not None else 0, tw.d_lo.data_ptr() if tw.d_lo is not None else 0,
                       r * s_, c, k, tw.f_hi.numel() // k, (tw.d_hi.numel() // c) if tw.d_hi is not None else 0, 0, 0, 0, 0, 0, 0)
        self.segs_plain = segs.copy()
        for i, (tw, w) in enumerate(items):
            r, s_, c, k = w.shape if w.dim() == 4 else (1, 1) + tuple(w.shape)
            if i in self.levels:
                w0, al, be, ra, ncols, bits = self.levels[i]
                if ncols not in (1, k) or not 1 <= int(bits) <= 8:
                    raise ValueError('weight levels need per-layer or per-output-channel buckets and 1..8 bits')
                segs[i]['w'], segs[i]['q_bits'], segs[i]['q_ncols'] = w0.data_ptr(), int(bits), int(ncols)
                segs[i]['q_alpha'], segs[i]['q_beta'], segs[i]['q_ralpha'] = al.data_ptr(), be.data_ptr(), ra.data_ptr()
            for k0 in range(0, r * s_ * c, 32):                 # 32 x 64 tiles of the [R*S*Cin, Cout] matrix
                for co0 in range(0, k, 64):
                    rows.append((i, 0, k0, 0, co0, 0, 0))
        self.keep = items
        self.segs = segs
        self.device = device
        self.work = np.array(rows, dtype=WORK) if rows else np.zeros(0, dtype=WORK)
        self.segs_dev = torch.from_numpy(segs.view(np.uint8).copy()).to(device)
        self.segs_plain_dev = torch.from_numpy(self.segs_plain.view(np.uint8).copy()).to(device) if self.levels else self.segs_dev
        self.work_dev = torch.from_numpy(self.work.view(np.uint8)).to(device)

    def set_bits(self, bits_of):
        """{item index: bits} for the level-prepared kernels (the RL bit search changes them between roll-outs);
        above 8 bits a kernel goes back to split-bf16 planes of its quantized values"""
        for i, b in bits_of.items():
            if i in self.levels:
                if 1 <= int(b) <= 8:
                    self.segs[i]['q_bits'], self.segs[i]['w'] = int(b), self.levels[i][0].data_ptr()
                else:
                    self.segs[i]['q_bits'], self.segs[i]['w'] = 0, self.segs_plain[i]['w']
        self.segs_dev = torch.from_numpy(self.segs.view(np.uint8).copy()).to(self.device)

    def prepare(self, levels=True):
        """levels=False: every kernel as split-bf16 planes of the tensors given at construction (evaluation passes)"""
        segs = self.segs_dev if levels else self.segs_plain_dev
        _lib.check(_lib.load().pf_conv2d_tc_prep_weights_multi(_p(segs), _p(self.work_dev), len(self.work),
                                                               _stream()), 'pf_conv2d_tc_prep_weights_multi')


def conv2d_tc_fwd(d, x, tw, bias, relu, y, residual=None, bn_out=None):
    """bn_out (TcBnOut): also apply that inference batch norm to the output in the epilogue (y is still written)"""
    if bn_out is None:
        _lib.check(_lib.load().pf_conv2d_tc_fwd(ctypes.byref(d), _p(x), _p(tw.f_hi), _p(tw.f_lo), _p(bias),
                                                int(bool(relu)), _p(residual), _p(y), _stream()), 'pf_conv2d_tc_fwd')
    else:
        _lib.check(_lib.load().pf_conv2d_tc_fwd_bn(ctypes.byref(d), _p(x), _p(tw.f_hi), _p(tw.f_lo), _p(bias),
                                                   int(bool(relu)), _p(residual), _p(y), ctypes.byref(bn_out),
                                                   _stream()), 'pf_conv2d_tc_fwd_bn')


class TcBnOut(_lib.TcBnOut):
    """pf_tc_bn_out of tensors: act(bn(.)) with the moving statistics (pf_bn_apply_eval's arithmetic), written to the
    fp32 tensor y and / or the operand planes `planes` by the forward conv whose output it normalizes"""

    def __init__(self, mean, var, eps, gamma, beta, act, y=None, planes=None):
        super().__init__(mean.data_ptr(), var.data_ptr(), gamma.data_ptr(), beta.data_ptr(), float(eps), int(act),
                         y.data_ptr() if y is not None else None, planes.hi.data_ptr() if planes is not None else None,
                         planes.lo.data_ptr() if planes is not None else None)
        self._keep = (mean, var, gamma, beta, y, planes)


def conv2d_tc_dgrad(d, dy, tw, accumulate, dx):
    _lib.check(_lib.load().pf_conv2d_tc_dgrad(ctypes.byref(d), _p(dy), _p(tw.d_hi), _p(tw.d_lo),
                                              int(bool(accumulate)), _p(dx), _stream()), 'pf_conv2d_tc_dgrad')


def conv2d_tc_wgrad_supported(d):
    return bool(_lib.load().pf_conv2d_tc_wgrad_supported(ctypes.byref(d)))


def conv2d_tc_wgrad_workspace_floats(d):
    return int(_lib.load().pf_conv2d_tc_wgrad_workspace_bytes(ctypes.byref(d))) // 4


def conv2d_tc_wgrad(d, x, dy, ws, dw):
    _lib.check(_lib.load().pf_conv2d_tc_wgrad(ctypes.byref(d), _p(x), _p(dy), _p(ws), _p(dw), _stream()),
               'pf_conv2d_tc_wgrad')


class Planes:
    """A tensor in the operand format of the tensor-core kernels: x = hi + lo, two bf16 planes with the layout of
    the fp32 tensor.  `buf` (optional) = one bf16 buffer of >= 2*numel elements to carve the planes from."""

    def __init__(self, numel, device, buf=None):
        assert numel % 8 == 0
        if buf is None:
            buf = torch.empty(2 * numel, dtype=torch.bfloat16, device=device)
            if os.environ.get('PF_POISON', '0') == '1':
                buf.fill_(float('nan'))
        assert buf.dtype == torch.bfloat16 and buf.numel() >= 2 * numel
        self.numel, self.buf = numel, buf
        self.hi, self.lo = buf[:numel], buf[numel:2 * numel]


def split_bf16(src, planes):
    """fp32 -> (hi, lo) bf16 planes."""
    _lib.check(_lib.load().pf_split_bf16(_p(src), _p(planes.hi), _p(planes.lo), src.numel(), _stream()), 'pf_split_bf16')


def conv2d_tc_fwd_planes(d, xp, tw, bias, relu, y, residual=None, bn_out=None):
    """bn_out: as conv2d_tc_fwd"""
    if bn_out is None:
        _lib.check(_lib.load().pf_conv2d_tc_fwd_planes(ctypes.byref(d), _p(xp.hi), _p(xp.lo), _p(tw.f_hi), _p(tw.f_lo),
                                                       _p(bias), int(bool(relu)), _p(residual), _p(y), _stream()),
                   'pf_conv2d_tc_fwd_planes')
    else:
        _lib.check(_lib.load().pf_conv2d_tc_fwd_planes_bn(ctypes.byref(d), _p(xp.hi), _p(xp.lo), _p(tw.f_hi), _p(tw.f_lo),
                                                          _p(bias), int(bool(relu)), _p(residual), _p(y),
                                                          ctypes.byref(bn_out), _stream()), 'pf_conv2d_tc_fwd_planes_bn')


def conv2d_tc_dgrad_planes(d, dyp, tw, accumulate, dx):
    _lib.check(_lib.load().pf_conv2d_tc_dgrad_planes(ctypes.byref(d), _p(dyp.hi), _p(dyp.lo), _p(tw.d_hi), _p(tw.d_lo),
                                                     int(bool(accumulate)), _p(dx), _stream()), 'pf_conv2d_tc_dgrad_planes')


def conv2d_tc_wgrad_planes_workspace_floats(d):
    return int(_lib.load().pf_conv2d_tc_wgrad_planes_workspace_bytes(ctypes.byref(d))) // 4


TC_REDUCE_SEG = np.dtype([('partial', np.uint64), ('out', np.uint64), ('n', np.int64), ('splits', np.int32),
                          ('reserved', np.int32)], align=True)


def conv2d_tc_wgrad_splits(d):
    return int(_lib.load().pf_conv2d_tc_wgrad_splits(ctypes.byref(d)))


class TcWgradReduceBatch:
    """Deferred split-K reduction of many weight gradients in one launch."""

    def __init__(self, items, device):
        """items: list of (partials tensor [splits*n], out tensor [n], splits)."""
        segs = np.zeros(len(items), dtype=TC_REDUCE_SEG)
        for i, (part, out, splits) in enumerate(items):
            segs[i] = (part.data_ptr(), out.data_ptr(), out.numel(), splits, 0)
        self.keep = items
        self.work = flat_works([o.numel() for _, o, _ in items], 1 << 14)
        self.segs_dev = torch.from_numpy(segs.view(np.uint8)).to(device)
        self.work_dev = torch.from_numpy(self.work.view(np.uint8)).to(device)

    def reduce(self):
        _lib.check(_lib.load().pf_conv2d_tc_wgrad_reduce_multi(_p(self.segs_dev), _p(self.work_dev), len(self.work),
                                                               _stream()), 'pf_conv2d_tc_wgrad_reduce_multi')


def conv2d_tc_wgrad_planes(d, xp, dyp, ws, dw):
    _lib.check(_lib.load().pf_conv2d_tc_wgrad_planes(ctypes.byref(d), _p(xp.hi), _p(xp.lo), _p(dyp.hi), _p(dyp.lo), _p(ws),
                                                     _p(dw), _stream()), 'pf_conv2d_tc_wgrad_planes')


# ---- TMA-fed kernels, operands as quantizer levels (include/pf_b200.h: pf_tc_act / pf_tc_wt)
ACT_HDR = np.dtype([('scale', np.float32), ('nplanes', np.int32)])


def conv2d_tc_set_feed(mode):
    """1: TMA kernels where eligible (default), 0: cp.async kernels everywhere, -1: PF_TC_FEED environment default."""
    _lib.check(_lib.load().pf_conv2d_tc_set_feed(int(mode)), 'pf_conv2d_tc_set_feed')


def conv2d_tc_tma_supported(d, which):
    """which: 0 fwd, 1 dgrad, 2 wgrad"""
    return bool(_lib.load().pf_conv2d_tc_tma_supported(ctypes.byref(d), int(which)))


def tc_act(planes, hdr=None, csum=None, nseg=0, single=False):
    """pf_tc_act of a Planes object (+ the producer's device header / channel sums); single: only plane0 is valid"""
    return _lib.TcAct(planes.hi.data_ptr(), 0 if single else planes.lo.data_ptr(), hdr.data_ptr() if hdr is not None else 0,
                      csum.data_ptr() if csum is not None else 0, int(nseg), 0)


def tc_wt(p0, p1=None, alpha=None, beta=None, per_channel=False, bits=0):
    return _lib.TcWt(p0.data_ptr(), p1.data_ptr() if p1 is not None else 0, alpha.data_ptr() if alpha is not None else 0,
                     beta.data_ptr() if beta is not None else 0, int(bool(per_channel)), int(bits))


def conv2d_tc_fwd_ex(d, act, wt, bias, relu, y, residual=None):
    _lib.check(_lib.load().pf_conv2d_tc_fwd_ex(ctypes.byref(d), ctypes.byref(act), ctypes.byref(wt), _p(bias), int(bool(relu)),
                                               _p(residual), _p(y), _stream()), 'pf_conv2d_tc_fwd_ex')


def conv2d_tc_dgrad_ex(d, act, wt, accumulate, dx):
    _lib.check(_lib.load().pf_conv2d_tc_dgrad_ex(ctypes.byref(d), ctypes.byref(act), ctypes.byref(wt), int(bool(accumulate)),
                                                 _p(dx), _stream()), 'pf_conv2d_tc_dgrad_ex')


def conv2d_tc_wgrad_ex(d, x_act, dy_act, ws, dw):
    _lib.check(_lib.load().pf_conv2d_tc_wgrad_ex(ctypes.byref(d), ctypes.byref(x_act), ctypes.byref(dy_act), _p(ws), _p(dw),
                                                 _stream()), 'pf_conv2d_tc_wgrad_ex')


def conv2d_u8_supported(d):
    """the shapes pf_conv2d_u8_fwd runs: Cin and Cout multiples of 64, strides <= 8, filters <= 16 x 16"""
    return bool(_lib.load().pf_conv2d_u8_supported(ctypes.byref(d)))


def conv2d_u8_narrow_supported(d):
    """the shapes pf_conv2d_u8_fwd runs on either of its kernels: those of conv2d_u8_supported, and any Cin and Cout
    that are multiples of 16 with R*S*Cin <= 32768 (the cp.async-fed kernel)"""
    return bool(_lib.load().pf_conv2d_u8_narrow_supported(ctypes.byref(d)))


def conv2d_u8_fwd(d, x_levels, hdr, csum, w_levels, alpha, beta, bits, y, bias=None, relu=False, residual=None,
                  bn_out=None):
    """y = the fake-quantized conv from u8 levels (pf_conv2d_u8_fwd): x_levels uint8 [N, H, W, Cin] with its header and
    channel sums (bn_eval_levels_u8), w_levels uint8 [Cout, R*S*Cin], alpha / beta the weight bucket scales ([1] per
    layer or [Cout] per channel); bn_out: a TcBnOut folded into the epilogue"""
    if x_levels.dtype != torch.uint8 or w_levels.dtype != torch.uint8:
        raise ValueError('conv2d_u8_fwd: the levels are uint8 tensors')
    _check_f32(csum, alpha, beta, y, bias, residual)
    act = _lib.TcAct(x_levels.data_ptr(), 0, hdr.data_ptr(), csum.data_ptr(), (d.c + 127) // 128, 0)
    wt = _lib.TcWt(w_levels.data_ptr(), 0, alpha.data_ptr(), beta.data_ptr(), int(alpha.numel() > 1), int(bits))
    _lib.check(_lib.load().pf_conv2d_u8_fwd(ctypes.byref(d), ctypes.byref(act), ctypes.byref(wt), _p(bias),
                                            int(bool(relu)), _p(residual), _p(y),
                                            ctypes.byref(bn_out) if bn_out is not None else None, _stream()),
               'pf_conv2d_u8_fwd')


def bn_eval_levels_u8(x, m, c, mov_mean, mov_var, eps, gamma, beta, act, bits, rng, levels, hdr, csum, have_range=False):
    """u8 levels of Q(act(bn(x))) with the moving statistics and this batch's range (pf_bn_eval_levels_u8): levels
    uint8 [m * c], hdr int32 [2] (pf_tc_act_hdr), csum float32 [m * ceil(c / 128)], rng int32 [2] (the range, ordered
    encoding); have_range: rng already holds the range of act(bn(x))"""
    if levels.dtype != torch.uint8:
        raise ValueError('bn_eval_levels_u8: levels must be uint8')
    _check_f32(x, mov_mean, mov_var, gamma, beta, csum)
    _lib.check(_lib.load().pf_bn_eval_levels_u8(_p(x), m, c, _p(mov_mean), _p(mov_var), float(eps), _p(gamma), _p(beta),
                                                int(act), int(bits), _p(rng), int(bool(have_range)), _p(levels), _p(hdr),
                                                _p(csum), _stream()), 'pf_bn_eval_levels_u8')


def bn_eval_levels_u8_static(x, m, c, mov_mean, mov_var, eps, gamma, beta, act, bits, rng, levels, hdr, csum):
    """bn_eval_levels_u8 with a static range rng (range_slots; read only): y clamped to it, one pass, no range pass
    (pf_bn_eval_levels_u8_static)"""
    if levels.dtype != torch.uint8:
        raise ValueError('bn_eval_levels_u8_static: levels must be uint8')
    _check_f32(x, mov_mean, mov_var, gamma, beta, csum)
    _lib.check(_lib.load().pf_bn_eval_levels_u8_static(_p(x), m, c, _p(mov_mean), _p(mov_var), float(eps), _p(gamma),
                                                       _p(beta), int(act), int(bits), _p(rng), _p(levels), _p(hdr),
                                                       _p(csum), _stream()), 'pf_bn_eval_levels_u8_static')


def conv2d_tc_last_plan():
    """Host-side plan of the most recent tensor-core conv launch (pf_tc_plan) as a dict: which feed, pass and kernel
    variant ran, and with what tile width, ring depth, stages, grid and split-K."""
    plan = _lib.TcPlan()
    _lib.check(_lib.load().pf_conv2d_tc_last_plan(ctypes.byref(plan)), 'pf_conv2d_tc_last_plan')
    out = {n: int(getattr(plan, n)) for n, _ in _lib.TcPlan._fields_}
    out['pass'] = out.pop('pass_')
    return out


def s2d_planes(x, pad_t, pad_l, hp, wp, cpad, planes):
    """space-to-depth of a stride-2 first layer's input [n,h,w,c] into operand planes [n,hp,wp,cpad]"""
    n, h, w, c = x.shape
    _lib.check(_lib.load().pf_s2d_planes(_p(x), n, h, w, c, int(pad_t), int(pad_l), int(hp), int(wp), int(cpad),
                                         _p(planes.hi), _p(planes.lo), _stream()), 'pf_s2d_planes')


def gather_rows(src, idx, dst, row_len):
    """dst[j] = src[idx[j]] (zero row where idx[j] < 0); rows of `row_len` floats"""
    _lib.check(_lib.load().pf_gather_rows(_p(src), _p(idx), idx.numel(), int(row_len), _p(dst), _stream()), 'pf_gather_rows')


def s2d_weight_maps(r, s, c, cpad):
    """Row maps between the HWIO kernel [r,s,c,K] of a stride-2 conv and its space-to-depth form [r2,s2,cpad,K]:
    fwd[j] = source row of s2d row j (-1: zero), bwd[i] = s2d row holding the gradient of source row i."""
    r2, s2 = (r + 1) // 2, (s + 1) // 2
    fwd = -np.ones(r2 * s2 * cpad, np.int32)
    bwd = np.zeros(r * s * c, np.int32)
    for rr in range(r):
        for ss in range(s):
            for cc in range(c):
                j = ((rr // 2) * s2 + (ss // 2)) * cpad + ((rr % 2) * 2 + (ss % 2)) * c + cc
                i = (rr * s + ss) * c + cc
                fwd[j], bwd[i] = i, j
    return r2, s2, fwd, bwd


def im2col_planes(d, x, kpad, planes):
    _lib.check(_lib.load().pf_im2col_planes(ctypes.byref(d), _p(x), int(kpad), _p(planes.hi), _p(planes.lo), _stream()),
               'pf_im2col_planes')


# ----------------------------------------------------------------------------- depthwise conv
def dwconv_fwd(d, x, w, y):
    _lib.check(_lib.load().pf_dwconv_fwd(ctypes.byref(d), _p(x), _p(w), _p(y), _stream()), 'pf_dwconv_fwd')


def dwconv_dgrad(d, dy, w, accumulate, dx):
    _lib.check(_lib.load().pf_dwconv_dgrad(ctypes.byref(d), _p(dy), _p(w), int(bool(accumulate)), _p(dx), _stream()),
               'pf_dwconv_dgrad')


def dwconv_wgrad_workspace_floats(d):
    return int(_lib.load().pf_dwconv_wgrad_workspace_bytes(ctypes.byref(d))) // 4


def dwconv_wgrad(d, x, dy, ws, dw):
    _lib.check(_lib.load().pf_dwconv_wgrad(ctypes.byref(d), _p(x), _p(dy), _p(ws), _p(dw), _stream()),
               'pf_dwconv_wgrad')


# pf_dwconv_last_variant codes (include/pf_b200.h: PF_DW_*), 1-based
DW_VARIANTS = ('fwd rows', 'fwd 3x3 s1', 'fwd 3x3 s2', 'fwd generic',
               'dgrad rows', 'dgrad 3x3 s1', 'dgrad block p0', 'dgrad block p1', 'dgrad 3x3 s2', 'dgrad generic',
               'wgrad rows', 'wgrad 3x3 s1', 'wgrad 3x3 s2', 'wgrad generic')


def dwconv_last_variant():
    """Name of the kernel the most recent depthwise launch ran (DW_VARIANTS), None before the first one."""
    v = int(_lib.load().pf_dwconv_last_variant())
    return DW_VARIANTS[v - 1] if v else None


def dwconv_u8_supported(d):
    """the shapes pf_dwconv_u8_fwd runs: depth multiplier 1, C % 16 == 0, <= 9 taps, strides 1 or 2"""
    return bool(_lib.load().pf_dwconv_u8_supported(ctypes.byref(d)))


def dwconv_u8_fwd(d, x_levels, hdr, w_levels, alpha, beta, bits, y):
    """y = the fake-quantized depthwise conv from u8 levels (pf_dwconv_u8_fwd): x_levels uint8 [N, H, W, C] with its
    header (bn_eval_levels_u8), w_levels uint8 [R*S, C], alpha / beta the weight bucket scales ([1] per layer or [C]
    per channel)"""
    if x_levels.dtype != torch.uint8 or w_levels.dtype != torch.uint8:
        raise ValueError('dwconv_u8_fwd: the levels are uint8 tensors')
    _check_f32(alpha, beta, y)
    act = _lib.TcAct(x_levels.data_ptr(), 0, hdr.data_ptr(), 0, 0, 0)
    wt = _lib.TcWt(w_levels.data_ptr(), 0, alpha.data_ptr(), beta.data_ptr(), int(alpha.numel() > 1), int(bits))
    _lib.check(_lib.load().pf_dwconv_u8_fwd(ctypes.byref(d), ctypes.byref(act), ctypes.byref(wt), _p(y), _stream()),
               'pf_dwconv_u8_fwd')


def preprocess_images(crops_u8, desc, out, mean=(123.68, 116.78, 103.94)):
    """ILSVRC-12 preprocessing of a packed mini-batch on the device (pf_preprocess_images): crops_u8 = uint8 CUDA buffer
    holding every decoded crop back to back, desc = uint8 CUDA view of n pf_img_desc records
    (datasets/ilsvrc12_dataset.py:IMG_DESC), out = fp32 [n, out_h, out_w, 3]."""
    L = _lib.load()
    _check_f32(out)
    if crops_u8.dtype != torch.uint8 or desc.dtype != torch.uint8 or not crops_u8.is_cuda or not desc.is_cuda:
        raise ValueError('expected uint8 CUDA buffers for the crops and the descriptor table')
    n, out_h, out_w, c = out.shape
    if c != 3 or desc.numel() != n * 40:
        raise ValueError('out must be [n, h, w, 3] with one 40-byte descriptor per image')
    _lib.check(L.pf_preprocess_images(_p(crops_u8), _p(desc), n, out_h, out_w, float(mean[0]), float(mean[1]),
                                      float(mean[2]), _p(out), _stream()), 'pf_preprocess_images')
    return out


def jpeg_decode(data_u8, desc, n, coef_ws, crops_u8, status):
    """Baseline JPEG decoding on the device (pf_jpeg_decode): data_u8 = uint8 CUDA buffer of the images' entropy-coded
    segments, desc = uint8 CUDA view of n pf_jpeg_desc records (datasets/jpeg.py:JPEG_DESC), coef_ws = int16 CUDA
    workspace of at least sum(jpeg.workspace_elems(d)) elements, crops_u8 = uint8 CUDA buffer the RGB crops are written
    into, status = int32 CUDA [n] (0: decoded; otherwise the host has to decode that image, datasets/jpeg.py:STATUS)."""
    L = _lib.load()
    for t, dt in ((data_u8, torch.uint8), (desc, torch.uint8), (coef_ws, torch.int16), (crops_u8, torch.uint8),
                  (status, torch.int32)):
        if t.dtype != dt or not t.is_cuda or not t.is_contiguous():
            raise ValueError('jpeg_decode: expected contiguous CUDA buffers (uint8 data / desc / crops, int16 workspace, '
                             'int32 status)')
    if desc.numel() < n * 4144 or status.numel() < n:
        raise ValueError('jpeg_decode: %d images need %d descriptor bytes and %d status words' % (n, n * 4144, n))
    _lib.check(L.pf_jpeg_decode(_p(data_u8), _p(desc), int(n), _p(coef_ws), _p(crops_u8), _p(status), _stream()),
               'pf_jpeg_decode')
    return status



# ----------------------------------------------------------------------------- f4 channel selection (pf_cpg.cu)
def cpg_diff_l2(a, b, diff, loss, partial_ws):
    """diff = a - b, loss[0] = sum(diff^2) / 2 — tf.nn.l2_loss of two conv outputs
    (learners/channel_pruning_gpu/learner.py:352); partial_ws: L2_PARTIALS floats."""
    _check_f32(a, b, diff, loss, partial_ws)
    if a.numel() != b.numel() or a.numel() != diff.numel():
        raise ValueError('cpg_diff_l2: size mismatch')
    _lib.check(_lib.load().pf_cpg_diff_l2(_p(a), _p(b), a.numel(), _p(diff), _p(loss), _p(partial_ws), _stream()),
               'pf_cpg_diff_l2')


def _rs_cin_cout(w):
    if w.dim() == 4:
        return w.shape[0] * w.shape[1], w.shape[2], w.shape[3]
    if w.dim() == 2:
        return 1, w.shape[0], w.shape[1]
    raise ValueError('kernel must be [R,S,Cin,Cout] or [Cin,Cout]')


def cpg_group_norms(w, g, lr, norms):
    """norms[c] = sqrt(sum_{r,s,k} (w - lr*g)^2) (learner.py:378-379); g None: norm of w itself (:256)."""
    _check_f32(w, g, norms)
    rs, cin, cout = _rs_cin_cout(w)
    _lib.check(_lib.load().pf_cpg_group_norms(_p(w), _p(g), float(lr), rs, cin, cout, _p(norms), _stream()),
               'pf_cpg_group_norms')


def cpg_prox_step(w, g, lr, prune_perctl, norms=None):
    """One proximal (group soft-threshold) step of the channel selection, in place on w (learner.py:375-383):
    w' = w - lr g ; n_c = ||w'[:, :, c, :]|| ; t = percentile(n, prune_perctl) ('nearest') ; w = w' max(1 - t/n_c, 0).
    Returns the threshold (device tensor [1])."""
    rs, cin, cout = _rs_cin_cout(w)
    if norms is None:
        norms = torch.empty(cin, dtype=torch.float32, device=w.device)
    lr = float(np.float32(lr))
    cpg_group_norms(w, g, lr, norms)
    # the percentile is fed through a float32 placeholder (learner.py:365) and widened to double by percentile()
    thr = select_desc([norms], [(0, percentile_rank_desc(cin, np.float32(prune_perctl)))])
    _lib.check(_lib.load().pf_cpg_prox_apply(_p(w), _p(g), float(lr), _p(norms), _p(thr), rs, cin, cout, _stream()),
               'pf_cpg_prox_apply')
    return thr


def cpg_channel_mask(w, mask, norms=None):
    """mask = tile(||w[:, :, c, :]|| > 0) (learner.py:256-259)."""
    _check_f32(w, mask)
    rs, cin, cout = _rs_cin_cout(w)
    if norms is None:
        norms = torch.empty(cin, dtype=torch.float32, device=w.device)
    cpg_group_norms(w, None, 0.0, norms)
    _lib.check(_lib.load().pf_cpg_channel_mask(_p(norms), rs, cin, cout, _p(mask), _stream()), 'pf_cpg_channel_mask')
    return norms


def mul(a, b, out):
    _check_f32(a, b, out)
    _lib.check(_lib.load().pf_mul(_p(a), _p(b), a.numel(), _p(out), _stream()), 'pf_mul')


# ----------------------------------------------------------------------------- f5 remastered channel selection (pf_cpr.cu)
def cpr_sample(d, x, y, rows, X, Y, planes=None, bias=None):
    """Gather pruned-model input patches into rows of X [*, R*S*Cin] (HWIO order) and conv outputs into rows of Y
    [*, Cout] (channel_pruning_rmt/learner.py:679-703).  rows: int32 CUDA tensor [n, 4] = (n, oh, ow, dst row; < 0
    skips the row).  The input is `x` (fp32 NHWC) or, when x is None, hi + lo of `planes` (an ops.Planes).  `bias`:
    subtracted from the output (a conv whose bias is fused into its epilogue)."""
    _check_f32(x, y, X, Y, bias)
    if rows.dtype != torch.int32 or not rows.is_cuda or not rows.is_contiguous() or rows.dim() != 2 or rows.shape[1] != 4:
        raise ValueError('cpr_sample: rows must be a contiguous int32 CUDA tensor [n, 4]')
    _lib.check(_lib.load().pf_cpr_sample(ctypes.byref(d), _p(x), _p(planes.hi) if planes is not None else None,
                                         _p(planes.lo) if planes is not None else None, _p(y), _p(bias), _p(rows),
                                         rows.shape[0], _p(X), _p(Y), _stream()), 'pf_cpr_sample')


def cpr_gram_ws_doubles(cin, cout, chunk_rows):
    return int(_lib.load().pf_cpr_gram_ws_doubles(int(cin), int(cout), int(chunk_rows)))


def cpr_gram_chunk_rows(cin, cout, n_idx, budget_bytes=1 << 30):
    """rows of X per chunk of the float64 feature matrix so that it stays within `budget_bytes`"""
    return int(max(1, min(n_idx, budget_bytes // (8 * (cin + 1) * cout))))


def cpr_gram(X, Y, idx, w, g, gf, bf, ws=None, chunk_rows=None):
    """G = F^T F, b = F^T y over the rows idx of X / Y, normalised by ||G||_F (channel_pruning_rmt/learner.py:751-769).
    g: float64 [(Cin+1)^2 + 1] (G | b columns, then the norm); gf / bf: float32 G [Cin, Cin] / b [Cin]."""
    rs, cin, cout = _rs_cin_cout(w)
    _check_f32(X, Y, w, gf, bf)
    if idx.dtype != torch.int32 or g.dtype != torch.float64 or g.numel() < (cin + 1) ** 2 + 1:
        raise ValueError('cpr_gram: idx must be int32 and g float64 [(Cin+1)^2 + 1]')
    if chunk_rows is None:
        chunk_rows = cpr_gram_chunk_rows(cin, cout, idx.numel())
    need = cpr_gram_ws_doubles(cin, cout, chunk_rows)
    if ws is None or ws.numel() < need:
        ws = torch.empty(need, dtype=torch.float64, device=X.device)
    _lib.check(_lib.load().pf_cpr_gram(_p(X), _p(Y), _p(idx), idx.numel(), _p(w), rs, cin, cout, _p(ws), int(chunk_rows),
                                       _p(g), _p(gf), _p(bf), _stream()), 'pf_cpr_gram')
    return ws


def cpr_ista(gf, bf, m0, lr, gamma, iters, m, ws, nnz):
    """iters ISTA steps at one gamma in one launch (channel_pruning_rmt/learner.py:449-452, :780-781); m = result,
    nnz (int32 [1]) = its count of non-zeros; ws: 2*Cin floats.  gamma / lr are rounded to float32 as the LASSO graph's
    placeholder / constant are."""
    _check_f32(gf, bf, m0, m, ws)
    cin = m0.numel()
    if gf.numel() != cin * cin or bf.numel() != cin or m.numel() != cin or ws.numel() < 2 * cin or nnz.dtype != torch.int32:
        raise ValueError('cpr_ista: shape mismatch')
    _lib.check(_lib.load().pf_cpr_ista(_p(gf), _p(bf), _p(m0), cin, float(np.float32(lr)), float(np.float32(gamma)),
                                       int(iters), _p(m), _p(ws), _p(nnz), _stream()), 'pf_cpr_ista')


def cpr_mask_channels(a, m, rs, cin, inner):
    """a[row, t, c, k] *= (|m[c]| > 0), a viewed as [rows, rs, cin, inner] (channel_pruning_rmt/learner.py:817-820)"""
    _check_f32(a, m)
    per = rs * cin * inner
    if a.numel() % per or m.numel() != cin:
        raise ValueError('cpr_mask_channels: shape mismatch')
    _lib.check(_lib.load().pf_cpr_mask_channels(_p(a), a.numel() // per, rs, cin, inner, _p(m), _stream()),
               'pf_cpr_mask_channels')



# ----------------------------------------------------------------------------- f5b LASSO channel selection (pf_cpr.cu)
def _check_f64(*ts):
    for t in ts:
        if t is not None and (t.dtype != torch.float64 or not t.is_cuda or not t.is_contiguous()):
            raise ValueError('expected a contiguous float64 CUDA tensor')


def cp_sample(d, x, y, rows, X, Y, planes=None, bias=None, res_full=None, res_cur=None):
    """Gather input patches into rows of X [*, R*S*Cin] (fp32) and conv outputs into rows of Y [*, Cout] (float64)
    (channel_pruner.py:263-341, :391-412).  rows: int32 CUDA tensor [n, 8] = (n, oh, ow, dst row (< 0 skips it), rh,
    rw, 0, 0).  The input is `x` (fp32 NHWC) or, when x is None, hi + lo of `planes`; `bias` is subtracted from the
    output; res_full / res_cur [N, H', W', Cout]: Y += res_full - res_cur at (n, rh, rw), in float64 (:579-586)."""
    _check_f32(x, y, X, bias, res_full, res_cur)
    _check_f64(Y)
    if rows.dtype != torch.int32 or not rows.is_cuda or not rows.is_contiguous() or rows.dim() != 2 or rows.shape[1] != 8:
        raise ValueError('cp_sample: rows must be a contiguous int32 CUDA tensor [n, 8]')
    rh, rw = (res_full.shape[1], res_full.shape[2]) if res_full is not None else (0, 0)
    if res_full is not None and (res_cur is None or res_cur.shape != res_full.shape or res_full.shape[0] != d.n
                                 or res_full.shape[3] != d.k):
        raise ValueError('cp_sample: the residual tensors must both be [N, H, W, Cout]')
    _lib.check(_lib.load().pf_cp_sample(ctypes.byref(d), _p(x), _p(planes.hi) if planes is not None else None,
                                        _p(planes.lo) if planes is not None else None, _p(y), _p(bias), _p(res_full),
                                        _p(res_cur), rh, rw, _p(rows), rows.shape[0], _p(X), _p(Y), _stream()),
               'pf_cp_sample')


def cp_gram(X, Y, idx, w, g, ws=None, chunk_rows=None, budget_bytes=1 << 30):
    """G_aug = [P | y]^T [P | y] in float64 over the rows idx of X / Y, P[(j, o), c] = sum_t X[idx j, t, c] W[t, c, o]
    (channel_pruner.py:468-476).  g: float64 [(Cin+1)^2 + 1]: G = g[:Cin, :Cin], P^T y = g[:Cin, Cin]."""
    rs, cin, cout = _rs_cin_cout(w)
    _check_f32(X, w)
    _check_f64(Y, g)
    if idx.dtype != torch.int32 or g.numel() < (cin + 1) ** 2 + 1:
        raise ValueError('cp_gram: idx must be int32 and g float64 [(Cin+1)^2 + 1]')
    if chunk_rows is None:
        chunk_rows = cpr_gram_chunk_rows(cin, cout, idx.numel(), budget_bytes)
    need = (cin + 1) * int(chunk_rows) * cout
    if ws is None or ws.numel() < need:
        ws = torch.empty(need, dtype=torch.float64, device=X.device)
    _lib.check(_lib.load().pf_cp_gram(_p(X), _p(Y), _p(idx), idx.numel(), _p(w), rs, cin, cout, _p(ws), int(chunk_rows),
                                      _p(g), _stream()), 'pf_cp_gram')
    return ws


def cp_normal_eq(X, Y, cols, g, ws=None, chunk_rows=None, budget_bytes=1 << 30):
    """[X_k | Y]^T [X_k | Y] in float64 over every row, X_k = the columns `cols` (int32) of X [N, K] (fp32), Y [N, Cout]
    (float64): A = g[:k, :k], B = g[:k, k:] are the normal equations of the refit (channel_pruner.py:569-573)."""
    _check_f32(X)
    _check_f64(Y, g)
    nrows, K = X.shape
    cout = Y.shape[1]
    ncols = cols.numel()
    n = ncols + cout
    if cols.dtype != torch.int32 or Y.shape[0] != nrows or g.numel() < n * n + 1:
        raise ValueError('cp_normal_eq: cols must be int32, Y [N, Cout] and g float64 [(k + Cout)^2 + 1]')
    if chunk_rows is None:
        chunk_rows = int(max(1, min(nrows, budget_bytes // (8 * n))))
    need = n * int(chunk_rows)
    if ws is None or ws.numel() < need:
        ws = torch.empty(need, dtype=torch.float64, device=X.device)
    _lib.check(_lib.load().pf_cp_normal_eq(_p(X), _p(Y), int(nrows), int(K), int(cout), _p(cols), int(ncols), _p(ws),
                                           int(chunk_rows), _p(g), _stream()), 'pf_cp_normal_eq')
    return ws


class CprLstsq:
    """The least-squares refit of one layer (channel_pruning_rmt/learner.py:470-523, :814-842): min_W ||X W - Y||^2 /
    (2N) + wd ||W||^2 / 2 by `iters` Adam steps from the current kernel.  X W is a 1x1 conv over N "pixels" of
    K = R*S*Cin channels and X^T (X W - Y) is its weight gradient, so the conv kernels do the GEMMs: tensor-core
    (split-bf16) where `conv_path` is 'tc' and the pass's shape rule holds (fwd: K, Cout multiples of 16; wgrad: also
    Cout a multiple of 64), exact fp32 otherwise.  The update is pf_adam_step with
    hp = (lr, beta1^t, beta2^t), the powers as float32 pow as tf.pow(beta, train_step) (:504-505).  Deviation: its
    moment update is TF's m += (g - m)(1 - beta1) instead of the reference's beta1 m + (1 - beta1) g (:499-500) —
    equal up to rounding."""

    def __init__(self, X, Y, conv_path='tc'):
        n, k = X.shape
        cout = Y.shape[1]
        self.X, self.Y, self.n = X, Y, n
        self.d = conv_desc(n, 1, 1, k, cout, 1, 1, 1, 1, 1, 1, 0, 0)
        self.tc_fwd = conv_path == 'tc' and conv2d_tc_supported(self.d)
        self.tc_wgrad = conv_path == 'tc' and conv2d_tc_wgrad_supported(self.d)
        dev = X.device
        self.P = torch.empty(n, cout, dtype=torch.float32, device=dev)
        self.R = torch.empty(n, cout, dtype=torch.float32, device=dev)
        self.g = torch.empty(k * cout, dtype=torch.float32, device=dev)
        self.loss = torch.zeros(1, dtype=torch.float32, device=dev)
        self.l2ws = torch.empty(L2_PARTIALS, dtype=torch.float32, device=dev)
        self.tw = TcWeights(self.d, dev, need_dgrad=False) if self.tc_fwd else None
        ws = conv2d_tc_wgrad_workspace_floats(self.d) if self.tc_wgrad else conv2d_wgrad_workspace_floats(self.d)
        self.ws = torch.empty(max(ws, 4), dtype=torch.float32, device=dev)

    def residual(self, w):
        """R = X W - Y; returns loss = ||R||^2 / 2 (device [1])"""
        if self.tc_fwd:
            self.tw.prepare(w)
            conv2d_tc_fwd(self.d, self.X, self.tw, None, False, self.P)
        else:
            conv2d_fwd(self.d, self.X, w, None, False, self.P)
        cpg_diff_l2(self.P, self.Y, self.R, self.loss, self.l2ws)
        return self.loss

    def run(self, w, iters, lr, wd, beta1=0.9, beta2=0.999, eps=1e-8):
        """w: [R, S, Cin, Cout] fp32 (updated in place).  Returns (loss before, loss after) / N: the reference's loss_reg."""
        m, v = torch.zeros_like(w), torch.zeros_like(w)
        b1, b2 = np.float32(beta1), np.float32(beta2)
        t = np.arange(1, iters + 1, dtype=np.float32)
        hp = np.zeros((max(iters, 1), 4), dtype=np.float32)
        hp[:iters, 0] = np.float32(lr)
        hp[:iters, 1] = np.power(b1, t)
        hp[:iters, 2] = np.power(b2, t)
        hp = torch.from_numpy(hp).to(w.device)
        inv_n = float(np.float32(1.0) / np.float32(self.n))
        first = float(self.residual(w).item()) / self.n
        for i in range(iters):
            if i:
                self.residual(w)
            if self.tc_wgrad:
                conv2d_tc_wgrad(self.d, self.X, self.R, self.ws, self.g)
            else:
                conv2d_wgrad(self.d, self.X, self.R, self.ws, self.g)
            adam_step(w.reshape(-1), m.reshape(-1), v.reshape(-1), self.g, hp[i], beta1, beta2, eps, wd=wd,
                      grad_scale=inv_n)
        last = float(self.residual(w).item()) / self.n
        return first, last
