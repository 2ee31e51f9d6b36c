"""CPU oracle of the bucketed codebook quantizer — NonUniformQuantization.__bucket_quantize
(learners/nonuniform_quantization/utils.py:196-243 with __split_bucket / __channel_bucket :435-476, __scale /
__inv_scale :388-433, __quantile_init :349-366, __build_bucket_norm_quant_point :309-347, __updt_bucket_storage
:487-494).

TEST INFRASTRUCTURE ONLY, like pf_oracle.py, and a module of its own so that the per-layer restatement there stays as
it is.  The numpy functions restate the reference's op chain in its op order in float32; they are pinned bit for bit
against the reference's own code executed on numpy-backed tensors (tests/golden/make_golden_nuq_buckets.py).  The
torch function is the same forward with the reference's STE overrides, for StepOracle-style autograd.
"""
import numpy as np
import torch

from . import pf_oracle as O
from .step_oracle import StepOracle, codebook_quant

F32 = np.float32


def bucket_view(x, bucket_type, bucket_size):
    """[rows, nb] view, nb, padded count: __split_bucket (pad with copies of the last element, reshape
    [bucket_size, -1]) or __channel_bucket (reshape [-1, cout])."""
    if bucket_type == 'split':
        if bucket_size <= 0:
            raise ValueError('split buckets need a positive bucket size')
        return O.split_bucket(x, bucket_size)
    if bucket_type == 'channel':
        return O.channel_bucket(np.asarray(x, F32))
    raise ValueError("Unrecognized bucket type, must be 'weight' or 'channel'.")


def bucket_quantile_init(x_normalized, nb_clusters):
    """__quantile_init with axis=0: [nb_clusters, nb], centroid j of bucket b = percentile(x_n[:, b],
    (j+1)*100/(k+1)), 'nearest' (padding rows included)."""
    return O.nuq_quantile_init(x_normalized, nb_clusters, axis=0)


def bucket_assign(x_normalized, clusters):
    """__build_bucket_norm_quant_point: idx = argmin over axis 1 of |tile(x_n)^T - c| ([rows, k, nb]; first index on
    ties), q = c[idx, b] * sign(x_n + 1e-6)."""
    xn = np.asarray(x_normalized, F32)
    c = np.asarray(clusters, F32)
    d = np.abs((xn[:, None, :] - c[None, :, :]).astype(F32))
    idx = np.argmin(d, axis=1)
    q = (np.take_along_axis(c, idx, axis=0) * np.sign((xn + F32(1e-6)).astype(F32))).astype(F32)
    return q, idx


def nonuniform_quantize_buckets(x, bits, bucket_type, bucket_size=256, clusters=None):
    """__bucket_quantize, 'weight' mode.  Returns (qx with x's shape, clusters [2^bits, nb], idx of the real elements in
    flat order, alpha [nb], beta [nb]).  clusters: a given codebook matrix (only its first 2^bits rows are used)."""
    x = np.ascontiguousarray(x, dtype=F32)
    xb, nb, padded = bucket_view(x, bucket_type, bucket_size)
    xn, alpha, beta = O.uq_scale(xb, 0)
    k = int(2 ** bits)
    if clusters is None:
        clusters = bucket_quantile_init(xn, k)
    c = np.asarray(clusters, F32)[:k]
    q, idx = bucket_assign(xn, c)
    qw = O.uq_inv_scale(q, alpha, beta).reshape(-1)
    n = x.size
    return qw[:n].reshape(x.shape), c, idx.reshape(-1)[:n], alpha, beta


def bucket_nuq_grads(g, idx, nb_clusters, alpha):
    """Codebook gradient: dL/dc[j, b] = alpha_b * sum_{i in b, real, idx_i = j} g_i (float64 sums), [k, nb].  Element i
    of the flat tensor lies in bucket i % nb."""
    g = np.asarray(g, F32).reshape(-1)
    idx = np.asarray(idx).reshape(-1)
    nb = np.asarray(alpha).size
    col = np.arange(g.size) % nb
    gc = np.zeros((nb_clusters, nb), np.float64)
    np.add.at(gc, (idx, col), g.astype(np.float64))
    return (gc * np.asarray(alpha, np.float64)[None, :]).astype(F32)


def bucket_storage_bits(shapes, bucket_type, bucket_size):
    """sum of nb * 64 over the quantized kernels (alpha and beta of every bucket)."""
    tot = 0
    for s in shapes:
        _, nb, _ = bucket_view(np.zeros(s, F32), bucket_type, bucket_size)
        tot += O.bucket_storage_bits(nb)
    return tot


def codebook_quant_buckets(w, clusters, bits, bucket_type, bucket_size):
    """torch forward of __bucket_quantize with the overrides of the per-layer codebook_quant: min/max under
    stop_gradient, Mul -> Add and Sign -> Identity, so the upstream gradient reaches both the gathered centroids (a
    segment sum per bucket) and x_n.  Padding copies are sliced off: they get no gradient."""
    shape, n = w.shape, w.numel()
    if bucket_type == 'channel':
        xb = w.reshape(-1, shape[-1])
    else:
        flat = w.reshape(-1)
        rest = n % bucket_size
        if rest:
            flat = torch.cat([flat, torch.ones(bucket_size - rest) * flat[-1]])
        xb = flat.reshape(bucket_size, -1)
    with torch.no_grad():
        w_max, w_min = xb.max(dim=0).values, xb.min(dim=0).values
    alpha = w_max - w_min + torch.tensor(1e-10)
    beta = w_min
    xn = (xb - beta) / alpha
    c = clusters if torch.is_tensor(clusters) else torch.as_tensor(np.asarray(clusters, F32))
    c = c[:2 ** int(bits)]
    with torch.no_grad():
        idx = torch.argmin(torch.abs(xn.unsqueeze(1) - c.unsqueeze(0)), dim=1)
        sgn = torch.sign(xn + 1e-6)
    q = torch.gather(c, 0, idx) * sgn + (xn - xn.detach())
    return (alpha * q + beta).reshape(-1)[:n].reshape(shape)


class BucketStepOracle(StepOracle):
    """StepOracle whose codebook-quantized kernels (conv, dense and depthwise alike) go through
    codebook_quant_buckets — weight_quant['use_buckets'] set — or, without buckets, through the per-layer
    codebook_quant also for depthwise kernels (as the device quantizes them).  Codebooks: the op's `clusters` variable,
    else self.clusters[op name]."""

    def forward(self, params, images, training=True, stats_out=None, force=None, local_out=None):
        if self.wq.get('kind', 'uniform') == 'uniform':
            return StepOracle.forward(self, params, images, training, stats_out, force, local_out)
        p = dict(params)
        for op in self.wq.get('ops', []):
            name = op.vars['kernel'].name
            cv = op.vars.get('clusters')
            c = params[cv.name] if cv is not None and cv.name in params else self.clusters[op.name]
            bits = self.wq_bits[op.name]
            if self.wq.get('use_buckets', False):
                p[name] = codebook_quant_buckets(params[name], c, bits, self.wq.get('bucket_type', 'split'),
                                                 self.wq.get('bucket_size', 256))
            else:
                p[name] = codebook_quant(params[name], c if torch.is_tensor(c) else
                                         torch.as_tensor(np.asarray(c, F32)[:2 ** bits]))
        saved = self.wq_bits
        self.wq_bits = {}
        try:
            return StepOracle.forward(self, p, images, training, stats_out, force, local_out)
        finally:
            self.wq_bits = saved
