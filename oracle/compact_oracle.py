"""Float64 restatement of fine-tuning a channel-pruned model at its pruned width (pocketflow_b200/compact.py).

The argument that the compact training step is sound, on the smallest net that has every ingredient: a producer layer
W1 whose output only partly survives, a channel gather, and a consumer layer W2 whose pruned input channels are zero,
masked rows:
    h = relu(x W1)        [n, c]           full width
    y = h W2              W2 [c, k], rows outside `keep` are zero and masked
    L = 0.5 sum (y - t)^2
Compact: W1c = W1[:, lay1] (the live columns, padded with zero columns), hc = relu(x W1c), W2c = W2[lay2] (rows in the
order of lay2 = positions in lay1's layout, -1 padding), y = gather(hc, idx) W2c.  In exact arithmetic the two steps give
the same logits, the same gradient on every kept entry and, after one masked Momentum step (pf_oracle.momentum_step's
formula), the same kept weights and slots; a dead column of W1 has gradient 0 in the masked model, so it only decays.
"""
import numpy as np


def gather(x, idx):
    """y[:, j] = x[:, idx[j]], 0 where idx[j] < 0 (pf_gather_channels)"""
    idx = np.asarray(idx)
    return np.where(idx >= 0, x[:, np.maximum(idx, 0)], 0.0)


def scatter(dy, idx, cin):
    """backward of gather: dx[:, idx[j]] = dy[:, j] for idx[j] >= 0, zeros elsewhere (pf_scatter_channels)"""
    idx = np.asarray(idx)
    dx = np.zeros((dy.shape[0], cin))
    dx[:, idx[idx >= 0]] = dy[:, idx >= 0]
    return dx


def momentum_step(w, acc, g, mask, lr, momentum, wd):
    """g_tot = (g + wd w) mask; acc = momentum acc + g_tot; w = w - lr acc (pf_momentum_step)"""
    acc = momentum * acc + (g + wd * w) * mask
    return w - lr * acc, acc


def two_layer_grads(x, w1, w2, t, idx=None):
    """(y, dW1, dW2) of the net above; idx: the gather between the layers (None: full width)"""
    a = x @ w1
    h = np.maximum(a, 0.0)
    hg = h if idx is None else gather(h, idx)
    y = hg @ w2
    dy = y - t
    dw2 = hg.T @ dy
    dhg = dy @ w2.T
    dh = dhg if idx is None else scatter(dhg, idx, h.shape[1])
    dw1 = x.T @ (dh * (a > 0))
    return y, dw1, dw2
