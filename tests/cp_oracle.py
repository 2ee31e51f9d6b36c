"""float64 numpy restatement of one layer of the LASSO channel-pruning learner's selection
(/root/reference/learners/channel_pruning/channel_pruner.py), for the tests: sampling, design matrix, residual
difference, selection, refit, W1 / W2 masks.  The LASSO itself is the package's LarsLassoPath, which the CPU tests check
against sklearn's LassoLars."""
import numpy as np

from pocketflow_b200.learners.channel_pruning import lars


def extract_patches(x, kh, kw, stride, pads, p, q):
    """tf.extract_image_patches on NHWC x with explicit leading pads: [N, P, Q, kh*kw*C] (h, w, c order)"""
    n, h, w, c = x.shape
    xp = np.zeros((n, h + kh + p * stride[0], w + kw + q * stride[1], c), x.dtype)
    xp[:, pads[0]:pads[0] + h, pads[1]:pads[1] + w, :] = x
    out = np.empty((n, p, q, kh * kw * c), x.dtype)
    for i in range(p):
        for j in range(q):
            out[:, i, j, :] = xp[:, i * stride[0]:i * stride[0] + kh, j * stride[1]:j * stride[1] + kw, :].reshape(n, -1)
    return out


def sample(x, y, pos, kh, kw, stride, pads, add_full=None, add_cur=None, pos_add=None):
    """one batch's rows (:317-337, :403-412, :579-586): X [bs * k, kh*kw*C], Y [bs * k, Cout] in float64"""
    xs, ys = pos
    patches = extract_patches(x, kh, kw, stride, pads, y.shape[1], y.shape[2])
    X = patches[:, xs, ys, :].reshape(-1, patches.shape[-1]).astype(np.float64)
    Y = y[:, xs, ys, :].reshape(-1, y.shape[-1]).astype(np.float64)
    if add_full is not None:
        xa, ya = pos_add
        Y = Y + (add_full[:, xa, ya, :].reshape(Y.shape).astype(np.float64)
                 - add_cur[:, xa, ya, :].reshape(Y.shape).astype(np.float64))
    return X, Y


def design_matrix(X, W2, Y, samples):
    """compute_pruned_kernel's product and reshape_Y (:468-476); X [N, kh*kw*C] in (h, w, c) order"""
    kh, kw, c_in, c_out = W2.shape
    nb = X.shape[0]
    X4 = X.reshape(nb, kh, kw, c_in)
    reshape_X = np.rollaxis(np.transpose(X4, (0, 3, 1, 2)).reshape((nb, c_in, -1))[samples], 1, 0)
    reshape_W2 = np.transpose(np.transpose(W2, (3, 2, 0, 1)).reshape((c_out, c_in, -1)), [1, 2, 0])
    product = np.matmul(reshape_X, reshape_W2.astype(np.float64)).reshape((c_in, -1)).T
    return product, Y[samples].reshape(-1)


def refit(X, Y, idxs, kh, kw):
    """featuremap_reconstruction (:442-454, :571-573): min-norm lstsq of Y on the kept columns; [kh, kw, k, Cout]"""
    nb = X.shape[0]
    c_in = X.shape[1] // (kh * kw)
    Xk = X.reshape(nb, kh, kw, c_in)[:, :, :, idxs].reshape(nb, -1)
    coef = np.linalg.lstsq(Xk, Y, rcond=None)[0]
    return coef.reshape(kh, kw, int(np.sum(idxs)), Y.shape[1])


def select_layer(X, Y, W2, c_new, samples, lasso=True, quadruple=False):
    """prune_kernel (:588-640): (kept mask, new W2 [kh, kw, Cin, Cout] with the dropped channels zero, solve log)"""
    kh, kw, c_in, c_out = W2.shape
    log = []
    if lasso:
        P, y = design_matrix(X, W2, Y, samples)
        path = lars.LarsLassoPath(P.T.dot(P), P.T.dot(y), P.shape[0])
        idxs, log = lars.select_channels(path.coef_at, c_in, c_new, quadruple=quadruple)
    else:
        idxs = lars.l1_select(W2, c_new)
    w = np.zeros(W2.shape, np.float64)
    w[:, :, idxs, :] = refit(X, Y, idxs, kh, kw)
    return idxs, w, log


def prune_w1(W1, bias, idxs, depthwise=False):
    """prune_W1 (:665-699): the producer's dropped output channels (a depthwise producer's channels) and bias zeroed"""
    W1 = W1.copy()
    if depthwise:
        W1[:, :, ~idxs, :] = 0
    else:
        W1[:, :, :, ~idxs] = 0
    if bias is not None:
        bias = bias.copy()
        bias[~idxs] = 0
    return W1, bias
