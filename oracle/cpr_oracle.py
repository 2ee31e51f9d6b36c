"""CPU oracle of the remastered channel-pruning learner's channel selection
(/root/reference/learners/channel_pruning_rmt/learner.py:432-523, 546-842).

TEST INFRASTRUCTURE ONLY, like pf_oracle.py: tests/ and the measurement tool import it, pocketflow_b200 never does.
Each function restates one piece of the reference in its op order and precision: the sampling and the regression
matrices in numpy float64 (the reference's np.zeros buffers), ISTA and the least-squares refit in float32 (its TF
graphs).  Random draws come from a caller-supplied np.random.RandomState, in the reference's order.
All citations are file:line into the reference's learners/channel_pruning_rmt/learner.py.
"""
import math

import numpy as np

F32 = np.float32

FLAG_DEFAULTS = dict(cpr_save_path='./models_cpr/model.ckpt', cpr_save_path_eval='./models_cpr_eval/model.ckpt',
                     cpr_save_path_ws='./models_cpr_ws/model.ckpt', cpr_prune_ratio=0.5, cpr_skip_frst_layer=True,
                     cpr_skip_last_layer=False, cpr_skip_op_names=None, cpr_nb_smpls=5000, cpr_nb_crops_per_smpl=10,
                     cpr_ista_lrn_rate=1e-2, cpr_ista_nb_iters=100, cpr_lstsq_lrn_rate=1e-3, cpr_lstsq_nb_iters=100,
                     cpr_warm_start=False)                                                          # (:33-52)


def cpr_prune_ratios(kernel_names, prune_ratio, skip_frst_layer=True, skip_last_layer=False, skip_op_names=None):
    """Per-layer ratios of __choose_channels (:549-567).  A ratio of 0 does not skip the layer."""
    ratios = [prune_ratio] * len(kernel_names)
    if skip_frst_layer:
        ratios[0] = 0.0
    if skip_last_layer:
        ratios[-1] = 0.0
    skip_names = skip_op_names.split(',') if skip_op_names is not None else []
    for i, name in enumerate(kernel_names):
        if any(s in name for s in skip_names):
            ratios[i] = 0.0
    return ratios


def cpr_pads(ih, iw, kh, kw, sh, sw, padding):
    """(top, left) leading pads of __smpl_inputs_n_outputs (:665-672)"""
    if padding == 'VALID':
        return 0, 0
    ph = max(kh - (sh if ih % sh == 0 else ih % sh), 0)
    pw = max(kw - (sw if iw % sw == 0 else iw % sw), 0)
    return ph // 2, pw // 2


def cpr_sample(rng, krnl_full, krnl_prnd, inputs_full, inputs_prnd, outputs_full, outputs_prnd, strides, padding,
               nb_crops, pads=None):
    """__smpl_inputs_n_outputs (:651-725), float64 like the reference's np.zeros buffers.
    Returns (X [bs*nb_crops, kh*kw*ic]: pruned patches in HWIO order, the layout of :819-820; Y [bs*nb_crops, oc]: full
    outputs; [(oh, ow)] drawn; (err_full, err_prnd) of :715-723).  Rows are crop-major.  `pads` overrides the SAME
    formula (the explicit padding of ResNet's strided convs)."""
    bs = inputs_full.shape[0]
    kh, kw = krnl_full.shape[0], krnl_full.shape[1]
    ih, iw, ic = inputs_full.shape[1], inputs_full.shape[2], inputs_full.shape[3]
    oh, ow, oc = outputs_full.shape[1], outputs_full.shape[2], outputs_full.shape[3]
    sh, sw = strides
    pt, pl = pads if pads is not None else cpr_pads(ih, iw, kh, kw, sh, sw, padding)
    xs_f, xs_p, ys_f, ys_p, pos = [], [], [], [], []
    for _ in range(nb_crops):
        idx_oh = rng.randint(oh)
        idx_ow = rng.randint(ow)
        pos.append((idx_oh, idx_ow))
        ih_lo, iw_lo = idx_oh * sh - pt, idx_ow * sw - pl
        ih_hi, iw_hi = ih_lo + kh, iw_lo + kw
        sh_lo, sh_hi = max(-ih_lo, 0), kh - max(ih_hi - ih, 0)
        sw_lo, sw_hi = max(-iw_lo, 0), kw - max(iw_hi - iw, 0)
        ih_lo, ih_hi, iw_lo, iw_hi = max(ih_lo, 0), min(ih_hi, ih), max(iw_lo, 0), min(iw_hi, iw)
        f, p = np.zeros((bs, kh, kw, ic)), np.zeros((bs, kh, kw, ic))
        f[:, sh_lo:sh_hi, sw_lo:sw_hi, :] = inputs_full[:, ih_lo:ih_hi, iw_lo:iw_hi, :]
        p[:, sh_lo:sh_hi, sw_lo:sw_hi, :] = inputs_prnd[:, ih_lo:ih_hi, iw_lo:iw_hi, :]
        xs_f.append(f)
        xs_p.append(p)
        ys_f.append(np.reshape(outputs_full[:, idx_oh, idx_ow, :], [bs, -1]))
        ys_p.append(np.reshape(outputs_prnd[:, idx_oh, idx_ow, :], [bs, -1]))
    x_f, x_p = np.concatenate(xs_f, axis=0), np.concatenate(xs_p, axis=0)
    y_f, y_p = np.vstack(ys_f), np.vstack(ys_p)
    err_f = float(np.sum((y_f - x_f.reshape(len(x_f), -1) @ np.reshape(krnl_full, [-1, oc])) ** 2) / y_f.size)
    err_p = float(np.sum((y_p - x_p.reshape(len(x_p), -1) @ np.reshape(krnl_prnd, [-1, oc])) ** 2) / y_p.size)
    return x_p.reshape(len(x_p), -1), y_f, pos, (err_f, err_p)


def cpr_gram(X, Y, w, idxs):
    """Feature matrix, response vector, <F^T F> and <F^T y> normalised by ||F^T F||_F (:751-769), float64.
    X: [N, kh*kw*ic] patches (HWIO order), Y: [N, oc], w: [kh, kw, ic, oc], idxs: the secondary sample's rows.
    Returns (G [ic, ic], b [ic, 1], ||F^T F||_F)."""
    kh, kw, ic, oc = w.shape
    x = np.asarray(X, np.float64).reshape(len(X), kh * kw, ic)[idxs]
    feat = np.zeros((ic, len(idxs) * oc))
    for c in range(ic):
        feat[c] = np.matmul(x[:, :, c], np.reshape(w[:, :, c, :], [kh * kw, oc]).astype(np.float64)).ravel()
    feat = feat.T
    rspn = np.reshape(np.asarray(Y, np.float64)[idxs], [-1, 1])
    g = feat.T @ feat
    b = feat.T @ rspn
    nrm = np.sqrt(np.sum(g * g))
    return g / nrm, b / nrm, nrm


def cpr_ista(g, b, m0, gamma, lr, nb_iters):
    """The meta-LASSO graph (:432-468) run nb_iters times at one gamma (:780-781), float32: the float64 G / b / m0 are fed
    to float32 placeholders; m <- prox(m - lr (G m - b), gamma lr).  Returns (mask [ic, 1], nnz).  The order of TF's
    matmul sum is not pinned: device results are compared with a tolerance."""
    g, b, m = np.asarray(g, F32), np.asarray(b, F32).reshape(-1, 1), np.asarray(m0, F32).reshape(-1, 1)
    lr, thr = F32(lr), F32(F32(gamma) * F32(lr))
    for _ in range(nb_iters):
        x = (m - lr * (np.matmul(g, m).astype(F32) - b)).astype(F32)
        m = np.where(x > thr, x - thr, np.where(x < -thr, x + thr, np.zeros_like(x))).astype(F32)
    return m, int(np.count_nonzero(m))


def cpr_gamma_search(solve, nnz_target):
    """The γ search of __solve_sparse_regression (:787-812): double ubnd from 0.1 until nnz <= target, then bisect
    while nnz != target and ubnd - lbnd > 1e-8.  solve(gamma) -> (mask, nnz).  Returns (mask, [(gamma, nnz)])."""
    log = []
    ubnd = 0.1
    while True:
        mask, nnz = solve(ubnd)
        log.append((ubnd, nnz))
        if nnz <= nnz_target:
            break
        ubnd *= 2.0
    lbnd = 0.0
    while nnz != nnz_target and ubnd - lbnd > 1e-8:
        val = (lbnd + ubnd) / 2.0
        mask, nnz = solve(val)
        log.append((val, nnz))
        if nnz < nnz_target:
            ubnd = val
        elif nnz > nnz_target:
            lbnd = val
        else:
            break
    return mask, log


def cpr_lstsq(X, Y, w, bnry, lr, nb_iters, wd, beta1=0.9, beta2=0.999, eps=1e-8):
    """The meta least-square graph (:470-523) run nb_iters times (:834-835) in float32 with the reference's own Adam:
    X = patches with the dropped channels zeroed (:817-820), grad = X^T (X W - Y) / N + wd W, moments
    beta m + (1 - beta) g (:499-500), step lr sqrt(1 - b2^t) / (1 - b1^t) * m / (sqrt(v) + eps) (:504-506); then
    W * bnry (:839).  Returns the new kernel [kh, kw, ic, oc]."""
    kh, kw, ic, oc = w.shape
    n = len(X)
    x = (np.asarray(X, F32).reshape(n, kh * kw, ic) * np.asarray(bnry, F32).reshape(1, 1, -1)).reshape(n, -1).astype(F32)
    y = np.asarray(Y, F32)
    wm = np.asarray(w, F32).reshape(-1, oc).copy()
    m, v = np.zeros_like(wm), np.zeros_like(wm)
    b1, b2, nf = F32(beta1), F32(beta2), F32(n)
    for t in range(1, nb_iters + 1):
        grad = ((x.T @ (x @ wm - y)).astype(F32) / nf + F32(wd) * wm).astype(F32)
        m = (b1 * m + (F32(1) - b1) * grad).astype(F32)
        v = (b2 * v + (F32(1) - b2) * grad ** 2).astype(F32)
        step = F32(F32(lr) * np.sqrt(F32(1) - np.power(b2, F32(t))) / (F32(1) - np.power(b1, F32(t))))
        wm = (wm - step * m / (np.sqrt(v) + F32(eps))).astype(F32)
    return (wm.reshape(w.shape) * np.asarray(bnry, F32).reshape(1, 1, -1, 1)).astype(F32)


def cpr_secondary_rows(bs, oc):
    """N' = ceil(min(N, N / Cout * 10)) (:751)"""
    return int(math.ceil(min(bs, bs / oc * 10.0)))


def cpr_solve_sparse_regression(rng, X, Y, w, prune_ratio, ista_lr=1e-2, ista_iters=100, lstsq_lr=1e-3,
                                lstsq_iters=100, wd=0.0):
    """__solve_sparse_regression (:727-842) with the draws from `rng` in the reference's order (choice, then uniform).
    Returns (new kernel, [(gamma, nnz)], mask)."""
    kh, kw, ic, oc = w.shape
    bs = len(Y)
    target = int(ic * (1.0 - prune_ratio))
    idxs = rng.choice(bs, size=(cpr_secondary_rows(bs, oc)), replace=False)
    g, b, _ = cpr_gram(X, Y, w, idxs)
    m0 = rng.uniform(size=(ic, 1))
    mask, log = cpr_gamma_search(lambda x: cpr_ista(g, b, m0, x, ista_lr, ista_iters), target)
    bnry = (np.abs(mask) > 0.0).astype(F32)
    return cpr_lstsq(X, Y, w, bnry, lstsq_lr, lstsq_iters, wd), log, mask
