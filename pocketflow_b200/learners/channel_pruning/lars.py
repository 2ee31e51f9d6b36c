"""The LASSO channel selection of the channel-pruning learner, on the Gram matrix, in float64, on the host.

The reference (/root/reference/learners/channel_pruning/channel_pruner.py:456-577) fits
sklearn's LassoLars(alpha, fit_intercept=False, max_iter=3000) on the design matrix P [S*Cout, Cin] and the flattened
outputs y, inside a bisection on alpha.  LassoLars minimises

    1 / (2 n) ||y - P b||^2 + alpha ||b||_1,     n = S * Cout,

by following the LARS-Lasso path (Efron, Hastie, Johnstone & Tibshirani, "Least Angle Regression", 2004) from
alpha = max|P^T y| / n down to the requested alpha.  Only G = P^T P and P^T y enter that path, so the learner forms them
on the GPU (pf_cp_gram) and follows the path here.  Cin is at most 2048: the path costs O(Cin^3) host flops at most.

The path is piecewise linear in alpha, and the reference's bisection solves the same problem at a dozen or more values
of alpha: `LarsLassoPath` therefore walks the path once, lazily, and answers every `coef(alpha)` from its breakpoints,
with the same end-of-path interpolation, tolerances and early stops as LassoLars.

No sklearn import: the GPU machines are not guaranteed to have it."""
import numpy as np
from scipy import linalg

EQ_TOL = float(np.finfo(np.float32).eps)          # equality_tolerance of the path's stop test
TINY32 = float(np.finfo(np.float32).tiny)         # keeps the step-length ratios finite
EPS = float(np.finfo(np.float64).eps)             # LassoLars' default eps: the smallest Cholesky pivot
DIGITS = int(np.finfo(np.float64).precision)      # corr_eq_dir is rounded to this many decimals
BIG = float(np.finfo(np.float64).max)


def _min_pos(x):
    pos = x[x > 0]
    return float(pos.min()) if pos.size else BIG


class LarsLassoPath(object):
    """The LARS-Lasso path of min 1/(2 n) ||y - P b||^2 + alpha ||b||_1 given G = P^T P and xy = P^T y."""

    def __init__(self, gram, xy, n_samples, max_iter=3000):
        self.G = np.array(gram, dtype=np.float64)
        self.xy = np.array(xy, dtype=np.float64).reshape(-1)
        self.n = float(n_samples)
        self.nf = self.xy.size
        self.max_iter = int(max_iter)
        self.cov = self.xy.copy()                     # P^T (y - P coef) of the inactive features
        self.inactive = np.ones(self.nf, dtype=bool)
        self.active = []                              # feature indices, in the order of L's rows
        self.sign = []
        self.L = np.zeros((0, 0))
        self.coef = np.zeros(self.nf)
        self.n_iter = 0
        self.drop = False
        self.done = False
        self.alphas, self.coefs = [], []              # breakpoints: alpha at the top of each step, coef there
        self.prev_alpha = None

    # ------------------------------------------------------------------ one step of the path
    def _top(self):
        """alpha at the current coef; returns False when the path ends here"""
        cand = np.where(self.inactive)[0]
        if cand.size:
            j = int(cand[np.argmax(np.abs(self.cov[cand]))])
            C_ = self.cov[j]
            C = abs(C_)
        else:
            j, C_, C = -1, 0.0, 0.0
        alpha = C / self.n
        self.alphas.append(alpha)
        self.coefs.append(self.coef.copy())
        return j, C_, C, alpha

    def _advance(self):
        """one LARS-Lasso step; sets self.done at the end of the path"""
        while True:
            j, C_, C, alpha = self._top()
            if alpha <= EQ_TOL:                       # below float32's eps every alpha_min has its breakpoint
                self.done = True
                return
            if self.n_iter >= self.max_iter or len(self.active) >= self.nf:
                self.done = True
                return
            if not self.drop:
                k = len(self.active)
                c = self.G[j, j]
                row = self.G[j, self.active] if k else np.zeros(0)
                if k:
                    row = linalg.solve_triangular(self.L, row, lower=True, check_finite=False)
                diag = max(np.sqrt(abs(c - np.dot(row, row))), EPS)
                if diag < 1e-7:                       # degenerate regressor: never again a candidate at this step
                    self.cov[j] = 0.0
                    self.alphas.pop()
                    self.coefs.pop()
                    continue
                L = np.zeros((k + 1, k + 1))
                L[:k, :k] = self.L
                L[k, :k] = row
                L[k, k] = diag
                self.L = L
                self.active.append(j)
                self.sign.append(float(np.sign(C_)))
                self.inactive[j] = False
            if self.n_iter > 0 and self.prev_alpha < alpha:
                self.done = True                      # alpha rose: the residues are too small to steer the path
                return
            break
        act = np.array(self.active)
        sgn = np.array(self.sign)
        ls = linalg.cho_solve((self.L, True), sgn, check_finite=False)
        if ls.size == 1 and ls[0] == 0:
            ls[...] = 1
            AA = 1.0
        else:
            AA = 1.0 / np.sqrt(np.sum(ls * sgn))
            if not np.isfinite(AA):
                i = 0
                L_ = self.L.copy()
                while not np.isfinite(AA):
                    L_.flat[::len(act) + 1] += (2 ** i) * EPS
                    ls = linalg.cho_solve((L_, True), sgn, check_finite=False)
                    AA = 1.0 / np.sqrt(max(np.sum(ls * sgn), EPS))
                    i += 1
            ls = ls * AA
        inact = np.where(self.inactive)[0]
        corr = np.around(self.G[np.ix_(inact, act)].dot(ls), decimals=DIGITS)
        cov_in = self.cov[inact]
        g1 = _min_pos((C - cov_in) / (AA - corr + TINY32))
        g2 = _min_pos((C + cov_in) / (AA + corr + TINY32))
        gamma = min(g1, g2, C / AA)
        self.drop = False
        z = -self.coef[act] / (ls + TINY32)
        z_pos = _min_pos(z)
        drop_pos = []
        if z_pos < gamma:
            drop_pos = list(np.where(z == z_pos)[0][::-1])
            gamma = z_pos
            self.drop = True
        self.n_iter += 1
        self.prev_alpha = alpha
        coef = np.zeros(self.nf)
        coef[act] = self.coef[act] + gamma * ls
        self.coef = coef
        self.cov[inact] = cov_in - gamma * corr
        if self.drop:
            for p in drop_pos:                        # highest position first
                jd = self.active.pop(p)
                self.sign.pop(p)
                self.inactive[jd] = True
                self.cov[jd] = self.xy[jd] - np.dot(self.G[jd], self.coef)   # its correlation, from scratch
            act = np.array(self.active, dtype=np.int64)
            self.L = np.linalg.cholesky(self.G[np.ix_(act, act)]) if act.size else np.zeros((0, 0))

    # ------------------------------------------------------------------ the solution at one alpha
    def coef_at(self, alpha_min):
        """LassoLars(alpha_min, fit_intercept=False, max_iter).coef_: the first breakpoint whose alpha is within
        float32's eps of alpha_min or below it, linearly interpolated back to alpha_min from the breakpoint before"""
        k = 0
        while True:
            while k >= len(self.alphas) and not self.done:
                self._advance()
            if k >= len(self.alphas):
                return self.coefs[-1].copy()
            a = self.alphas[k]
            if a <= alpha_min + EQ_TOL:
                coef = self.coefs[k].copy()
                if abs(a - alpha_min) > EQ_TOL and k > 0:
                    pa, pc = self.alphas[k - 1], self.coefs[k - 1]
                    ss = (pa - alpha_min) / (pa - a)
                    coef = pc + ss * (coef - pc)
                return coef
            if self.done and k == len(self.alphas) - 1:
                return self.coefs[-1].copy()
            k += 1


def select_channels(solve, c_in, c_new, alpha=1e-4, tolerance=0.02, quadruple=False):
    """The reference's bisection on alpha (channel_pruner.py:496-565), statement by statement.
    solve(alpha) -> coef; returns (kept mask, [(alpha, nnz)] of every solve)."""
    log = []

    def nnz_of(a):
        coef = solve(a)
        idxs = coef != 0.
        log.append((float(a), int(idxs.sum())))
        return idxs, int(idxs.sum())

    if c_new == c_in:
        return np.ones(c_in, dtype=bool), log
    left = 0
    right = alpha
    lbound = c_new - tolerance * c_in / 2
    rbound = c_new + tolerance * c_in / 2
    while True:
        _, tmp = nnz_of(right)
        if tmp < c_new:
            break
        right *= 2
    while True:
        if lbound < 0:
            lbound = 1
        idxs, tmp = nnz_of(alpha)
        if quadruple:
            if tmp % 4 == 0 and abs(tmp - lbound) <= 2:
                break
        if lbound <= tmp and tmp <= rbound:
            if quadruple:
                if tmp % 4 == 0:
                    break
                elif tmp % 4 <= 2:
                    rbound = tmp - 1
                    lbound = lbound - 2
                else:
                    lbound = tmp + 1
                    rbound = rbound + 2
            else:
                break
        elif abs(left - right) <= right * 0.1:
            if lbound > 1:
                lbound = lbound - 1
            if rbound < c_in:
                rbound = rbound + 1
            left = left / 1.2
            right = right * 1.2
        elif tmp > rbound:
            left = left + (alpha - left) / 2
        else:
            right = right - (right - alpha) / 2
        if alpha < 1e-10:
            break
        alpha = (left + right) / 2
    return idxs, log


def lasso_select(gram, xy, n_samples, c_new, alpha=1e-4, tolerance=0.02, quadruple=False, max_iter=3000):
    """compute_pruned_kernel's channel selection on G = P^T P and xy = P^T y: (kept mask, solve log)"""
    path = LarsLassoPath(gram, xy, n_samples, max_iter)
    return select_channels(path.coef_at, len(xy), c_new, alpha, tolerance, quadruple)


def l1_select(w2, c_new):
    """prune_kernel without cp_lasso (channel_pruner.py:623-626): the c_new input channels of W2 [kh, kw, Cin, Cout]
    with the largest L1 norms (np.argsort's order among equal norms)"""
    idxs = np.argsort(-np.abs(w2).sum((0, 1, 3)))
    mask = np.zeros(len(idxs), bool)
    mask[idxs[:c_new]] = True
    return mask


def solve_normal_equations(A, B):
    """argmin_W ||X W - Y||^2 from A = X^T X and B = X^T Y, in float64: Cholesky, or, where A is singular to working
    precision, the minimum-norm least-squares solution of A W = B (numpy.linalg.lstsq, whose default cut-off drops the
    singular values below n * eps * the largest), which is also the minimum-norm solution of X W = Y.
    A is taken as singular when a Cholesky pivot squared falls below n * eps * max(diag A): collinear columns of X
    (a constant channel, such as relu(beta) of a producer channel another consumer pruned) factor with a rounding-sized
    pivot and would give huge, cancelling weights.
    sklearn's LinearRegression(fit_intercept=False) solves X W = Y with lstsq directly: on a well-conditioned X the two
    agree to the conditioning of A times float64's eps, the square of that of X."""
    A = np.asarray(A, dtype=np.float64)
    B = np.asarray(B, dtype=np.float64)
    n = A.shape[0]
    tiny = n * EPS * float(np.max(np.diag(A))) if n else 0.0
    try:
        c = linalg.cho_factor(A, lower=True, check_finite=False)
        d = np.diag(c[0])
        if np.all(np.isfinite(c[0])) and np.all(d > 0) and float(np.min(d)) ** 2 >= tiny:
            return linalg.cho_solve(c, B, check_finite=False), 'cholesky'
    except linalg.LinAlgError:
        pass
    return np.linalg.lstsq(A, B, rcond=None)[0], 'lstsq'
