"""Float64 NumPy reference of the softmax focal loss (``SSDFocalLoss``, csrc/focal_loss.cu), and the per-element bound the kernel is
held to, in the style of oracle/opexact.py: the reference takes the float32 operands the kernel reads and computes in float64;
the bound adds up the documented errors of what the kernel computes in float32.

The loss of image b (the batch's layout is SSDLoss's, (B, P, C+12)):
    cls[b,p] = sum_c t_c w_c (1 - q_c)^gamma (-log max(q_c, 1e-15)),   w_0 = 1 - focal_alpha, w_c = focal_alpha (c >= 1),
    pos[b,p] = max_{c=1..C-1} t_c,   loc[b,p] = sum_j smooth_L1(t_{C+j} - q_{C+j}),
    L_b = B_global (sum_p cls + alpha sum_p loc pos) / max(1, N),   N = sum_{b,p} pos over the global batch;
the gradient is d(sum_b u_b L_b) / d q with u_b = upstream[b], or 1 / B_global; the clamp passes gradient where q >= 1e-15;
gamma (1-q)^(gamma-1) log q is 0 at q = 1, its limit, for every gamma.

The bound (u = 2**-24, the unit roundoff of float32; an error of k ulps is at most 2k u relative).  The CUDA Math API documents
logf within 1 ulp and powf within 4 ulps.  Per class term T = fl(fl(w t) pw) (-lg): the rounding of w_0 = 1 - focal_alpha, the
products (3), 1 - q (which moves pw by gamma u), powf (8 u) and logf (2 u): |dT| <= (gamma + 14) u |T|.  Per offset term
v = smooth_L1 pos: the difference's rounding enters twice in 0.5 d d (or once, at most 2 u v, in |d| - 0.5), one rounding for
the value and one for the product with pos: |dv| <= 4 u |v|.  The terms are summed in double (per thread, per tile, per image):
at most (n + 4) 2**-53 of the sum of their absolute values.  N is counted in 32.32 fixed point: each row's pos moves by at most
2**-33, so 1 / max(1, N) moves by at most rel_N = rows 2**-33 / max(1, N).  The loss is rounded to float32 once (u).
Gradient of a class entry: G = s w t (D1 - D2), D1 = gamma (1-q)^(gamma-1) log q (powf, 1 - q, the product and logf:
(|gamma - 1| + 12) u), D2 = (1-q)^gamma / q (powf, 1 - q and the division: (gamma + 9) u), D1 <= 0 <= D2 so the difference
does not cancel (one more rounding); w t (2 u), the two products and the rounding of s = u_b B_global / max(1, N) (3 u) and
rel_N.  Gradient of an offset: slope(q - t) pos s alpha, four roundings and the rounding of s: (6 u + rel_N) |G|.  Everything
else the kernel writes is an exact zero.  All first-order; SLACK covers the second-order terms.
"""
import numpy as np

U = 2.0 ** -24
SLACK = 1.0 + 2.0 ** -10
EPS = float(np.float32(1e-15))
PERTURBATIONS = ('no_gamma', 'swap_alpha', 'per_image_n', 'drop_box', 'no_clamp_grad')


def _f64(a):
    return np.asarray(a, np.float32).astype(np.float64)


def _class_parts(t, q, gamma):
    """(1-q)^gamma, log max(q, eps), D1, D2 on the class entries (any shape), float64."""
    omq = 1.0 - q
    lg = np.log(np.maximum(q, EPS))
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        pw = np.power(omq, gamma)
        d1 = np.where((lg != 0) & (gamma != 0), gamma * np.power(omq, gamma - 1.0) * lg, 0.0)
        d2 = np.where(q >= EPS, pw / np.where(q > 0, q, 1.0), 0.0)
    return pw, lg, d1, d2


def focal_parts(y_true, y_pred, gamma=2.0, focal_alpha=0.25, alpha=1.0, upstream=None, global_B=None, n_pos=None, perturb=None):
    """The reference -> {'loss': (B,), 'grad': (B, P, C+12), 'cls': (B, P), 'pos': (B, P), 'n_pos': float}, float64.
    gamma, focal_alpha, alpha: as the kernel receives them (rounded to float32).  upstream: (B,) or None (1 / global_B);
    global_B: the batch size of the normalisation (default B); n_pos: the global N (default the sum over this batch).
    perturb: one of PERTURBATIONS or None: gamma taken as 0, the two weights swapped, N per image, the box with the largest
    contribution to image 0 left out, the clamp's gradient ignored (1 / q below 1e-15 too)."""
    yt, yp = _f64(y_true), _f64(y_pred)
    B, P, W = yt.shape
    C = W - 12
    g = 0.0 if perturb == 'no_gamma' else float(np.float32(gamma))
    fa = float(np.float32(focal_alpha))
    wb, wf = (fa, 1.0 - fa) if perturb == 'swap_alpha' else (1.0 - fa, fa)
    w = np.full(C, wf)
    w[0] = wb
    a32 = float(np.float32(alpha))
    gB = B if global_B is None else int(global_B)
    t, q = yt[..., :C], yp[..., :C]
    nz = t != 0
    pw, lg, d1, d2 = _class_parts(t, q, g)
    if perturb == 'no_clamp_grad':
        with np.errstate(divide='ignore'):
            d2 = np.where(q >= EPS, d2, pw / q)
    wt = w * t
    cls = np.where(nz, wt * pw * -lg, 0.0).sum(-1)
    pos = yt[..., 1:C].max(-1)
    d = yt[..., C:C + 4] - yp[..., C:C + 4]
    ad = np.abs(d)
    loc = np.where(ad < 1.0, 0.5 * d * d, ad - 0.5).sum(-1)
    keep = np.ones((B, P))
    if perturb == 'drop_box':
        keep[0, np.argmax(np.abs(cls[0]) + abs(a32) * loc[0] * np.abs(pos[0]))] = 0.0
    N = float(pos.sum()) if n_pos is None else float(n_pos)
    norm = np.full(B, max(1.0, N)) if perturb != 'per_image_n' else np.maximum(1.0, pos.sum(-1))
    loss = gB * ((cls * keep).sum(-1) + a32 * (loc * pos * keep).sum(-1)) / norm
    up = np.full(B, 1.0 / gB) if upstream is None else _f64(upstream)
    s = (up * gB / norm)[:, None, None] * keep[..., None]
    grad = np.zeros((B, P, W))
    with np.errstate(invalid='ignore'):
        grad[..., :C] = np.where(nz, s * wt * (d1 - d2), 0.0)
    e = -d
    grad[..., C:C + 4] = np.clip(e, -1.0, 1.0) * (s * (pos * a32)[..., None])
    return {'loss': loss, 'grad': grad, 'cls': cls, 'pos': pos, 'n_pos': N}


def focal_loss(y_true, y_pred, gamma=2.0, focal_alpha=0.25, alpha=1.0, global_B=None, n_pos=None):
    """(B,) float64 per-image losses."""
    return focal_parts(y_true, y_pred, gamma, focal_alpha, alpha, global_B=global_B, n_pos=n_pos)['loss']


def focal_loss_grad(y_true, y_pred, gamma=2.0, focal_alpha=0.25, alpha=1.0, upstream=None, global_B=None, n_pos=None):
    """(B, P, C+12) float64: d(sum_b u_b loss_b) / d y_pred."""
    return focal_parts(y_true, y_pred, gamma, focal_alpha, alpha, upstream, global_B, n_pos)['grad']


def focal_bound(y_true, y_pred, gamma=2.0, focal_alpha=0.25, alpha=1.0, upstream=None, global_B=None, n_pos=None, rows=None):
    """The kernel's error bound (module docstring) -> {'loss': (B,), 'grad': (B, P, C+12)}.  rows: the rows N was counted over
    (default B * P)."""
    yt, yp = _f64(y_true), _f64(y_pred)
    B, P, W = yt.shape
    C = W - 12
    g = float(np.float32(gamma))
    fa = float(np.float32(focal_alpha))
    w = np.full(C, fa)
    w[0] = 1.0 - fa
    a32 = float(np.float32(alpha))
    gB = B if global_B is None else int(global_B)
    ref = focal_parts(y_true, y_pred, gamma, focal_alpha, alpha, upstream, global_B, n_pos)
    norm = max(1.0, ref['n_pos'])
    rel_n = (B * P if rows is None else rows) * 2.0 ** -33 / norm
    t, q = yt[..., :C], yp[..., :C]
    nz = t != 0
    pw, lg, d1, d2 = _class_parts(t, q, g)
    wt = w * t
    T = np.abs(np.where(nz, wt * pw * lg, 0.0))
    d = yt[..., C:C + 4] - yp[..., C:C + 4]
    ad = np.abs(d)
    v = np.where(ad < 1.0, 0.5 * d * d, ad - 0.5) * np.abs(ref['pos'])[..., None]
    n_terms = nz.sum((1, 2)) + 4 * P
    s_abs = T.sum((1, 2)) + abs(a32) * v.sum((1, 2))
    e = (g + 14) * U * T.sum((1, 2)) + abs(a32) * 4 * U * v.sum((1, 2)) + (n_terms + 4) * 2.0 ** -53 * s_abs
    loss_b = (gB / norm * e + (rel_n + U + 2.0 ** -50) * np.abs(ref['loss'])) * SLACK
    up = np.full(B, 1.0 / gB) if upstream is None else _f64(upstream)
    s = np.abs(up * gB / norm)[:, None, None]
    grad_b = np.zeros((B, P, W))
    G = np.abs(ref['grad'])
    with np.errstate(invalid='ignore'):
        grad_b[..., :C] = np.where(nz, s * np.abs(wt) * ((abs(g - 1) + 12) * U * np.abs(d1) + (g + 9) * U * np.abs(d2))
                                   + (7 * U + rel_n) * G[..., :C], 0.0) * SLACK
    grad_b[..., C:C + 4] = (6 * U + rel_n) * G[..., C:C + 4] * SLACK
    return {'loss': loss_b, 'grad': grad_b}


def ratio(got, ref, bnd):
    """max |got - ref| / bound; equal values pass a zero bound, a NaN or an infinite difference is an infinite ratio."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape == bnd.shape, (got.shape, ref.shape, bnd.shape)
    with np.errstate(invalid='ignore', divide='ignore', over='ignore'):
        d = np.abs(got - ref)
        r = np.where(d == 0, 0.0, d / np.maximum(bnd, np.finfo(np.float64).tiny))
    r = np.where(np.isnan(r), np.inf, r)
    return float(r.max()) if r.size else 0.0
