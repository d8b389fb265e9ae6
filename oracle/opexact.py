"""Operand-exact float64 references of the tensor-core convolutions, with a per-element error bound.

The convolution kernels do not multiply float32 operands.  They multiply the 16-bit split of each operand,
``hi = bf16_rne(x)``, ``lo = bf16_rne(x - hi)`` (pack_kernel, repack_kernel, first_weight_image, the hi/lo activation planes),
and issue hi*hi + hi*lo + lo*hi per k-step in bf16x3 mode, hi*hi in bf16 mode.  A reference that multiplies the unrounded
float32 operands has to absorb the representation error of the split as well as the arithmetic, which needs bars of 1e-4 of
the tensor's max (bf16x3) or 5e-2 (bf16).  The references here multiply the same split operands in float64.  The kernel's
products are then exact (8-bit x 8-bit significands), and only two things separate it from the reference:

1. fp32 accumulation.  One wgmma k-step adds 16 products to the fp32 accumulator.  The tensor core aligns the terms to the
   largest exponent and truncates, so one step loses at most 2 ulps of fp32 (2**-22 relative) of a value no larger than the
   running sum of absolute products, which is bounded by A, the float64 sum of |product| over the whole dot product.  The
   epilogue's fp32 operations (cross-term add, bias, BatchNorm scale and shift, activation) add one more such term.  Hence
        |y_fp32 - y_ref| <= kappa * A,   kappa = 2**-22 * (n_steps + 1),
   with n_steps the k-steps the kernel issues on one accumulator (``n_steps_*`` below).  The fp32 FMAs of
   conv_direct_kernel lose at most 1/2 ulp each, so the same form with n_steps = taps * cin is a bound there too.
   kappa is derived from this worst case and is not fitted to any measurement.  Linear maps pass the bound through
   unchanged.  ReLU and ELU are 1-Lipschitz, so they do too.
2. The output store.  EPI_SPLIT keeps hi + lo of the fp32 result (16 significant bits).  A bf16 plan keeps hi only (8 bits).
   EPI_F32 and EPI_HEAD keep fp32.  One unit of the stored format is added to the bound:
        |y - y_ref| <= kappa * A + unit * |y_ref|,   unit = 2**-15 (hi + lo), 2**-7 (bf16), 2**-23 (fp32).

Softmax rows: if every logit of a row moves by at most delta, every probability moves by at most a factor e**(+-2 delta).
fp32 exp, the row sum and the division add a relative (C + 8) * 2**-23.  delta also carries the fp32 rounding of the
logit itself and of its difference to the row max (2**-22 * max|logit|).

Gradients over a chain of GEMMs use the same bound.  A is the float64 autograd of the same graph run on absolute values:
|x|, |w|, |dy|, with the ReLU masks as 0/1.

The module is CPU only: NumPy for the bit-level rounding, torch float64 for the convolutions.
"""
import numpy as np
import torch
import torch.nn.functional as Fn

UNIT = {'split': 2.0 ** -15, 'bf16': 2.0 ** -7, 'f32': 2.0 ** -23}


def bf16_rne(x):
    """float32 -> float32 values rounded to bfloat16, round to nearest even (the f2bf of conv.cuh, __float2bfloat16_rn)."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    u = x.view(np.uint32).astype(np.uint64)
    nan = (u & 0x7fffffff) > 0x7f800000
    r = ((u + 0x7fff + ((u >> 16) & 1)) >> 16) << 16
    r = np.where(nan, ((u >> 16) | 0x40) << 16, r)
    return (r & 0xffffffff).astype(np.uint32).view(np.float32).reshape(x.shape)


def split(x):
    """-> (hi, lo) float32 arrays, hi = bf16_rne(x), lo = bf16_rne(x - hi)."""
    x = np.asarray(x, dtype=np.float32)
    hi = bf16_rne(x)
    lo = bf16_rne((x - hi).astype(np.float32))
    return hi, lo


def kappa(n_steps):
    return 2.0 ** -22 * (n_steps + 1)


def n_steps_gemm(taps, kblocks):
    """k-steps of conv_wgmma_kernel on its main accumulator: every k-block issues all 4 k-steps of 16."""
    return taps * kblocks * 4


def n_steps_first(kblocks, split_mode):
    """conv_first_kernel: all three products of a k-step go into the same accumulator."""
    return kblocks * 4 * (3 if split_mode else 1)


def n_steps_direct(taps, cin):
    return taps * cin


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64))


def conv64(x, w, stride=1, dil=1, pads=(0, 0, 0, 0)):
    """float64 NHWC x (B,H,W,Cin), HWIO w -> NHWC (B,Ho,Wo,Cout); pads = (top, left, bottom, right)."""
    pt, pl, pb, pr = pads
    xt = Fn.pad(_t(x).permute(0, 3, 1, 2), (pl, pr, pt, pb))
    return Fn.conv2d(xt, _t(w).permute(3, 2, 0, 1), stride=stride, dilation=dil).permute(0, 2, 3, 1).numpy()


def _tap64(x, w, t, stride, dil, pads, c0=0, c1=None):
    """Contribution of tap t (input channels [c0, c1)) to conv64(x, w): one shifted window times one (cin, cout) slice."""
    pt, pl, pb, pr = pads
    KH, KW, cin, _ = w.shape
    kh, kw = divmod(t, KW)
    c1 = cin if c1 is None else min(c1, cin)
    xp = np.pad(np.asarray(x, np.float64), ((0, 0), (pt, pb), (pl, pr), (0, 0)))
    Ho = (xp.shape[1] - dil * (KH - 1) - 1) // stride + 1
    Wo = (xp.shape[2] - dil * (KW - 1) - 1) // stride + 1
    win = xp[:, kh * dil:kh * dil + stride * (Ho - 1) + 1:stride, kw * dil:kw * dil + stride * (Wo - 1) + 1:stride, c0:c1]
    return np.einsum('bhwc,co->bhwo', win, np.asarray(w[kh, kw, c0:c1], np.float64))


def conv_ref(x, w, bias=None, stride=1, dil=1, pads=(0, 0, 0, 0), mode='bf16x3', act=None, bn_scale=None, bn_shift=None,
             perturb=()):
    """Operand-exact reference of one convolution + epilogue -> (y_ref, A, {perturbation: perturbed y_ref}), float64 NHWC.

    x: the layer's input as the kernel reads it, float32 NHWC (split here exactly as the kernel's planes were).
    w: the float32 HWIO kernel the plan was given.  mode: 'bf16x3' | 'bf16' (split products) or 'fp32' (conv_direct_kernel).
    perturb: perturbations for the sensitivity checks, each a tuple -- ('cross',) drops hi*lo; ('tap', t) drops tap t;
    ('taps', t0, t1) drops taps [t0, t1) (one 64-column K block of conv_first_kernel: 16 taps x 4 channels);
    ('kblock', t, kb) drops input channels [64 kb, 64 kb + 64) of tap t; ('kcols', k0, k1) drops the columns [k0, k1) of an
    im2col row (k = tap * cin + c); ('bias', o) drops output channel o's bias.
    A perturbed reference differs from y_ref by the dropped products only; it is judged with the unperturbed bound."""
    geo = dict(stride=stride, dil=dil, pads=pads)
    if mode == 'fp32':
        x32, w32 = np.asarray(x, np.float32), np.asarray(w, np.float32)
        terms = [(x32, w32)]
        z = conv64(x32, w32, **geo)
        A = conv64(np.abs(x32), np.abs(w32), **geo)
    else:
        xh, xl = split(x)
        wh, wl = split(w)
        if mode == 'bf16x3':
            terms = [(xh, wh), (xh, wl), (xl, wh)]
            wsum = wh.astype(np.float64) + wl                              # exact: hi*hi + hi*lo in one float64 convolution
            z = conv64(xh, wsum, **geo) + conv64(xl, wh, **geo)
            A = conv64(np.abs(xh), np.abs(wh).astype(np.float64) + np.abs(wl), **geo) + conv64(np.abs(xl), np.abs(wh), **geo)
        else:
            terms = [(xh, wh)]
            z = conv64(xh, wh, **geo)
            A = conv64(np.abs(xh), np.abs(wh), **geo)
    b = np.zeros(w.shape[3]) if bias is None else np.asarray(bias, np.float64)

    def epilogue(z, b):
        y = z + b
        if bn_scale is not None:
            y = y * np.asarray(bn_scale, np.float64) + np.asarray(bn_shift, np.float64)
        if act == 'relu':
            y = np.maximum(y, 0.0)
        elif act == 'elu':
            y = np.where(y > 0, y, np.expm1(np.minimum(y, 0.0)))
        return y

    A = A + np.abs(b)
    if bn_scale is not None:
        A = A * np.abs(np.asarray(bn_scale, np.float64)) + np.abs(np.asarray(bn_shift, np.float64))
    out = {}
    for p in perturb:
        bp, dz = b, 0.0
        if p[0] == 'cross':
            dz = conv64(terms[1][0], terms[1][1], **geo)
        elif p[0] == 'tap':
            dz = sum(_tap64(a, k, p[1], **geo) for a, k in terms)
        elif p[0] == 'taps':
            dz = sum(_tap64(a, k, t, **geo) for t in range(p[1], min(p[2], w.shape[0] * w.shape[1])) for a, k in terms)
        elif p[0] == 'kblock':
            dz = sum(_tap64(a, k, p[1], c0=64 * p[2], c1=64 * p[2] + 64, **geo) for a, k in terms)
        elif p[0] == 'kcols':                                              # im2col row columns k = tap * cin + c in [k0, k1)
            cin = w.shape[2]
            dz = sum(_tap64(a, k, t, c0=max(p[1] - t * cin, 0), c1=min(p[2] - t * cin, cin), **geo)
                     for t in range(w.shape[0] * w.shape[1]) if t * cin < p[2] and (t + 1) * cin > p[1] for a, k in terms)
        elif p[0] == 'bias':
            bp = b.copy()
            bp[p[1]] = 0.0
        out[p] = epilogue(z - dz, bp)
    return epilogue(z, b), A, out


def bound(y_ref, A, n_steps, store):
    """Per-element bound |y - y_ref| <= kappa(n_steps) * A + UNIT[store] * |y_ref|."""
    return kappa(n_steps) * A + UNIT[store] * np.abs(y_ref)


def err_ratio(y, y_ref, bnd):
    """max |y - y_ref| / bound over all elements (<= 1: within the bound)."""
    y = np.asarray(y, np.float64)
    assert y.shape == y_ref.shape == bnd.shape, (y.shape, y_ref.shape, bnd.shape)
    return float(np.max(np.abs(y - y_ref) / bnd))


def softmax_ref(z, A_z, n_steps, n_classes):
    """Softmax over the last axis of float64 logits z with their magnitudes -> (p_ref, bound on |p - p_ref|)."""
    z = np.asarray(z, np.float64)
    e = np.exp(z - z.max(axis=-1, keepdims=True))
    p = e / e.sum(axis=-1, keepdims=True)
    delta = (kappa(n_steps) * A_z).max(axis=-1, keepdims=True) + 2.0 ** -22 * np.abs(z).max(axis=-1, keepdims=True)
    return p, p * (np.expm1(2.0 * delta) + (n_classes + 8) * 2.0 ** -23)
