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

Backward launches (``*_bwd_ref``, ``dgrad_ref``, ``wgrad_ref``) take the operands the kernel reads: the stored forward planes
(hi + lo, as float32), the stored gradient planes (hi and lo separately, so no re-split is needed), the float32 masters.  Each
returns (ref, A, {perturbation: ref'}) and is judged with the same form |g - ref| <= kappa * A + unit * |ref|:

3. GEMMs (data and weight gradients) follow 1. with their own k-step counts.  dgrad: ``n_steps_gemm(taps, kblocks of dZ)``, and
   one more for the old value a second consumer already wrote.  The strided data gradient stores the one-tap column GEMM in fp32
   and col2im adds up to ``taps`` of those, one fp32 rounding each: ``n_steps_gemm(1, kblocks) + taps``.  The weight gradient
   puts all three products of a k-step on one accumulator (wgrad_wgmma_kernel: ``4 * patches per split * products`` k-steps)
   or runs the pixel axis through conv_wgmma_kernel (cross terms apart: ``4 * K blocks per split``); the ``k_split`` partial
   sums meet in fp32 atomics (``n_steps_wgrad``).  The X operand is the stored planes themselves, not a re-split of hi + lo.
4. fp32 sums (wgrad_direct, bias_grad_kernel, col2im, pool routing, the gamma gradient).  Adding N terms in
   any order loses at most (N - 1) * 2**-24 * sum |term| (every partial sum is bounded by the sum of absolute terms); a
   rounded product adds 2**-24 * |term|.  So n_steps = N + 1 in kappa = 2**-22 * (n_steps + 1) is a bound, whatever order
   the atomics take.
5. Pointwise chains (softmax backward, L2Normalization backward) carry a relative error per fp32 operation; each is
   written as kappa * A with A the sum of the absolute values of the terms, see the functions.

The optimiser updates and the training-phase forward launches that are not convolutions (``sgd_ref``, ``adam_ref``,
``bn_fwd_ref``, ``l2norm_fwd_ref``, ``pool_fwd_ref``, ``preprocess_ref``) take the operands the launch read and return
per-element bounds.  train.cu, bn.cu and conv.cu build with --fmad=true, so the compiler may contract a product and an add into
one FMA: every bound counts a product and an add as two roundings, which covers the contracted form (one rounding) as well.
u = 2**-24 is the unit roundoff of fp32; a rounding of a value t loses at most u |t|.  expm1f is within 1 ulp, rsqrtf within
2 ulps, sqrtf and division are correctly rounded.

6. SGD (sgd_kernel<true> / sgd_kernel<false>): grad = g s + 2 l2 w, v' = mom v - lr grad, w' = w + v'.  Six roundings (g s, 2 l2 w,
   their sum, lr grad, mom v, the difference), each at most u times A_v = |mom v| + |lr| (|g s| + 2 l2 |w|), which bounds every
   intermediate:  |v' - v'_ref| <= 8 u A_v.  w' adds one rounding of its own, the store; as everywhere in this module one unit
   of the stored format (2**-23 for fp32) is added:  |v' - v'_ref| <= 8 u A_v + 2**-23 |v'_ref|, the same for w'.
7. Adam (adam_kernel<true> / adam_kernel<false>): grad as in 6.; m' = b1 m + (1 - b1) grad (1 - b1 is exact for b1 in [1/2, 1]);
   v' = b2 v + (1 - b2) grad^2; w' = w - lr_t m' / (sqrtf(v') + eps), lr_t = fp32(fp32(sqrt(1 - b2^t) / (1 - b1^t)) lr).
   m' carries the 3 roundings of grad and 3 of its own: |m' - m'_ref| <= 8 u A_m, A_m = |b1 m| + (1 - b1) G, G = |g s| + 2 l2 |w|.
   v' has no cancellation but grad's error enters squared (6 u) and v' adds 4 roundings: |v' - v'_ref| <= 16 u A_v,
   A_v = b2 v + (1 - b2) G^2.  The denominator D = sqrt(v') + eps moves by E_D = e_v / (sqrt(v'_ref) + sqrt(max(v'_ref - e_v, 0)))
   + 2 u D (|sqrt x - sqrt y| = |x - y| / (sqrt x + sqrt y), the square root and the add).  The numerator N = lr_t m' moves by
   lr_t e_m + 3 u |N| (lr_t's two roundings and the product).  The quotient adds one rounding: |N/D - N_ref/D_ref| <=
   e_N / (D - E_D) + |N| E_D / (D (D - E_D)) + u |N/D|, and w' one more, the store (one unit, 2**-23 |w'_ref|, for each array).
8. BatchNormalization forward (bn_stats_kernel, bn_finalize_kernel, bn_apply_kernel): the batch sums are float64; mean and
   rstd = 1 / sqrt(var + eps) are rounded to fp32 once (u each).  var = E[z^2] - mean^2 from float64 sums of N terms loses at
   most (N + 4) 2**-53 (E[z^2] + 2 |mean| E|z|); rstd then carries that over 2 (var + eps) as a relative r on top.  a = act(gamma ((z - mean) rstd) + beta): with
   X = (|z - mean| + |mean|) rstd, the subtraction, the mean's rounding, rstd's rounding and the product lose 4 u X, the
   gamma product and the beta add 2 u (|gamma| X + |beta|); ReLU and ELU are 1-Lipschitz, expm1f adds 2 u |a|.
   |a - a_ref| <= 8 u (|gamma| X (1 + r / 8u) + |beta|) + 2 u |a_ref| + unit |a_ref|.  The moving statistics follow the
   recurrence of bn_finalize_kernel, x' = mom x + (1 - mom) s with s the fp32 batch mean or the unbiased variance var N / (N - 1):
   four roundings of at most A = |mom x| + |(1 - mom) s|, |x' - x'_ref| <= 8 u A + 2**-23 |x'_ref| (the batch variance's own r
   included).
9. L2Normalization forward (l2norm_kernel, l2norm8_kernel): y = x s gamma, s = rsqrtf(max(sum x^2, 1e-12)).  The sum of C
   non-negative squares loses at most (C + 1) u of itself whatever the order; rsqrtf adds 4 u and halves the sum's error; the two
   products 2 u.  |y - y_ref| <= ((C + 1) / 2 + 8) u |y_ref| + unit |y_ref|.  A clamped pixel (sum x^2 <= 1e-12 in fp32) takes
   s = rsqrt(1e-12): max is continuous, so the reference uses the same formula in float64.
10. Max-pooling and the input preprocessing move or compute values without an accumulation: ``pool_fwd_ref`` (the hi and lo
   planes of the first maximum of hi + lo) and ``preprocess_ref`` ((x - mean) / std in fp32, channel swap, split) are bit-exact.
11. The SSD loss (ssd_loss_kernel, ssd_loss_phase_kernel; loss.cu builds with --fmad=false, so every product and every add is
   one rounding).  ``loss_ref`` takes y_true, y_pred and the per-box losses the kernel stored (ssdk_ssd_loss_read_box_losses):
   cls = -sum_c tv_c logf(max(p_c, 1e-15f)) and negl = cls * y_true[..., 0].
   - negl must be fl(cls * yt0) bit for bit.  cls: logf is within 1 ulp (2 u relative), the product with tv one rounding, the
     first add to 0 exact and the n - 1 others one each, every partial sum bounded by S = sum |tv log p| (1 + 3u):
        |cls - cls_ref| <= (n + 2) u S (1 + 2**-20),   n = the non-zero tv of the box.
   - The hard-negative selection is exact on the kernel's negl: k = min(max(ratio n_pos, n_neg_min), nnz) over the whole batch
     (n_pos = int(fp32 sum of the positive flags), nnz = the non-zero negl), ordered by value descending, then flat index
     ascending, -0 == +0 (tf.nn.top_k).  n_pos, nnz, k and `want` (the boxes equal to the k-th value that are kept) are exact.
   - Smooth L1 is not stored: d = fl(yt - yp) is off by u |d|, and f(x) = 0.5 x^2 (|x| < 1) or |x| - 0.5 has |f'| <= min(|x|, 1)
     (both branches give 0.5 at |d| = 1, so a d that rounds onto the other side moves f by the same amount); each f adds one
     rounding, the three adds one each:  |l - l_ref| <= (u sum_j |d_j| min(1, |d_j|) + 4 u l_ref) (1 + 2**-20).
   - The per-image loss (pc + ng + alpha loc) inv_norm global_B is summed in float64 from fp32 products: cls pmax and l pmax
     one rounding each (u of the term; l carries its bound into the sum), the float64 sums (N + 8) 2**-53 of the absolute
     sum, inv_norm = fp32(1 / max(1, n_pos)) is an operand, and the store one unit (2**-23) of the result.
   - The gradient of a class entry is (-tv / q) w_cls, w_cls = (pmax + take) (up global_B inv_norm): up * global_B, * inv_norm,
     pmax + take, * scale, the division and the last product are six roundings; a loc entry slope(fl(yp - yt)) (pmax scale alpha)
     has six too (the difference, the two of scale, * pmax, * alpha, the product; slope = clip(d, -1, 1) is 1-Lipschitz and
     exact at |d| = 1).  Each is a product of exactly rounded factors:  |g - g_ref| <= 6 u |g_ref| (1 + 2**-20).  q < 1e-15f
     gives 0.  upstream is read as float32 operands (NULL: fp32(1 / global_B)).

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
    return np.einsum('bhwc,co->bhwo', win, np.asarray(w[kh, kw, c0:c1], np.float64), optimize=True)    # a BLAS product


def conv_ref(x, w, bias=None, stride=1, dil=1, pads=(0, 0, 0, 0), mode='bf16x3', act=None, bn_scale=None, bn_shift=None,
             perturb=()):
    """Operand-exact reference of one convolution + epilogue -> (y_ref, A, {perturbation: perturbed y_ref}), float64 NHWC.

    x: the layer's input as the kernel reads it, float32 NHWC (split here exactly as the kernel's planes were), or the stored
    planes (hi, lo) of a layer output as float32 (lo None in bf16 mode), multiplied as they are.
    w: the float32 HWIO kernel the plan was given.  mode: 'bf16x3' | 'bf16' (split products) or 'fp32' (conv_direct_kernel).
    perturb: perturbations for the sensitivity checks, each a tuple -- ('cross',) drops hi*lo; ('tap', t) drops tap t;
    ('taps', t0, t1) drops taps [t0, t1) (one 64-column K block of conv_first_kernel: 16 taps x 4 channels);
    ('kblock', t, kb) drops input channels [64 kb, 64 kb + 64) of tap t; ('kcols', k0, k1) drops the columns [k0, k1) of an
    im2col row (k = tap * cin + c); ('bias', o) drops output channel o's bias; ('bias_live',) drops the largest |bias| of the
    output channels the activation does not zero everywhere (a ReLU channel that is zero on every pixel hides its bias).
    A perturbed reference differs from y_ref by the dropped products only; it is judged with the unperturbed bound."""
    geo = dict(stride=stride, dil=dil, pads=pads)
    if mode == 'fp32':
        x32 = np.sum(_planes(x), axis=0, dtype=np.float32) if isinstance(x, tuple) else np.asarray(x, np.float32)
        w32 = np.asarray(w, np.float32)
        terms = [(x32, w32)]
        z = conv64(x32, w32, **geo)
        A = conv64(np.abs(x32), np.abs(w32), **geo)
    else:
        xh, xl = _planes(x) if isinstance(x, tuple) else split(x)
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
    y = epilogue(z, b)
    out = {}
    for p in perturb:
        bp, dz = b, 0.0
        if p[0] == 'bias_live':
            live = np.any(y != 0, axis=tuple(range(y.ndim - 1)))
            bp = b.copy()
            bp[int(np.argmax(np.abs(b) * live))] = 0.0
        elif p[0] == 'cross':
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
    return y, A, out


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


# ------------------------------------------------------------------------------------------------------------------------------
# backward launches
# ------------------------------------------------------------------------------------------------------------------------------
def bf16_bits_to_f32(u16):
    """uint16 bf16 bit patterns -> float32 values."""
    return (np.asarray(u16, np.uint16).astype(np.uint32) << 16).view(np.float32)


def n_steps_wgrad(plan, products):
    """k-steps behind one weight-gradient element, from ssdk_trainer_layer_plan.  NATIVE (wgrad_wgmma_kernel): ``kv`` 64-pixel
    patches, all ``products`` of a k-step on one accumulator.  TRANSPOSED / IM2COL (conv_wgmma_kernel on a K axis of ``kv``
    pixels, ceil(kv / 64) K blocks): the cross products have accumulators of their own, added in the epilogue, so the main
    accumulator takes 4 k-steps per K block.  Either way the axis is cut into k_split ranges of at most ceil(units /
    (k_split - 1)) units each, whose partial sums meet in fp32 atomics."""
    ks = plan['k_split']
    units, per_unit = (plan['kv'], 4 * products) if plan['wgrad'] == 'native' else (-(-plan['kv'] // 64), 4)
    per = units if ks == 1 else min(units, -(-units // (ks - 1)))
    return per_unit * per + ks


def direct_wgrad_rows(B, Ho, sm_count):
    """train.cu, the launch of wgrad_direct_kernel / wgrad_direct3x3_kernel -> (rows_per_block, grid, rows of the last block):
    each block owns ceil(B Ho / (8 SMs)) consecutive output rows (image-major)."""
    rows = B * Ho
    rpb = max(1, -(-rows // (8 * sm_count)))
    grid = -(-rows // rpb)
    return rpb, grid, rows - (grid - 1) * rpb


def n_steps_wgrad_direct(B, Ho, Wo, cout, fast, sm_count):
    """Roundings behind one element of the direct weight gradient, in the kernels' summation order (section 4): a thread adds
    its products over the block's rows in fp32 (wgrad_direct3x3_kernel: every 256 / (cout / 2)-th pixel of a row, the pixel
    lanes then meet in shared-memory atomics; wgrad_direct_kernel: every pixel, one add into shared memory), and each block adds
    its sum into the flat gradient with one fp32 atomic.  A sum whose partial sums are formed this way loses at most
    (longest chain of roundings) * 2**-24 * sum |term|, so this count replaces the B Ho Wo + 1 of one flat sum."""
    rpb, grid, _ = direct_wgrad_rows(B, Ho, sm_count)
    if fast:
        lanes = 256 // (cout // 2)
        per_thread = rpb * -(-Wo // lanes)
    else:
        lanes, per_thread = 1, rpb * Wo
    return per_thread + lanes + grid + 1


def _dconv_tap(dz, w, t, in_hw, stride, dil, pads, c0=0, c1=None):
    """Contribution of tap t (dZ channels [c0, c1)) to the data gradient: dz (B,Ho,Wo,Cout) x w[kh,kw,:,c0:c1]^T scattered
    onto the (B,H,W,Cin) input grid."""
    pt, pl, _, _ = pads
    KH, KW, cin, cout = w.shape
    kh, kw = divmod(t, KW)
    c1 = cout if c1 is None else min(c1, cout)
    B, Ho, Wo, _ = dz.shape
    H, W = in_hw
    out = np.zeros((B, H + 2 * (pt + dil * KH + stride), W + 2 * (pl + dil * KW + stride), cin))
    v = np.asarray(dz[..., c0:c1], np.float64) @ np.asarray(w[kh, kw, :, c0:c1], np.float64).T
    y0, x0 = kh * dil, kw * dil                                    # padded-input position of output (0, 0) under this tap
    out[:, y0:y0 + stride * (Ho - 1) + 1:stride, x0:x0 + stride * (Wo - 1) + 1:stride] += v
    return out[:, pt:pt + H, pl:pl + W]


def _dconv(dz, w, in_hw, stride, dil, pads):
    return sum(_dconv_tap(dz, w, t, in_hw, stride, dil, pads) for t in range(w.shape[0] * w.shape[1]))


def _planes(p):
    """(hi, lo) float32 planes; lo None -> zeros (single-pass bf16 gradients)."""
    hi, lo = p
    return np.asarray(hi, np.float32), (np.zeros_like(hi, np.float32) if lo is None else np.asarray(lo, np.float32))


def _terms(a, b, mode):
    """Products the kernel issues for split operands a = (hi, lo), b = (hi, lo)."""
    return [(a[0], b[0]), (a[0], b[1]), (a[1], b[0])] if mode == 'bf16x3' else [(a[0], b[0])]


def _mask_acc(v, A, mask, old):
    if mask is not None:
        v, A = v * (mask > 0), A * (mask > 0)
    if old is not None:
        v, A = v + old, A + np.abs(old)
    return v, A


def dgrad_ref(dz, w, in_hw, stride=1, dil=1, pads=(0, 0, 0, 0), mode='bf16x3', mask=None, old=None, perturb=()):
    """Data gradient of one convolution -> (ref, A, {perturbation: ref'}), float64 (B,H,W,Cin).

    dz: the layer's gradient planes (hi, lo) as float32 (B,Ho,Wo,Cout), lo None in bf16 mode.  w: float32 HWIO master (split
    here as the data-gradient planes are packed).  mask: the ReLU producer's stored output (the gradient is zeroed where it is
    not > 0) or None.  old: the producer's gradient before the launch (accumulation) or None.  perturb: ('cross',) drops
    dZ_hi * W_lo; ('tap', t) drops tap t; ('kblock', t, kb) drops dZ channels [64 kb, 64 kb + 64) of tap t (one K block of
    the GEMM); ('mask',) leaves the mask out; ('old',) leaves the old value out."""
    d = _planes(dz)
    terms = _terms(d, split(w), mode)
    geo = dict(in_hw=in_hw, stride=stride, dil=dil, pads=pads)
    z = sum(_dconv(a, k, **geo) for a, k in terms)
    A = sum(_dconv(np.abs(a), np.abs(k), **geo) for a, k in terms)
    out = {}
    for p in perturb:
        zp, mp, op = z, mask, old
        if p[0] == 'cross':
            zp = z - _dconv(*terms[1], **geo)
        elif p[0] == 'tap':
            zp = z - sum(_dconv_tap(a, k, p[1], **geo) for a, k in terms)
        elif p[0] == 'kblock':
            zp = z - sum(_dconv_tap(a, k, p[1], c0=64 * p[2], c1=64 * p[2] + 64, **geo) for a, k in terms)
        elif p[0] == 'mask':
            mp = None
        elif p[0] == 'old':
            op = None
        out[p] = _mask_acc(zp, A, mp, op)[0]
    ref, A = _mask_acc(z, A, mask, old)
    return ref, A, out


def n_steps_dgrad(plan, taps, kblocks):
    """k-steps behind one data-gradient element (section 3)."""
    if plan['dgrad'] == 'strided':
        return n_steps_gemm(1, kblocks) + taps + plan['dgrad_accumulate']
    return n_steps_gemm(taps, kblocks) + plan['dgrad_accumulate']


def _wgrad_tap(x, dz, t, KH, KW, stride, dil, pads, pix=None):
    """dW[:, tap t, :] = sum over output pixels of dz (B,Ho,Wo,Cout) x the tap's window of x -> (Cout, Cin); pix: optional
    (B,Ho,Wo) 0/1 weights of the output pixels."""
    pt, pl, pb, pr = pads
    kh, kw = divmod(t, KW)
    B, Ho, Wo, _ = dz.shape
    xp = np.pad(np.asarray(x, np.float64), ((0, 0), (pt, pb + stride + dil * KH), (pl, pr + stride + dil * KW), (0, 0)))
    win = xp[:, kh * dil:kh * dil + stride * (Ho - 1) + 1:stride, kw * dil:kw * dil + stride * (Wo - 1) + 1:stride]
    d = np.asarray(dz, np.float64) if pix is None else np.asarray(dz, np.float64) * pix[..., None]
    return np.tensordot(d, win, axes=([0, 1, 2], [0, 1, 2]))         # one BLAS product: full-size layers stay cheap


def wgrad_ref(x, dz, KH, KW, stride=1, dil=1, pads=(0, 0, 0, 0), mode='bf16x3', perturb=()):
    """Weight gradient -> (ref, A, {perturbation: ref'}), float64 (Cout, KH, KW, Cin) (the flat buffer's OHWI layout).

    x: the layer's input as stored: its planes (hi, lo) as float32 (lo None in bf16 mode), or float32 hi + lo values to be
    split here.  Pass the planes: where lo is exactly half an ulp of hi, split(hi + lo) may trade that half ulp between the
    planes, which moves hi * dZ_lo by 2**-16 of the product -- more than the accumulation bound when a sparse (ReLU) input
    channel has few non-zero products.  dz: the gradient planes (hi, lo).  mode 'fp32':
    wgrad_direct_kernel, fp32 products of the unsplit hi + lo values.  perturb: ('cross',) drops X_hi * dZ_lo; ('tap', t);
    ('kblock', kb) drops input channels [64 kb, 64 kb + 64) of every tap (one wgmma N block); ('pixels', n, y0, x0, h, w)
    drops an h x w block of output pixels of image n (with h x w = bh x bw at the origin: one K block of the native kernel);
    ('first', n, m) drops the first m output pixels of image n in row-major order (the first K block of the im2col GEMM)."""
    g = _planes(dz)
    xs = _planes(x) if isinstance(x, tuple) else split(x)
    if mode == 'fp32':
        terms = [(xs[0].astype(np.float64) + xs[1], g[0].astype(np.float64) + g[1])]
    else:
        terms = _terms(xs, g, mode)
    taps = KH * KW
    geo = dict(KH=KH, KW=KW, stride=stride, dil=dil, pads=pads)

    def full(pix=None, skip_tap=None, which=None):
        out = np.zeros((dz[0].shape[-1], taps, xs[0].shape[-1]))
        for a, d in (terms if which is None else which):
            for t in range(taps):
                if t != skip_tap:
                    out[:, t] += _wgrad_tap(a, d, t, pix=pix, **geo)
        return out
    ref = full()
    A = full(which=[(np.abs(a), np.abs(d)) for a, d in terms])
    out = {}
    for p in perturb:
        if p[0] == 'cross':
            out[p] = ref - full(which=[terms[1]])
        elif p[0] == 'tap':
            out[p] = full(skip_tap=p[1])
        elif p[0] == 'kblock':
            out[p] = ref.copy()
            out[p][:, :, 64 * p[1]:64 * p[1] + 64] = 0.0
        elif p[0] == 'pixels':
            pix = np.ones(dz[0].shape[:3])
            pix[p[1], p[2]:p[2] + p[4], p[3]:p[3] + p[5]] = 0
            out[p] = full(pix=pix)
        elif p[0] == 'first':
            pix = np.ones(dz[0].shape[:3])
            pix[p[1]].reshape(-1)[:p[2]] = 0
            out[p] = full(pix=pix)
    shape = (-1, KH, KW, xs[0].shape[-1])
    return ref.reshape(shape), A.reshape(shape), {k: v.reshape(shape) for k, v in out.items()}


def bias_grad_ref(dz, perturb=()):
    """Bias gradient (bias_grad_kernel): fp32 sum of hi and lo over all pixels -> (ref, A, n_steps, {...}).
    perturb: ('lo',) leaves the lo plane out; ('row', n, y) leaves pixel row y of image n out."""
    g = _planes(dz)
    ref = g[0].astype(np.float64).sum(axis=(0, 1, 2)) + g[1].astype(np.float64).sum(axis=(0, 1, 2))
    A = np.abs(g[0]).astype(np.float64).sum(axis=(0, 1, 2)) + np.abs(g[1]).astype(np.float64).sum(axis=(0, 1, 2))
    out = {}
    for p in perturb:
        if p[0] == 'lo':
            out[p] = g[0].astype(np.float64).sum(axis=(0, 1, 2))
        elif p[0] == 'row':
            out[p] = ref - g[0][p[1], p[2]].astype(np.float64).sum(0) - g[1][p[1], p[2]].astype(np.float64).sum(0)
    return ref, A, 2 * int(np.prod(g[0].shape[:3])), out


def pool_route(x, gout, KH, KW, stride, pad_t, pad_l, last=False):
    """Max-pool backward routing in float64: each output's gradient goes to the FIRST maximum of its window (row-major scan,
    strict '>', out-of-range taps skipped); last=True routes ties to the last maximum.  -> (routed, sum of |routed|,
    windows per input element)."""
    x = np.asarray(x, np.float64)
    B, H, W, Cc = x.shape
    _, Ho, Wo, _ = gout.shape
    g = np.asarray(gout, np.float64)
    out, A, cnt = np.zeros_like(x), np.zeros_like(x), np.zeros_like(x)
    bi, ci = np.meshgrid(np.arange(B), np.arange(Cc), indexing='ij')
    for yo in range(Ho):
        for xo in range(Wo):
            ys = [y for y in range(yo * stride - pad_t, yo * stride - pad_t + KH) if 0 <= y < H]
            xs = [xx for xx in range(xo * stride - pad_l, xo * stride - pad_l + KW) if 0 <= xx < W]
            pos = [(y, xx) for y in ys for xx in xs]                   # row-major scan order
            win = np.stack([x[:, y, xx] for y, xx in pos], axis=-1)     # (B, C, taps)
            k = win.shape[-1] - 1 - np.argmax(win[..., ::-1], axis=-1) if last else np.argmax(win, axis=-1)
            py = np.array([p[0] for p in pos])[k]
            px = np.array([p[1] for p in pos])[k]
            np.add.at(out, (bi, py, px, ci), g[:, yo, xo])
            np.add.at(A, (bi, py, px, ci), np.abs(g[:, yo, xo]))
            np.add.at(cnt, (bi, py, px, ci), 1.0)
    return out, A, cnt


def pool_bwd_ref(x, gout, KH, KW, stride, pad_t, pad_l, relu_mask=False, old=None, perturb=()):
    """pool_bwd_kernel -> (ref, A, n_steps, {...}).  x: the pool's input as stored (hi + lo); gout: the pool's gradient (hi + lo).
    n_steps: the most windows that route to one element, plus the accumulation.  perturb: ('last',) ties to the last
    maximum; ('mask',), ('old',)."""
    r, A, cnt = pool_route(x, gout, KH, KW, stride, pad_t, pad_l)
    mask = x if relu_mask else None
    out = {}
    for p in perturb:
        if p[0] == 'last':
            out[p] = _mask_acc(pool_route(x, gout, KH, KW, stride, pad_t, pad_l, last=True)[0], A, mask, old)[0]
        elif p[0] == 'mask':
            out[p] = _mask_acc(r, A, None, old)[0]
        elif p[0] == 'old':
            out[p] = _mask_acc(r, A, mask, None)[0]
    ref, A = _mask_acc(r, A, mask, old)
    return ref, A, int(cnt.max()) + (old is not None), out


def l2norm_bwd_ref(x, gy, gamma, relu_mask=False, old=None, perturb=()):
    """l2norm_bwd_kernel -> (gx_ref, A, kappa, gamma_ref, A_gamma, n_steps_gamma, {...}), float64.

    y_c = gamma_c x_c s, s = rsqrt(max(sum x^2, 1e-12)): gx_c = s gamma_c d_c - x_c s^3 dot, dot = sum_c gamma_c d_c x_c; a
    clamped pixel (sum x^2 <= 1e-12) keeps s gamma_c d_c only.  dgamma_c = sum over pixels of d_c x_c s.
    Bound of gx: sum x^2 and dot are fp32 sums of C products (relative (C + 1) 2**-24 of their absolute sums); rsqrtf adds
    2 ulps, so s carries (C/2 + 3) 2**-23 and s^3 three times that; the remaining multiplies, the subtraction and the
    accumulation add a few roundings.  kappa = (3 C + 32) 2**-23 with A = s |gamma d| + |x| s^3 sum|gamma d x| (+ |old|)
    covers all of them.  dgamma: a product of three factors (s as above) summed over N pixels in fp32 atomics ->
    n_steps = N + C/2 + 6.  perturb: ('proj',) drops the projection term x s^3 dot."""
    x = np.asarray(x, np.float64)
    d = np.asarray(gy, np.float64)
    gm = np.asarray(gamma, np.float64)
    Cc = x.shape[-1]
    ss = (x * x).sum(-1, keepdims=True)
    clamped = ~(ss > 1e-12)
    s = 1.0 / np.sqrt(np.maximum(ss, 1e-12))
    dot = (gm * d * x).sum(-1, keepdims=True)
    t1 = s * gm * d
    t2 = np.where(clamped, 0.0, x * s ** 3 * dot)
    A = np.abs(t1) + np.where(clamped, 0.0, np.abs(x) * s ** 3 * (np.abs(gm * d * x)).sum(-1, keepdims=True))
    mask = x if relu_mask else None
    out = {}
    for p in perturb:
        if p[0] == 'proj':
            out[p] = _mask_acc(t1, A, mask, old)[0]
        elif p[0] == 'mask':
            out[p] = _mask_acc(t1 - t2, A, None, old)[0]
        elif p[0] == 'old':
            out[p] = _mask_acc(t1 - t2, A, mask, None)[0]
    ref, A = _mask_acc(t1 - t2, A, mask, old)
    gg = (d * x * s).reshape(-1, Cc).sum(0)
    Ag = np.abs(d * x * s).reshape(-1, Cc).sum(0)
    npix = int(np.prod(x.shape[:-1]))
    return ref, A, (3 * Cc + 32) * 2.0 ** -23, gg, Ag, npix + Cc // 2 + 6, out


def head_bwd_ref(logits, dy, n_boxes, n_classes, perturb=()):
    """head_bwd_kernel -> (ref, A, kappa, {...}), float64 (B,H,W,n_boxes*(C+4)).

    logits: the head's stored fp32 output (B,H,W,n_boxes*(C+4)); dy: d loss / d y_pred rows of this head, (B,H,W,n_boxes,>=C+4).
    Class columns: p_c (d_c - dot), dot = sum p d; offsets pass d through.  Bound: expf is within 2 ulps, so each p carries a
    relative e_p = (C + 8) 2**-22 (C exponentials in the sum, the max, the quotient); dot adds (C + 2) 2**-23 of S = sum p|d|;
    the difference and the product one rounding each.  |err| <= (2 e_p + (C + 4) 2**-23) p (|d| + S): kappa = (5 C + 36) 2**-23,
    A = p (|d| + S).  perturb: ('dot',) drops the dot term."""
    Cc = n_classes
    B, H, W, _ = logits.shape
    z = np.asarray(logits, np.float64).reshape(B, H, W, n_boxes, Cc + 4)
    d = np.asarray(dy, np.float64)[..., :Cc + 4]
    e = np.exp(z[..., :Cc] - z[..., :Cc].max(-1, keepdims=True))
    p = e / e.sum(-1, keepdims=True)
    dot = (p * d[..., :Cc]).sum(-1, keepdims=True)
    S = (p * np.abs(d[..., :Cc])).sum(-1, keepdims=True)

    def rows(cls):
        return np.concatenate([cls, d[..., Cc:]], axis=-1).reshape(B, H, W, -1)
    ref = rows(p * (d[..., :Cc] - dot))
    A = rows(p * (np.abs(d[..., :Cc]) + S)) * np.tile(np.concatenate([np.ones(Cc), np.zeros(4)]), n_boxes)
    out = {}
    for q in perturb:
        if q[0] == 'dot':
            out[q] = rows(p * d[..., :Cc])
    return ref, A, (5 * Cc + 36) * 2.0 ** -23, out


def bn_bwd_ref(z, a, da, gamma, act=None, eps=1e-3, perturb=()):
    """BatchNormalization backward (bn_bwd_reduce_kernel + bn_bwd_apply_kernel) -> (dz_ref, A, kappa, dgamma_ref, dbeta_ref,
    A_dgamma, A_dbeta, kappa_params, {...}), float64.

    z: the stored raw convolution output (hi + lo); a: the stored activation output; da: d loss / d a (the gradient planes the
    launch read).  The batch statistics are recomputed in float64 from z (biased variance over B, H, W).
        dy = da * act'(a)  (ReLU: a > 0; ELU: a + 1 where a <= 0, written through the output like the kernel),
        x^ = (z - mean) * rstd,  m1 = mean(dy),  m2 = mean(dy x^),  dz = gamma rstd (dy - m1 - x^ m2),
        dgamma = sum dy x^,  dbeta = sum dy.
    Bound: the kernel holds mean and rstd in fp32 (2**-24 relative each, from float64 statistics), forms dy with one rounding,
    x^ with two (the subtraction and the product; the mean's rounding adds 2**-24 |mean| rstd), m1 and m2 as float64 sums rounded
    once to fp32, and dz with three more roundings.  dy - m1 - x^ m2 cancels, so every term is bounded on absolute values:
    with X = (|z - mean| + |mean|) rstd >= |x^| and its error, S1 = mean |dy| and S2 = mean(|dy| X),
        |dz - dz_ref| <= 16 * 2**-23 * |gamma| rstd (|dy| + S1 + X (S2 + |m2|))  (kappa = 2**-19, A the factor after it).
    The parameter gradients are float64 sums of fp32 terms dy x^ (each within 6 * 2**-23 of |dy| X) and dy, rounded once:
    kappa_params = 8 * 2**-23 with A = sum |dy| X and sum |dy|.  perturb: ('m1',) and ('m2',) drop those terms; ('elu1',)
    replaces act' by 1."""
    z = np.asarray(z, np.float64)
    a = np.asarray(a, np.float64)
    da = np.asarray(da, np.float64)
    gm = np.asarray(gamma, np.float64)
    axes = tuple(range(z.ndim - 1))
    mean = z.mean(axes)
    rstd = 1.0 / np.sqrt(z.var(axes) + float(np.float32(eps)))
    xh = (z - mean) * rstd
    X = (np.abs(z - mean) + np.abs(mean)) * rstd

    def deriv(unit_elu=False):
        if act == 'relu':
            return (a > 0).astype(np.float64)
        if act == 'elu' and not unit_elu:
            return np.where(a > 0, 1.0, a + 1.0)
        return np.ones_like(a)

    def dz_of(dy, drop=None):
        m1, m2 = dy.mean(axes), (dy * xh).mean(axes)
        return gm * rstd * (dy - (0 if drop == 'm1' else m1) - (0 if drop == 'm2' else xh * m2))
    dy = da * deriv()
    ref = dz_of(dy)
    m2 = (dy * xh).mean(axes)
    A = np.abs(gm) * rstd * (np.abs(dy) + np.abs(dy).mean(axes) + X * ((np.abs(dy) * X).mean(axes) + np.abs(m2)))
    out = {}
    for p in perturb:
        if p[0] in ('m1', 'm2'):
            out[p] = dz_of(dy, p[0])
        elif p[0] == 'elu1':
            out[p] = dz_of(da * deriv(unit_elu=True))
    dgamma, dbeta = (dy * xh).sum(axes), dy.sum(axes)
    Ag, Ab = (np.abs(dy) * X).sum(axes), np.abs(dy).sum(axes)
    return ref, A, 16 * 2.0 ** -23, dgamma, dbeta, Ag, Ab, 8 * 2.0 ** -23, out


# ------------------------------------------------------------------------------------------------------------------------------
# optimiser updates and the training-phase forward launches that are not convolutions (sections 6 - 10)
# ------------------------------------------------------------------------------------------------------------------------------
U32 = 2.0 ** -24


def _f64(a):
    """float32 operands (or Python scalars the launch receives as float) -> their float64 values."""
    return np.asarray(a, np.float32).astype(np.float64)


def state_ratio(got, ref, bnd):
    """max |got - ref| / bound over the arrays of an update ({'w': ..., 'm': ...}); a zero bound admits only exact values."""
    r = 0.0
    for k in ref:
        b = np.maximum(np.asarray(bnd[k], np.float64), np.finfo(np.float64).tiny)
        r = max(r, err_ratio(np.asarray(got[k], np.float64).reshape(ref[k].shape), ref[k], b))
    return r


def _grad(g, w, l2, scale, kernel_shape, p):
    """The gradient an update reads (section 6) and G = |g s| + 2 l2 |w|; p: the perturbation that changes it, or None."""
    g, w = _f64(g), _f64(w)
    if p == ('hwio',):                                               # the flat gradient indexed like the HWIO master
        cout, kh, kw, cin = kernel_shape
        g = g.reshape(kh, kw, cin, cout).transpose(3, 0, 1, 2).reshape(g.shape)
    s = 1.0 if p == ('no_scale',) else float(np.float32(scale))
    l2 = float(np.float32(l2))
    if kernel_shape is None:
        l2 = l2 if p == ('l2_all',) else 0.0
    elif p == ('no_l2',):
        l2 = 0.0
    return g * s + 2.0 * l2 * w, np.abs(g * s) + 2.0 * l2 * np.abs(w)


def sgd_ref(w, v, g, lr, momentum, l2=0.0, scale=1.0, kernel_shape=None, perturb=()):
    """One SGD update of one parameter span (sgd_kernel<true> / sgd_kernel<false>) -> (ref, bound, {perturbation: ref'}), each a dict
    {'w': new master, 'v': new velocity}, float64.

    w, v, g: the master, the velocity and the gradient as the launch read them, in the gradient's layout (kernels OHWI, as
    ssdk_trainer_read_params / ssdk_trainer_read_opt_state return them).  kernel_shape: (cout, kh, kw, cin) of a conv / head kernel,
    whose update carries the l2 term; None for biases and gammas.  Bound: section 6.  perturb: ('no_l2',) drops the l2 term;
    ('l2_all',) applies it to a bias / gamma span; ('no_scale',) ignores grad_scale; ('no_momentum',) drops the carried velocity;
    ('hwio',) reads the gradient at the HWIO index."""
    lr, mom = float(np.float32(lr)), float(np.float32(momentum))
    w64, v64 = _f64(w), _f64(v)

    def update(p=None):
        grad, G = _grad(g, w, l2, scale, kernel_shape, p)
        nv = (0.0 if p == ('no_momentum',) else mom * v64) - lr * grad
        return {'w': w64 + nv, 'v': nv}, G
    ref, G = update()
    A = np.abs(mom * v64) + abs(lr) * G
    unit = UNIT['f32']
    bnd = {'v': 8 * U32 * A + unit * np.abs(ref['v']), 'w': 8 * U32 * A + unit * np.abs(ref['w'])}
    return ref, bnd, {p: update(p)[0] for p in perturb}


def adam_lr_t(lr, beta1, beta2, t):
    """Keras' lr_t = lr sqrt(1 - b2^t) / (1 - b1^t) in float64 from the float32 operands."""
    b1, b2 = float(np.float32(beta1)), float(np.float32(beta2))
    return float(np.float32(lr)) * np.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t)


def adam_ref(w, m, v, g, lr, beta1, beta2, eps, t, l2=0.0, scale=1.0, kernel_shape=None, perturb=()):
    """One Adam update of one parameter span (adam_kernel<true> / adam_kernel<false>) -> (ref, bound, {perturbation: ref'}), each a dict
    {'w': new master, 'm': new first moment, 'v': new second moment}, float64.

    w, m, v, g: as read before the launch, in the gradient's layout; t: the step the update was given (from 1).  Bound: section
    7.  perturb: the perturbations of sgd_ref that change the gradient, and ('t-1',), ('t+1',) (lr_t of the neighbouring step),
    ('eps_in_root',) (w -= lr_t m / sqrt(v + eps)), ('no_m',), ('no_v',) (a moment not carried)."""
    b1, b2, e = float(np.float32(beta1)), float(np.float32(beta2)), float(np.float32(eps))
    w64, m64, v64 = _f64(w), _f64(m), _f64(v)

    def update(p=None):
        grad, G = _grad(g, w, l2, scale, kernel_shape, p)
        a = (0.0 if p == ('no_m',) else b1 * m64) + (1.0 - b1) * grad
        b = (0.0 if p == ('no_v',) else b2 * v64) + (1.0 - b2) * grad * grad
        tt = t - 1 if p == ('t-1',) else t + 1 if p == ('t+1',) else t
        den = np.sqrt(b + e) if p == ('eps_in_root',) else np.sqrt(b) + e
        return {'w': w64 - adam_lr_t(lr, b1, b2, tt) * a / den, 'm': a, 'v': b}, G
    ref, G = update()
    lr_t = adam_lr_t(lr, b1, b2, t)
    e_m = 8 * U32 * (np.abs(b1 * m64) + (1.0 - b1) * G)
    e_v = 16 * U32 * (b2 * v64 + (1.0 - b2) * G * G)
    vr = ref['v']
    D = np.sqrt(vr) + e
    with np.errstate(divide='ignore', invalid='ignore'):
        e_sqrt = np.minimum(np.sqrt(e_v), np.where(e_v > 0, e_v / (np.sqrt(vr) + np.sqrt(np.maximum(vr - e_v, 0.0))), 0.0))
    e_D = e_sqrt + 2 * U32 * D
    N = lr_t * np.abs(ref['m'])
    e_N = lr_t * e_m + 3 * U32 * N
    D_lo = D - e_D
    e_step = e_N / D_lo + N * e_D / (D * D_lo) + U32 * N / D
    unit = UNIT['f32']
    bnd = {'w': e_step + unit * np.abs(ref['w']), 'm': e_m + unit * np.abs(ref['m']), 'v': e_v + unit * np.abs(vr)}
    return ref, bnd, {p: update(p)[0] for p in perturb}


def bn_fwd_ref(z, gamma, beta, mmean, mvar, act=None, eps=1e-3, momentum=0.99, z_prev=None, perturb=()):
    """BatchNormalization forward in the training phase (bn_stats_kernel, bn_finalize_kernel, bn_apply_kernel) -> (a_ref, A,
    kappa, stats_ref, stats_bound, {perturbation: (a', stats')}), float64.  |a - a_ref| <= kappa A + unit |a_ref| (section 8).

    z: the raw convolution output the pass normalised (ssdk_trainer_read_bn_input); mmean, mvar: the moving statistics read
    before the pass.  stats: {'mean': moving mean after the pass, 'var': moving variance}.  perturb: ('acc',) the accumulator of
    the previous pass (whose input was z_prev) is not cleared, so its sums are added in; ('biased',) the moving average takes the
    biased variance; ('no_eps',) rstd = 1 / sqrt(var)."""
    z = _f64(z)
    axes = tuple(range(z.ndim - 1))
    N = float(np.prod(z.shape[:-1]))
    gm, bt, e, mom = _f64(gamma), _f64(beta), float(np.float32(eps)), float(np.float32(momentum))
    mm, mv = _f64(mmean), _f64(mvar)

    def run(p=None):
        s1, s2 = z.sum(axes), (z * z).sum(axes)
        if p == ('acc',):
            zp = _f64(z_prev)
            s1, s2 = s1 + zp.sum(axes), s2 + (zp * zp).sum(axes)
        mean = s1 / N
        var = np.maximum(s2 / N - mean * mean, 0.0)
        rstd = 1.0 / np.sqrt(var + (0.0 if p == ('no_eps',) else e))
        y = gm * (z - mean) * rstd + bt
        a = np.maximum(y, 0.0) if act == 'relu' else np.where(y > 0, y, np.expm1(np.minimum(y, 0.0))) if act == 'elu' else y
        unb = var if p == ('biased',) else var * N / (N - 1.0) if N > 1 else var
        return a, {'mean': mom * mm + (1.0 - mom) * mean, 'var': mom * mv + (1.0 - mom) * unb}, mean, var, rstd
    a, stats, mean, var, rstd = run()
    ez2 = (z * z).mean(axes)
    r = (N + 4) * 2.0 ** -53 * (ez2 + 2 * np.abs(mean) * np.abs(z).mean(axes)) / (var + e) / 2
    X = (np.abs(z - mean) + np.abs(mean)) * rstd
    kap = 8 * U32
    A = np.abs(gm) * X * (1.0 + r / kap) + np.abs(bt) + (2 * U32 / kap) * np.abs(a)
    unb = var * N / (N - 1.0) if N > 1 else var
    sb = {'mean': kap * (np.abs(mom * mm) + (1.0 - mom) * np.abs(mean)) + UNIT['f32'] * np.abs(stats['mean']),
          'var': kap * (np.abs(mom * mv) + (1.0 - mom) * unb * (1.0 + 2 * r / kap)) + UNIT['f32'] * np.abs(stats['var'])}
    out = {}
    for p in perturb:
        ap, sp = run(p)[:2]
        out[p] = (ap, sp)
    return a, A, kap, stats, sb, out


def l2norm_fwd_ref(x, gamma, perturb=()):
    """L2Normalization forward (l2norm_kernel, l2norm8_kernel) -> (y_ref, kappa * |y_ref|, {perturbation: y'}), float64; add
    unit |y_ref| of the store (section 9).  x: the layer's input as stored (hi + lo).  perturb: ('no_gamma',);
    ('gamma_shift',) channel c takes gamma[c + 1]; ('gamma_at', c) only channel c takes gamma[c + 1]."""
    x = _f64(x)
    gm = _f64(gamma)
    Cc = x.shape[-1]
    s = 1.0 / np.sqrt(np.maximum((x * x).sum(-1, keepdims=True), float(np.float32(1e-12))))
    y = x * s * gm
    out = {}
    for p in perturb:
        if p == ('no_gamma',):
            out[p] = x * s
        elif p == ('gamma_shift',):
            out[p] = x * s * np.roll(gm, -1)
        elif p[0] == 'gamma_at':
            g2 = gm.copy()
            g2[p[1]] = gm[(p[1] + 1) % Cc]
            out[p] = x * s * g2
    return y, ((Cc + 1) / 2.0 + 8) * U32 * np.abs(y), out


def pool_fwd_ref(hi, lo, KH, KW, stride, pad_t, pad_l, Ho, Wo, perturb=()):
    """Max-pool forward (maxpool_kernel, maxpool2x2_kernel), bit-exact -> (hi_out, lo_out, {perturbation: (hi', lo')}), float32.

    hi, lo: the input planes' values (B,H,W,C) (lo None in bf16 mode).  Each output takes both planes of the FIRST maximum of
    hi + lo in its window (row-major scan, strict '>', taps outside the input skipped: TF 'same' padding).  perturb: ('hi_only',)
    compares hi alone; ('lo_tie',) keeps the hi plane but takes lo from the last tap whose hi is the window's largest hi."""
    hi = np.asarray(hi, np.float32)
    lo = np.zeros_like(hi) if lo is None else np.asarray(lo, np.float32)
    v = hi.astype(np.float64) + lo
    B, H, W, Cc = hi.shape
    bi, ci = np.meshgrid(np.arange(B), np.arange(Cc), indexing='ij')
    res = {k: (np.zeros((B, Ho, Wo, Cc), np.float32), np.zeros((B, Ho, Wo, Cc), np.float32)) for k in [None] + list(perturb)}
    for yo in range(Ho):
        for xo in range(Wo):
            pos = [(y, xx) for y in range(yo * stride - pad_t, yo * stride - pad_t + KH) if 0 <= y < H
                   for xx in range(xo * stride - pad_l, xo * stride - pad_l + KW) if 0 <= xx < W]
            py, px = np.array([p[0] for p in pos]), np.array([p[1] for p in pos])

            def pick(vals, last=False):
                win = np.stack([vals[:, y, xx] for y, xx in pos], axis=-1)
                k = win.shape[-1] - 1 - np.argmax(win[..., ::-1], axis=-1) if last else np.argmax(win, axis=-1)
                return (bi, py[k], px[k], ci)
            first = pick(v)
            for key, (ho, lo_) in res.items():
                if key == ('hi_only',):
                    at = pick(hi.astype(np.float64))
                    ho[:, yo, xo], lo_[:, yo, xo] = hi[at], lo[at]
                elif key == ('lo_tie',):
                    ho[:, yo, xo], lo_[:, yo, xo] = hi[first], lo[pick(hi.astype(np.float64), last=True)]
                else:
                    ho[:, yo, xo], lo_[:, yo, xo] = hi[first], lo[first]
    out = res.pop(None)
    return out[0], out[1], res


def preprocess_ref(img, mean=None, std=None, swap=None):
    """The input layer (preprocess_kernel), bit-exact -> (hi, lo) float32 (B,H,W,3): t = x - mean, t = t / std in fp32 (each
    correctly rounded), output channel c = t[swap[c]], split into the two planes."""
    x = np.asarray(img, np.float32)
    t = x - (np.zeros(3, np.float32) if mean is None else np.asarray(mean, np.float32))
    if std is not None:
        t = (t / np.asarray(std, np.float32)).astype(np.float32)
    t = t[..., list(swap) if swap is not None else [0, 1, 2]]
    return split(t)


# ------------------------------------------------------------------------------------------------------------------------------
# the SSD loss (section 11)
# ------------------------------------------------------------------------------------------------------------------------------
LOSS_PERTURBATIONS = ('drop_last', 'add_next', 'tie_reverse', 'per_image', 'signed_zero', 'no_max1', 'no_alpha', 'loc_by_yt0',
                      'no_upstream', 'local_B', 'k_no_cap')
_SLACK = 1.0 + 2.0 ** -20


def okey(x):
    """The selection's order key of float32 values (okey of csrc/loss.cu): a larger value has a larger key; -0 and +0 share
    0x80000000."""
    x = np.ascontiguousarray(x, np.float32)
    b = x.view(np.uint32)
    k = np.where(b & np.uint32(0x80000000), ~b, b | np.uint32(0x80000000)).astype(np.uint32)
    return np.where(x == 0, np.uint32(0x80000000), k).astype(np.uint32)


def loss_box_ref(y_true, y_pred):
    """Per-box float64 references and bounds -> (cls, cls_bound, loc, loc_bound), each (B, P) (section 11)."""
    yt, yp = _f64(y_true), _f64(y_pred)
    C = yt.shape[-1] - 12
    tv = yt[..., :C]
    nz = tv != 0
    terms = np.where(nz, tv * np.log(np.maximum(yp[..., :C], float(np.float32(1e-15)))), 0.0)
    cls = -terms.sum(-1)
    cls_b = (nz.sum(-1) + 2) * U32 * np.abs(terms).sum(-1) * _SLACK
    d = yt[..., C:C + 4] - yp[..., C:C + 4]
    ad = np.abs(d)
    loc = np.where(ad < 1.0, 0.5 * d * d, ad - 0.5).sum(-1)
    loc_b = (U32 * (ad * np.minimum(ad, 1.0)).sum(-1) + 4 * U32 * loc) * _SLACK
    return cls, cls_b, loc, loc_b


def _order(v, signed_zero=False):
    """Flat indices by value descending, then index ascending (tf.nn.top_k); signed_zero orders -0 below +0."""
    v = np.ascontiguousarray(v, np.float32).reshape(-1)
    if signed_zero:
        b = v.view(np.uint32)
        key = np.where(b & np.uint32(0x80000000), ~b, b | np.uint32(0x80000000)).astype(np.int64)
    else:
        key = okey(v).astype(np.int64)
    return np.lexsort((np.arange(v.size), -key))


def loss_select(negl, n_pos, ratio, n_neg_min, perturb=None, img_pos=None):
    """The hard-negative mask over the batch -> (mask (B, P) bool, stats [n_pos, nnz, k, want]).  perturb: one selection
    perturbation of LOSS_PERTURBATIONS or None (the stats stay those of the exact selection, except k for 'k_no_cap');
    img_pos: per-image n_pos for 'per_image'."""
    negl = np.ascontiguousarray(negl, np.float32)
    B, P = negl.shape
    flat = negl.reshape(-1)
    nnz = int(np.count_nonzero(flat))
    k = min(max(int(ratio) * int(n_pos), int(n_neg_min)), nnz)
    mask = np.zeros(flat.size, bool)
    stats = [int(n_pos), nnz, 0, 0]
    if k > 0:
        order = _order(flat)
        mask[order[:k]] = True
        ties = np.flatnonzero(okey(flat) == okey(flat[order[k - 1]]))
        stats[2:] = [k, int(mask[ties].sum())]
    if perturb == 'drop_last' and k > 0:
        mask[order[k - 1]] = False
    elif perturb == 'add_next' and k < flat.size:
        mask[_order(flat)[k]] = True
    elif perturb == 'tie_reverse' and k > 0:
        mask[ties] = False
        mask[ties[ties.size - stats[3]:]] = True
    elif perturb == 'signed_zero' and k > 0:
        mask[:] = False
        mask[_order(flat, signed_zero=True)[:k]] = True
    elif perturb == 'k_no_cap':
        kk = min(max(int(ratio) * int(n_pos), int(n_neg_min)), flat.size)
        mask[:] = False
        mask[_order(flat)[:kk]] = True
        stats[2] = kk
    elif perturb == 'per_image':
        mask[:] = False
        for b in range(B):
            vb = flat[b * P:(b + 1) * P]
            kb = min(max(int(ratio) * int(img_pos[b]), int(n_neg_min)), int(np.count_nonzero(vb)))
            mask[b * P + _order(vb)[:kb]] = True
    return mask.reshape(B, P), stats


def loss_ref(y_true, y_pred, cls, negl, ratio=3, n_neg_min=0, alpha=1.0, upstream=None, global_B=None, local_B=None, perturb=()):
    """The SSD loss of one fused call (or of the whole batch of a phase-wise run) from the kernel's own per-box losses
    (section 11) -> (ref, bound, {perturbation: ref'}).

    ref: {'mask': (B, P) bool, 'stats': [n_pos, nnz, k, want], 'loss': (B,), 'grad': (B, P, C+12), 'cls': (B, P)}, float64;
    bound: {'cls', 'loss', 'grad'} of the same shapes.  cls, negl: the kernel's (B, P) float32 arrays (their consistency,
    negl == fl(cls * yt0), is the caller's check).  upstream: (B,) float32 or None (fp32(1 / global_B)); global_B: the batch
    size of the normalisation (default B); local_B: one rank's B, for the 'local_B' perturbation.  perturb: names of
    LOSS_PERTURBATIONS: the mask without its last kept box / with the first unkept one, ties kept from the highest index, top-k
    per image, -0 below +0, no max(1, n_pos), alpha = 1, the loc term weighted by yt0, upstream ignored, local_B for global_B,
    k not capped at nnz."""
    yt, yp = np.asarray(y_true, np.float32), np.asarray(y_pred, np.float32)
    B, P, W = yt.shape
    C = W - 12
    gB = B if global_B is None else int(global_B)
    cls_k = _f64(cls)
    cls_ref, cls_b, loc, loc_b = loss_box_ref(yt, yp)
    pmax = _f64(yt[..., 1:C].max(-1))
    n_pos_f = float(np.float32(np.sum(pmax)))
    img_pos = [int(np.float32(pmax[b].sum())) for b in range(B)]
    a32 = float(np.float32(alpha))
    tv, q = _f64(yt[..., :C]), _f64(yp[..., :C])
    live = (tv != 0) & (q >= float(np.float32(1e-15)))
    dlog = np.where(live, -tv / np.where(live, q, 1.0), 0.0)
    d = _f64(yp[..., C:C + 4]) - _f64(yt[..., C:C + 4])
    slope = np.clip(d, -1.0, 1.0)

    def run(p=None):
        sel = p if p in ('drop_last', 'add_next', 'tie_reverse', 'per_image', 'signed_zero', 'k_no_cap') else None
        mask, stats = loss_select(negl, int(n_pos_f), ratio, n_neg_min, sel, img_pos)
        den = n_pos_f if p == 'no_max1' else max(1.0, n_pos_f)
        inv = float(np.float32(1.0) / np.float32(den)) if den else np.inf
        nb = local_B if p == 'local_B' else gB
        al = 1.0 if p == 'no_alpha' else a32
        wl = _f64(yt[..., 0]) if p == 'loc_by_yt0' else pmax
        if upstream is None or p == 'no_upstream':
            up = np.full(B, float(np.float32(1) / np.float32(nb)))
        else:
            up = _f64(upstream)
        with np.errstate(invalid='ignore'):
            tot = ((cls_k * pmax).sum(-1) + (cls_k * mask).sum(-1) + al * (loc * wl).sum(-1)) * inv * nb
            scale = (up * nb * inv)[:, None]
            g = np.zeros((B, P, W))
            g[..., :C] = dlog * ((pmax + mask) * scale)[..., None]
            g[..., C:C + 4] = slope * (wl * scale * al)[..., None]
        return {'mask': mask, 'stats': stats, 'loss': tot, 'grad': g, 'cls': cls_ref}
    ref = run()
    inv = float(np.float32(1.0) / np.float32(max(1.0, n_pos_f)))
    cp = np.abs(cls_k * pmax)
    lp = loc * pmax
    s_abs = cp.sum(-1) + (np.abs(cls_k) * ref['mask']).sum(-1) + abs(a32) * lp.sum(-1)
    e = U32 * cp.sum(-1) + abs(a32) * (pmax * (loc_b + U32 * (loc + loc_b))).sum(-1) + (P + 8) * 2.0 ** -53 * s_abs
    bnd = {'cls': cls_b, 'loss': e * inv * gB * _SLACK + UNIT['f32'] * np.abs(ref['loss']),
           'grad': 6 * U32 * _SLACK * np.abs(ref['grad'])}
    return ref, bnd, {p: run(p) for p in perturb}


def loss_ratio(got, ref, bnd):
    """max |got - ref| / bound; equal values pass a zero bound, and a NaN or an infinite difference is an infinite ratio."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape == bnd.shape, (got.shape, ref.shape, bnd.shape)
    with np.errstate(invalid='ignore', divide='ignore', over='ignore'):
        d = np.abs(got - ref)
        r = np.where(d == 0, 0.0, d / np.maximum(bnd, np.finfo(np.float64).tiny))
    r = np.where(np.isnan(r), np.inf, r)
    return float(r.max()) if r.size else 0.0
