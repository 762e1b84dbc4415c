"""oracle/mask_chain.py — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Float64 restatement, with per-pixel certainty, of the library calls that decide the reference's segmentation pixels:

    instance masks   deformable_detr_segm_vl.py:569-610
      mask = F.interpolate(mask_pred, padded, "bilinear", align_corners=False).sigmoid() > 0.5
      BitMasks(mask).crop_and_resize(boxes, 128)       torchvision roi_align(aligned=True, scale 1, sampling_ratio 0) >= 0.5
      paste_masks_in_image(masks, boxes, out, 0.5)     detectron2 _do_paste_mask: grid_sample(bilinear, zeros,
                                                       align_corners=False) >= 0.5  (detector_postprocess)
    panoptic maps    deformable_detr_segm_vl.py:919-998 with detectron2 sem_seg_postprocess
      p = sigmoid(resize2(crop(resize1(logit))));  id = first argmax_k score_k * p_k;  solid = p_id >= prob;  three areas.

Torch tensors throughout, so the same code runs on the host in CPU tests and on the device in GPU tests.  Every resample is
separable, so each stage is a product of small weight matrices: W_y @ plane @ W_x^T.

Discrete quantities are the reference's fp32 expressions: the scales in / out, roi_align's grid count ceil(roi / S), its
"sample outside the image" test and its sample count.  Continuous values (lambdas, bilinear sums, roi averages, sigmoid,
score * p) are float64.  The integer part of a source coordinate enters only a bilinear value, which is continuous in the
coordinate, so the weights are formed at the exact coordinate and the fp32 rounding of the coordinate goes into the band.

Each thresholded stage returns (decision, certain).  A value is certain when it lies outside a band around the threshold;
the band is a bound on |fp32 value - float64 value| built from its causes (u = 2^-24, the fp32 unit roundoff):
  * coordinates: e = bound on the fp32 rounding of a source coordinate (upsample: 2u * scale * (dst + 0.5); roi_align sample:
    8u * (|y1| + |y2| + 1); paste: u * (S * (6|q| + 3) + |i| + 1) with q the box-relative position, i the grid coordinate),
    times the largest difference of neighbouring taps within two texels of the sample (G below);
  * sums: a few ulps of sum |w * t| (upsample 4u sum |w t|, roi_align (n + 8) u per summed value, paste 12u);
  * panoptic: resize1 and resize2 coordinates as above (a resize2 coordinate error moves the resize1 map by scale1 times
    the logit slope), 10u * sum |w * t| for the two resamples and the fp32 resize1 map the reference stores, and
    p (1 - p) band e^band (sigmoid' changes by at most e^|dv|) + 8u * p + 2^-140 for the sigmoid (p = 0 exactly where fp32 expf(-v) overflows), u * s
    for score * p.
A pixel has band 0 only when no evaluation order can round: its source coordinates are exact in fp32, every weight is a
multiple of 2^-kw and every tap of 2^-kt, and the largest partial sum a bilinear or roi sum can reach (max |t| for a
resample, the sample count for roi_align) is below 2^(24 - kw - kt).  Then every product and every partial sum, in any order
and with or without fused multiply-adds, is a multiple of 2^-(kw + kt) below 2^(24 - kw - kt) in magnitude, which fp32 holds
exactly (`_exact_in_fp32`).  The dyadic constructors below make such pixels, which is what lets exact ties (a value exactly
on the threshold, two equal scores) be certain.

Uncertainty propagates by interval arithmetic: every stage is monotone with non-negative weights, so the next stage runs with
the uncertain bits as 0 (lo) and as 1 (hi), and a pixel is certain only if both fall on the same side outside the band."""
import math

import numpy as np
import torch
import torch.nn.functional as F

U = 2.0 ** -24
F64 = torch.float64
F32 = torch.float32


# ---- shared pieces --------------------------------------------------------------------------------------------------------
def _slope_bound(lo, hi, axis, pad):
    """A bound on |t[i + 1] - t[i]| along `axis` within two cells of every point, for any plane t with lo <= t <= hi
    ([..., H, W]); pad: the plane is zero outside (grid_sample) rather than clamped (upsample, roi_align), so the first and last
    cells are the steps to zero."""
    if pad:
        lo, hi = F.pad(lo, (1, 1, 1, 1)), F.pad(hi, (1, 1, 1, 1))
    n = lo.shape[axis] - 1

    def step(a, b):
        return (a.narrow(axis, 1, n) - b.narrow(axis, 0, n)).abs()

    d = torch.maximum(step(hi, lo), step(lo, hi))
    d = F.pad(d, (0, 1) if axis == -1 else (0, 0, 0, 1))
    return F.max_pool2d(d.reshape(-1, 1, *d.shape[-2:]), 5, 1, 2).reshape(d.shape)


def _dyadic_exp(x, kmax=48):
    """The least k <= kmax such that every value of x is a multiple of 2^-k, or None."""
    x = x.detach().double().flatten()
    if x.numel() == 0:
        return 0
    if not torch.isfinite(x).all():
        return None
    for k in range(kmax + 1):
        if ((x * 2.0 ** k).frac() == 0).all():
            return k
    return None


def _exact_in_fp32(largest, *exps):
    """True when sums whose terms are products of multiples of 2^-k (k in exps) and whose partial sums stay within `largest` in
    magnitude are exact in fp32 in every order."""
    if any(k is None for k in exps):
        return False
    return float(largest) * 2.0 ** sum(exps) < 2.0 ** 24


def _f32(x):
    return torch.as_tensor(x, dtype=F32)


def _resize_axis(in_size, out_size, device):
    """upsample_bilinear2d (align_corners=False) along one axis: (A [out, in], e [out], scale, kw).  src = max(scale *
    (dst + 0.5) - 0.5, 0) with scale the fp32 in / out; e = 0 where the fp32 source coordinate is exact; kw: the dyadic
    exponent of the lambdas of those exact rows."""
    scale = float(np.float32(in_size) / np.float32(out_size))
    d = torch.arange(out_size, dtype=F64, device=device) + 0.5
    p64 = scale * d  # exact: 24 x 17 bits
    p32 = _f32(scale).to(device) * d.to(F32)
    src64 = (p64 - 0.5).clamp(min=0.0)
    src32 = (p32 - 0.5).clamp(min=0.0)
    exact = (p32.double() == p64) & (src32.double() == src64)
    e = torch.where(exact, torch.zeros_like(p64), 2 * U * p64)
    i0 = src64.floor()
    l1 = src64 - i0
    l0 = 1 - l1
    i0 = i0.long()
    i1 = torch.where(i0 < in_size - 1, i0 + 1, i0)
    A = torch.zeros((out_size, in_size), dtype=F64, device=device)
    r = torch.arange(out_size, device=device)
    A.index_put_((r, i0), l0, accumulate=True)
    A.index_put_((r, i1), l1, accumulate=True)
    return A, e, scale, _dyadic_exp(l1[exact])


def _mm3(a, t, b):
    """a @ t @ b^T for t [..., H, W]."""
    return torch.matmul(torch.matmul(a, t), b.transpose(-1, -2))


def _certain_ge(lo, hi, band, thr, strict=False):
    """(decision, certain) of `value >= thr` (or `> thr`) for a value known to lie in [lo - band, hi + band]."""
    if strict:
        on, off = lo - band > thr, hi + band <= thr
    else:
        on, off = lo - band >= thr, hi + band < thr
    return on, on | off


# ---- stage 1: F.interpolate to the padded size, sigmoid > 0.5 (as logit > 0) ----------------------------------------------
def binarize(planes, padded_hw):
    """planes [K, h, w] (any float dtype) -> (on, certain) bool [K, Hp, Wp]: bilinear upsample > 0."""
    K, h, w = planes.shape
    Hp, Wp = padded_hw
    dev = planes.device
    Ay, ey, _, ky = _resize_axis(h, Hp, dev)
    Ax, ex, _, kx = _resize_axis(w, Wp, dev)
    on = torch.empty((K, Hp, Wp), dtype=torch.bool, device=dev)
    cert = torch.empty_like(on)
    exact_coord = (ey == 0)[:, None] & (ex == 0)[None, :]
    for k in range(K):
        L = planes[k].to(F64)
        v = _mm3(Ay, L, Ax)
        band = (ey[:, None] * _mm3(Ay, _slope_bound(L, L, -2, False), Ax) + ex[None, :] * _mm3(Ay, _slope_bound(L, L, -1, False), Ax)
                + 4 * U * _mm3(Ay, L.abs(), Ax))
        if _exact_in_fp32(L.abs().max(), ky, kx, _dyadic_exp(L)):
            band = torch.where(exact_coord, torch.zeros_like(band), band)
        on[k], cert[k] = _certain_ge(v, v, band, 0.0, strict=True)
    return on, cert


# ---- stage 2: roi_align(aligned=True, spatial_scale 1, sampling_ratio 0) >= 0.5 -----------------------------------------
def _roi_axis(a, b, S, size, device):
    """One axis of torchvision roi_align for the box edges a < b (fp32 values): (W [S, size]: the bilinear weights of the
    samples that are inside, summed over the grid; W_hi: also the samples within rounding of the outside test; We: W_hi with
    every sample weighted by its coordinate error; grid count g; the dyadic exponent of the lambdas when every sample coordinate
    is exact in fp32, else None)."""
    a32, b32 = np.float32(a), np.float32(b)
    start32 = np.float32(a32 - np.float32(0.5))
    roi32 = np.float32(np.float32(b32 - np.float32(0.5)) - start32)
    bin32 = np.float32(roi32 / np.float32(S))
    g = int(math.ceil(float(np.float32(roi32 / np.float32(S)))))
    n = max(g, 0)
    ph = torch.arange(S, device=device, dtype=F64)[:, None]
    iy = torch.arange(n, device=device, dtype=F64)[None, :] + 0.5
    # the reference's fp32 expression: start + ph * bin + (iy + .5) * bin / g
    t1 = _f32(bin32).to(device) * ph.to(F32)
    t2 = (iy.to(F32) * _f32(bin32).to(device)) / _f32(float(max(g, 1))).to(device)
    y32 = (_f32(start32).to(device) + t1) + t2
    t1_64 = float(bin32) * ph
    t2_64 = (iy * float(bin32)) / float(max(g, 1))
    y64 = (float(start32) + t1_64) + t2_64
    exact = ((t1.double() == t1_64) & (t2.double() == t2_64) & (y32.double() == y64) & (float(a32) - 0.5 == float(start32))
             & (float(b32) - float(a32) == float(roi32)) & (float(roi32) / S == float(bin32)))
    # the exact value (from the fp32 box) and a bound on the fp32 rounding of it
    yx = (float(a32) - 0.5) + (float(b32) - float(a32)) * ((ph + iy / max(g, 1)) / S)
    e = torch.where(exact, torch.zeros_like(yx), torch.full_like(yx, 8 * U * (abs(float(a32)) + abs(float(b32)) + 1)))
    outside = (y32 < -1) | (y32 > size)
    unsure = ~exact & (((yx + 1).abs() <= e) | ((yx - size).abs() <= e))
    y = yx.clamp(min=0.0)
    low = y.floor().clamp(max=size - 1)
    y = torch.where(low >= size - 1, low, y)
    l1 = y - low
    low = low.long()
    high = torch.where(low >= size - 1, low, low + 1)
    rows = torch.arange(S, device=device)[:, None].expand_as(low)

    def mat(keep, scale=None):
        W = torch.zeros((S, size), dtype=F64, device=device)
        w0, w1 = (1 - l1) * keep, l1 * keep
        if scale is not None:
            w0, w1 = w0 * scale, w1 * scale
        W.index_put_((rows, low), w0, accumulate=True)
        W.index_put_((rows, high), w1, accumulate=True)
        return W

    keep_lo = (~outside & ~unsure).to(F64)
    keep_hi = (~outside | unsure).to(F64)
    return mat(keep_lo), mat(keep_hi), mat(keep_hi, e), g, _dyadic_exp(l1) if bool(exact.all()) else None


def roi_align(on, cert, boxes, S):
    """on, cert bool [K, Hp, Wp] (binarize) and boxes fp32 [K, 4] -> (on, certain) bool [K, S, S]."""
    K, Hp, Wp = on.shape
    dev = on.device
    out_on = torch.empty((K, S, S), dtype=torch.bool, device=dev)
    out_cert = torch.empty_like(out_on)
    bx = boxes.detach().to("cpu", F32).numpy()
    for k in range(K):
        B_lo = (on[k] & cert[k]).to(F64)
        B_hi = (on[k] | ~cert[k]).to(F64)
        x1, y1, x2, y2 = (float(v) for v in bx[k])
        Wy_lo, Wy_hi, Wy_e, gh, ky = _roi_axis(y1, y2, S, Hp, dev)
        Wx_lo, Wx_hi, Wx_e, gw, kx = _roi_axis(x1, x2, S, Wp, dev)
        count = float(max(gh * gw, 1))
        acc_lo = _mm3(Wy_lo, B_lo, Wx_lo)
        acc_hi = _mm3(Wy_hi, B_hi, Wx_hi)
        Gy, Gx = _slope_bound(B_lo, B_hi, -2, False), _slope_bound(B_lo, B_hi, -1, False)
        n = max(gh, 0) * max(gw, 0)
        band = _mm3(Wy_e, Gy, Wx_hi) + _mm3(Wy_hi, Gx, Wx_e) + (n + 8) * U * (acc_hi + n)
        # exact sample coordinates, and sums of up to n bits times weights in multiples of 2^-(ky + kx): no rounding
        exact = (acc_lo == acc_hi) & _exact_in_fp32(max(n, 1), ky, kx)
        avg = acc_lo / count
        exact = exact & (avg * count == acc_lo) & (avg.to(F32).double() == avg)  # an exact quotient: no rounding either
        band = torch.where(exact, torch.zeros_like(band), band / count + U * acc_hi / count)
        out_on[k], out_cert[k] = _certain_ge(acc_lo / count, acc_hi / count, band, 0.5)
    return out_on, out_cert


def crop_and_resize(planes, boxes, padded_hw, S):
    """BitMasks(interpolate(planes, padded).sigmoid() > 0.5).crop_and_resize(boxes, S): (on, certain) bool [K, S, S]."""
    return roi_align(*binarize(planes, padded_hw), boxes, S)


# ---- stage 3: detectron2 paste_masks_in_image (grid_sample, zeros padding, align_corners=False) >= threshold -------------
def _paste_axis(a, b, n, S, device):
    """One axis of _do_paste_mask for box edges a, b (fp32) over n output pixels: (W [n, S + 2], the bilinear weights on the
    zero-padded mask (tap -1 .. S), e [n], and the dyadic exponent of the weights of the rows whose coordinate is exact)."""
    a32, b32 = _f32(float(a)).to(device), _f32(float(b)).to(device)
    y = torch.arange(n, device=device, dtype=F64)
    t32 = (y.to(F32) + 0.5) - a32
    den32 = b32 - a32
    q32 = t32 / den32
    g32 = q32 * 2 - 1
    i32 = ((g32 + 1) * S - 1) / 2
    t64 = (y + 0.5) - float(a32)
    den64 = float(b32) - float(a32)
    finite = torch.isfinite(i32) & (den64 != 0)
    q64 = t64 / den64 if den64 != 0 else torch.full_like(t64, float("nan"))
    g64 = q64 * 2 - 1
    i64 = ((g64 + 1) * S - 1) / 2
    exact = ((t32.double() == t64) & (float(den32) == den64) & (q32.double() == q64) & (q64 * den64 == t64) & (g32.double() == g64)
             & (i32.double() == i64))
    e = torch.where(exact, torch.zeros_like(t64), U * (S * (6 * q64.abs() + 3) + i64.abs() + 1))
    i = torch.where(finite, i64, torch.full_like(i64, -10.0))  # non-finite coordinates sample nothing
    f = i.floor()
    w1 = i - f
    w0 = (f + 1) - i
    f = f.long() + 1  # padded tap index of the "north" / "west" tap
    inside0 = (f >= 0) & (f <= S + 1)
    inside1 = (f + 1 >= 0) & (f + 1 <= S + 1)
    W = torch.zeros((n, S + 2), dtype=F64, device=device)
    r = torch.arange(n, device=device)
    W.index_put_((r[inside0], f[inside0]), w0[inside0], accumulate=True)
    W.index_put_((r[inside1], f[inside1] + 1), w1[inside1], accumulate=True)
    e = torch.where(finite, e, torch.zeros_like(e))
    return W, e, _dyadic_exp(w1[finite & exact])


def paste(on, cert, boxes, out_hw, threshold=0.5, rows=None):
    """on, cert bool [N, S, S] and boxes fp32 [N, 4] (output pixels) -> (on, certain) bool [N, H, W] (rows: only these output
    rows, a slice)."""
    N, S, _ = on.shape
    H, W = out_hw
    dev = on.device
    r0, r1 = (0, H) if rows is None else (rows.start, rows.stop)
    out_on = torch.empty((N, r1 - r0, W), dtype=torch.bool, device=dev)
    out_cert = torch.empty_like(out_on)
    bx = boxes.detach().to("cpu", F32).numpy()
    for k in range(N):
        x1, y1, x2, y2 = (float(v) for v in bx[k])
        Wy, ey, ky = _paste_axis(y1, y2, r1, S, dev)
        Wx, ex, kx = _paste_axis(x1, x2, W, S, dev)
        Wy, ey = Wy[r0:], ey[r0:]
        M_lo = F.pad((on[k] & cert[k]).to(F64), (1, 1, 1, 1))
        M_hi = F.pad((on[k] | ~cert[k]).to(F64), (1, 1, 1, 1))
        v_lo = _mm3(Wy, M_lo, Wx)
        v_hi = _mm3(Wy, M_hi, Wx)
        m_lo, m_hi = M_lo[1:-1, 1:-1], M_hi[1:-1, 1:-1]
        band = (ey[:, None] * _mm3(Wy, _slope_bound(m_lo, m_hi, -2, True), Wx)
                + ex[None, :] * _mm3(Wy, _slope_bound(m_lo, m_hi, -1, True), Wx) + 12 * U)
        # taps of 0 / 1 and partial sums of at most 1
        exact = (ey == 0)[:, None] & (ex == 0)[None, :] & (v_lo == v_hi) & _exact_in_fp32(1, ky, kx)
        band = torch.where(exact, torch.zeros_like(band), band)
        out_on[k], out_cert[k] = _certain_ge(v_lo, v_hi, band, threshold)
    return out_on, out_cert


# ---- panoptic: per-pixel winners and the three areas -------------------------------------------------------------------
def _panoptic_axis(in_size, padded, img, out, dev):
    """R [out, in] = resize2 (img -> out) after resize1 (in -> padded) cropped to img, and E [out, in]: R weighted by the
    coordinate errors (resize1's, and resize2's times scale1); exact [out]: the output rows read only exact coordinates of both
    resizes; k: the dyadic exponent of their weights (resize1's plus resize2's)."""
    A1, e1, s1, k1 = _resize_axis(in_size, padded, dev)
    A2, e2, _, k2 = _resize_axis(img, out, dev)
    A1c = A1[:img]
    R = A2 @ A1c
    E = A2 @ (e1[:img, None] * A1c) + (s1 * e2)[:, None] * R
    exact = (e2 == 0) & ((A2 != 0).to(F64) @ (e1[:img] != 0).to(F64) == 0)
    return R, E, None if k1 is None or k2 is None else k1 + k2, exact


def panoptic(logits, index, scores, padded_hw, img_hw, out_hw, prob, chunk=1 << 24):
    """ops.panoptic_winners' quantities in float64 with certainty.  logits [Q, h, w]; index int64 [K]; scores fp32 [K] (-inf:
    the query takes no part).  Returns a dict:
      ids int64 [oh, ow] (the float64 decision, -1 where not solid), ids_certain bool [oh, ow],
      lo, hi int64 [3, K] (bounds of mask_area, inter_area, original_area), count int64 [3, K] (the float64 decisions),
      unsure_pairs int, unsure_pixels int."""
    dev = logits.device
    K = int(index.numel())
    h, w = logits.shape[1:]
    oh, ow = out_hw
    Ry, Ey, ky, exy = _panoptic_axis(h, padded_hw[0], img_hw[0], oh, dev)
    Rx, Ex, kx, exx = _panoptic_axis(w, padded_hw[1], img_hw[1], ow, dev)
    sc = scores.detach().to(dev, F32).double()
    live = sc != float("-inf")
    idx = index.to(dev).long()
    # duplicates: the same plane and the same score give the kernel bit-identical values, and the lower index wins
    first = {}
    gid = torch.tensor([first.setdefault(key, k) for k, key in enumerate(zip(idx.tolist(), sc.tolist()))], dtype=torch.long,
                       device=dev)
    L = logits[idx].to(F64)
    Gy = _slope_bound(L, L, -2, False) if K else L
    Gx = _slope_bound(L, L, -1, False) if K else L
    # both resamples and the stored resize1 map: every partial sum is within max |L|
    exact_sums = K > 0 and _exact_in_fp32(L.abs().max(), ky, kx, _dyadic_exp(L))
    ids = torch.full((oh, ow), -1, dtype=torch.long, device=dev)
    ids_c = torch.ones((oh, ow), dtype=torch.bool, device=dev)
    lo = torch.zeros((3, K), dtype=torch.long, device=dev)
    hi = torch.zeros_like(lo)
    count = torch.zeros_like(lo)
    pairs = 0
    step = max(1, min(oh, chunk // max(K * ow, 1)))
    kk = torch.arange(K, device=dev)[:, None, None]
    any_live = bool(live.any())
    for y0 in range(0, oh, step if any_live else oh):
        y1 = min(oh, y0 + step)
        if not any_live:
            break
        v = _mm3(Ry[y0:y1], L, Rx)
        band = _mm3(Ey[y0:y1], Gy, Rx) + _mm3(Ry[y0:y1], Gx, Ex) + 10 * U * _mm3(Ry[y0:y1], L.abs(), Rx)
        if exact_sums:
            band = torch.where(exy[y0:y1, None] & exx[None, :], torch.zeros_like(band), band)
        p = torch.sigmoid(v)
        bp = p * (1 - p) * band * torch.exp(band) + torch.where((band == 0) & (v == 0), 0.0, 8 * U) * p + torch.where(v < -80, 2.0 ** -140, 0.0)
        # fp32 expf(-v) overflows past ln(FLT_MAX) = 88.7228...: p is exactly 0 there, and ties between such queries are real
        sat = v + band < -88.7229
        unsure = ~sat & (v - band < -88.7228)
        bp = torch.where(sat, 0.0, torch.where(unsure, p + bp, bp))
        p = torch.where(sat, 0.0, p)
        s = sc[:, None, None] * p
        bs = sc[:, None, None].clamp(min=0) * bp + torch.where(bp == 0, 0.0, U) * s.abs()
        s = torch.where(live[:, None, None], s, float("-inf"))
        top = s.argmax(0)  # first maximum
        s_top = s.gather(0, top[None])[0]
        b_top = bs.gather(0, top[None])[0]
        rivals = live[:, None, None] & (gid[:, None, None] != top[None])
        beaten = (s_top - b_top > s + bs) | ((b_top == 0) & (bs == 0) & ((s_top > s) | ((s_top == s) & (top < kk))))
        win_c = (~rivals | beaten).all(0)
        cand = live[:, None, None] & (gid[:, None, None] == kk) & ((kk == top[None]) | ~beaten)
        ge, ge_c = _certain_ge(p, p, bp, prob)
        ge = ge & live[:, None, None]
        ge_c = ge_c | ~live[:, None, None]
        p_top_c = ge_c.gather(0, top[None])[0]
        win = kk == top[None]
        ids[y0:y1] = torch.where((p >= prob).gather(0, top[None])[0], top, -1)
        ids_c[y0:y1] = win_c & p_top_c
        unsure_win = (~win_c)[None] & cand
        lo[0] += (win & win_c[None]).flatten(1).sum(1)
        hi[0] += (win & win_c[None]).flatten(1).sum(1) + unsure_win.flatten(1).sum(1)
        lo[1] += (win & win_c[None] & ge & ge_c).flatten(1).sum(1)
        hi[1] += ((win & win_c[None]) | unsure_win).logical_and(ge | ~ge_c).flatten(1).sum(1)
        lo[2] += (ge & ge_c).flatten(1).sum(1)
        hi[2] += (ge | ~ge_c).flatten(1).sum(1)
        count[0] += win.flatten(1).sum(1)
        count[1] += (win & (p >= prob)).flatten(1).sum(1)
        count[2] += ((p >= prob) & live[:, None, None]).flatten(1).sum(1)
        pairs += int(unsure_win.sum()) + int((~ge_c).sum())
    return {"ids": ids, "ids_certain": ids_c, "lo": lo, "hi": hi, "count": count, "unsure_pairs": pairs,
            "unsure_pixels": int((~ids_c).sum())}


def segments(lo, hi, classes, thing_ids, num_thing_classes, stuff_first_is_things, overlap_threshold):
    """The reference's loop over the kept queries (deformable_detr_segm_vl.py:958-995) on area bounds lo, hi [3, K] (mask,
    inter, original): segments_info, or None when some decision (an area > 0, mask_area / original_area < threshold) differs
    between counts within the bounds."""
    thing_ids = set(int(t) for t in thing_ids)
    lo, hi = lo.tolist(), hi.tolist()
    info, stuff, current = [], {}, 0
    for k, c in enumerate(int(c) for c in classes):
        a, i, o = (lo[0][k], hi[0][k]), (lo[1][k], hi[1][k]), (lo[2][k], hi[2][k])
        if any((x[0] > 0) != (x[1] > 0) for x in (a, i, o)):
            return None
        if not (a[0] > 0 and o[0] > 0 and i[0] > 0):
            continue
        low, high = a[0] / o[1] < overlap_threshold, a[1] / o[0] < overlap_threshold
        if low != high:
            return None
        if low:
            continue
        isthing = c in thing_ids
        if not isthing:
            if c in stuff:
                continue
            stuff[c] = current + 1
        current += 1
        if not isthing and stuff_first_is_things:
            c = c - num_thing_classes + 1
        info.append({"id": current, "isthing": bool(isthing), "category_id": int(c)})
    return info


# ---- adversarial inputs, from seeds ----------------------------------------------------------------------------------------
def smooth_logits(Q, h, w, seed, dtype=torch.float32, amp=4.0):
    """[Q, h, w] logits that change sign along smooth curves (bicubic upsample of a coarse normal grid)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(Q, 1, max(h // 8, 1), max(w // 8, 1), generator=g)
    return (F.interpolate(x, size=(h, w), mode="bicubic", align_corners=False)[:, 0] * amp).to(dtype).contiguous()


def edge_boxes(Hp, Wp, S, seed, n=24):
    """fp32 [n, 4] boxes in padded pixels whose edges fall where roi_align goes wrong: integers and half-integers (roi_start =
    x - 0.5 on a texel), roi sizes of exactly m * S and one fp32 ulp above, boxes smaller than a pixel, degenerate boxes
    (x1 == x2, y1 == y2), boxes past the image on every side, boxes that touch only the last row or the last column, the
    whole image, then random boxes with half-integer edges."""
    g = torch.Generator().manual_seed(seed)
    up = lambda v: float(np.nextafter(np.float32(v), np.float32(np.inf)))  # noqa: E731
    b = [[0.0, 0.0, Wp, Hp],                                  # the whole padded image: the largest grid
         [-3.0, -2.5, Wp + 4.0, Hp + 3.5],                    # past the image on every side
         [0.5, 0.5, 0.5 + S, 0.5 + S],                        # roi of exactly S, starting on a texel centre
         [2.0, 1.0, 2.0 + min(2 * S, Wp), 1.0 + min(2 * S, Hp)],  # roi of exactly 2S
         [1.0, 1.0, up(1.0 + S), up(1.0 + S)],                # one ulp above S: the grid count steps to 2
         [3.25, 4.5, 3.75, 4.75],                             # smaller than a pixel
         [5.0, 6.0, 5.0, 30.0],                               # x1 == x2
         [5.0, 6.0, 30.0, 6.0],                               # y1 == y2
         [0.0, Hp - 1.0, Wp, Hp],                             # only the last row
         [Wp - 1.0, 0.0, Wp, Hp],                             # only the last column
         [Wp - 0.5, Hp - 0.5, Wp + 0.5, Hp + 0.5],            # the last texel and past it
         [-1.5, -1.5, 0.5, 0.5]]                              # the first texel and before it
    while len(b) < n:
        c = torch.rand(2, generator=g) * torch.tensor([Wp, Hp])
        wh = (torch.rand(2, generator=g) * torch.tensor([Wp, Hp]) * 0.6 + 1.0)
        lo_, hi_ = ((c - wh / 2) * 2).round() / 2, ((c + wh / 2) * 2).round() / 2
        b.append([float(lo_[0]), float(lo_[1]), float(hi_[0]), float(hi_[1])])
    return torch.tensor(b[:n], dtype=F32)


def dyadic_crop_case(seed=0):
    """Logits, boxes and geometry on which every fp32 operation of interpolate + roi_align is exact: Hp = 4h (scale 1/4, lambdas in
    odd eighths), logits small dyadic values, boxes with half-integer edges and roi sizes of S and 2S (samples on texels or half
    way between them, averages exact).  Plane 0 is all zeros and plane 2 alternates columns of 1/8 and -7/8, so that some
    upsampled values are exactly 0 (they must come out off); plane 1 is a half plane whose box puts samples half way across its
    edge, so that roi averages are exactly 0.5 (they must come out on)."""
    g = torch.Generator().manual_seed(seed)
    h, w, S = 16, 24, 16
    Hp, Wp = 4 * h, 4 * w
    L = (torch.randint(-3, 4, (6, h, w), generator=g).float() / 8)
    L[0] = 0.0
    L[1, :, : w // 2], L[1, :, w // 2:] = 1.0, -1.0   # on up to padded column Wp / 2 - 1, off from Wp / 2
    L[2] = torch.where(torch.arange(w) % 2 == 0, 0.125, -0.875).expand(h, w)  # 7/8 * 1/8 + 1/8 * -7/8 = 0
    L[3] = 1.0
    x1 = Wp / 2 - S / 2 + 0.5
    boxes = torch.tensor([[0.5, 0.5, 0.5 + S, 0.5 + S],
                          [x1, 8.0, x1 + S, 8.0 + S],                        # samples at x = Wp / 2 - 0.5: averages of 0.5
                          [0.0, 0.0, Wp, Hp],
                          [4.5, 2.5, 4.5 + 2 * S, 2.5 + 2 * S],
                          [Wp - S / 2, Hp - S / 2, Wp + S / 2, Hp + S / 2],  # samples exactly on the last texel and past it
                          [-S / 2, -S / 2, S / 2, S / 2]],  # samples exactly on -1
                         dtype=F32)
    return L, boxes, (Hp, Wp), S


def dyadic_paste_case():
    """An all-ones and an all-zeros 128 x 128 mask pasted exactly: a 128-wide box starting at 16.5 puts column 16 at ixf = -0.5 with
    weight exactly 1/2, which must come out on; boxes of 64 and 256 pixels (weights in halves and quarters)."""
    S = 128
    masks = torch.zeros((4, S, S), dtype=torch.bool)
    masks[0] = True
    masks[2] = True
    masks[3, :, : S // 2] = True
    boxes = torch.tensor([[16.5, 16.5, 144.5, 144.5], [16.5, 16.5, 144.5, 144.5], [3.5, 40.0, 259.5, 104.0],
                          [10.0, 10.0, 138.0, 138.0]], dtype=F32)
    return masks, boxes, (160, 272)


def paste_boxes(H, W, seed, n=17):
    """fp32 [n, 4] output-image boxes: the whole image, past every side, degenerate (x1 == x2 and y1 == y2), touching only the
    last row / column, smaller than a pixel, half-integer edges, then random ones."""
    g = torch.Generator().manual_seed(seed)
    b = [[0.0, 0.0, W, H], [-5.0, -5.0, W + 5.0, H + 5.0], [3.0, 2.0, 3.0, H - 1.0], [2.0, 3.0, W - 1.0, 3.0],
         [0.0, H - 1.0, W, H], [W - 1.0, 0.0, W, H], [1.25, 1.5, 1.75, 1.75], [16.5, 0.5, 16.5 + 128, 0.5 + 128]]
    while len(b) < n:
        c = torch.rand(2, generator=g) * torch.tensor([W, H])
        wh = torch.rand(2, generator=g) * torch.tensor([W, H]) * 0.8 + 1.0
        b.append([float(v) for v in torch.cat([c - wh / 2, c + wh / 2])])
    return torch.tensor(b[:n], dtype=F32)


def panoptic_logits(Q, h, w, seed, dtype=torch.float32):
    """Overlapping blobs as mask logits [Q, h, w]."""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(h).float(), torch.arange(w).float(), indexing="ij")
    c = torch.rand(Q, 2, generator=g) * torch.tensor([h, w]).float()
    r = torch.rand(Q, generator=g) * (h / 5) + h / 32
    out = torch.empty(Q, h, w)
    for i in range(0, Q, 64):
        d = ((yy[None] - c[i:i + 64, 0, None, None]) ** 2 + (xx[None] - c[i:i + 64, 1, None, None]) ** 2).sqrt()
        out[i:i + 64] = (r[i:i + 64, None, None] - d) * (75.0 / h) + torch.randn(d.shape, generator=g) * 0.3
    return out.to(dtype)


def panoptic_queries(Q, K, seed):
    """(index int64 [K], scores fp32 [K]): distinct queries, except that query 1 repeats query 0 (same plane, same score) and
    query 2 has the score -inf (it takes no part)."""
    g = torch.Generator().manual_seed(seed)
    index = torch.randperm(Q, generator=g)[:K]
    scores = torch.rand(K, generator=g) * 0.9 + 0.1
    if K >= 2:
        index[1], scores[1] = index[0], scores[0]
    if K >= 3:
        scores[2] = float("-inf")
    return index, scores


def dyadic_panoptic_case():
    """Planes on which resize1, crop and resize2 are exact (Hp = 4h, image = pad / 2, output = image): plane 0 is all zeros, so
    v == 0 and p == 0.5 exactly, solid at prob = 0.5; queries 0 and 1 are that plane with equal scores (query 0 must win), query
    2 a dyadic blob (+2 inside, -2 outside) with a higher score that wins inside it, query 3 a copy of plane 0 with a lower score."""
    h = w = 16
    L = torch.zeros((3, h, w))
    L[1] = -2.0
    L[1, 4:12, 4:12] = 2.0
    L[2, :, 8:] = -0.25
    index = torch.tensor([0, 0, 1, 2])
    scores = torch.tensor([0.5, 0.5, 0.75, 0.25])
    return L, index, scores, (4 * h, 4 * w), (2 * h + 8, 2 * w), (2 * h + 8, 2 * w), 0.5


def crop_edge_panoptic_case():
    """One query whose plane changes sign at the right edge of the image crop, upsampled 2.56 x by resize2 (600 -> 1536, a dyadic
    scale of 25 / 64): padded columns 599 and 600 hold exactly +2 and -12, so the last output column (source 599.3) is +2 when
    resize2 clamps to the crop, as sem_seg_postprocess does, and negative if it reads past the crop."""
    L = torch.full((1, 256, 256), 23.0)  # 5/8 * 23 + 3/8 * -33 = 2, 3/8 * 23 + 5/8 * -33 = -12
    L[0, :, 150:] = -33.0
    return L, torch.tensor([0]), torch.tensor([1.0]), (1024, 1024), (600, 600), (64, 1536), 0.5
