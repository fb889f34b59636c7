"""Lossless frames (quantizer 0, the reference's Haar-wavelet path) restated in numpy: what the keyframe engine's lossless
step (config.lossless, csrc/lossless.cu) computes, and what a host tree coder reads from it.

At quantizer 0 (OD_LOSSLESS, reference src/internal.h:131) every superblock is one block, n = 64 in luma and 32 in
4:2:0 chroma, with no lapping and no deringing.  Per block, planes 0, 1, 2 of each superblock in raster order:
  1. c = pixel - 128.  P and B frames: mc = prediction - 128, and every sample of c outside the picture
     (x >= pic_w >> xdec or y >= pic_h >> ydec) is mc's (src/encode.c:2589-2602).  Keyframes keep their padding.
  2. d = od_haar(c) (src/dct.c:4822); P and B frames also md = od_haar(mc).
  3. DC: keyframes code dc0 = d[0] - the superblock DC predictor of the left, up, up-left and up-right superblocks'
     d[0] (od_quantize_haar_dc_sb, src/encode.c:1537-1590, dc_quant = 1); P and B frames code d[0] - md[0].
  4. AC: out = d - pred with q = 1 (od_wavelet_quantize, src/encode.c:1012-1027), pred = 0 on keyframes and md else.
  5. The coder starts from the root sums of od_compute_max_tree (src/encode.c:899-919) at (1, 0), (0, 1), (1, 1).
  6. The decoder adds pred back, runs od_haar_inv and + 128 with a clamp; the result is c, i.e. the (padded) input.
"""
import numpy as np

from .frame import Geometry


def _kernel(ll, lh, hl, hh):
    """OD_HAAR_KERNEL (reference src/tf.h:34) on int64 arrays."""
    ll = ll + hl
    hh = hh - lh
    m = (ll - hh) >> 1
    lh = m - lh
    hl = m - hl
    ll = ll - lh
    hh = hh + hl
    return ll, lh, hl, hh


def haar(x, ln):
    """od_haar of every n x n block in the last two axes of x (n = 1 << ln)."""
    n = 1 << ln
    t = np.array(x, np.int64)
    y = np.zeros_like(t)
    for level in range(ln):
        m = n >> level >> 1
        a, b = t[..., 0:2 * m:2, 0:2 * m:2], t[..., 1:2 * m:2, 0:2 * m:2]
        c, d = t[..., 0:2 * m:2, 1:2 * m:2], t[..., 1:2 * m:2, 1:2 * m:2]
        a, b, c, d = _kernel(a, b, c, d)
        t[..., :m, :m] = a
        y[..., :m, m:2 * m] = b
        y[..., m:2 * m, :m] = c
        y[..., m:2 * m, m:2 * m] = d
    y[..., 0, 0] = t[..., 0, 0]
    return y


def haar_inv(y, ln):
    """od_haar_inv of every n x n block in the last two axes of y."""
    y = np.asarray(y, np.int64)
    x = np.zeros_like(y)
    x[..., 0, 0] = y[..., 0, 0]
    for level in range(ln - 1, -1, -1):
        m = 1 << (ln - 1 - level)
        a, b, c, d = _kernel(x[..., :m, :m].copy(), y[..., :m, m:2 * m], y[..., m:2 * m, :m], y[..., m:2 * m, m:2 * m])
        x[..., 0:2 * m:2, 0:2 * m:2] = a
        x[..., 1:2 * m:2, 0:2 * m:2] = b
        x[..., 0:2 * m:2, 1:2 * m:2] = c
        x[..., 1:2 * m:2, 1:2 * m:2] = d
    return x


def tree_map(ln):
    """[n, n] int8: the root tree each coefficient belongs to (0: (1, 0) = tree_sum[0][1], 1: (0, 1) = tree_sum[1][0],
    2: (1, 1) = tree_sum[1][1]); -1 at the DC."""
    n = 1 << ln
    r, c = np.mgrid[0:n, 0:n]
    top = np.maximum(r, c)
    s = np.where(top > 0, 1 << np.floor(np.log2(np.maximum(top, 1))).astype(np.int64), 1)
    out = np.where(r < s, 0, np.where(c < s, 1, 2)).astype(np.int8)
    out[0, 0] = -1
    return out


def dc_predictor(dc, sbx, sby):
    """The superblock DC predictor of od_quantize_haar_dc_sb from dc[sby][sbx] of the neighbours (at quantizer 0 their
    d[0], unquantised); has_ur = sby > 0 && sbx < nhsb - 1 (src/encode.c:2640)."""
    nhsb = dc.shape[1]
    L = lambda y, x: int(dc[y, x])
    if sby > 0 and sbx > 0:
        if sbx < nhsb - 1:
            return (22 * L(sby, sbx - 1) - 9 * L(sby - 1, sbx - 1) + 15 * L(sby - 1, sbx) + 4 * L(sby - 1, sbx + 1)
                    + 16) >> 5
        return (23 * L(sby, sbx - 1) - 10 * L(sby - 1, sbx - 1) + 19 * L(sby - 1, sbx) + 16) >> 5
    if sby > 0:
        return L(sby - 1, sbx)
    if sbx > 0:
        return L(sby, sbx - 1)
    return 0


def _blocks(plane, n):
    """[H, W] -> [nvsb, nhsb, n, n] view order."""
    h, w = plane.shape
    return plane.reshape(h // n, n, w // n, n).swapaxes(1, 2)


def _unblocks(b):
    nv, nh, n, _ = b.shape
    return b.swapaxes(1, 2).reshape(nv * n, nh * n)


def padded_input(geom, planes, pred=None):
    """Step 1: c = pixel - 128 per plane (int64), with the P / B padding rule when pred is given."""
    out = []
    for p in range(3):
        c = np.asarray(planes[p], np.int64) - 128
        if pred is not None:
            pw, ph = geom.pic_w >> (1 if p else 0), geom.pic_h >> (1 if p else 0)
            mc = np.asarray(pred[p], np.int64) - 128
            c = c.copy()
            c[:, pw:] = mc[:, pw:]
            c[ph:, :] = mc[ph:, :]
        out.append(c)
    return out


def encode_frame(geom, planes, pred=None):
    """One frame (planes: three [h, w] u8 arrays of the padded geometry; pred: the prediction planes of a P / B frame,
    None for a keyframe).  Returns dict(coeffs=[3 x [h, w] int64]: the residual with the coded DC in each block's DC
    slot, d=[3 x [h, w]]: the transform of the (padded) input, blocks=[nvsb, nhsb, 3, 4] int64: the three root sums
    and a 0)."""
    c = padded_input(geom, planes, pred)
    coeffs, ds = [], []
    blocks = np.zeros((geom.nvsb, geom.nhsb, 3, 4), np.int64)
    for p in range(3):
        ln = 5 if p else 6
        n = 1 << ln
        d = haar(_blocks(c[p], n), ln)
        if pred is None:
            out = d.copy()
            dc = d[:, :, 0, 0]
            for sby in range(geom.nvsb):
                for sbx in range(geom.nhsb):
                    out[sby, sbx, 0, 0] = dc[sby, sbx] - dc_predictor(dc, sbx, sby)
        else:
            md = haar(_blocks(np.asarray(pred[p], np.int64) - 128, n), ln)
            out = d - md
        tm = tree_map(ln)
        for k in range(3):
            blocks[:, :, p, k] = np.abs(np.where(tm == k, out, 0)).sum(axis=(2, 3))
        coeffs.append(_unblocks(out))
        ds.append(_unblocks(d))
    return dict(coeffs=coeffs, d=ds, blocks=blocks)


def decode_frame(geom, coeffs, pred=None):
    """Step 6, as the decoder makes it: the reconstruction planes (u8) from the residual planes of encode_frame (and
    the prediction of a P / B frame).  Keyframe DCs are rebuilt in coding order from the decoded neighbours."""
    rec = []
    for p in range(3):
        ln = 5 if p else 6
        n = 1 << ln
        y = _blocks(np.asarray(coeffs[p], np.int64), n).copy()
        if pred is None:
            dc = np.zeros(y.shape[:2], np.int64)
            for sby in range(geom.nvsb):
                for sbx in range(geom.nhsb):
                    dc[sby, sbx] = y[sby, sbx, 0, 0] + dc_predictor(dc, sbx, sby)
            y[:, :, 0, 0] = dc
        else:
            y = y + haar(_blocks(np.asarray(pred[p], np.int64) - 128, n), ln)
        rec.append(np.clip(_unblocks(haar_inv(y, ln)) + 128, 0, 255).astype(np.uint8))
    return rec


def bounds(ln):
    """Value ranges of the lossless step for 8-bit input and block size n = 1 << ln, from the closed form of
    OD_HAAR_KERNEL (DESIGN.md): ll = ceil((a+b+c+d)/2), lh = floor((a-b+c-d)/2), hl = floor((a+b-c-d)/2),
    hh = floor((a-b-c+d)/2).  With inputs in [lo, hi], ll lies in [2 lo, 2 hi] and each detail in [lo - hi, hi - lo].
    Returns dict(dc=(lo, hi) of d[0], detail=max |detail| over all levels, resid=max |d - md| (P / B frames, DC
    included), dc0=(lo, hi) of a keyframe's dc0)."""
    lo, hi, det = -128, 127, 0
    for _ in range(ln):
        det = max(det, hi - lo)
        lo, hi = 2 * lo, 2 * hi
    # the predictor's extremes: positive weights take one end of [lo, hi], negative ones the other
    preds = []
    for w in ((22, -9, 15, 4), (23, -10, 19)):
        top = sum(k * (hi if k > 0 else lo) for k in w)
        bot = sum(k * (lo if k > 0 else hi) for k in w)
        preds += [(top + 16) >> 5, (bot + 16) >> 5]
    preds += [lo, hi, 0]
    resid = max(det, hi - lo)
    return dict(dc=(lo, hi), detail=det, resid=resid, dc0=(lo - max(preds), hi - min(preds)))
