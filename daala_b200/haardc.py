"""Quantised keyframe DCs (config.haar_dc_quant) restated in numpy: what the keyframe engine's DC chain
(csrc/haar_dc.cu) computes, and what a host coder reads from it.

The forward transform leaves the unquantised Haar DC pyramid in the `d` planes (od_compute_dcts): the superblock DC at
the superblock's origin, and at every split node the three Haar coefficients of its children's DCs at the origins of
children 1..3 (TR, BL, BR).  The reference codes them per plane, in od_encode_recursive's order (reference
src/encode.c:2605-2656, :1537-1657, :1765-1787):
  1. Models reset for the keyframe (od_adapt_ctx_reset): one generic model per plane, ex_sb_dc, ex_dc[5][3] at 32768
     (luma) or 8 (chroma).
  2. Superblocks in raster order.  The SB DC is predicted from the quantised DCs of the left, up, up-left and (has_ur
     = sby > 0 && sbx < nhsb - 1) up-right superblocks and quantised with OD_DIV_R0 by
     dc_quant = max(1, q0 * pvq_qm_q4[pli][20] >> 4); generic_encode on (model, ex_sb_dc).  The gradients start at 0
     and take the differences to the up and left superblock DCs where those exist.
  3. Every split node depth-first (TL, TR, BL, BR) with the gradients its parent returned, by value: x[1] -= hgrad / 5,
     x[2] -= vgrad / 5, |x[i]| / q with q = ac_quant[i == 3] = (dc_quant * OD_DC_QM[bsi - xdec][.] + 8) >> 4, one RDO
     increment rated by generic_encode_cost, generic_encode on (model, ex_dc[bsi][i - 1]); the gradients become the
     reconstructed x[1], x[2]; OD_HAAR_KERNEL gives the children their DCs.
The result: every leaf DC final in `d`, and the signed indices in a grid of 4x4 units per plane, the SB index at the
superblock origin, a split node's three at the origins of its children 1..3.
"""
import math

import numpy as np

from .symbols import HDC_DTYPE

GENERIC_TABLES = 12
OD_DC_QM = ((21, 25), (18, 20), (17, 18), (17, 17))   # src/state.c:48
M_LOG2E = 1.4426950408889634074


def _tdiv(a, b):
    """C integer division (truncation toward zero)."""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


def div_r0(x, y):
    """OD_DIV_R0 (src/odintrin.h:123)."""
    h = ((y + 1) >> 1) - 1
    return _tdiv(x + (-h if x < 0 else h), y)


def _ilog(v):
    return int(v).bit_length()


def log_ex(ex_q16):
    """log_ex (src/generic_code.c:109)."""
    lg = _ilog(ex_q16)
    if lg < 15:
        odd = ex_q16 * ex_q16 > 2 << 2 * lg
    else:
        tmp = ex_q16 >> (lg - 8)
        odd = tmp * tmp > (1 << 15)
    return max(0, 2 * lg - 33 + int(odd))


class Model:
    """One plane's DC symbol state after od_adapt_ctx_reset: the generic model (12 CDFs of 16), ex_sb_dc and
    ex_dc[bsi][3].  `stats` counts what the chain reached: RDO increments and xs >= 15 tails."""

    def __init__(self, pli):
        self.cdf = [[(j + 1) * 64 for j in range(16)] for _ in range(GENERIC_TABLES)]
        e = 8 if pli > 0 else 32768
        self.ex_sb_dc = [e]
        self.ex_dc = [[[e] for _ in range(3)] for _ in range(5)]
        self.stats = dict(rdo_inc=0, tail=0, symbols=0)

    def _id_shift(self, ex):
        lg_q1 = log_ex(ex[0])
        return min(GENERIC_TABLES - 1, lg_q1), max(0, (lg_q1 - 5) >> 1)

    def cost(self, x, ex):
        """generic_encode_cost with max = -1 (src/generic_encoder.c:161)."""
        i, shift = self._id_shift(ex)
        cdf = self.cdf[i]
        xs = (x + (1 << shift >> 1)) >> shift
        extra = shift - (xs == 0) if shift else 0
        xs = min(15, xs)
        if xs == 15:
            extra += 2
        return extra - M_LOG2E * math.log(float(cdf[xs] - (cdf[xs - 1] if xs else 0)) / cdf[15])

    def encode(self, x, ex):
        """The model adaptation of generic_encode with max = -1 and integration 2 (src/generic_encoder.c:99,
        generic_model_update :136)."""
        i, shift = self._id_shift(ex)
        cdf = self.cdf[i]
        xs = (x + (1 << shift >> 1)) >> shift
        self.stats["symbols"] += 1
        if xs >= 15:
            self.stats["tail"] += 1
        if cdf[15] + 64 > 32767:
            for j in range(16):
                cdf[j] = (cdf[j] >> 1) + j + 1
        for j in range(min(15, xs), 16):
            cdf[j] += 64
        x = min(x, 32767)
        ex[0] += ((x << 16) - ex[0]) >> 2


def sb_dc_pred(mem, sbx, sby, has_ur):
    """The superblock DC predictor of od_quantize_haar_dc_sb (src/encode.c:1563-1582)."""
    if sby > 0 and sbx > 0:
        if has_ur:
            return (22 * mem[sby][sbx - 1] - 9 * mem[sby - 1][sbx - 1] + 15 * mem[sby - 1][sbx]
                    + 4 * mem[sby - 1][sbx + 1] + 16) >> 5
        return (23 * mem[sby][sbx - 1] - 10 * mem[sby - 1][sbx - 1] + 19 * mem[sby - 1][sbx] + 16) >> 5
    if sby > 0:
        return mem[sby - 1][sbx]
    if sbx > 0:
        return mem[sby][sbx - 1]
    return 0


def dc_quant(q0, pvq_qm_q4, pli):
    return max(1, int(q0) * int(pvq_qm_q4[pli][20]) >> 4)


def quantize_plane(d, bsize, pli, xdec, q0, pvq_qm_q4, lam, nhsb, nvsb):
    """The chain of one plane.  d: [h, w] the unquantised pyramid (not modified); bsize: [nvsb * 8, nhsb * 8].
    Returns (d with every coded DC position replaced by its reconstruction, [h / 4, w / 4] int32 indices, stats)."""
    d = np.array(d, np.int64)
    idx = np.zeros((d.shape[0] >> 2, d.shape[1] >> 2), np.int32)
    m = Model(pli)
    dq = dc_quant(q0, pvq_qm_q4, pli)
    mem = [[0] * nhsb for _ in range(nvsb)]
    lam = float(lam)

    def level(bx, by, bsi, hgrad, vgrad):
        ln = bsi - xdec + 2
        acq = ((dq * OD_DC_QM[bsi - xdec][0] + 8) >> 4, (dq * OD_DC_QM[bsi - xdec][1] + 8) >> 4)
        pos = ((by << ln, bx << ln), (by << ln, (bx + 1) << ln), ((by + 1) << ln, bx << ln),
               ((by + 1) << ln, (bx + 1) << ln))
        x = [int(d[p]) for p in pos]
        x[1] -= _tdiv(hgrad, 5)
        x[2] -= _tdiv(vgrad, 5)
        for i in (1, 2, 3):
            q = acq[i == 3]
            sign = x[i] < 0
            a = abs(x[i])
            quant = a // q
            ex = m.ex_dc[bsi][i - 1]
            cost = m.cost(quant + 1, ex) - m.cost(quant, ex)
            if quant == 0:
                cost += 1
            if (q * q - 2 * q * (a - quant * q)) + float(q * q) * lam * cost < 0:
                quant += 1
                m.stats["rdo_inc"] += 1
            m.encode(quant, ex)
            idx[pos[i][0] >> 2, pos[i][1] >> 2] = -quant if sign else quant
            x[i] = -quant * q if sign else quant * q
        x[1] += _tdiv(hgrad, 5)
        x[2] += _tdiv(vgrad, 5)
        hgrad, vgrad = x[1], x[2]
        ll, lh, hl, hh = x
        ll += hl
        hh -= lh
        t = (ll - hh) >> 1
        lh = t - lh
        hl = t - hl
        ll -= lh
        hh += hl
        for p, v in zip(pos, (ll, lh, hl, hh)):
            d[p] = v
        return hgrad, vgrad

    def recurse(bx, by, bsi, hgrad, vgrad):
        obs = int(bsize[(by << bsi) >> 1, (bx << bsi) >> 1])
        if max(obs, xdec) >= bsi:
            return
        hgrad, vgrad = level(2 * bx, 2 * by, bsi - 1, hgrad, vgrad)
        for cy in (0, 1):
            for cx in (0, 1):
                recurse(2 * bx + cx, 2 * by + cy, bsi - 1, hgrad, vgrad)

    ln = 6 - xdec
    for sby in range(nvsb):
        for sbx in range(nhsb):
            has_ur = sby > 0 and sbx < nhsb - 1
            pred = sb_dc_pred(mem, sbx, sby, has_ur)
            quant = div_r0(int(d[sby << ln, sbx << ln]) - pred, dq)
            m.encode(abs(quant), m.ex_sb_dc)
            cur = quant * dq + pred
            d[sby << ln, sbx << ln] = cur
            mem[sby][sbx] = cur
            idx[(sby << ln) >> 2, (sbx << ln) >> 2] = quant
            hgrad = vgrad = 0
            if sby > 0:
                vgrad = mem[sby - 1][sbx] - cur
            if sbx > 0:
                hgrad = mem[sby][sbx - 1] - cur
            recurse(sbx, sby, 4, hgrad, vgrad)
    return d, idx, m.stats


def quantize_frame(geom, d_planes, bsize, q0, pvq_qm_q4, lam):
    """All three planes of one keyframe.  Returns dict(d=[3 x [h, w] int64], idx=[3 x [h / 4, w / 4] int32],
    stats=[3 x dict])."""
    out = dict(d=[], idx=[], stats=[])
    for p in range(3):
        d, idx, st = quantize_plane(d_planes[p], bsize, p, geom.xdec[p], q0, pvq_qm_q4, lam, geom.nhsb, geom.nvsb)
        out["d"].append(d)
        out["idx"].append(idx)
        out["stats"].append(st)
    return out


# What a host coder reads of the chain (config.symbol_stream = 1 with haar_dc_quant = 1; include/daala_b200.h,
# daala_b200_kf_sym_hdc): per superblock in raster order, planes 0, 1, 2, the superblock DC and then every split node's
# three indices in od_encode_recursive's pre-order, each record naming the block record the coder emits it before.
# The records are symbols.HDC_DTYPE.


def _walk_records(bsize, geom, visit):
    """The DC symbols of one frame in coding order: visit(pli, gy, gx, bsi, child, block) per symbol, with (gy, gx) the
    index grid position of the symbol (4x4 units of the plane), bsi the record's size index and block the frame-relative
    index of the leaf the symbol precedes.  Returns the frame's leaf count."""
    bsize = np.asarray(bsize)
    leaves = [0]

    def recurse(pli, xdec, bx, by, bsi):
        obs = int(bsize[(by << bsi) >> 1, (bx << bsi) >> 1])
        if max(obs, xdec) >= bsi:
            leaves[0] += 1
            return
        first = leaves[0]
        sh = bsi - 1 - xdec             # child edge in 4x4 units of the plane: 2 ** sh
        gx, gy = (2 * bx) << sh, (2 * by) << sh
        half = 1 << sh
        for c in (1, 2, 3):
            visit(pli, gy + (c >> 1) * half, gx + (c & 1) * half, bsi - 1, c, first)
        for cy in (0, 1):
            for cx in (0, 1):
                recurse(pli, xdec, 2 * bx + cx, 2 * by + cy, bsi - 1)

    for sby in range(geom.nvsb):
        for sbx in range(geom.nhsb):
            for pli in range(3):
                xdec = geom.xdec[pli]
                g = 16 >> xdec                   # superblock edge in 4x4 units of the plane
                visit(pli, sby * g, sbx * g, 4, 0, leaves[0])
                recurse(pli, xdec, sbx, sby, 4)
    return leaves[0]


def stream_records(idx_planes, bsize, geom):
    """One frame's keyframe DC records (HDC_DTYPE, one per leaf block, in coding order) from its index grids
    (idx_planes: 3 x [h / 4, w / 4], what quantize_frame returns as idx and the engine as dc_index0..2) and its
    block-size map."""
    out = []
    _walk_records(bsize, geom, lambda pli, gy, gx, bsi, c, blk: out.append(
        (int(idx_planes[pli][gy, gx]), blk, pli, bsi, c, 0)))
    return np.array(out, HDC_DTYPE)


def grids_from_records(records, bsize, geom):
    """The inverse of stream_records: the three index grids (int32, 0 where no symbol is coded) from one frame's
    records.  Asserts that the records are those of the map (count, order, sizes and blocks)."""
    idx = [np.zeros((h >> 2, w >> 2), np.int32) for h, w in (geom.plane_shape(p) for p in range(3))]
    it = iter(np.asarray(records, HDC_DTYPE))

    def visit(pli, gy, gx, bsi, c, blk):
        r = next(it, None)
        assert r is not None, "fewer records than the map's symbols"
        assert (int(r["pli"]), int(r["bsi"]), int(r["child"]), int(r["block"])) == (pli, bsi, c, blk), \
            "record does not fit the map: %r against %r" % (r, (pli, bsi, c, blk))
        idx[pli][gy, gx] = r["value"]

    n = _walk_records(bsize, geom, visit)
    assert len(records) == n, "%d records for %d leaves" % (len(records), n)
    return idx
