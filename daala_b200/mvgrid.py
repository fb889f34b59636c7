"""Host logic: MV grid -> OBMC block list (the control flow of od_state_mc_predict,
od_state_pred_block and od_state_pred_block_from_setup, reference src/state.c:932,
:673, :627), vectorised over the whole frame.

The grid has one vertex per 8x8 luma pixels: (nvmvbs+1) x (nhmvbs+1) points with a
`valid` flag and a motion vector in 1/8 luma pixels.  A 64x64 motion-vector block
is split recursively wherever the vertex at its centre is valid; every leaf is
predicted from the MVs of four vertices chosen by its outside corner `oc` and
split state `s` (OD_VERT_SETUP_DX/DY, src/state.c:592-625) and blended by OBMC.
"""
import numpy as np

from . import mc

# OD_VERT_D, src/state.c:585; OD_VERT_DX = D + 1, OD_VERT_DY = D + 0 (src/state.h:93-96)
_D = [0, 0, 1, 1, 0, 0, 1, 2, 0, 0, 2, 1, 0, -1, 1, 1, 0, -1, 0, 1, 1, -1]
_DX = _D[1:5]
_DY = _D[0:4]
_SETUP_DX = [[9, 1, 9, 1], [13, 13, 1, 1], [18, 1, 18, 1], [5, 5, 1, 1]]   # offsets into OD_VERT_D
_SETUP_DY = [[4, 4, 0, 0], [8, 0, 8, 0], [12, 12, 0, 0], [17, 0, 17, 0]]   # offsets into OD_VERT_DY (= D)
LOG_MVB_DELTA0 = 3   # OD_LOG_MVBSIZE_MAX - OD_LOG_MVBSIZE_MIN
# daala_b200_mv_pt (include/daala_b200.h): one vertex as od_mv_grid_pt holds it; ref 0 = OD_FRAME_GOLD, 1 = _PREV,
# 2 = _NEXT (B frames, mc_next engines: the vertex's second vector mv1 travels beside the grid)
MV_PT_DTYPE = np.dtype([("mv", "<i4", 2), ("valid", "u1"), ("ref", "u1"), ("pad_", "u1", 2)])
assert MV_PT_DTYPE.itemsize == 12


def _div_pow2_re(x, shift):
    """OD_DIV_POW2_RE (src/odintrin.h:150): divide by 2^shift rounding to even."""
    if shift == 0:
        return x
    return (x + (((1 << shift) + ((x >> shift) & 1) - 1) >> 1)) >> shift


def leaves(valid):
    """All leaf MV blocks as arrays (vx, vy, log_mvb_sz, oc, s)."""
    nv, nh = valid.shape[0] - 1, valid.shape[1] - 1
    vy, vx = np.mgrid[0:nv:8, 0:nh:8]
    cur = (vx.ravel(), vy.ravel())
    out = []
    for l in range(LOG_MVB_DELTA0, -1, -1):
        x, y = cur
        half = (1 << l) >> 1
        if l > 0:
            split = valid[y + half, x + half].astype(bool)
        else:
            split = np.zeros(len(x), bool)
        lx, ly = x[~split], y[~split]
        if l < LOG_MVB_DELTA0:
            mask = (1 << (l + 1)) - 1
            oc = ((lx & mask) != 0).astype(np.int64)
            oc = np.where((ly & mask) != 0, 3 - oc, oc)
            dx = np.array(_DX)
            dy = np.array(_DY)
            s1x, s1y = lx + (dx[(oc + 1) & 3] << l), ly + (dy[(oc + 1) & 3] << l)
            s3x, s3y = lx + (dx[(oc + 3) & 3] << l), ly + (dy[(oc + 3) & 3] << l)
            s = valid[s1y, s1x].astype(np.int64) | (valid[s3y, s3x].astype(np.int64) << 1)
        else:
            oc = np.zeros(len(lx), np.int64)
            s = np.full(len(lx), 3, np.int64)
        out.append((lx, ly, np.full(len(lx), l, np.int64), oc, s))
        sx, sy = x[split], y[split]
        cur = (np.concatenate([sx, sx + half, sx, sx + half]), np.concatenate([sy, sy, sy + half, sy + half]))
    return tuple(np.concatenate([o[i] for o in out]) for i in range(5))


REF_NEXT = 2   # OD_FRAME_NEXT


def vectors(mv, ref, mv1=None):
    """The vector each vertex is predicted with (od_state_pred_block_from_setup, src/state.c:647-660): mv1 where
    ref == 2 (OD_FRAME_NEXT), mv elsewhere.  mv1 is never taken on a GOLD / PREV vertex, where the encoder leaves
    stale values; without mv1 (P frames) this is mv."""
    if mv1 is None:
        return np.asarray(mv)
    return np.where((np.asarray(ref) == REF_NEXT)[..., None], mv1, mv)


def block_list(valid, mv, xdec=0):
    """daala_b200_mc_block records (mc.MC_BLOCK_DTYPE) of one plane: `valid` bool
    [(nvmvbs+1), (nhmvbs+1)], `mv` int32 [.., .., 2] in 1/8 luma pixel."""
    return blocks_for(*leaves(valid), mv, xdec)


def corners(vx, vy, l, oc, s):
    """The grid vertices (gx, gy) of the four corners of given MV blocks, in od_mc_predict's rotational order."""
    vx, vy, l, oc, s = (np.asarray(a, np.int64) for a in (vx, vy, l, oc, s))
    d = np.array(_D)
    sdx = np.array(_SETUP_DX)[oc, s]   # offsets
    sdy = np.array(_SETUP_DY)[oc, s]
    return [(vx + (d[sdx + k] << l), vy + (d[sdy + k] << l)) for k in range(4)]


def blocks_for(vx, vy, l, oc, s, mv, xdec=0, ref=None, mv1=None):
    """Block records of given MV blocks (vertex position, log size, outside corner, split state): what
    od_state_pred_block_from_setup (src/state.c:627) derives for one plane.  With ref and mv1 (B frames) a corner on
    a NEXT vertex takes mv1 (see vectors)."""
    vx, vy, l, oc, s = (np.asarray(a, np.int64) for a in (vx, vy, l, oc, s))
    if mv1 is not None:
        mv = vectors(mv, ref, mv1)
    blocks = np.zeros(len(vx), mc.MC_BLOCK_DTYPE)
    for k, (gx, gy) in enumerate(corners(vx, vy, l, oc, s)):
        blocks["mvx"][:, k] = _div_pow2_re(mv[gy, gx, 0].astype(np.int64), xdec)
        blocks["mvy"][:, k] = _div_pow2_re(mv[gy, gx, 1].astype(np.int64), xdec)
    blocks["x0"] = vx << (3 - xdec)
    blocks["y0"] = vy << (3 - xdec)
    blocks["log_xblk"] = blocks["log_yblk"] = l + 3 - xdec
    blocks["oc"], blocks["s"] = oc, s
    return blocks


def pack(valid, mv, ref):
    """MV_PT_DTYPE records of grids given as `valid` [..., nv+1, nh+1] (bool / 0-1), `mv` [..., nv+1, nh+1, 2]
    (1/8 luma pixel) and `ref` (0 = GOLD, 1 = PREV), any leading (frame) dimensions."""
    valid = np.asarray(valid)
    out = np.zeros(valid.shape, MV_PT_DTYPE)
    out["valid"] = valid
    out["mv"] = mv
    out["ref"] = ref
    return out


def unpack(grid):
    """(valid, mv, ref) arrays of MV_PT_DTYPE records: the inverse of pack."""
    return grid["valid"].copy(), grid["mv"].copy(), grid["ref"].copy()
