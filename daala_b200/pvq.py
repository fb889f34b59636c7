"""Host side of the PVQ stage: block / band list construction from the
block-size map and the device buffers + launches of the batch entry points
(include/daala_b200.h, "PVQ" section).

Band geometry follows OD_BAND_OFFSETS (reference src/partition.c:85-91):
4x4 -> {15}; 8x8 -> {15, 8, 8, 32}; 16x16 -> {15, 8, 8, 32, 32, 32, 128};
32x32 and 64x64 -> {15, 8, 8, 32, 32, 32, 128, 128, 128} (only the first 512
coefficients in coding order are coded).
"""
import ctypes
import os

import numpy as np
import torch

from . import _native

BAND_EDGES = [1, 16, 24, 32, 64, 96, 128, 256, 384, 512]
NBANDS = {0: 1, 1: 4, 2: 7, 3: 9, 4: 9}
OD_QM_STRIDE = 5456
PVQ_LAMBDA = 0.147  # OD_PVQ_LAMBDA, src/pvq.h:51

BLOCK_DTYPE = np.dtype([("coef_off", "<i4"), ("x0", "<u2"), ("y0", "<u2"), ("bs", "u1"), ("pli", "u1"),
                        ("xdec", "u1"), ("frame", "u1")])


class PvqParams(ctypes.Structure):
    """struct daala_b200_pvq_params"""
    _fields_ = [
        ("blocks", ctypes.c_void_p), ("in_", ctypes.c_void_p), ("ref", ctypes.c_void_p),
        ("out", ctypes.c_void_p), ("y", ctypes.c_void_p), ("res_gain", ctypes.c_void_p),
        ("res_theta", ctypes.c_void_p), ("res_max_theta", ctypes.c_void_p), ("res_k", ctypes.c_void_p),
        ("res_skip_term", ctypes.c_void_p), ("res_skip_diff", ctypes.c_void_p), ("res_flip", ctypes.c_void_p),
        ("res_dc", ctypes.c_void_p), ("y16", ctypes.c_void_p), ("qm", ctypes.c_void_p), ("qm_inv", ctypes.c_void_p),
        ("coef_plane", ctypes.c_void_p * 3), ("pred_plane", ctypes.c_void_p * 3),
        ("plane_frame_pitch", ctypes.c_longlong * 3), ("plane_stride", ctypes.c_int * 3),
        ("qm_stride", ctypes.c_int), ("q0", ctypes.c_int), ("is_keyframe", ctypes.c_int),
        ("use_masking", ctypes.c_int), ("pad_", ctypes.c_int), ("pvq_norm_lambda", ctypes.c_double),
        ("pvq_qm_q4", (ctypes.c_ubyte * 32) * 3),
    ]


def _bind():
    L = _native.lib()
    if getattr(L, "_pvq_bound", False):
        return L
    pp = ctypes.POINTER(PvqParams)
    L.daala_b200_pvq_encode_bands.argtypes = [pp, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    L.daala_b200_pvq_encode_bands_mode.argtypes = [pp, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                   ctypes.c_void_p]
    for name in ("daala_b200_pvq_block_finish", "daala_b200_pvq_cfl_flip", "daala_b200_coding_order_scatter"):
        getattr(L, name).argtypes = [pp, ctypes.c_int, ctypes.c_void_p]
    L.daala_b200_coding_order_gather.argtypes = [pp, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    L.daala_b200_pvq_intra_band_ref.argtypes = [pp, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                                                  ctypes.c_void_p]
    L.daala_b200_pvq_order_by_work.argtypes = [pp, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                 ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    L.daala_b200_pvq_cfl_pred.argtypes = [pp, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_int,
                                          ctypes.c_void_p]
    L._pvq_bound = True
    return L


def default_qm(hvs=True):
    """state->qm / qm_inv for the default (HVS or flat) 8x8 base matrix."""
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "data", "qm_%s.npy" % ("hvs" if hvs else "flat"))
    a = np.load(path)
    return a[0].copy(), a[1].copy()


def qm_inputs():
    """The data od_init_qm starts from, exported from the reference build by tools/extract_tables.py:
    basis magnitudes OD_BASIS_MAG per decimation and size, the 8x8 base matrices, the scan tables."""
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "data", "qm_inputs.npz")
    return dict(np.load(path))


def raster_to_coding_order(block, scans):
    """od_raster_to_coding_order (src/partition.c:123) of a full n x n block: DC, then for every nested
    size m = 4, 8, .. n the m-size stage's scan (entries are raster indices y*m + x)."""
    n = block.shape[0]
    out = [block[0:1, 0]]
    m = 4
    while m <= n:
        idx = scans[m]
        out.append(block[idx // m, idx % m])
        m *= 2
    return np.concatenate(out)


def init_qm(qm8, inputs=None):
    """Host restatement of od_init_qm (src/pvq.c:322, fixed-point branch): magnitude-compensated
    quantisation matrix and its inverse for every block size and both decimations, in coding order,
    Q11 / Q12 int16.  qm8: the 64 entries of an 8x8 base matrix in Q4 (OD_QM8_Q4_HVS / _FLAT)."""
    inputs = qm_inputs() if inputs is None else inputs
    scans = {m: inputs["scan%d" % m].astype(np.int64) for m in (4, 8, 16, 32, 64)}
    qm8 = np.asarray(qm8, np.int64)
    qm = np.zeros(2 * OD_QM_STRIDE, np.int16)
    qm_inv = np.zeros(2 * OD_QM_STRIDE, np.int16)
    for bs in range(5):
        n = 4 << bs
        off0 = (((1 << (2 * bs)) - 1) << 4) // 3           # OD_QM_OFFSET(bs), src/pvq.h:71
        i, j = np.mgrid[0:n, 0:n]
        qmv = qm8[((i << 1) >> bs) * 8 + ((j << 1) >> bs)]
        for xydec in range(2):
            bm = inputs["mag_%d_%d" % (xydec, bs)]
            mag = np.floor(.5 + (2048. * bm[i]) * bm[j]).astype(np.int64)     # OD_ROUND32(OD_QM_SCALE * m_i * m_j)
            mag = (mag * 16 + (qmv >> 1)) // qmv
            mag[0, 0] = 2048
            y = np.minimum(32767, mag)
            y_inv = (2048 * 4096 + (y >> 1)) // y
            off = xydec * OD_QM_STRIDE + off0
            # od_raster_to_coding_order_16 writes the coded prefix only: 512 entries for 32x32 / 64x64
            # (src/partition.c:216); the rest of the table stays zero
            ncoded = min(n * n, 512)
            qm[off:off + ncoded] = raster_to_coding_order(y, scans)[:ncoded].astype(np.int16)
            qm_inv[off:off + ncoded] = raster_to_coding_order(y_inv, scans)[:ncoded].astype(np.int16)
    return qm, qm_inv


def block_list(bsize, geom, frame=0, sb_row0=0, sb_rows=None):
    """Leaf transform blocks of one frame for every plane, from the block-size
    map (one byte per 8x8 luma unit).  Returns a BLOCK_DTYPE array (coef_off
    not yet assigned), ordered by transform size so warps see uniform work."""
    sb_rows = geom.nvsb - sb_row0 if sb_rows is None else sb_rows
    u0, u1 = sb_row0 * 8, (sb_row0 + sb_rows) * 8
    out = []
    bh, bw = bsize.shape
    uy, ux = np.mgrid[0:bh, 0:bw]
    inrows = (uy >= u0) & (uy < u1)
    for pli in range(geom.nplanes):
        xdec = geom.xdec[pli]
        eff = np.maximum(bsize, xdec).astype(np.int32)  # bs = max(obs, xdec), src/encode.c:1467
        for L in range(xdec, 5):
            if L == 0:
                sel = (eff == 0) & inrows
                ys, xs = uy[sel], ux[sel]
                # four 4x4 luma blocks per 8x8 unit
                for dy in (0, 4):
                    for dx in (0, 4):
                        a = np.zeros(len(ys), BLOCK_DTYPE)
                        a["x0"], a["y0"] = xs * 8 + dx, ys * 8 + dy
                        a["bs"], a["pli"], a["xdec"], a["frame"] = 0, pli, xdec, frame
                        out.append(a)
                continue
            span = 1 << (L - 1)  # units per block side
            sel = (eff == L) & (uy % span == 0) & (ux % span == 0) & inrows
            ys, xs = uy[sel], ux[sel]
            a = np.zeros(len(ys), BLOCK_DTYPE)
            a["x0"], a["y0"] = (xs * 8) >> xdec, (ys * 8) >> xdec
            a["bs"], a["pli"], a["xdec"], a["frame"] = L - xdec, pli, xdec, frame
            out.append(a)
    blocks = np.concatenate(out)
    order = np.argsort(blocks["bs"], kind="stable")
    return blocks[order]


def mark_luma4x4(blocks, bsize_maps):
    """Sets bit 7 of `xdec` on chroma blocks whose luma area is coded as 4x4 blocks
    (od_resample_luma_coeffs' chroma_bs == 0 case, src/intra.c:78)."""
    maps = np.stack([np.asarray(m) for m in bsize_maps])
    cand = np.nonzero((blocks["pli"] != 0) & (blocks["bs"] == 0))[0]
    b = blocks[cand]
    hit = maps[b["frame"].astype(np.int64), b["y0"].astype(np.int64) >> 2, b["x0"].astype(np.int64) >> 2] == 0
    blocks["xdec"][cand[hit]] |= 0x80
    return blocks


def intra_dependencies(blocks, bsize_maps, geom):
    """For luma blocks in raster order of their origin (per frame): index of the top / left
    neighbour of the same size (od_hv_intra_pred's `top` / `left`, src/intra.c:46-47) or -1."""
    n = len(blocks)
    top = np.full(n, -1, np.int32)
    left = np.full(n, -1, np.int32)
    h4, w4 = geom.frame_h // 4, geom.frame_w // 4
    nframes = int(blocks["frame"].max()) + 1 if n else 0
    index = np.full((nframes, h4, w4), -1, np.int32)
    index[blocks["frame"], blocks["y0"] >> 2, blocks["x0"] >> 2] = np.arange(n, dtype=np.int32)
    fr = blocks["frame"].astype(np.int64)
    x4 = (blocks["x0"] >> 2).astype(np.int64)
    y4 = (blocks["y0"] >> 2).astype(np.int64)
    bs = blocks["bs"].astype(np.int64)
    n4 = 1 << bs
    maps = np.stack(bsize_maps)
    has_top = y4 > 0
    ty = np.maximum(y4 - 1, 0)
    same_top = has_top & (maps[fr, ty >> 1, x4 >> 1] == bs)
    top[same_top] = index[fr[same_top], (y4 - n4)[same_top], x4[same_top]]
    has_left = x4 > 0
    lx = np.maximum(x4 - 1, 0)
    same_left = has_left & (maps[fr, y4 >> 1, lx >> 1] == bs)
    left[same_left] = index[fr[same_left], y4[same_left], (x4 - n4)[same_left]]
    assert (top[same_top] >= 0).all() and (left[same_left] >= 0).all()
    assert (top < np.arange(n)).all() and (left < np.arange(n)).all()
    return top, left


def dependency_depth(top, left):
    """Longest chain ending at each block (1 = no dependency): iterated relaxation, one
    vectorised pass per wavefront (a few dozen for real block-size maps)."""
    depth = np.ones(len(top), np.int32)
    ht, hl = top >= 0, left >= 0
    while True:
        new = np.ones_like(depth)
        new[ht] = np.maximum(new[ht], depth[top[ht]] + 1)
        new[hl] = np.maximum(new[hl], depth[left[hl]] + 1)
        if np.array_equal(new, depth):
            return depth
        depth = new


def sort_by_depth(luma, bsize_maps, geom):
    """Luma blocks (raster order) -> (blocks sorted by dependency depth, top, left, depth) with the
    neighbour indices remapped to the new order.  Still a topological order: a neighbour's depth is
    smaller, so it comes earlier."""
    top, left = intra_dependencies(luma, bsize_maps, geom)
    depth = dependency_depth(top, left)
    order = np.argsort(depth, kind="stable")
    inv = np.empty(len(order), np.int32)
    inv[order] = np.arange(len(order), dtype=np.int32)
    t, l = top[order], left[order]
    t = np.where(t >= 0, inv[np.maximum(t, 0)], -1).astype(np.int32)
    l = np.where(l >= 0, inv[np.maximum(l, 0)], -1).astype(np.int32)
    return luma[order], t, l, depth[order]


def raster_order(blocks):
    """Sort by (frame, y0, x0): the order the intra wavefront kernel requires."""
    return blocks[np.lexsort((blocks["x0"], blocks["y0"], blocks["frame"]))]


def assign_offsets(blocks):
    n2 = (16 << (2 * blocks["bs"].astype(np.int64)))
    length = np.minimum(n2, 512)
    off = np.concatenate([[0], np.cumsum(length)])
    if int(off[-1]) >= 1 << 31:
        raise ValueError("batch holds %d coded coefficients; coef_off is 32-bit: split the batch" % int(off[-1]))
    blocks["coef_off"] = off[:-1]
    return int(off[-1])


def band_lists(blocks):
    """(block << 4 | band) lists per size class {16: n in (15, 8), 32, 128}."""
    idx = np.arange(len(blocks), dtype=np.uint32)
    bs = blocks["bs"]
    cls = {16: [], 32: [], 128: []}
    for band in range(9):
        n = BAND_EDGES[band + 1] - BAND_EDGES[band]
        has = np.array([NBANDS[b] > band for b in range(5)])[bs]
        key = 16 if n <= 16 else (32 if n == 32 else 128)
        cls[key].append((idx[has] << 4) | band)
    # keep equal band sizes together inside the class-16 list (15s then 8s)
    return {k: (np.concatenate(v) if v else np.zeros(0, np.uint32)) for k, v in cls.items()}


def band_wave_lists(blocks, top, left, depth):
    """Band-granular intra wavefront of a luma block list (see k_intra_band_ref): per size class
    {16, 32, 128} -> (bulk, chain, slices).  `bulk[k]`: entries of the dependency-free bands 3 / 6;
    `chain[k]`: the other entries sorted by (wave, band, block), where the wave of band 0 is the
    block's depth over both neighbour chains, of bands 1/4/7 its depth over the top chain and of
    2/5/8 over the left chain; `slices[k][w]` = (first, count) of wave w + 1 inside chain[k]."""
    none = np.full(len(top), -1, np.int32)
    dh, dv = dependency_depth(top, none), dependency_depth(none, left)
    per_band = [depth, dh, dv, None, dh, dv, None, dh, dv]
    bulk, chain, slices = {}, {}, {}
    for k, v in band_lists(blocks).items():
        blk, band = (v >> 4).astype(np.int64), (v & 15).astype(np.int64)
        free = (band == 3) | (band == 6)
        bulk[k] = v[free]
        v, blk, band = v[~free], blk[~free], band[~free]
        d = np.ones(len(v), np.int32)
        for b in (0, 1, 2, 4, 5, 7, 8):
            m = band == b
            d[m] = per_band[b][blk[m]]
        order = np.lexsort((blk, band, d))
        v, d = v[order], d[order]
        chain[k] = v
        top_d = int(d.max()) if len(d) else 0
        cuts = np.searchsorted(d, np.arange(1, top_d + 2))
        slices[k] = [(int(a), int(b - a)) for a, b in zip(cuts[:-1], cuts[1:])]
    return bulk, chain, slices


class _KeyframeLists(ctypes.Structure):
    """struct daala_b200_keyframe_lists"""
    _fields_ = [
        ("n_luma", ctypes.c_int), ("n_chroma", ctypes.c_int),
        ("luma", ctypes.c_void_p), ("chroma", ctypes.c_void_p),
        ("dep_top", ctypes.c_void_p), ("dep_left", ctypes.c_void_p), ("depth", ctypes.c_void_p),
        ("luma_total", ctypes.c_longlong), ("chroma_total", ctypes.c_longlong),
        ("chain", ctypes.c_void_p * 3), ("chain_wave", ctypes.c_void_p * 3),
        ("wave_first", ctypes.c_void_p * 3), ("wave_count", ctypes.c_void_p * 3),
        ("bulk", ctypes.c_void_p * 3), ("chroma_list", ctypes.c_void_p * 3),
        ("n_chain", ctypes.c_int * 3), ("n_waves", ctypes.c_int * 3), ("n_bulk", ctypes.c_int * 3),
        ("n_chroma_list", ctypes.c_int * 3),
    ]


def native_keyframe_lists(bsize_maps, geom, nthreads=8):
    """The work lists of a keyframe batch built by the library's host code
    (daala_b200_host_keyframe_lists, csrc/host_lists.cu): the same arrays, in the same order, as
    block_list + raster_order + sort_by_depth + band_wave_lists (luma) and mark_luma4x4 + the stable
    size sort + band_lists (chroma) produce in numpy -- about two orders of magnitude faster, which
    matters because a real encoder rebuilds them for every frame.  No GPU involved."""
    L = _native.lib()
    fn = L.daala_b200_host_keyframe_lists
    fn.restype = ctypes.POINTER(_KeyframeLists)
    fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                   ctypes.c_int]
    L.daala_b200_host_keyframe_lists_free.argtypes = [ctypes.POINTER(_KeyframeLists)]
    maps = np.ascontiguousarray(np.stack([np.asarray(b, np.uint8) for b in bsize_maps]))
    assert maps.shape[1:] == tuple(geom.bsize_shape)
    p = fn(maps.ctypes.data, len(maps), maps.strides[0], maps.strides[1], geom.nhsb, geom.nvsb, nthreads)
    if not p:
        raise RuntimeError("daala_b200_host_keyframe_lists failed")
    k = p.contents

    def arr(ptr, count, dtype):
        if count == 0:
            return np.zeros(0, dtype)
        nbytes = count * np.dtype(dtype).itemsize
        return np.frombuffer((ctypes.c_char * nbytes).from_address(ptr), dtype=dtype).copy()

    try:
        out = dict(
            luma=arr(k.luma, k.n_luma, BLOCK_DTYPE), chroma=arr(k.chroma, k.n_chroma, BLOCK_DTYPE),
            dep_top=arr(k.dep_top, k.n_luma, np.int32), dep_left=arr(k.dep_left, k.n_luma, np.int32),
            depth=arr(k.depth, k.n_luma, np.int32), luma_total=int(k.luma_total), chroma_total=int(k.chroma_total),
            chain={}, chain_wave={}, chain_slices={}, bulk={}, chroma_lists={})
        for c, key in enumerate((16, 32, 128)):
            out["chain"][key] = arr(k.chain[c], k.n_chain[c], np.uint32)
            out["chain_wave"][key] = arr(k.chain_wave[c], k.n_chain[c], np.uint16)
            first = arr(k.wave_first[c], k.n_waves[c], np.int32)
            count = arr(k.wave_count[c], k.n_waves[c], np.int32)
            out["chain_slices"][key] = [(int(a), int(b)) for a, b in zip(first, count)]
            out["bulk"][key] = arr(k.bulk[c], k.n_bulk[c], np.uint32)
            out["chroma_lists"][key] = arr(k.chroma_list[c], k.n_chroma_list[c], np.uint32)
    finally:
        L.daala_b200_host_keyframe_lists_free(p)
    return out


# Luma chain waves of fewer bands than this (per size class) use the group-cooperative kernels: shorter latency
# than the default mix (measured crossover of the scalar and 16-lane kernels).
COOP_WAVE_BANDS = {16: 32768, 32: 65536, 128: 0}
COOP_WAVE_MODE = 3


class PvqBatch:
    """Device state of one PVQ batch: coding-order buffers, result arrays and
    the launch sequence gather -> [CfL flip] -> bands -> finish -> scatter."""

    def __init__(self, blocks, coef_planes, pred_planes=None, q0=38, is_keyframe=1, use_masking=1,
                 lam=PVQ_LAMBDA, qm=None, qm_inv=None, pvq_qm_q4=None, device="cuda:0"):
        self.device = torch.device(device)
        dev = self.device
        if isinstance(blocks, dict):
            # descriptors and band lists already on the device (daala_b200/lists_torch.py):
            # {"records": [n, 12] uint8, "total": coefficients, "lists": {16 / 32 / 128: int32 entries}}
            self.blocks_np = None
            self.total = int(blocks["total"])
            self.nblocks = int(blocks["records"].shape[0])
            self.blocks = blocks["records"].reshape(-1).to(dev)
            self.lists = {k: v.to(dev) for k, v in blocks["lists"].items()}
        else:
            self.blocks_np = blocks.copy()
            self.total = assign_offsets(self.blocks_np)
            self.nblocks = len(blocks)
            self.blocks = torch.from_numpy(self.blocks_np.view(np.uint8).reshape(-1)).to(dev)
            lists = band_lists(self.blocks_np)
            self.lists = {k: torch.from_numpy(v.view(np.int32)).to(dev) for k, v in lists.items()}
        z = lambda n, dt=torch.int32: torch.zeros(max(n, 1), dtype=dt, device=dev)  # noqa: E731
        self.in_, self.ref, self.out, self.y = z(self.total), z(self.total), z(self.total), z(self.total)
        nb9 = self.nblocks * 9
        self.res_gain, self.res_theta, self.res_max_theta, self.res_k = z(nb9), z(nb9), z(nb9), z(nb9)
        self.res_skip_term = z(nb9, torch.float64)
        self.res_skip_diff = z(self.nblocks, torch.float64)
        self.res_flip, self.res_dc = z(self.nblocks), z(self.nblocks)
        self.y16 = z(self.total, torch.int16)
        if qm is None:
            qm, qm_inv = default_qm(True)
        self.qm = torch.from_numpy(qm).to(dev)
        self.qm_inv = torch.from_numpy(qm_inv).to(dev)
        self.coef_planes = coef_planes      # list of [F, h, w] int32 tensors
        self.pred_planes = pred_planes      # same or None
        p = PvqParams()
        p.blocks = self.blocks.data_ptr()
        p.in_, p.ref, p.out, p.y = (t.data_ptr() for t in (self.in_, self.ref, self.out, self.y))
        p.res_gain, p.res_theta = self.res_gain.data_ptr(), self.res_theta.data_ptr()
        p.res_max_theta, p.res_k = self.res_max_theta.data_ptr(), self.res_k.data_ptr()
        p.res_skip_term, p.res_skip_diff = self.res_skip_term.data_ptr(), self.res_skip_diff.data_ptr()
        p.res_flip, p.res_dc = self.res_flip.data_ptr(), self.res_dc.data_ptr()
        p.y16 = self.y16.data_ptr()
        p.qm, p.qm_inv, p.qm_stride = self.qm.data_ptr(), self.qm_inv.data_ptr(), OD_QM_STRIDE
        for i, t in enumerate(coef_planes):
            p.coef_plane[i] = t.data_ptr()
            p.plane_stride[i] = t.stride(1)
            p.plane_frame_pitch[i] = t.stride(0)
            p.pred_plane[i] = pred_planes[i].data_ptr() if pred_planes is not None else None
        p.q0, p.is_keyframe, p.use_masking = int(q0), int(is_keyframe), int(use_masking)
        p.pvq_norm_lambda = float(lam)
        if pvq_qm_q4 is None:
            pvq_qm_q4 = np.full((3, 30), 16, np.uint8)
        for pli in range(3):
            for i in range(30):
                p.pvq_qm_q4[pli][i] = int(pvq_qm_q4[pli][i])
        self.params = p
        self.is_keyframe = int(is_keyframe)
        # kernel choice of daala_b200_pvq_encode_bands_mode (0 = measured-best mix)
        self.mode = 0
        # bucket every launch's entries by expected search work (daala_b200_pvq_order_by_work)
        self.order_by_work = True
        self._order_bins = torch.zeros(_bind().daala_b200_pvq_order_bins(), dtype=torch.int32, device=dev)
        self._order_keys = torch.zeros(max(1, max(v.numel() for v in self.lists.values())), dtype=torch.int16,
                                       device=dev)
        self.ordered = {k: torch.empty_like(v) for k, v in self.lists.items()}

    def symbol_tensors(self):
        """What the host entropy coder consumes: per-band indices, flags and the packed pulses."""
        return [self.res_gain, self.res_theta, self.res_max_theta, self.res_k, self.res_skip_diff, self.res_flip,
                self.res_dc, self.y16]

    def _s(self, stream):
        s = stream if stream is not None else torch.cuda.current_stream(self.device)
        return ctypes.c_void_p(s.cuda_stream)

    def gather(self, stream=None):
        L = _bind()
        p = ctypes.byref(self.params)
        _native.check(L.daala_b200_coding_order_gather(p, self.nblocks, 0, self._s(stream)), "gather(in)")
        _native.check(L.daala_b200_coding_order_gather(p, self.nblocks, 1, self._s(stream)), "gather(ref)")

    def _order(self, src, dst, nmax, s, waves=None, nwaves=1):
        """dst <- src bucketed by (wave, work); 3 launches.  Needs `in` gathered."""
        if not src.numel():
            return 0
        assert src.numel() <= self._order_keys.numel()
        _native.check(_bind().daala_b200_pvq_order_by_work(
            ctypes.byref(self.params), src.data_ptr(), waves.data_ptr() if waves is not None else None, src.numel(),
            nwaves, nmax, dst.data_ptr(), self._order_keys.data_ptr(), self._order_bins.data_ptr(), s), "order_by_work")
        return 3

    def quantise(self, stream=None):
        L = _bind()
        p = ctypes.byref(self.params)
        s = self._s(stream)
        n = 0
        if self.is_keyframe:
            _native.check(L.daala_b200_pvq_cfl_flip(p, self.nblocks, s), "cfl_flip")
            n += 1
        for nmax in (128, 32, 16):
            lst = self.lists[nmax]
            if self.order_by_work and lst.numel():
                n += self._order(lst, self.ordered[nmax], nmax, s)
                lst = self.ordered[nmax]
            if lst.numel():
                _native.check(L.daala_b200_pvq_encode_bands_mode(p, lst.data_ptr(), lst.numel(), nmax, self.mode, s),
                              "pvq_bands")
                n += 1
        _native.check(L.daala_b200_pvq_block_finish(p, self.nblocks, s), "block_finish")
        return n + 1

    def scatter(self, stream=None):
        L = _bind()
        _native.check(L.daala_b200_coding_order_scatter(ctypes.byref(self.params), self.nblocks, self._s(stream)),
                      "scatter")

    # --- keyframe predictors -------------------------------------------------
    def _intra_streams(self):
        dev = self.device
        if dev.type == "cuda":
            self.chain_streams = {k: torch.cuda.Stream(device=dev, priority=-1) for k in (16, 32, 128)}
            self.bulk_stream = torch.cuda.Stream(device=dev)
        else:                       # host-side dry runs of the list plumbing (tests)
            self.chain_streams, self.bulk_stream = {}, None

    def setup_intra_device(self, lists):
        """setup_intra for descriptors built on the device (lists_torch.keyframe_lists output)."""
        dev = self.device
        self.dep_top, self.dep_left = lists["dep_top"].to(dev), lists["dep_left"].to(dev)
        self.max_depth = int(lists["depth"].max().item()) if self.nblocks else 0
        self.chain_lists = {k: lists["chain"][k].to(dev) for k in (16, 32, 128)}
        self.bulk_lists = {k: lists["bulk"][k].to(dev) for k in (16, 32, 128)}
        self.chain_waves = {k: lists["chain_wave"][k].to(dev) for k in (16, 32, 128)}
        self.chain_slices = {k: list(lists["chain_slices"][k]) for k in (16, 32, 128)}
        self.chain_ordered = {k: torch.empty_like(v) for k, v in self.chain_lists.items()}
        self.bulk_ordered = {k: torch.empty_like(v) for k, v in self.bulk_lists.items()}
        need = max([v.numel() for v in self.chain_lists.values()] + [v.numel() for v in self.bulk_lists.values()] + [1])
        if need > self._order_keys.numel():
            self._order_keys = torch.zeros(need, dtype=torch.int16, device=dev)
        self._intra_streams()

    def setup_intra(self, top, left, depth):
        """Luma-only batch whose blocks are sorted by dependency depth (see
        `sort_by_depth`): neighbour indices and the band-granular wave lists."""
        dev = self.device
        self.dep_top = torch.from_numpy(np.ascontiguousarray(top)).to(dev)
        self.dep_left = torch.from_numpy(np.ascontiguousarray(left)).to(dev)
        self.max_depth = int(depth.max()) if len(depth) else 0
        # band b of a block depends on band b of the same-size top (bands 1/4/7), left (2/5/8),
        # both (0) or no (3/6) neighbour -- see k_intra_band_ref.  Every size class is a closed
        # dependency system, so each gets its own stream and wave sequence.
        bulk, chain, self.chain_slices = band_wave_lists(self.blocks_np, top, left, depth)
        as_dev = lambda v: torch.from_numpy(np.ascontiguousarray(v).view(np.int32)).to(dev)  # noqa: E731
        self.bulk_lists = {k: as_dev(v) for k, v in bulk.items()}
        self.chain_lists = {k: as_dev(v) for k, v in chain.items()}
        self.chain_waves, self.chain_ordered, self.bulk_ordered = {}, {}, {}
        for k, sl in self.chain_slices.items():
            assert len(sl) < 65536
            w = np.repeat(np.arange(len(sl), dtype=np.uint16), [c for _, c in sl])
            self.chain_waves[k] = torch.from_numpy(w.view(np.int16)).to(dev)
            self.chain_ordered[k] = torch.empty_like(self.chain_lists[k])
            self.bulk_ordered[k] = torch.empty_like(self.bulk_lists[k])
        self._intra_streams()

    def run_luma_intra(self, stream=None):
        L = _bind()
        p = ctypes.byref(self.params)
        main = stream if stream is not None else torch.cuda.current_stream(self.device)
        _native.check(L.daala_b200_coding_order_gather(p, self.nblocks, 0, self._s(main)), "gather(in)")
        n = 1
        top, left = self.dep_top.data_ptr(), self.dep_left.data_ptr()
        chain_lists, bulk_lists = self.chain_lists, self.bulk_lists
        if self.order_by_work:
            for k in (128, 32, 16):
                n += self._order(self.chain_lists[k], self.chain_ordered[k], k, self._s(main),
                                 self.chain_waves[k], max(1, len(self.chain_slices[k])))
                n += self._order(self.bulk_lists[k], self.bulk_ordered[k], k, self._s(main))
            chain_lists, bulk_lists = self.chain_ordered, self.bulk_ordered
        # latency-bound chains first (high-priority streams), the dependency-free bands fill the GPU behind
        for k in (128, 32, 16):
            st = self.chain_streams[k]
            st.wait_stream(main)
            sp = ctypes.c_void_p(st.cuda_stream)
            for w, (a, c) in enumerate(self.chain_slices[k]):
                if not c:
                    continue
                ptr = chain_lists[k].data_ptr() + 4 * a
                if w > 0:
                    _native.check(L.daala_b200_pvq_intra_band_ref(p, top, left, ptr, c, sp), "intra_band_ref")
                    n += 1
                mode = COOP_WAVE_MODE if c < COOP_WAVE_BANDS[k] else self.mode
                _native.check(L.daala_b200_pvq_encode_bands_mode(p, ptr, c, k, mode, sp), "pvq_bands")
                n += 1
        self.bulk_stream.wait_stream(main)
        sp = ctypes.c_void_p(self.bulk_stream.cuda_stream)
        for k in (128, 32):
            lst = bulk_lists[k]
            if lst.numel():
                _native.check(L.daala_b200_pvq_encode_bands_mode(p, lst.data_ptr(), lst.numel(), k, self.mode, sp),
                              "pvq_bands")
                n += 1
        for st in list(self.chain_streams.values()) + [self.bulk_stream]:
            main.wait_stream(st)
        _native.check(L.daala_b200_pvq_block_finish(p, self.nblocks, self._s(main)), "block_finish")
        _native.check(L.daala_b200_coding_order_scatter(p, self.nblocks, self._s(main)), "scatter")
        return n + 2

    def cfl_pred(self, pred_plane, stream=None):
        """Fill the chroma prediction plane ([F, h/2, w/2] int32) from the quantised luma."""
        L = _bind()
        _native.check(L.daala_b200_pvq_cfl_pred(ctypes.byref(self.params), pred_plane.data_ptr(),
                                                pred_plane.stride(0), pred_plane.stride(1), self.nblocks,
                                                self._s(stream)), "pvq_cfl_pred")
        return 1

    def run(self, stream=None):
        """gather -> quantise -> scatter; returns the number of kernel launches."""
        self.gather(stream)
        n = self.quantise(stream)
        self.scatter(stream)
        return n + 3
