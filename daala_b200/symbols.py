"""The keyframe engine's symbol stream (include/daala_b200.h, "Symbol stream"; config.symbol_stream = 1): per
frame the PVQ symbols the serial entropy coder reads, in bitstream order.  The P-frame stream (symbol_stream = 2,
inter = 1) is the same with flip = 0 and a DC_DTYPE record per block record (sym_dc, same index): the step's scalar
DC index and the unquantised DC residual; with late_skip = 1 also a LATE_SKIP_DTYPE record (sym_late_skip).  The
mixed stream (symbol_stream = 3, frame_types = 1) has both record kinds: each frame's block records in the kind of its
frame, a keyframe's with its CfL flips, HDC_DTYPE records and zero DC_DTYPE records, a P / B frame's with flip 0,
DC_DTYPE records and zero HDC_DTYPE records (no keyframe record is all zero: bsi = 4 or child >= 1).

For each frame of a batch the index (int64[6]: first block, block count, first band, band count, first pulse
byte, pulse byte count) locates three parts inside batch-wide arrays:
  blocks  one BLOCK_DTYPE record per leaf block, in coding order;
  bands   per block NBANDS[bs] records {coded gain index, itheta, max_theta, K} (int16[4]), in band order;
  pulses  per band with K > 0 the n - (itheta != -1) values od_encode_pvq_codeword codes, int8 when K <= 127,
          little-endian int16 otherwise.
Coding order: superblocks in raster order, planes 0, 1, 2, inside a plane the quadtree leaves depth-first with
the children top-left, top-right, bottom-left, bottom-right (od_encode_recursive, reference src/encode.c).

This module holds the dtypes, a reader, `coding_order` (a walk of that recursion over a block-size map),
`pack_reference` (the expected stream built with numpy from the engine's classic outputs) and `stream_to_classic`
(each stream record's index in the classic block order)."""
import numpy as np

BLOCK_DTYPE = np.dtype([("skip_diff", "<f8"), ("pulse_off", "<u4"), ("band_off", "<u4"), ("x0", "<u2"),
                        ("y0", "<u2"), ("bs", "u1"), ("pli", "u1"), ("flip", "u1"), ("reserved", "u1")])
assert BLOCK_DTYPE.itemsize == 24
INDEX_FIELDS = ("first_block", "n_blocks", "first_band", "n_bands", "first_byte", "n_bytes")
NBANDS = np.array([1, 4, 7, 9, 9])
BAND_EDGES = np.array([1, 16, 24, 32, 64, 96, 128, 256, 384, 512])   # OD_BAND_OFFSETS in coding order
ORDER_DTYPE = np.dtype([("pli", "u1"), ("x0", "<u2"), ("y0", "<u2"), ("bs", "u1")])
DC_DTYPE = np.dtype([("qdc", "<i4"), ("dc_resid", "<i4")])
assert DC_DTYPE.itemsize == 8
# symbol_stream = 1 with haar_dc_quant = 1: daala_b200_kf_sym_hdc, the keyframe's DC symbols in coding order, one per
# block record (sym_hdc, same index range; haardc.stream_records)
HDC_DTYPE = np.dtype([("value", "<i4"), ("block", "<u4"), ("pli", "u1"), ("bsi", "u1"), ("child", "u1"),
                      ("reserved", "u1")])
assert HDC_DTYPE.itemsize == 12
# config.late_skip: daala_b200_kf_late_skip, one per block (block order) or per block record (sym_late_skip)
LATE_SKIP_DTYPE = np.dtype([("dist_skip", "<f8"), ("noskip_coded_dc0", "<f8"), ("noskip_coded_dcq", "<f8"),
                            ("noskip_pred_dcq", "<f8")])
assert LATE_SKIP_DTYPE.itemsize == 32


def _excl(a):
    out = np.zeros(len(a), np.int64)
    if len(a):
        np.cumsum(a[:-1], out=out[1:])
    return out


def _band_sizes(band_no, rec):
    """Values and bytes per value of each band's pulses in the stream."""
    k, itheta = rec[:, 3].astype(np.int64), rec[:, 1].astype(np.int64)
    n = BAND_EDGES[band_no + 1] - BAND_EDGES[band_no] - (itheta != -1)
    n = np.where(k > 0, n, 0)
    width = np.where(k > 127, 2, 1)
    return n, width


def _band_numbers(bs):
    """Band number inside its block of every band of blocks with sizes `bs` (in order)."""
    nb = NBANDS[bs.astype(np.int64)]
    return np.arange(int(nb.sum())) - np.repeat(_excl(nb), nb), nb


def read_frame(out, f):
    """Frame f of a submit's stream outputs (sym_index, sym_blocks, sym_bands, sym_pulses[, sym_dc][, sym_hdc]): dict
    with `blocks` (BLOCK_DTYPE), `bands` (int16[B, 4]), `band_block` (block of each band), `band_no` (band number
    inside its block), `pulses` (per band an int32 vector of its coded values; empty when K = 0) and, when the outputs
    have sym_dc, `dc` (DC_DTYPE, one record per block), when they have sym_hdc, `hdc` (HDC_DTYPE, one record per
    block)."""
    idx = out["sym_index"][f]
    b0, nb, n0, nn, y0, ny = (int(v) for v in idx)
    blocks = out["sym_blocks"][b0:b0 + nb]
    bands = out["sym_bands"][n0:n0 + nn]
    data = out["sym_pulses"][y0:y0 + ny]
    band_no, per = _band_numbers(blocks["bs"])
    assert len(band_no) == nn, "band count does not match the blocks' sizes"
    band_block = np.repeat(np.arange(nb), per)
    n, width = _band_sizes(band_no, bands)
    nbytes = n * width
    start = _excl(nbytes)
    assert int(nbytes.sum()) == ny, "pulse byte count does not match the band records"
    # every block's pulse_off / band_off is where its first band's data starts
    assert np.array_equal(blocks["band_off"].astype(np.int64), _excl(per))
    assert np.array_equal(blocks["pulse_off"].astype(np.int64), start[_excl(per)] if nb else np.zeros(0, np.int64))
    vi = np.repeat(np.arange(nn), n)
    t = np.arange(int(n.sum())) - np.repeat(_excl(n), n)
    w = width[vi]
    pos = start[vi] + t * w
    lo = data[pos].astype(np.int64)
    hi = data[np.minimum(pos + 1, max(ny - 1, 0))].astype(np.int64) if ny else lo
    v = np.where(w == 2, (lo | (hi << 8)).astype(np.uint16).view(np.int16), lo.astype(np.uint8).view(np.int8))
    v = v.astype(np.int32)
    pulses = np.split(v, np.cumsum(n)[:-1]) if nn else []
    r = dict(blocks=blocks, bands=bands, band_block=band_block, band_no=band_no, pulses=pulses)
    if "sym_dc" in out:
        r["dc"] = out["sym_dc"][b0:b0 + nb]
    if "sym_hdc" in out:
        r["hdc"] = out["sym_hdc"][b0:b0 + nb]
    return r


def coding_order(bsize, geom, sb_row0=0, sb_rows=None):
    """Leaf blocks of one frame in bitstream order: superblock raster order, planes 0 .. nplanes-1, the
    od_encode_recursive quadtree walk (src/encode.c:1669-1787: the size is read at the block's top-left 8x8 unit,
    bs = max(obs, xdec), children TL, TR, BL, BR).  Returns an ORDER_DTYPE array (plane coordinates, plane bs)."""
    bsize = np.asarray(bsize)
    sb_rows = geom.nvsb - sb_row0 if sb_rows is None else sb_rows
    out = []

    def walk(pli, xdec, bx, by, bsi):
        obs = int(bsize[(by << bsi) >> 1, (bx << bsi) >> 1])
        bs = max(obs, xdec)
        if bs == bsi:
            sh = 2 + bsi - xdec
            out.append((pli, bx << sh, by << sh, bsi - xdec))
            return
        for dy in (0, 1):
            for dx in (0, 1):
                walk(pli, xdec, 2 * bx + dx, 2 * by + dy, bsi - 1)

    for sby in range(sb_row0, sb_row0 + sb_rows):
        for sbx in range(geom.nhsb):
            for pli in range(geom.nplanes):
                walk(pli, geom.xdec[pli], sbx, sby, 4)
    return np.array(out, ORDER_DTYPE)


def _zrank(x0, y0, pli):
    """Sort key of bitstream order inside a frame: (superblock row, superblock column, plane, Z order of the
    block's origin inside the superblock in 4-sample units)."""
    x0, y0 = x0.astype(np.int64), y0.astype(np.int64)
    sh = np.where(pli > 0, 5, 6)                # superblock edge in plane samples (4:2:0 chroma: 32)
    ux, uy = (x0 & ((1 << sh) - 1)) >> 2, (y0 & ((1 << sh) - 1)) >> 2
    z = np.zeros_like(x0)
    for bit in range(4):
        z |= ((ux >> bit) & 1) << (2 * bit)
        z |= ((uy >> bit) & 1) << (2 * bit + 1)
    return y0 >> sh, x0 >> sh, z


def pack_blocks(x0, y0, bs, pli, flip, skip_diff, res, y, y_off, qdc=None, dc_resid=None):
    """One frame's stream parts from its blocks listed in coding order: band records res[i, :nbands] and
    pulse vectors in coding order at y[y_off[i]:] (DC at index 0).  Returns (blocks, bands, pulses), and with qdc
    and dc_resid (P frames) also the DC records."""
    n = len(bs)
    bs = np.asarray(bs).astype(np.int64)
    band_no, per = _band_numbers(bs)
    band_block = np.repeat(np.arange(n), per)
    bands = np.ascontiguousarray(res[band_block, band_no], np.int16).reshape(-1, 4)
    nv, width = _band_sizes(band_no, bands)
    nbytes = nv * width
    start = _excl(nbytes)
    blocks = np.zeros(n, BLOCK_DTYPE)
    blocks["skip_diff"] = skip_diff
    blocks["band_off"] = _excl(per)
    blocks["pulse_off"] = start[_excl(per)] if n else 0
    blocks["x0"], blocks["y0"], blocks["bs"], blocks["pli"], blocks["flip"] = x0, y0, bs, pli, flip
    vi = np.repeat(np.arange(len(nv)), nv)
    t = np.arange(int(nv.sum())) - np.repeat(_excl(nv), nv)
    v = np.asarray(y)[np.asarray(y_off, np.int64)[band_block[vi]] + BAND_EDGES[band_no[vi]] + t].astype(np.int64)
    w = width[vi]
    pos = start[vi] + t * w
    pulses = np.zeros(int(nbytes.sum()), np.uint8)
    pulses[pos] = (v & 0xff).astype(np.uint8)
    m = w == 2
    pulses[pos[m] + 1] = ((v[m] >> 8) & 0xff).astype(np.uint8)
    if qdc is None:
        return blocks, bands, pulses
    dc = np.zeros(n, DC_DTYPE)
    dc["qdc"], dc["dc_resid"] = qdc, dc_resid
    return blocks, bands, pulses, dc


def concat_frames(parts):
    """Batch-wide (index, blocks, bands, pulses[, dc]) from per-frame (blocks, bands, pulses[, dc])."""
    index = np.zeros((len(parts), 6), np.int64)
    pos = np.zeros(3, np.int64)
    for f, (b, n, p) in enumerate(q[:3] for q in parts):
        index[f] = (pos[0], len(b), pos[1], len(n), pos[2], len(p))
        pos += (len(b), len(n), len(p))
    cat = (lambda xs, dt, shape: np.concatenate(xs) if xs else np.zeros(shape, dt))
    r = dict(sym_index=index, sym_blocks=cat([p[0] for p in parts], BLOCK_DTYPE, (0,)),
             sym_bands=cat([p[1] for p in parts], np.int16, (0, 4)),
             sym_pulses=cat([p[2] for p in parts], np.uint8, (0,)))
    if parts and len(parts[0]) == 4:
        r["sym_dc"] = cat([p[3] for p in parts], DC_DTYPE, (0,))
    return r


def pack_reference(out, frames, frame_type=None):
    """The stream the engine must produce, built from a submit's classic outputs (luma_/chroma_blocks, _res,
    _y16, _skip_diff, chroma_flip) for the frames `frames` (list, or a count = frames 0 .. count-1).  Blocks are
    put in bitstream order by sorting on (superblock, plane, Z order of the origin), independently of how the
    device ranks them.  Returns dict(sym_index, sym_blocks, sym_bands, sym_pulses) over those frames.  The outputs of
    a P-frame step (they have luma_dc / chroma_dc, and luma_dc_resid / chroma_dc_resid must be there too) give the
    P-frame stream: flip 0 and sym_dc from *_dc and *_dc_resid.  Those of a haar_dc_quant keyframe step with the index
    grids (dc_index0..2) give sym_hdc too (haardc.stream_records over the map the luma blocks tile).
    frame_type (the type of every frame of the step, 1 = keyframe) gives the mixed stream (symbol_stream = 3) from a
    frame_types step's outputs, which have both: each keyframe's records as the keyframe stream has them with a zero
    sym_dc record, each P / B frame's as the P-frame stream has them with a zero sym_hdc record."""
    frames = list(range(frames)) if np.isscalar(frames) else list(frames)
    inter = "luma_dc" in out
    hdc = (frame_type is not None or not inter) and "dc_index0" in out
    lb, cb = out["luma_blocks"], out["chroma_blocks"]
    nl_coefs = len(out["luma_y16"])
    y = np.concatenate([out["luma_y16"], out["chroma_y16"]])
    parts, hdcs = [], []
    for f in frames:
        key = not inter if frame_type is None else bool(frame_type[f])
        sl, sc = np.nonzero(lb["frame"] == f)[0], np.nonzero(cb["frame"] == f)[0]
        blk = np.concatenate([lb[sl], cb[sc]])
        res = np.concatenate([out["luma_res"][sl], out["chroma_res"][sc]])
        skip = np.concatenate([out["luma_skip_diff"][sl], out["chroma_skip_diff"][sc]])
        flip = np.zeros(len(blk), np.int64)
        if key:
            flip[len(sl):] = out["chroma_flip"][sc]
        y_off = np.concatenate([lb["coef_off"][sl].astype(np.int64), cb["coef_off"][sc].astype(np.int64) + nl_coefs])
        pli = blk["pli"].astype(np.int64)
        sby, sbx, z = _zrank(blk["x0"], blk["y0"], pli)
        o = np.lexsort((z, pli, sbx, sby))
        dc = {}
        if inter:
            for k in ("dc", "dc_resid"):
                v = np.concatenate([out["luma_" + k][sl], out["chroma_" + k][sc]])[o]
                dc[k] = np.zeros_like(v) if key else v
        parts.append(pack_blocks(blk["x0"][o], blk["y0"][o], blk["bs"][o], pli[o], flip[o], skip[o], res[o], y,
                                 y_off[o], dc.get("dc"), dc.get("dc_resid")))
        if hdc:
            hdcs.append(_hdc_reference(out, lb[sl], f) if key else np.zeros(len(blk), HDC_DTYPE))
    r = concat_frames(parts)
    if hdc:
        r["sym_hdc"] = np.concatenate(hdcs) if hdcs else np.zeros(0, HDC_DTYPE)
    return r


def _hdc_reference(out, luma, f):
    """Frame f's keyframe DC records from the index grids dc_index0..2 and the map its luma blocks tile."""
    from . import haardc
    from .frame import Geometry
    idx = [np.asarray(out["dc_index%d" % p][f]) for p in range(3)]
    gh, gw = idx[0].shape
    geom = Geometry(gw * 4, gh * 4)
    bsize = np.zeros(geom.bsize_shape, np.uint8)
    for x0, y0, bs in zip(luma["x0"].astype(np.int64), luma["y0"].astype(np.int64), luma["bs"].astype(np.int64)):
        n = max(1, 1 << (bs - 1))            # 8x8 units the block spans (a 4x4 block: its unit, value 0)
        bsize[y0 >> 3:(y0 >> 3) + n, x0 >> 3:(x0 >> 3) + n] = bs
    return haardc.stream_records(idx, bsize, geom)


def stream_to_classic(out):
    """For every block record of a submit's stream (sym_index, sym_blocks), in the order of sym_blocks (frames one
    after the other), the index of the same block in the classic block order (luma_blocks i -> i, chroma_blocks
    i -> n_luma + i).  A decision array `d` in classic order is `d[stream_to_classic(out)]` in stream order (what
    KeyframeEngine.finish_stream takes)."""

    def key(frame, pli, x0, y0):
        return ((np.asarray(frame, np.int64) * 3 + pli) << 32) | (np.asarray(y0, np.int64) << 16) | np.asarray(x0, np.int64)

    lb, cb = out["luma_blocks"], out["chroma_blocks"]
    classic = np.concatenate([key(b["frame"], b["pli"].astype(np.int64), b["x0"], b["y0"]) for b in (lb, cb)])
    idx = out["sym_index"]
    n = int(idx[:, 1].sum())
    sb = out["sym_blocks"][:n]
    stream = key(np.repeat(np.arange(len(idx)), idx[:, 1]), sb["pli"].astype(np.int64), sb["x0"], sb["y0"])
    o = np.argsort(classic, kind="stable")
    pos = np.minimum(np.searchsorted(classic[o], stream), max(len(o) - 1, 0))
    assert n == len(classic) and np.array_equal(classic[o][pos], stream), \
        "the stream's blocks are not the classic lists' blocks"
    return o[pos]


def stream_equal(got, want, frames_got, frames_want=None):
    """Frame by frame byte equality of two streams (dicts of sym_* arrays); returns a list of differences."""
    frames_want = frames_got if frames_want is None else frames_want
    bad = []
    for fg, fw in zip(frames_got, frames_want):
        ig, iw = got["sym_index"][fg], want["sym_index"][fw]
        for name, col in (("n_blocks", 1), ("n_bands", 3), ("n_bytes", 5)):
            if ig[col] != iw[col]:
                bad.append((fg, name, int(ig[col]), int(iw[col])))
        if bad:
            continue
        parts = (("sym_blocks", 0, 1), ("sym_bands", 2, 3), ("sym_pulses", 4, 5))
        if "sym_dc" in got or "sym_dc" in want:
            parts += (("sym_dc", 0, 1),)
        if "sym_hdc" in got or "sym_hdc" in want:
            parts += (("sym_hdc", 0, 1),)
        for key, c0, c1 in parts:
            if key not in got or key not in want:
                bad.append((fg, key, "missing"))
                continue
            a = got[key][ig[c0]:ig[c0] + ig[c1]]
            b = want[key][iw[c0]:iw[c0] + iw[c1]]
            if a.tobytes() != b.tobytes():
                diff = np.nonzero(a.view(np.uint8).reshape(len(a), -1) != b.view(np.uint8).reshape(len(b), -1))[0]
                bad.append((fg, key, "first differing entry %d of %d" % (int(diff[0]), len(a))))
    return bad
