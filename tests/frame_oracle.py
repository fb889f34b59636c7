"""Frame-level CPU oracle calls (test infrastructure): drives
oracle/pipeline_driver.inc through either the real reference build
(oracle/_ref) or the plain-C port."""
import ctypes

import numpy as np  # noqa: E402

from tests.oracle_lib import addr


def forward_plane(lib, prefix, src, geom, pli, bsize, haar_dc):
    ph, pw = geom.plane_shape(pli)
    src = np.ascontiguousarray(src, dtype=np.uint8)
    assert src.shape == (ph, pw)
    c = np.zeros((ph, pw), np.int32)
    d = np.zeros((ph, pw), np.int32)
    bs = np.ascontiguousarray(bsize, dtype=np.uint8)
    fn = getattr(lib, "oracle_%s_forward_plane" % prefix)
    fn(addr(src), pw, addr(c), addr(d), geom.nhsb, geom.nvsb, geom.xdec[pli], addr(bs),
       bs.shape[1], geom.pic_w, geom.pic_h, int(haar_dc))
    return d


def inverse_plane(lib, prefix, d, geom, pli, bsize, haar_dc, lapped_only=False):
    ph, pw = geom.plane_shape(pli)
    d = np.ascontiguousarray(d, dtype=np.int32).copy()
    c = np.zeros((ph, pw), np.int32)
    out = np.zeros((ph, pw), np.uint8)
    bs = np.ascontiguousarray(bsize, dtype=np.uint8)
    fn = getattr(lib, "oracle_%s_inverse_plane" % prefix)
    fn(addr(d), addr(c), addr(out), pw, geom.nhsb, geom.nvsb, geom.xdec[pli], addr(bs), bs.shape[1],
       geom.pic_w, geom.pic_h, int(haar_dc), int(lapped_only))
    return c if lapped_only else out


def pvq_plane(lib, prefix, d, md, geom, pli, bsize, q0, is_keyframe, use_masking, lam, qm, qm_inv, qm_q4):
    """Quantises a coefficient plane in place (a copy is returned) with the
    oracle's per-block PVQ driver; returns (d_quantised, stats[5])."""
    d = np.ascontiguousarray(d, dtype=np.int32).copy()
    bs = np.ascontiguousarray(bsize, dtype=np.uint8)
    stats = np.zeros(5, np.float64)
    q4 = np.ascontiguousarray(qm_q4[pli], dtype=np.uint8)
    mdp = addr(np.ascontiguousarray(md, dtype=np.int32)) if md is not None else None
    fn = getattr(lib, "oracle_%s_pvq_plane" % prefix)
    fn(addr(d), mdp, geom.nhsb, geom.nvsb, geom.xdec[pli], pli, addr(bs), bs.shape[1], int(q0),
       int(is_keyframe), int(use_masking), ctypes.c_double(lam), addr(np.ascontiguousarray(qm)),
       addr(np.ascontiguousarray(qm_inv)), addr(q4), addr(stats))
    return d, stats


def pvq_plane_pred(lib, prefix, d, geom, pli, bsize, q0, use_masking, lam, qm, qm_inv, qm_q4, luma_d=None):
    """Keyframe quantisation WITH the reference's predictors: luma (pli == 0) uses
    od_hv_intra_pred from already quantised neighbours, chroma uses CfL from the
    quantised luma plane `luma_d`.  Returns (d_quantised, stats[5])."""
    d = np.ascontiguousarray(d, dtype=np.int32).copy()
    bs = np.ascontiguousarray(bsize, dtype=np.uint8)
    stats = np.zeros(5, np.float64)
    q4 = np.ascontiguousarray(qm_q4[pli], dtype=np.uint8)
    lp = addr(np.ascontiguousarray(luma_d, dtype=np.int32)) if luma_d is not None else None
    fn = getattr(lib, "oracle_%s_pvq_plane_pred" % prefix)
    fn(addr(d), None, geom.nhsb, geom.nvsb, geom.xdec[pli], pli, addr(bs), bs.shape[1], int(q0), 1,
       int(use_masking), ctypes.c_double(lam), addr(np.ascontiguousarray(qm)), addr(np.ascontiguousarray(qm_inv)),
       addr(q4), addr(stats), 1 if pli == 0 else 0, lp)
    return d, stats


def keyframe_chain(lib, prefix, planes, geom, bsize, q0, qm_q4, use_masking=1, lam=0.147, qm=None, qm_inv=None,
                   record=True, dering_levels=None, dering_search=None, symbols=False):
    """One keyframe through the oracle's whole chain (forward -> PVQ with luma H/V intra prediction and
    chroma CfL -> inverse).  Returns per plane a dict: dq (quantised coefficient plane), recon (u8),
    stats, and with record=True rec ([h/4, w/4, 9, 4] int16 band decisions at each block's origin,
    -32768 where no band) and yplane (pulse vectors in raster order).
    symbols=True adds, at each block's origin in 4-sample units like rec, skip_diff ([h/4, w/4] float64,
    NaN where no block starts) and flip ([h/4, w/4] int32: the keyframe CfL sign flip, 0 or 1; -1 where no
    block starts).
    dering_levels: [nvsb, nhsb] levels -> reconstruction through the deringing application.
    dering_search: dict(coded_quantizer=, dering_lambda=, qm=1) -> the levels are searched the way the encoder does
    (src/encode.c:2708-2811, reference build only) and returned as out[0]["dering_levels"]."""
    from daala_b200 import pvq
    if qm is None:
        qm, qm_inv = pvq.default_qm(True)
    out = []
    luma_q = None
    for pli in range(3):
        ph, pw = geom.plane_shape(pli)
        d = forward_plane(lib, prefix, planes[pli], geom, pli, bsize, 1)
        d = np.ascontiguousarray(d, dtype=np.int32).copy()
        bs = np.ascontiguousarray(bsize, dtype=np.uint8)
        stats = np.zeros(5, np.float64)
        q4 = np.ascontiguousarray(qm_q4[pli], dtype=np.uint8)
        rec = np.full((ph // 4, pw // 4, 9, 4), -32768, np.int16) if record else None
        yplane = np.zeros((ph, pw), np.int32) if record else None
        lp = addr(np.ascontiguousarray(luma_q, dtype=np.int32)) if pli else None
        args = [addr(d), None, geom.nhsb, geom.nvsb, geom.xdec[pli], pli, addr(bs), bs.shape[1], int(q0), 1,
                int(use_masking), ctypes.c_double(lam), addr(np.ascontiguousarray(qm)),
                addr(np.ascontiguousarray(qm_inv)), addr(q4), addr(stats), 1 if pli == 0 else 0, lp,
                addr(rec) if record else None, addr(yplane) if record else None]
        if symbols:
            skip = np.full((ph // 4, pw // 4), np.nan, np.float64)
            flip = np.full((ph // 4, pw // 4), -1, np.int32)
            getattr(lib, "oracle_%s_pvq_plane_sym" % prefix)(*args, addr(skip), addr(flip))
        else:
            getattr(lib, "oracle_%s_pvq_plane_rec" % prefix)(*args)
        if pli == 0:
            luma_q = d
        recon = inverse_plane(lib, prefix, d, geom, pli, bsize, 1) if dering_levels is None and dering_search is None else None
        out.append(dict(dq=d, recon=recon, stats=stats, rec=rec, yplane=yplane))
        if symbols:
            out[-1].update(skip_diff=skip, flip=flip)
    if dering_levels is not None:
        # reconstruction with the deringing application (levels [nvsb, nhsb] given): oracle/pipeline_driver.inc
        ds = [np.ascontiguousarray(o["dq"], np.int32).copy() for o in out]
        recs = [np.zeros(geom.plane_shape(p), np.uint8) for p in range(3)]
        bs = np.ascontiguousarray(bsize, dtype=np.uint8)
        lv = np.ascontiguousarray(dering_levels, np.uint8)
        assert lv.shape == (geom.nvsb, geom.nhsb)
        getattr(lib, "oracle_%s_inverse_frame_dering" % prefix)(
            addr(ds[0]), addr(ds[1]), addr(ds[2]), addr(recs[0]), addr(recs[1]), addr(recs[2]), geom.nhsb, geom.nvsb,
            addr(bs), bs.shape[1], geom.pic_w, geom.pic_h, int(q0), addr(lv))
        for p in range(3):
            out[p]["recon"] = recs[p]
    if dering_search is not None:
        ds = [np.ascontiguousarray(o["dq"], np.int32).copy() for o in out]
        recs = [np.zeros(geom.plane_shape(p), np.uint8) for p in range(3)]
        bs = np.ascontiguousarray(bsize, dtype=np.uint8)
        lv = np.zeros((geom.nvsb, geom.nhsb), np.uint8)
        src = np.ascontiguousarray(planes[0], np.uint8)
        fn = getattr(lib, "oracle_%s_inverse_frame_dering_search" % prefix)
        fn.argtypes = [ctypes.c_void_p] * 6 + [ctypes.c_int] * 2 + [ctypes.c_void_p] + [ctypes.c_int] * 4 + [
            ctypes.c_void_p] + [ctypes.c_int] * 4 + [ctypes.c_double, ctypes.c_void_p]
        fn(addr(ds[0]), addr(ds[1]), addr(ds[2]), addr(recs[0]), addr(recs[1]), addr(recs[2]), geom.nhsb, geom.nvsb,
           addr(bs), bs.shape[1], geom.pic_w, geom.pic_h, int(q0), addr(src), src.shape[1],
           int(dering_search["coded_quantizer"]), int(dering_search.get("qm", 1)), int(use_masking),
           float(dering_search["dering_lambda"]), addr(lv))
        for p in range(3):
            out[p]["recon"] = recs[p]
        out[0]["dering_levels"] = lv
    return out
