"""Frame-level CPU oracle for non-key frames (test infrastructure), beside tests/frame_oracle.py: drives the
recording PVQ driver of oracle/pipeline_driver.inc with a prediction plane and is_keyframe = 0, through either the
real reference build (oracle/_ref) or the plain-C port."""
import ctypes

import numpy as np

from tests import frame_oracle
from tests.oracle_lib import addr


def inter_chain(lib, prefix, planes, pred, geom, bsize, q0, qm_q4, use_masking=1, lam=0.147, qm=None, qm_inv=None):
    """One non-key frame through the oracle's residual chain as od_encode_coefficients codes it: source and
    motion-compensated prediction `pred` (u8 planes like `planes`) through the forward transform without the DC
    Haar pyramid, every band quantised against the transformed prediction md (is_keyframe = 0: no intra
    prediction, no CfL, no flip), scalar DC, inverse.  Returns per plane a dict: md, dq, recon, stats, rec, yplane,
    skip_diff (as frame_oracle.keyframe_chain with record and symbols) and qdc ([h/4, w/4] int32 at each block's origin: the
    scalar-quantised DC index, (dq[0] - md[0]) / dc_quant with the band-0 quantiser; 0 where no block starts)."""
    from daala_b200 import pvq
    if qm is None:
        qm, qm_inv = pvq.default_qm(True)
    bs = np.ascontiguousarray(bsize, dtype=np.uint8)
    out = []
    for pli in range(3):
        ph, pw = geom.plane_shape(pli)
        d = np.ascontiguousarray(frame_oracle.forward_plane(lib, prefix, planes[pli], geom, pli, bsize, 0), np.int32).copy()
        md = np.ascontiguousarray(frame_oracle.forward_plane(lib, prefix, pred[pli], geom, pli, bsize, 0), np.int32)
        stats = np.zeros(5, np.float64)
        q4 = np.ascontiguousarray(qm_q4[pli], dtype=np.uint8)
        rec = np.full((ph // 4, pw // 4, 9, 4), -32768, np.int16)
        yplane = np.zeros((ph, pw), np.int32)
        skip = np.full((ph // 4, pw // 4), np.nan, np.float64)
        flip = np.full((ph // 4, pw // 4), -1, np.int32)
        getattr(lib, "oracle_%s_pvq_plane_sym" % prefix)(
            addr(d), addr(md), geom.nhsb, geom.nvsb, geom.xdec[pli], pli, addr(bs), bs.shape[1], int(q0), 0,
            int(use_masking), ctypes.c_double(lam), addr(np.ascontiguousarray(qm)), addr(np.ascontiguousarray(qm_inv)),
            addr(q4), addr(stats), 0, None, addr(rec), addr(yplane), addr(skip), addr(flip))
        # block sizes at the origins (4-sample units of this plane), from the band records: 1, 4, 7 bands = 4x4,
        # 8x8, 16x16; 9 bands = 32x32 or 64x64, told apart by the map
        origin = ~np.isnan(skip)
        ys, xs = np.nonzero(origin)
        sh = 1 - geom.xdec[pli]   # 4-sample units of this plane per map unit, log2
        obs = bs[ys >> sh, xs >> sh].astype(np.int64)
        pbs = np.maximum(obs, geom.xdec[pli]) - geom.xdec[pli]
        dcq = np.maximum((int(q0) * q4[pbs * (pbs + 1)].astype(np.int64)) >> 4, 1)
        diff = d[ys * 4, xs * 4].astype(np.int64) - md[ys * 4, xs * 4]
        assert not np.any(diff % dcq), "DC is not md + a multiple of the quantiser"
        qdc = np.zeros((ph // 4, pw // 4), np.int32)
        qdc[ys, xs] = diff // dcq
        recon = frame_oracle.inverse_plane(lib, prefix, d, geom, pli, bsize, 0)
        out.append(dict(md=md, dq=d, recon=recon, stats=stats, rec=rec, yplane=yplane, skip_diff=skip, qdc=qdc))
    return out
