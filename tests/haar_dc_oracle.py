"""CPU oracle of quantised keyframe DCs (test infrastructure): the driver oracle_ref_haar_dc_frame of
oracle/ref_hooks_haar_dc.c (the reference's own od_compute_dcts, od_quantize_haar_dc_sb and od_quantize_haar_dc_level
in od_encode_recursive's order on a real encoder), which oracle/haar_dc.mk links with the reference build's objects
into oracle/_ref/libdaala_ref_haar_dc.so."""
import ctypes
import os
import subprocess

import numpy as np

from tests import oracle_lib
from tests.oracle_lib import addr

_lib = []


def load():
    """The driver library: (re)built first when the reference sources are present, else used as it is; None when it
    is absent."""
    if not _lib:
        if oracle_lib.have_ref_sources():
            subprocess.run(["make", "-C", oracle_lib.ORACLE, "-f", "haar_dc.mk", "haar_dc", "-j8",
                            "REF=" + os.path.abspath(oracle_lib.REF_SRC)], check=True, stdout=subprocess.DEVNULL,
                           stderr=subprocess.PIPE)
        path = os.path.join(oracle_lib.ORACLE, "_ref", "libdaala_ref_haar_dc.so")
        lib = None
        if os.path.exists(path):
            lib = ctypes.CDLL(path)
            lib.oracle_ref_haar_dc_frame.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                                     ctypes.c_int, ctypes.c_void_p, ctypes.c_double, ctypes.c_void_p,
                                                     ctypes.c_void_p, ctypes.c_void_p]
        _lib.append(lib)
    return _lib[0]


def _unpack(geom, buf, shift=0):
    out, o = [], 0
    for p in range(3):
        h, w = (s >> shift for s in geom.plane_shape(p))
        out.append(buf[o:o + h * w].reshape(h, w))
        o += h * w
    return out


def frame(lib, geom, planes, bsize, quantizer, pvq_qm_q4, lam):
    """The driver on one keyframe (planes: three u8 arrays of the padded geometry; bsize: [nvsb * 8, nhsb * 8] u8;
    pvq_qm_q4: [3, 30] u8).  Returns dict(d_pre=, d_post= [3 x [h, w] int32]: the `d` planes before and after the DC
    chain, idx= [3 x [h / 4, w / 4] int32]: the signed coded indices)."""
    src = np.ascontiguousarray(np.concatenate([np.asarray(planes[p], np.uint8).reshape(-1) for p in range(3)]))
    bs = np.ascontiguousarray(bsize, np.uint8)
    q4 = np.ascontiguousarray(pvq_qm_q4, np.uint8)
    assert bs.shape == tuple(geom.bsize_shape) and q4.shape == (3, 30)
    d_pre = np.zeros(src.size, np.int32)
    d_post = np.zeros(src.size, np.int32)
    idx = np.zeros(src.size // 16, np.int32)
    rc = lib.oracle_ref_haar_dc_frame(geom.pic_w, geom.pic_h, addr(src), addr(bs), int(quantizer), addr(q4),
                                      float(lam), addr(d_pre), addr(d_post), addr(idx))
    assert rc == 0, rc
    return dict(d_pre=_unpack(geom, d_pre), d_post=_unpack(geom, d_post), idx=_unpack(geom, idx, 2))


def encode_keyframe(lib, geom, planes, quant, complexity=7):
    """The whole reference encoder on one keyframe (oracle_ref_haar_dc_encode_keyframe).  Returns dict(bsize= its map,
    d= [3 x [h, w] int32] the final pass's `d` planes, leaf DCs final at the leaf origins, quantizer=, pvq_qm_q4=
    [3, 30] u8, lam=): the settings the final pass coded with."""
    import ctypes
    src = np.ascontiguousarray(np.concatenate([np.asarray(planes[p], np.uint8).reshape(-1) for p in range(3)]))
    bs = np.zeros(tuple(geom.bsize_shape), np.uint8)
    d = np.zeros(src.size, np.int32)
    qz = np.zeros(1, np.int32)
    q4 = np.zeros((3, 30), np.uint8)
    lam = np.zeros(1, np.float64)
    rc = lib.oracle_ref_haar_dc_encode_keyframe(ctypes.c_int(geom.pic_w), ctypes.c_int(geom.pic_h), addr(src),
                                                ctypes.c_int(int(quant)), ctypes.c_int(int(complexity)), addr(bs),
                                                addr(d), addr(qz), addr(q4), addr(lam))
    assert rc == 0, rc
    return dict(bsize=bs, d=_unpack(geom, d), quantizer=int(qz[0]), pvq_qm_q4=q4, lam=float(lam[0]))


def leaf_origins(geom, bsize, pli):
    """[h / 4, w / 4] bool: the 4x4 units of plane pli where a block of the map starts (its leaf DC position)."""
    bs = np.asarray(bsize, np.int64)
    if pli == 0:
        b = np.repeat(np.repeat(bs, 2, axis=0), 2, axis=1)   # per luma 4x4 unit
    else:
        b = np.maximum(bs, 1) - 1                            # chroma 4x4 unit = luma 8x8 unit
    v, u = np.mgrid[0:b.shape[0], 0:b.shape[1]]
    n = 1 << b
    return (u % n == 0) & (v % n == 0)
