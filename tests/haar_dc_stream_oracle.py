"""CPU oracle of the keyframe DC records' coded bytes (test infrastructure): oracle/ref_hooks_haar_dc_stream.c, which
oracle/haar_dc_stream.mk links with the reference build's objects into oracle/_ref/libdaala_ref_haar_dc_stream.so.
`frame_bytes` is what the reference's own DC chain codes for a keyframe (the driver of tests/haar_dc_oracle.py), and
`replay` codes a list of symbols.HDC_DTYPE records through the reference's generic_encode and od_ec_enc_bits; equal
bytes mean the records carry the reference's values in its order with its model contexts."""
import ctypes
import os
import subprocess

import numpy as np

from tests import oracle_lib
from tests.oracle_lib import addr

_lib = []


def load():
    """The library: (re)built first when the reference sources are present, else used as it is; None when it is
    absent."""
    if not _lib:
        if oracle_lib.have_ref_sources():
            subprocess.run(["make", "-C", oracle_lib.ORACLE, "-f", "haar_dc_stream.mk", "haar_dc_stream", "-j8",
                            "REF=" + os.path.abspath(oracle_lib.REF_SRC)], check=True, stdout=subprocess.DEVNULL,
                           stderr=subprocess.PIPE)
        path = os.path.join(oracle_lib.ORACLE, "_ref", "libdaala_ref_haar_dc_stream.so")
        lib = None
        if os.path.exists(path):
            lib = ctypes.CDLL(path)
            lib.oracle_ref_haar_dc_frame_bytes.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                                           ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                                           ctypes.c_double, ctypes.c_void_p, ctypes.c_int]
            lib.oracle_ref_haar_dc_replay.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                                      ctypes.c_void_p, ctypes.c_int]
        _lib.append(lib)
    return _lib[0]


def _cap(geom):
    return 8 * sum(h * w for h, w in (geom.plane_shape(p) for p in range(3))) // 16 + 4096


def frame_bytes(lib, geom, planes, bsize, quantizer, pvq_qm_q4, lam):
    """The bytes the reference's DC chain codes for one keyframe (the arguments of haar_dc_oracle.frame)."""
    src = np.ascontiguousarray(np.concatenate([np.asarray(planes[p], np.uint8).reshape(-1) for p in range(3)]))
    bs = np.ascontiguousarray(bsize, np.uint8)
    q4 = np.ascontiguousarray(pvq_qm_q4, np.uint8)
    assert bs.shape == tuple(geom.bsize_shape) and q4.shape == (3, 30)
    out = np.zeros(_cap(geom), np.uint8)
    n = lib.oracle_ref_haar_dc_frame_bytes(geom.pic_w, geom.pic_h, addr(src), addr(bs), int(quantizer), addr(q4),
                                           float(lam), addr(out), out.size)
    assert n >= 0, n
    return out[:n].tobytes()


def replay(lib, geom, records):
    """The bytes one frame's records (symbols.HDC_DTYPE) code on a fresh encoder."""
    from daala_b200.symbols import HDC_DTYPE
    rec = np.ascontiguousarray(records, HDC_DTYPE)
    out = np.zeros(_cap(geom), np.uint8)
    n = lib.oracle_ref_haar_dc_replay(geom.pic_w, geom.pic_h, addr(rec) if len(rec) else None, len(rec), addr(out),
                                      out.size)
    assert n >= 0, n
    return out[:n].tobytes()
