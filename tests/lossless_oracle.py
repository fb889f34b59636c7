"""CPU oracle of lossless frames (test infrastructure): the quantizer-0 frame driver oracle_ref_lossless_frame of
oracle/ref_hooks_lossless.c (the reference's own od_compute_dcts, od_quantize_haar_dc_sb and od_compute_max_tree on a
real encoder), which oracle/lossless.mk links with the reference build's objects into
oracle/_ref/libdaala_ref_lossless.so."""
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
            subprocess.run(["make", "-C", oracle_lib.ORACLE, "-f", "lossless.mk", "lossless", "-j8",
                            "REF=" + os.path.abspath(oracle_lib.REF_SRC)], check=True, stdout=subprocess.DEVNULL,
                           stderr=subprocess.PIPE)
        path = os.path.join(oracle_lib.ORACLE, "_ref", "libdaala_ref_lossless.so")
        _lib.append(ctypes.CDLL(path) if os.path.exists(path) else None)
    return _lib[0]


def _pack(geom, planes):
    return np.ascontiguousarray(np.concatenate([np.asarray(planes[p], np.uint8).reshape(-1) for p in range(3)]))


def _unpack(geom, buf):
    out, o = [], 0
    for p in range(3):
        h, w = geom.plane_shape(p)
        out.append(buf[o:o + h * w].reshape(h, w))
        o += h * w
    return out


def frame(lib, geom, planes, pred=None):
    """The driver on one frame (planes / pred: three frame-sized u8 arrays; pred None = keyframe).  Returns dict(d=,
    coeffs= [3 x [h, w] int32]: the `d` planes and the residual with the coded DC, roots= [nvsb, nhsb, 3, 3] int32)."""
    src = _pack(geom, planes)
    prd = _pack(geom, pred) if pred is not None else np.zeros(1, np.uint8)
    d = np.zeros(src.size, np.int32)
    res = np.zeros(src.size, np.int32)
    roots = np.zeros((geom.nvsb, geom.nhsb, 3, 3), np.int32)
    rc = lib.oracle_ref_lossless_frame(geom.pic_w, geom.pic_h, int(pred is None), addr(src), addr(prd), addr(d),
                                       addr(res), addr(roots))
    assert rc == 0, rc
    return dict(d=_unpack(geom, d), coeffs=_unpack(geom, res), roots=roots)
