"""CPU oracle of the P-frame finishing pass (test infrastructure): the frame driver of oracle/inter_finish_driver.inc,
bound to the reference (oracle/ref_inter_finish.c, which oracle/inter_finish.mk links with the reference build's
objects into oracle/_ref/libdaala_ref_inter_finish.so) and to the plain-C port (oracle/port_inter_finish.c, part of
oracle/libdaala_port.so)."""
import ctypes
import os
import subprocess

import numpy as np

from tests import oracle_lib
from tests.oracle_lib import addr

_ref = []


def load_ref():
    """The reference-bound library: (re)built first when the reference sources are present, else used as it is; None
    when it is absent."""
    if not _ref:
        if oracle_lib.have_ref_sources():
            subprocess.run(["make", "-C", oracle_lib.ORACLE, "-f", "inter_finish.mk", "inter_finish", "-j8",
                            "REF=" + os.path.abspath(oracle_lib.REF_SRC)], check=True, stdout=subprocess.DEVNULL,
                           stderr=subprocess.PIPE)
        path = os.path.join(oracle_lib.ORACLE, "_ref", "libdaala_ref_inter_finish.so")
        _ref.append(ctypes.CDLL(path) if os.path.exists(path) else None)
    return _ref[0]


def load():
    """(library, prefix): the reference build when it exists, else the port."""
    ref = load_ref()
    return (ref, "ref") if ref is not None else (oracle_lib.load_port(), "port")


def finish(lib, prefix, dq, geom, bsize, q0, levels, bskip):
    """One frame through inverse_frame_inter_finish: patched coefficient planes dq, skip maps bskip
    ([plane_h / 4, nhsb * 16] each), levels [nvsb, nhsb] -> (u8 planes, levels applied)."""
    ds = [np.ascontiguousarray(x, np.int32).copy() for x in dq]
    recs = [np.zeros(geom.plane_shape(p), np.uint8) for p in range(3)]
    bs = np.ascontiguousarray(bsize, np.uint8)
    lv = np.ascontiguousarray(levels, np.uint8)
    assert lv.shape == (geom.nvsb, geom.nhsb)
    applied = np.zeros_like(lv)
    sk = [np.ascontiguousarray(b, np.uint8) for b in bskip]
    for p in range(3):
        assert sk[p].shape == (geom.plane_shape(p)[0] // 4, geom.nhsb * 16)
    getattr(lib, "oracle_%s_fin_inverse_frame_inter_finish" % prefix)(
        addr(ds[0]), addr(ds[1]), addr(ds[2]), addr(recs[0]), addr(recs[1]), addr(recs[2]), geom.nhsb, geom.nvsb,
        addr(bs), bs.shape[1], geom.pic_w, geom.pic_h, int(q0), addr(lv), addr(sk[0]), addr(sk[1]), addr(sk[2]),
        addr(applied))
    return recs, applied
