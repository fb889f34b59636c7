"""CPU oracle of the late-skip distortions (test infrastructure): the plane driver of oracle/late_skip_driver.inc,
bound to the reference (oracle/ref_late_skip.c, which oracle/late_skip.mk links with the reference build's objects into
oracle/_ref/libdaala_ref_late_skip.so) and to the plain-C port (oracle/port_late_skip.c, part of
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
            subprocess.run(["make", "-C", oracle_lib.ORACLE, "-f", "late_skip.mk", "late_skip", "-j8",
                            "REF=" + os.path.abspath(oracle_lib.REF_SRC)], check=True, stdout=subprocess.DEVNULL,
                           stderr=subprocess.PIPE)
        path = os.path.join(oracle_lib.ORACLE, "_ref", "libdaala_ref_late_skip.so")
        _ref.append(ctypes.CDLL(path) if os.path.exists(path) else None)
    return _ref[0]


def load():
    """(library, prefix): the reference build when it exists, else the port."""
    ref = load_ref()
    return (ref, "ref") if ref is not None else (oracle_lib.load_port(), "port")


def plane(lib, prefix, src, pred, dcoded, geom, bsize, pli, q0, q4, qm_is_flat, masking, coded_quantizer):
    """One plane of one frame: source and prediction u8 planes, the step's coded coefficient plane -> [h/4, w/4, 4]
    float64 with {dist_skip, noskip_coded_dc0, noskip_coded_dcq, noskip_pred_dcq} at each leaf's top-left 4x4 unit
    (zero elsewhere and at leaves with bs = 0)."""
    h, w = geom.plane_shape(pli)
    s = np.ascontiguousarray(src, np.uint8)
    p = np.ascontiguousarray(pred, np.uint8)
    d = np.ascontiguousarray(dcoded, np.int32)
    assert s.shape == p.shape == d.shape == (h, w)
    bs = np.ascontiguousarray(bsize, np.uint8)
    qq = np.ascontiguousarray(np.asarray(q4, np.uint8)[pli], np.uint8)
    out = np.zeros((h // 4, w // 4, 4), np.float64)
    getattr(lib, "oracle_%s_ls_late_skip_plane" % prefix)(
        addr(s), addr(p), addr(d), geom.nhsb, geom.nvsb, 1 if pli else 0, addr(bs), bs.shape[1], geom.pic_w,
        geom.pic_h, int(q0), addr(qq), int(qm_is_flat), int(masking), int(coded_quantizer), addr(out))
    return out
