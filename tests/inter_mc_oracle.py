"""CPU oracle of P-frame prediction from MV grids (test infrastructure): the two-picture od_state_mc_predict hook
(oracle_ref_state_mc_predict2) and real P frames captured from the whole reference encoder
(oracle_ref_capture_p_frames), both in oracle/ref_hooks_inter_mc.c, which oracle/inter_mc.mk links with the reference
build's objects into oracle/_ref/libdaala_ref_inter_mc.so."""
import ctypes
import os
import subprocess

import numpy as np

from tests import oracle_lib
from tests.oracle_lib import addr

_lib = []


def load():
    """The hook library: (re)built first when the reference sources are present, else used as it is; None when
    it is absent."""
    if not _lib:
        if oracle_lib.have_ref_sources():
            subprocess.run(["make", "-C", oracle_lib.ORACLE, "-f", "inter_mc.mk", "inter_mc", "-j8",
                            "REF=" + os.path.abspath(oracle_lib.REF_SRC)], check=True, stdout=subprocess.DEVNULL,
                           stderr=subprocess.PIPE)
        path = os.path.join(oracle_lib.ORACLE, "_ref", "libdaala_ref_inter_mc.so")
        _lib.append(ctypes.CDLL(path) if os.path.exists(path) else None)
    return _lib[0]


def _planes(geom, buf):
    """Frame-sized Y, U, V views of one packed picture (Y then U then V)."""
    h, w = geom.plane_shape(0)
    ch, cw = geom.plane_shape(1)
    return [buf[:h * w].reshape(h, w), buf[h * w:h * w + ch * cw].reshape(ch, cw), buf[h * w + ch * cw:].reshape(ch, cw)]


def predict(lib, geom, gold, prev, valid, mv, ref, same=False, timed=False):
    """od_state_mc_predict with GOLD picture `gold` and PREV picture `prev` (per plane frame-sized u8; with
    same=True one picture, `gold`, for both) on the grid (valid, mv, ref) of mvgrid.pack's inputs.  Returns the
    three prediction planes, and with timed=True also the seconds od_state_mc_predict alone took."""
    out = [np.zeros(geom.plane_shape(p), np.uint8) for p in range(3)]
    g = [np.ascontiguousarray(a, np.uint8) for a in gold]
    q = g if same else [np.ascontiguousarray(a, np.uint8) for a in prev]
    v = np.ascontiguousarray(valid, np.uint8)
    m = np.ascontiguousarray(mv, np.int32)
    r = np.ascontiguousarray(ref, np.uint8)
    sec = np.zeros(1, np.float64)
    rc = lib.oracle_ref_state_mc_predict2(geom.pic_w, geom.pic_h, addr(g[0]), addr(g[1]), addr(g[2]), addr(q[0]),
                                          addr(q[1]), addr(q[2]), int(bool(same)), addr(v), addr(m), addr(r),
                                          addr(out[0]), addr(out[1]), addr(out[2]), addr(sec))
    assert rc == 0
    return (out, float(sec[0])) if timed else out


def capture_p_frames(lib, geom, nframes, quant=30, complexity=7):
    """Encodes a keyframe and nframes - 1 P frames with the reference encoder; per P frame a dict of src, gold,
    prev, pred (lists of frame-sized planes), same (GOLD and PREV were one picture), bsize, valid, ref, mv."""
    n = nframes - 1
    h, w = geom.plane_shape(0)
    pic = h * w * 3 // 2
    nv, nh = geom.nvsb * 8 + 1, geom.nhsb * 8 + 1
    src, gold, prev, pred = (np.zeros((n, pic), np.uint8) for _ in range(4))
    same = np.zeros(n, np.int32)
    bsize = np.zeros((n, geom.nvsb * 8, geom.nhsb * 8), np.uint8)
    valid = np.zeros((n, nv, nh), np.uint8)
    ref = np.zeros((n, nv, nh), np.uint8)
    mv = np.zeros((n, nv, nh, 2), np.int32)
    rc = lib.oracle_ref_capture_p_frames(geom.pic_w, geom.pic_h, nframes, quant, complexity, addr(src), addr(gold),
                                         addr(prev), addr(same), addr(pred), addr(bsize), addr(valid), addr(ref),
                                         addr(mv))
    assert rc == 0, rc
    return [dict(src=_planes(geom, src[f]), gold=_planes(geom, gold[f]), prev=_planes(geom, prev[f]),
                 pred=_planes(geom, pred[f]), same=bool(same[f]), bsize=bsize[f], valid=valid[f], ref=ref[f], mv=mv[f])
            for f in range(n)]
