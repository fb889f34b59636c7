"""CPU oracle of B-frame prediction (test infrastructure): od_state_mc_predict with GOLD, PREV and NEXT pictures
(oracle_ref_state_mc_predict3) and whole B-frame sequences captured from the reference encoder
(oracle_ref_capture_b_frames), both in oracle/ref_hooks_bframes.c, which oracle/bframes.mk links with the reference
build's objects into oracle/_ref/libdaala_ref_bframes.so."""
import ctypes
import os
import subprocess

import numpy as np

from tests import oracle_lib
from tests.inter_mc_oracle import _planes
from tests.oracle_lib import addr

_lib = []


def load():
    """The hook library: (re)built first when the reference sources are present, else used as it is; None when
    it is absent."""
    if not _lib:
        if oracle_lib.have_ref_sources():
            subprocess.run(["make", "-C", oracle_lib.ORACLE, "-f", "bframes.mk", "bframes", "-j8",
                            "REF=" + os.path.abspath(oracle_lib.REF_SRC)], check=True, stdout=subprocess.DEVNULL,
                           stderr=subprocess.PIPE)
        path = os.path.join(oracle_lib.ORACLE, "_ref", "libdaala_ref_bframes.so")
        _lib.append(ctypes.CDLL(path) if os.path.exists(path) else None)
    return _lib[0]


def predict3(lib, geom, gold, prev, nxt, valid, mv, mv1, ref):
    """od_state_mc_predict with GOLD / PREV / NEXT pictures (per plane frame-sized u8; pictures given as the same
    arrays share one reference buffer) on the grid (valid, mv, mv1, ref), ref 2 predicted with mv1."""
    out = [np.zeros(geom.plane_shape(p), np.uint8) for p in range(3)]
    keep, ptrs = [], []
    seen = {}
    for pic in (gold, prev, nxt):
        arr = seen.get(id(pic))
        if arr is None:
            arr = seen[id(pic)] = [np.ascontiguousarray(a, np.uint8) for a in pic]
        keep.append(arr)
        ptrs.append((ctypes.c_void_p * 3)(*(addr(a) for a in arr)))
    v = np.ascontiguousarray(valid, np.uint8)
    m = np.ascontiguousarray(mv, np.int32)
    m1 = np.ascontiguousarray(mv1, np.int32)
    r = np.ascontiguousarray(ref, np.uint8)
    rc = lib.oracle_ref_state_mc_predict3(geom.pic_w, geom.pic_h, ptrs[0], ptrs[1], ptrs[2], addr(v), addr(m), addr(m1),
                                          addr(r), addr(out[0]), addr(out[1]), addr(out[2]))
    assert rc == 0
    return out


def capture_b_frames(lib, geom, nframes, b_frames, keyframe_rate=256, quant=30, complexity=7):
    """Encodes nframes display frames with OD_SET_B_FRAMES = b_frames; per coded frame, in coding order, a dict of
    number, type (0 I, 1 P, 2 B), golden, refi (ref_imgi[GOLD, PREV, NEXT, SELF] the frame used), quantizer, src,
    gold, prev, next, pred (lists of frame-sized planes; zeros where refi is -1, pred zeros for keyframes), bsize,
    valid, ref, mv, mv1."""
    n = nframes
    h, w = geom.plane_shape(0)
    pic = h * w * 3 // 2
    nv, nh = geom.nvsb * 8 + 1, geom.nhsb * 8 + 1
    ints = {k: np.zeros(n, np.int32) for k in ("number", "type", "golden", "quantizer")}
    refi = np.zeros((n, 4), np.int32)
    src, gold, prev, nxt, pred = (np.zeros((n, pic), np.uint8) for _ in range(5))
    bsize = np.zeros((n, geom.nvsb * 8, geom.nhsb * 8), np.uint8)
    valid = np.zeros((n, nv, nh), np.uint8)
    ref = np.zeros((n, nv, nh), np.uint8)
    mv = np.zeros((n, nv, nh, 2), np.int32)
    mv1 = np.zeros((n, nv, nh, 2), np.int32)
    rc = lib.oracle_ref_capture_b_frames(geom.pic_w, geom.pic_h, nframes, b_frames, keyframe_rate, quant, complexity,
                                         addr(ints["number"]), addr(ints["type"]), addr(ints["golden"]), addr(refi),
                                         addr(ints["quantizer"]), addr(src), addr(gold), addr(prev), addr(nxt),
                                         addr(pred), addr(bsize), addr(valid), addr(ref), addr(mv), addr(mv1))
    assert rc == n, rc
    return [dict(number=int(ints["number"][k]), type=int(ints["type"][k]), golden=bool(ints["golden"][k]),
                 refi=tuple(int(x) for x in refi[k]), quantizer=int(ints["quantizer"][k]), src=_planes(geom, src[k]),
                 gold=_planes(geom, gold[k]), prev=_planes(geom, prev[k]), next=_planes(geom, nxt[k]),
                 pred=_planes(geom, pred[k]), bsize=bsize[k], valid=valid[k], ref=ref[k], mv=mv[k], mv1=mv1[k])
            for k in range(n)]
