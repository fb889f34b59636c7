#!/usr/bin/env python
"""Dev-time tool: block-size maps the WHOLE reference encoder decides (public API, OD_SET_QUANT 20,
complexity 7 -- BASELINE.json's configuration) for bench.py's four synthetic 3840x2160 frames, saved as
daala_b200/data/bench_bsize_4k.npz for `bench.py --block-sizes reference`.  Needs oracle/_ref
(i.e. the reference sources); the saved maps travel with the repository."""
import ctypes
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from daala_b200 import synth  # noqa: E402
from daala_b200.frame import Geometry  # noqa: E402
from tests import oracle_lib  # noqa: E402
from tests.oracle_lib import addr  # noqa: E402

W, H, QUANT, COMPLEXITY, DISTINCT = 3840, 2160, 20, 7, 4


def main():
    ref = oracle_lib.load_ref()
    assert ref is not None, "needs oracle/_ref"
    geom = Geometry(W, H)
    out = {}
    seed = 12345
    for f in range(DISTINCT):
        planes, seed = synth.frame(W, H, f=f, seed=seed)          # same frames as bench.make_host_frames
        bsize = np.zeros(geom.bsize_shape, np.uint8)
        dering = np.zeros((geom.nvsb, geom.nhsb), np.uint8)
        nbytes, csum = ctypes.c_long(0), ctypes.c_uint(0)
        t = time.time()
        rc = ref.oracle_ref_encode_keyframe(W, H, addr(np.ascontiguousarray(planes[0])),
                                            addr(np.ascontiguousarray(planes[1])), addr(np.ascontiguousarray(planes[2])),
                                            QUANT, COMPLEXITY, addr(bsize), addr(dering), ctypes.byref(nbytes),
                                            ctypes.byref(csum))
        assert rc == 0
        print("frame %d: %.1f s, packet %d bytes, sizes %s" % (f, time.time() - t, nbytes.value,
                                                               np.bincount(bsize.ravel(), minlength=5).tolist()))
        out["bsize_%d" % f] = bsize
        out["dering_%d" % f] = dering
        out["packet_%d" % f] = np.array([nbytes.value, csum.value], np.int64)
    np.savez_compressed(os.path.join(ROOT, "daala_b200", "data", "bench_bsize_4k.npz"), **out)


if __name__ == "__main__":
    main()
