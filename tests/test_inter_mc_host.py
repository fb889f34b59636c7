"""Host side of the engine's P-frame prediction from MV grids (config.inter_mc), without a GPU: the two-picture
od_state_mc_predict hook against the single-picture one and against the reference encoder's own prediction, the
ctypes mirrors of the new C fields, and the MV-grid packer."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from tests import inter_mc_oracle
from tests.oracle_lib import addr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ref():
    """The reference build with the prediction hooks (oracle/inter_mc.mk; may be absent)."""
    lib = inter_mc_oracle.load()
    if lib is None:
        pytest.skip("oracle/_ref/libdaala_ref_inter_mc.so not built (needs the reference sources)")
    return lib


def test_two_reference_hook_on_all_prev_grids_equals_the_single_reference_hook(ref):
    from daala_b200 import synth
    from daala_b200.frame import Geometry
    for w, h, seed in ((200, 130, 1), (328, 200, 2)):
        geom = Geometry(w, h)
        valid, mv, _ = synth.mv_grid(geom, seed=seed)
        rng = np.random.default_rng(seed)
        prev = [rng.integers(0, 256, size=geom.plane_shape(p), dtype=np.uint8) for p in range(3)]
        gold = [255 - a for a in prev]   # never read on an all-PREV grid
        got = inter_mc_oracle.predict(ref, geom, gold, prev, valid, mv, np.ones_like(valid))
        want = [np.zeros(geom.plane_shape(p), np.uint8) for p in range(3)]
        v, m = np.ascontiguousarray(valid), np.ascontiguousarray(mv)
        assert ref.oracle_ref_state_mc_predict(w, h, addr(prev[0]), addr(prev[1]), addr(prev[2]), addr(v), addr(m),
                                               addr(want[0]), addr(want[1]), addr(want[2])) == 0
        for p in range(3):
            assert np.array_equal(got[p], want[p]), (w, h, p)


def test_two_reference_hook_reproduces_the_encoders_prediction(ref):
    """On the captured P frames the hook, given the grid and the two pictures, makes the encoder's own prediction;
    from the third frame on the two pictures differ."""
    from daala_b200.frame import Geometry
    geom = Geometry(328, 200)
    caps = inter_mc_oracle.capture_p_frames(ref, geom, 4)
    assert [c["same"] for c in caps] == [True, False, False]
    for f, c in enumerate(caps):
        got = inter_mc_oracle.predict(ref, geom, c["gold"], c["prev"], c["valid"], c["mv"], c["ref"], same=c["same"])
        for p in range(3):
            assert np.array_equal(got[p], c["pred"][p]), (f, p)
        assert not np.array_equal(c["gold"][0], c["prev"][0]) or c["same"]


SRC = r"""
#include <stddef.h>
#include <stdio.h>
#include "daala_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\n",
         sizeof(daala_b200_kf_config), offsetof(daala_b200_kf_config, inter_mc), offsetof(daala_b200_kf_config, mc_refs),
         sizeof(daala_b200_kf_io), offsetof(daala_b200_kf_io, ref_pixels), offsetof(daala_b200_kf_io, nrefs),
         offsetof(daala_b200_kf_io, ref_slot), offsetof(daala_b200_kf_io, mv_grid),
         offsetof(daala_b200_kf_io, pred_pixels_out),
         sizeof(daala_b200_kf_buffers), offsetof(daala_b200_kf_buffers, ref_pixels),
         offsetof(daala_b200_kf_buffers, ref_slot), offsetof(daala_b200_kf_buffers, mv_grid),
         offsetof(daala_b200_kf_buffers, mc_refs),
         sizeof(daala_b200_mv_pt), offsetof(daala_b200_mv_pt, mv), offsetof(daala_b200_mv_pt, valid),
         offsetof(daala_b200_mv_pt, ref), offsetof(daala_b200_mv_pt, pad_));
  return 0;
}
"""


def test_ctypes_mirrors_of_the_prediction_fields_match_the_header(tmp_path):
    from daala_b200 import engine, mvgrid
    (tmp_path / "layout.c").write_text(SRC)
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(tmp_path / "layout.c"), "-o", exe], check=True)
    got = [int(v) for v in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()]
    d = mvgrid.MV_PT_DTYPE
    assert got == [ctypes.sizeof(engine.Config), engine.Config.inter_mc.offset, engine.Config.mc_refs.offset,
                   ctypes.sizeof(engine.IO), engine.IO.ref_pixels.offset, engine.IO.nrefs.offset,
                   engine.IO.ref_slot.offset, engine.IO.mv_grid.offset, engine.IO.pred_pixels_out.offset,
                   ctypes.sizeof(engine.Buffers), engine.Buffers.ref_pixels.offset, engine.Buffers.ref_slot.offset,
                   engine.Buffers.mv_grid.offset, engine.Buffers.mc_refs.offset,
                   d.itemsize, d.fields["mv"][1], d.fields["valid"][1], d.fields["ref"][1], d.fields["pad_"][1]]


def test_mvgrid_pack_round_trips():
    from daala_b200 import mvgrid, synth
    from daala_b200.frame import Geometry
    geom = Geometry(200, 130)
    grids = [synth.mv_grid(geom, seed=s) for s in range(3)]
    valid, mv, ref = (np.stack([g[i] for g in grids]) for i in range(3))
    packed = mvgrid.pack(valid, mv, ref)
    assert packed.dtype == mvgrid.MV_PT_DTYPE and packed.shape == valid.shape
    assert not packed["pad_"].any()
    for a, b in zip(mvgrid.unpack(packed), (valid, mv, ref)):
        assert np.array_equal(a, b)
    # the bytes are those of the C record: mv[2] little-endian int32, then valid, ref, two zero bytes
    raw = packed.reshape(-1)[:1].view(np.uint8)
    assert np.array_equal(raw[:8].view("<i4"), mv.reshape(-1, 2)[0]) and raw[8] == valid.reshape(-1)[0] \
        and raw[9] == ref.reshape(-1)[0]
