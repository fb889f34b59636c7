"""B frames on the host (no GPU): the appended C struct fields of config.mc_next, the vector each vertex is predicted
with, the synthetic B-frame grids, the reference's coding order and buffer rotation (daala_b200/gop.py) against the
reference encoder, and the three-picture od_state_mc_predict hook against the encoder's own prediction."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from tests import bframe_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SRC = r"""
#include <stddef.h>
#include <stdio.h>
#include "daala_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(daala_b200_kf_config), offsetof(daala_b200_kf_config, mc_next),
         sizeof(daala_b200_kf_io), offsetof(daala_b200_kf_io, ref_slot_next), offsetof(daala_b200_kf_io, mv1_grid),
         sizeof(daala_b200_kf_buffers), offsetof(daala_b200_kf_buffers, ref_slot_next),
         offsetof(daala_b200_kf_buffers, mv1_grid), sizeof(daala_b200_mv_pt));
  return 0;
}
"""


def _ref():
    lib = bframe_oracle.load()
    if lib is None:
        pytest.skip("oracle/_ref/libdaala_ref_bframes.so not built (needs the reference sources)")
    return lib


def test_struct_layout(tmp_path):
    from daala_b200 import engine, mvgrid
    (tmp_path / "layout.c").write_text(SRC)
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(tmp_path / "layout.c"), "-o", exe], check=True)
    got = [int(v) for v in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [ctypes.sizeof(engine.Config), engine.Config.mc_next.offset,
                   ctypes.sizeof(engine.IO), engine.IO.ref_slot_next.offset, engine.IO.mv1_grid.offset,
                   ctypes.sizeof(engine.Buffers), engine.Buffers.ref_slot_next.offset, engine.Buffers.mv1_grid.offset,
                   mvgrid.MV_PT_DTYPE.itemsize]
    # appended last: every earlier field keeps its offset
    assert engine.Config.mc_next.offset > engine.Config.late_skip.offset
    assert engine.IO.ref_slot_next.offset > engine.IO.sym_late_skip_cap.offset
    assert engine.Buffers.ref_slot_next.offset > engine.Buffers.mc_refs.offset


def test_vertex_vectors():
    from daala_b200 import mvgrid, synth
    from daala_b200.frame import Geometry
    rng = np.random.default_rng(3)
    ref = rng.integers(0, 4, (9, 17)).astype(np.uint8)
    mv = rng.integers(-256, 257, (9, 17, 2)).astype(np.int32)
    mv1 = rng.integers(-256, 257, (9, 17, 2)).astype(np.int32)
    got = mvgrid.vectors(mv, ref, mv1)
    assert np.array_equal(got[ref == 2], mv1[ref == 2])
    assert np.array_equal(got[ref != 2], mv[ref != 2])
    assert np.array_equal(mvgrid.vectors(mv, ref), mv)
    # blocks_for takes mv1 on the NEXT corners only
    valid = synth.mv_grid(Geometry(128, 64), seed=1)[0]
    lv = mvgrid.leaves(valid.astype(bool))
    b = mvgrid.blocks_for(*lv, mv, 0, ref=ref, mv1=mv1)
    for k, (gx, gy) in enumerate(mvgrid.corners(*lv)):
        want = np.where((ref[gy, gx] == 2)[:, None], mv1[gy, gx], mv[gy, gx])
        assert np.array_equal(b["mvx"][:, k], want[:, 0]) and np.array_equal(b["mvy"][:, k], want[:, 1])
    # the B-frame grids: every split level, all three refs, mv1 on every vertex; mv_grid's stream unchanged
    geom = Geometry(328, 200)
    valid, mv, mv1, ref = synth.mv_grid_b(geom, seed=4)
    assert valid.shape == ref.shape == mv.shape[:2] == mv1.shape[:2] == (geom.nvsb * 8 + 1, geom.nhsb * 8 + 1)
    assert (np.bincount(mvgrid.leaves(valid.astype(bool))[2], minlength=4) > 0).all()
    assert set(np.unique(ref)) == {0, 1, 2}
    assert (mv1 != 0).any(-1).mean() > 0.99
    assert np.array_equal(synth.mv_grid_b(geom, seed=4)[2], mv1)
    v0, m0, r0 = synth.mv_grid(geom, seed=4)
    rng = np.random.default_rng(4)   # mv_grid: valid, then mv, then ref from default_rng(seed)
    nv, nh = v0.shape
    rng.random((nv, nh))
    assert np.array_equal(m0, rng.integers(-256, 257, size=(nv, nh, 2)).astype(np.int32))


@pytest.mark.parametrize("nframes,b_frames,keyframe_rate",
                         [(7, 2, 256), (6, 2, 256), (5, 1, 256), (8, 1, 256), (9, 3, 256), (11, 3, 256),
                          (25, 2, 12), (23, 1, 7), (22, 3, 256), (12, 0, 256)])
def test_rotation_matches_reference(nframes, b_frames, keyframe_rate):
    """gop.coding_order equals the encoder record for record: display number, type, golden flag, ref_imgi.  The
    parameters cover short last groups (6, 8, 11 frames), golden P frames (25 / 2, 23 / 1, 22 / 3) and keyframes
    inside the sequence (keyframe_rate 12 and 7)."""
    from daala_b200 import gop
    from daala_b200.frame import Geometry
    lib = _ref()
    caps = bframe_oracle.capture_b_frames(lib, Geometry(64, 64), nframes, b_frames, keyframe_rate)
    want = gop.coding_order(nframes, b_frames, keyframe_rate)
    assert [(c["number"], c["type"], c["golden"], c["refi"], c["type"] != gop.B_FRAME) for c in caps] == \
        [(f.number, f.type, f.golden, f.refs, f.kept) for f in want]
    types = {f.type for f in want}
    assert (gop.B_FRAME in types) == (b_frames > 0) and gop.P_FRAME in types
    if keyframe_rate < nframes:
        assert sum(f.type == gop.I_FRAME for f in want) > 1
    if nframes > 20:
        assert any(f.golden and f.type == gop.P_FRAME for f in want)


def test_coding_order_facts():
    from daala_b200 import gop
    assert [f.number for f in gop.coding_order(7, 2)] == [0, 3, 1, 2, 6, 4, 5]
    assert [f.number for f in gop.coding_order(6, 2)] == [0, 3, 1, 2, 5, 4]
    assert [f.type for f in gop.coding_order(6, 2)] == [0, 1, 2, 2, 1, 2]
    assert all(not f.kept for f in gop.coding_order(12, 3) if f.type == gop.B_FRAME)
    # no B frames: the P-frame rotation (PREV is the last frame)
    order = gop.coding_order(4, 0)
    assert [f.number for f in order] == [0, 1, 2, 3] and [f.refs[1] for f in order] == [-1, 0, 1, 2]
    with pytest.raises(ValueError):
        gop.coding_order(4, 16)


def test_three_picture_hook_reproduces_the_encoder():
    """oracle_ref_state_mc_predict3 on each captured frame's pictures and grid gives the encoder's own pred; the B
    frames mix PREV and NEXT vertices, the P frames after the first carry stale mv1."""
    lib = _ref()
    from daala_b200.frame import Geometry
    geom = Geometry(328, 200)
    caps = bframe_oracle.capture_b_frames(lib, geom, 7, 2)
    mixed = stale = 0
    for c in caps:
        if c["type"] == 0:
            continue
        pics = {}
        g, p, n = (pics.setdefault(c["refi"][i], c[k]) for i, k in enumerate(("gold", "prev", "next")))
        out = bframe_oracle.predict3(lib, geom, g, p, n, c["valid"], c["mv"], c["mv1"], c["ref"])
        for pl in range(3):
            assert np.array_equal(out[pl], c["pred"][pl]), (c["number"], pl)
        v = c["valid"].astype(bool)
        assert not (c["ref"][v] == 3).any()
        mixed += c["type"] == 2 and (c["ref"][v] == 1).any() and (c["ref"][v] == 2).any()
        stale += c["type"] == 1 and bool(((c["mv1"] != 0).any(-1) & v & (c["ref"] != 2)).any())
    assert mixed >= 1 and stale >= 1
