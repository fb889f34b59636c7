"""The keyframe DC records of the symbol stream (symbol_stream = 1 with haar_dc_quant = 1) without a GPU: the numpy walk
haardc.stream_records over the reference driver's index grids gives one record per leaf of every (superblock, plane),
the records replayed through the reference's generic_encode code the same bytes as the reference's own DC chain
(tests/haar_dc_stream_oracle.py), and haardc.grids_from_records rebuilds the grids; the record's C layout."""
import os
import subprocess

import numpy as np
import pytest

from tests.test_haar_dc_host import content, maps, settings

SIZES = ((200, 130), (1920, 1080))


@pytest.fixture(scope="module")
def libs():
    from tests import haar_dc_oracle, haar_dc_stream_oracle
    drv, strm = haar_dc_oracle.load(), haar_dc_stream_oracle.load()
    if drv is None or strm is None:
        pytest.skip("needs oracle/_ref/libdaala_ref_haar_dc.so and libdaala_ref_haar_dc_stream.so (the reference sources)")
    return drv, strm


def check_structure(records, bsize, geom):
    """One record per leaf of every (superblock, plane), the superblock DC first, every block inside the (superblock,
    plane)'s range of block records, blocks non-decreasing; returns the leaf count."""
    from daala_b200 import symbols
    order = symbols.coding_order(bsize, geom)
    assert len(records) == len(order)
    sb = (order["y0"].astype(np.int64) >> np.where(order["pli"] > 0, 5, 6)) * geom.nhsb + \
         (order["x0"].astype(np.int64) >> np.where(order["pli"] > 0, 5, 6))
    group = sb * 3 + order["pli"]
    starts = np.nonzero(np.r_[True, group[1:] != group[:-1]])[0]
    ends = np.r_[starts[1:], len(group)]
    blk = records["block"].astype(np.int64)
    for s, e in zip(starts, ends):
        assert records["child"][s] == 0 and records["bsi"][s] == 4 and blk[s] == s
        assert np.all(records["child"][s + 1:e] > 0)
        assert np.all((blk[s:e] >= s) & (blk[s:e] < e))
        assert np.all(records["pli"][s:e] == order["pli"][s])
    assert np.all(np.diff(blk) >= 0)
    assert np.all(records["reserved"] == 0)
    return len(order)


@pytest.mark.parametrize("size", SIZES, ids=lambda s: "%dx%d" % s)
def test_records_replay_to_the_reference_bytes(libs, size):
    """For every map (uniform 4x4 .. 64x64, random quadtrees, a real encoder map) and a spread of the encoder's keyframe
    settings: one record per leaf, byte-equal coding against the reference's own chain, and the grids rebuilt."""
    from daala_b200 import haardc
    from daala_b200.frame import Geometry
    from tests import haar_dc_oracle, haar_dc_stream_oracle
    drv, strm = libs
    geom = Geometry(*size)
    sets = settings()
    kinds = ("random", "ramp", "checker")
    nonzero = 0
    for mi, (name, bs) in enumerate(maps(geom)):
        for j in range(2 if size[0] < 1000 else 1):
            kind = kinds[(mi + j) % len(kinds)]
            q0, q4, lam = sets[(3 * mi + 5 * j) % len(sets)]
            planes = content(geom, kind, seed=mi + 7 * j)
            want = haar_dc_oracle.frame(drv, geom, planes, bs, q0, q4, lam)
            rec = haardc.stream_records(want["idx"], bs, geom)
            check_structure(rec, bs, geom)
            nonzero += int(np.count_nonzero(rec["value"]))
            ref = haar_dc_stream_oracle.frame_bytes(strm, geom, planes, bs, q0, q4, lam)
            got = haar_dc_stream_oracle.replay(strm, geom, rec)
            assert got == ref, (name, kind, q0, len(got), len(ref))
            back = haardc.grids_from_records(rec, bs, geom)
            for p in range(3):
                assert np.array_equal(back[p], want["idx"][p]), (name, p)
    assert nonzero > 0


def test_replay_detects_a_changed_record(libs):
    """The byte comparison is sensitive: one value, one context (bsi) or one swapped pair changes the bytes."""
    from daala_b200 import haardc
    from daala_b200.frame import Geometry
    from tests import haar_dc_oracle, haar_dc_stream_oracle
    drv, strm = libs
    geom = Geometry(200, 130)
    bs = dict(maps(geom))["quadtree3"]
    q0, q4, lam = settings()[2]
    planes = content(geom, "random", seed=1)
    want = haar_dc_oracle.frame(drv, geom, planes, bs, q0, q4, lam)
    rec = haardc.stream_records(want["idx"], bs, geom)
    ref = haar_dc_stream_oracle.frame_bytes(strm, geom, planes, bs, q0, q4, lam)
    assert haar_dc_stream_oracle.replay(strm, geom, rec) == ref
    i = int(np.nonzero((rec["child"] > 0) & (rec["value"] != 0))[0][0])
    for change in ("value", "bsi", "swap"):
        r = rec.copy()
        if change == "value":
            r["value"][i] += 1
        elif change == "bsi":
            r["bsi"][i] = (r["bsi"][i] + 1) % 4
        else:
            r[[0, 1]] = r[[1, 0]]
        assert haar_dc_stream_oracle.replay(strm, geom, r) != ref, change


def test_uniform_maps_give_the_expected_counts():
    """No reference needed: an all-64x64 map gives only superblock DCs, an all-4x4 map one record per 4x4 luma block
    and per 4x4 chroma block, and the inverse walk refuses records that do not fit the map."""
    from daala_b200 import haardc, synth
    from daala_b200.frame import Geometry
    geom = Geometry(200, 130)
    nsb = geom.nhsb * geom.nvsb
    grids = [np.arange(np.prod(s) // 16, dtype=np.int32).reshape(s[0] // 4, s[1] // 4) - 7
             for s in (geom.plane_shape(p) for p in range(3))]
    rec = haardc.stream_records(grids, synth.block_size_map(geom, "64"), geom)
    assert len(rec) == 3 * nsb and np.all(rec["child"] == 0)
    rec = haardc.stream_records(grids, synth.block_size_map(geom, "4"), geom)
    assert len(rec) == nsb * (256 + 2 * 64)
    assert check_structure(rec, synth.block_size_map(geom, "4"), geom) == len(rec)
    back = haardc.grids_from_records(rec, synth.block_size_map(geom, "4"), geom)
    assert np.array_equal(back[0], grids[0])            # every 4x4 luma unit carries a symbol on an all-4x4 map
    with pytest.raises(AssertionError):
        haardc.grids_from_records(rec[:-1], synth.block_size_map(geom, "4"), geom)


SRC = r"""
#include <stddef.h>
#include <stdio.h>
#include "daala_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(daala_b200_kf_sym_hdc), offsetof(daala_b200_kf_sym_hdc, block),
         offsetof(daala_b200_kf_sym_hdc, pli), offsetof(daala_b200_kf_sym_hdc, bsi),
         offsetof(daala_b200_kf_sym_hdc, child), sizeof(daala_b200_kf_io), offsetof(daala_b200_kf_io, sym_hdc),
         offsetof(daala_b200_kf_io, sym_hdc_cap));
  return 0;
}
"""


def test_layout_matches_the_header(tmp_path):
    import ctypes
    from daala_b200 import engine, symbols
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    (tmp_path / "layout.c").write_text(SRC)
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), str(tmp_path / "layout.c"), "-o", exe], check=True)
    got = [int(v) for v in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()]
    d = symbols.HDC_DTYPE
    assert got == [d.itemsize, d.fields["block"][1], d.fields["pli"][1], d.fields["bsi"][1], d.fields["child"][1],
                   ctypes.sizeof(engine.IO), engine.IO.sym_hdc.offset, engine.IO.sym_hdc_cap.offset]
