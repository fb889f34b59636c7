"""Per-frame quantizers on the host (no GPU): the C record and the appended config / io / buffers fields against their
ctypes mirrors, the pipelined schedule of daala_b200/gop.py simulated slot by slot, and what submit derives from the
records (each frame's deringing thresholds, the finishing pass's DC limit)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SRC = r"""
#include <stddef.h>
#include <stdio.h>
#include "daala_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %d\n", sizeof(daala_b200_kf_frame_quant),
         offsetof(daala_b200_kf_frame_quant, q0), offsetof(daala_b200_kf_frame_quant, coded_quantizer),
         offsetof(daala_b200_kf_frame_quant, dering_lambda), offsetof(daala_b200_kf_frame_quant, pvq_qm_q4),
         sizeof(daala_b200_kf_config), offsetof(daala_b200_kf_config, frame_quant),
         sizeof(daala_b200_kf_io), offsetof(daala_b200_kf_io, frame_quant),
         sizeof(daala_b200_kf_buffers), offsetof(daala_b200_kf_buffers, frame_quant),
         _Alignof(daala_b200_kf_frame_quant), DAALA_B200_KF_MAX_Q0);
  return 0;
}
"""


def test_struct_layout(tmp_path):
    from daala_b200 import engine
    (tmp_path / "layout.c").write_text(SRC)
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(tmp_path / "layout.c"), "-o", exe], check=True)
    got = [int(v) for v in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()]
    d = engine.FRAME_QUANT_DTYPE
    assert got == [112, d.fields["q0"][1], d.fields["coded_quantizer"][1], d.fields["dering_lambda"][1],
                   d.fields["pvq_qm_q4"][1], ctypes.sizeof(engine.Config), engine.Config.frame_quant.offset,
                   ctypes.sizeof(engine.IO), engine.IO.frame_quant.offset,
                   ctypes.sizeof(engine.Buffers), engine.Buffers.frame_quant.offset, 8, engine.MAX_Q0]
    assert d.itemsize == 112
    # appended last: every earlier field keeps its offset
    assert engine.Config.frame_quant.offset > engine.Config.mc_next.offset
    assert engine.IO.frame_quant.offset > engine.IO.mv1_grid.offset
    assert engine.Buffers.frame_quant.offset > engine.Buffers.mv1_grid.offset


def test_records_from_per_frame_arrays():
    from daala_b200 import engine, pvq
    q4 = np.arange(2 * 3 * 30, dtype=np.uint8).reshape(2, 3, 30) + 1
    r = engine.frame_quant_records([12, 8191], [6, 63], None, q4)
    assert r.dtype == engine.FRAME_QUANT_DTYPE and r.shape == (2,)
    assert list(r["q0"]) == [12, 8191] and list(r["coded_quantizer"]) == [6, 63]
    assert np.array_equal(r["dering_lambda"], 0.67 * pvq.PVQ_LAMBDA * np.array([12.0, 8191.0]) ** 2)
    assert np.array_equal(r["pvq_qm_q4"][..., :30], q4) and not r["pvq_qm_q4"][..., 30:].any()
    one = engine.frame_quant_records([30, 40, 50], 20, 1.5, q4[0])
    assert (one["coded_quantizer"] == 20).all() and (one["dering_lambda"] == 1.5).all()
    assert all(np.array_equal(x[..., :30], q4[0]) for x in one["pvq_qm_q4"])


def _simulate(b_frames, n, keyframe_rate):
    """Steps of the pipelined schedule against the reference's sequential order, on a pool of the four buffers."""
    from daala_b200 import gop
    order = gop.coding_order(n, b_frames, keyframe_rate)
    steps = gop.pipelined_steps(order)
    # what each buffer holds when each frame is coded in the reference's own order
    held, want = [-1] * 4, {}
    for fr in order:
        want[fr.number] = tuple(held[r] if r >= 0 else None for r in fr.refs[:gop.SELF])
        if fr.kept:
            held[fr.refs[gop.SELF]] = fr.number
    pool, done = [-1] * 4, set()
    for step in steps:
        assert step
        kinds = [f.type for f in step]
        if gop.I_FRAME in kinds:
            assert step == [step[0]] and len(step) == 1
        else:
            assert sum(k == gop.P_FRAME for k in kinds) <= 1 and all(k == gop.B_FRAME for k in kinds[1:])
        for fr in step:
            # every picture the frame reads was finished in an earlier step, and is the one the reference reads
            assert tuple(pool[r] if r >= 0 else None for r in fr.refs[:gop.SELF]) == want[fr.number], fr
            for r in fr.refs[:gop.SELF]:
                assert r < 0 or pool[r] in done
            g, p, nx = gop.pool_slots(fr)
            assert (g, p) == (fr.refs[gop.GOLD], fr.refs[gop.PREV])
            assert nx == (fr.refs[gop.NEXT] if fr.type == gop.B_FRAME else fr.refs[gop.PREV])
        for fr in step:   # the step's finish stores its anchors after every frame of the step has read the pool
            if fr.kept:
                pool[fr.refs[gop.SELF]] = fr.number
        done.update(fr.number for fr in step)
    return order, steps


@pytest.mark.parametrize("b_frames", [0, 1, 2, 3])
def test_pipelined_schedule(b_frames):
    from daala_b200 import gop
    for n, rate in ((47, 17), (64, 256), (23, 6)):
        order, steps = _simulate(b_frames, n, rate)
        flat = [f.number for s in steps for f in s]
        assert sorted(flat) == list(range(n)) and len(flat) == len(order)   # every coded frame exactly once
        kinds = {f.type for f in order}
        assert gop.I_FRAME in kinds and (b_frames == 0) == (gop.B_FRAME not in kinds)
        if rate > 10 and n > 40:
            assert sum(f.golden and f.type == gop.P_FRAME for f in order) >= 1
        if b_frames and rate == 256:   # the steps that hold an anchor also hold the B frames coded before it
            assert max(len(s) for s in steps) == b_frames + 1


def test_derived_thresholds_and_dc_limit():
    """daala_b200_kf_frame_quant_derive: per frame (int)(OD_DERING_GAIN_TABLE[g] * q0^0.84182) (x 0.6 on chroma) as
    daala_b200_dering_threshold_table computes it, and the finishing pass's DC limit 2^30 / the largest dc_quant of the
    step over records, planes and block sizes (entries od_qm_get_index(bs, 0) = bs * (bs + 1))."""
    from daala_b200 import engine
    from tests.test_gpu_engine_quantizer_range import SETTINGS
    q0 = SETTINGS["quantizer"].reshape(-1)
    q4 = SETTINGS["pvq_qm_q4"].reshape(-1, 3, 30)
    rec = engine.frame_quant_records(q0, SETTINGS["coded_quantizer"].reshape(-1), None, q4)
    tbl, limit = engine.frame_quant_derive(rec)
    gain = (0, 0.5, 0.707, 1, 1.41, 2)
    for f in range(len(rec)):
        base = float(q0[f]) ** 0.84182
        assert list(tbl[f, 0]) == [int(g * base) for g in gain], f
        assert list(tbl[f, 1]) == [int(g * base * 0.6) for g in gain], f
    dq = [(int(r["q0"]) * int(r["pvq_qm_q4"][p][bs * (bs + 1)])) >> 4 for r in rec for p in range(3) for bs in range(5)]
    assert limit == (1 << 30) // max(dq)
    # one frame's limit is its own; the step's is the smallest of its frames'
    limits = [engine.frame_quant_derive(rec[f:f + 1])[1] for f in range(len(rec))]
    assert limit == min(limits) and len(set(limits)) > 1
