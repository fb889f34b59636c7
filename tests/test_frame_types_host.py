"""Host side of batches that mix keyframes and P / B frames (config.frame_types): gop.pipelined_steps with
keyframes_inline, the ctypes mirrors of the new config and io fields, and the Python wrapper's frame_type= rule.  No
GPU needed."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from daala_b200 import engine, gop

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("n,b,rate", [(20, 2, 7), (31, 3, 9), (12, 0, 5), (17, 1, 4)])
def test_keyframes_inline_puts_each_i_frame_with_its_b_frames(n, b, rate):
    frames = gop.coding_order(n, b, keyframe_rate=rate)
    steps = gop.pipelined_steps(frames, keyframes_inline=True)
    assert [fr for st in steps for fr in sorted(st, key=lambda fr: frames.index(fr))] == frames
    assert sum(fr.type == gop.I_FRAME for fr in frames) > 1
    pos = 0
    for st in steps:
        anchors = [fr for fr in st if fr.type != gop.B_FRAME]
        assert len(anchors) <= 1
        if anchors:
            # the anchor, I or P alike, first, then the B frames coded just before it
            assert st[0] is anchors[0] and st[1:] == frames[pos:pos + len(st) - 1]
        pos += len(st)
    # the default keeps an I frame in a step of its own
    default = gop.pipelined_steps(frames)
    assert gop.pipelined_steps(frames, keyframes_inline=False) == default
    for st in default:
        assert not any(fr.type == gop.I_FRAME for fr in st) or len(st) == 1
    # the two differ only where an I frame had B frames coded before it
    assert len(default) >= len(steps)


LAYOUT = r"""
#include <stddef.h>
#include <stdio.h>
#include "daala_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu\n", sizeof(daala_b200_kf_config), offsetof(daala_b200_kf_config, frame_types),
         sizeof(daala_b200_kf_io), offsetof(daala_b200_kf_io, frame_type));
  return 0;
}
"""


def test_frame_types_fields_match_the_header(tmp_path):
    (tmp_path / "layout.c").write_text(LAYOUT)
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(tmp_path / "layout.c"), "-o", exe], check=True)
    got = [int(v) for v in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [ctypes.sizeof(engine.Config), engine.Config.frame_types.offset, ctypes.sizeof(engine.IO),
                   engine.IO.frame_type.offset]


def _wrapper(F, frame_types):
    """The Python wrapper's host-buffer logic alone (no engine behind it)."""
    eng = engine.KeyframeEngine.__new__(engine.KeyframeEngine)
    eng.F, eng.frame_types, eng.pinned, eng._host, eng._ftype = F, frame_types, False, {}, None
    return eng


def test_frame_type_is_refused_without_the_mode_and_required_with_it():
    with pytest.raises(ValueError, match="frame_type"):
        _wrapper(3, 0).stage_frame_type([1, 0, 0])
    with pytest.raises(ValueError, match="frame_type"):
        _wrapper(3, 1).stage_frame_type(None)
    with pytest.raises(ValueError, match="frame_type"):
        _wrapper(3, 1).stage_frame_type([1, 0])
    eng = _wrapper(3, 1)
    eng.stage_frame_type([1, 0, 1])
    assert eng._ftype.dtype == np.uint8 and list(eng._ftype) == [1, 0, 1]
    _wrapper(3, 0).stage_frame_type(None)
