"""Per-frame quantizers in keyframe batches (config.keyframe_quant) without a GPU: the appended config field against its
ctypes mirror and the refusals of daala_b200_kf_create (before it looks for a device), among them the q0 range every
lossy engine's config must keep, since its records are made from it."""
import ctypes
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SRC = r"""
#include <stddef.h>
#include <stdio.h>
#include "daala_b200.h"
int main(void) {
  printf("%zu %zu %zu\n", sizeof(daala_b200_kf_config), offsetof(daala_b200_kf_config, keyframe_quant),
         offsetof(daala_b200_kf_config, haar_dc_quant));
  return 0;
}
"""


def test_struct_layout(tmp_path):
    from daala_b200 import engine
    (tmp_path / "layout.c").write_text(SRC)
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(tmp_path / "layout.c"), "-o", exe], check=True)
    got = [int(v) for v in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [ctypes.sizeof(engine.Config), engine.Config.keyframe_quant.offset, engine.Config.haar_dc_quant.offset]
    assert engine.Config.keyframe_quant.offset == engine.Config.haar_dc_quant.offset + 4   # appended after it


KQ = "keyframe_quant is not defined with "
Q0 = r"q0 is outside \[1, 8191\]"
REFUSED = (
    (dict(keyframe_quant=2), KQ + "a value other than 0 or 1"),
    (dict(keyframe_quant=-1), KQ + "a value other than 0 or 1"),
    (dict(inter=1), KQ + "inter"),
    (dict(lossless=1), KQ + "lossless"),
    (dict(sb_row0=0, sb_rows=1), KQ + r"a row shard \(sb_rows > 0\)"),
    (dict(q0=0), Q0),
    (dict(keyframe_quant=0, q0=0), Q0),
    (dict(keyframe_quant=0, q0=-3), Q0),
    (dict(keyframe_quant=0, q0=8192), Q0),
    (dict(keyframe_quant=0, inter=1, q0=0), Q0),
)


@pytest.mark.parametrize("kw,why", REFUSED, ids=lambda v: ",".join("%s=%s" % kv for kv in v.items())
                         if isinstance(v, dict) else "")
def test_create_refusals(kw, why):
    """daala_b200_kf_create refuses these with a message: keyframe_quant naming what it is not defined with, and a
    lossy engine's q0 outside the range of a record's."""
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    kw = dict(kw)
    kw.setdefault("keyframe_quant", 1)
    with pytest.raises(RuntimeError, match="daala_b200_kf_create: " + why):
        engine.KeyframeEngine(Geometry(200, 130), nframes=1, **kw)


def test_frame_quant_on_keyframes_stays_refused():
    """P and B frames keep their mode: frame_quant = 1 without inter is refused as before, and the message points to
    the keyframe field."""
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    with pytest.raises(RuntimeError, match="frame_quant is 0 or 1.*keyframe_quant"):
        engine.KeyframeEngine(Geometry(200, 130), nframes=1, frame_quant=1)
