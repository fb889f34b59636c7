"""Per-frame quantizers in keyframe batches (config.keyframe_quant) without a GPU: the appended config field against its
ctypes mirror, the refusals of daala_b200_kf_create (before it looks for a device), and the instruction footprint of
the luma chain kernel's per-frame instantiation, k_pvq_persist_fq<true> (nvcc cross-compiles)."""
import ctypes
import importlib.util
import os
import subprocess

import pytest

from daala_b200 import build as _build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HAVE_NVCC = os.path.exists(_build.NVCC)

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


REFUSED = (
    (dict(keyframe_quant=2), "a value other than 0 or 1"),
    (dict(keyframe_quant=-1), "a value other than 0 or 1"),
    (dict(inter=1), "inter"),
    (dict(lossless=1), "lossless"),
    (dict(noref_prepass=1), "noref_prepass"),
    (dict(level_chains=1), "level_chains"),
    (dict(sb_row0=0, sb_rows=1), r"a row shard \(sb_rows > 0\)"),
)


@pytest.mark.parametrize("kw,why", REFUSED, ids=lambda v: ",".join("%s=%s" % kv for kv in v.items())
                         if isinstance(v, dict) else "")
def test_create_refusals(kw, why):
    """daala_b200_kf_create refuses these with keyframe_quant, with a message naming what it is not defined with."""
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    kw = dict(kw)
    kw.setdefault("keyframe_quant", 1)
    with pytest.raises(RuntimeError, match="daala_b200_kf_create: keyframe_quant is not defined with " + why):
        engine.KeyframeEngine(Geometry(200, 130), nframes=1, **kw)


def test_frame_quant_on_keyframes_stays_refused():
    """P and B frames keep their mode: frame_quant = 1 without inter is refused as before, and the message points to
    the keyframe field."""
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    with pytest.raises(RuntimeError, match="frame_quant is 0 or 1.*keyframe_quant"):
        engine.KeyframeEngine(Geometry(200, 130), nframes=1, frame_quant=1)


# the budget of k_pvq_persist<true> (tests/test_sass_budget.py), which its per-frame instantiation holds too
MAX_SASS_BYTES = 96 * 1024
MAX_STACK_BYTES = 224
REGISTERS = 64


@pytest.mark.skipif(not HAVE_NVCC, reason="nvcc not available")
def test_per_frame_luma_chain_kernel_within_footprint_budget():
    path = os.path.join(_build.ROOT, "tools", "sass_footprint.py")
    spec = importlib.util.spec_from_file_location("sass_footprint", path)
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    rows, _ = tool.footprint()
    row = next(r for r in rows if r["kernel"] == "k_pvq_persist_fq<true>")
    assert row["sass_bytes"] <= MAX_SASS_BYTES, row
    assert row["stack"] <= MAX_STACK_BYTES, row
    assert row["regs"] == REGISTERS, row
    # the engine-wide kernel is still there under its own name, and the per-frame one is not larger by more than the
    # slack the budget leaves
    base = next(r for r in rows if r["kernel"] == "k_pvq_persist<true>")
    assert row["sass_bytes"] <= base["sass_bytes"] + 256, (row, base)
