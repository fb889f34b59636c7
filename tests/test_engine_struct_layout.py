"""The ctypes mirrors of the engine's C structs (daala_b200/engine.py) have the sizes and the offsets of the
fields appended last that include/daala_b200.h gives them."""
import ctypes
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SRC = r"""
#include <stddef.h>
#include <stdio.h>
#include "daala_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(daala_b200_kf_config), offsetof(daala_b200_kf_config, inter),
         sizeof(daala_b200_kf_io), offsetof(daala_b200_kf_io, pred_pixels), offsetof(daala_b200_kf_io, chroma_dc),
         sizeof(daala_b200_kf_buffers), offsetof(daala_b200_kf_buffers, pred_pixels),
         offsetof(daala_b200_kf_buffers, pred_coeffs), sizeof(daala_b200_kf_totals));
  return 0;
}
"""


def test_ctypes_mirrors_match_the_header(tmp_path):
    from daala_b200 import engine
    (tmp_path / "layout.c").write_text(SRC)
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(tmp_path / "layout.c"), "-o", exe], check=True)
    got = [int(v) for v in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [ctypes.sizeof(engine.Config), engine.Config.inter.offset,
                   ctypes.sizeof(engine.IO), engine.IO.pred_pixels.offset, engine.IO.chroma_dc.offset,
                   ctypes.sizeof(engine.Buffers), engine.Buffers.pred_pixels.offset, engine.Buffers.pred_coeffs.offset,
                   ctypes.sizeof(engine.Totals)]
