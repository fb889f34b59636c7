"""Lossless frames (quantizer 0) without a GPU: the numpy restatement daala_b200/lossless.py against the reference's
own statics (tests/lossless_oracle.py, oracle/ref_hooks_lossless.c) on keyframes and P frames over extreme content, its
round trip, the int16 bound of the engine's residual planes, the C struct layout and the refusals of
daala_b200_kf_create."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONTENT = ("random", "flat", "saturated", "checker")
SIZES = ((200, 130), (128, 192))


def content(geom, kind, seed=0):
    """Three frame-sized u8 planes: random, flat (one value), saturated (255 above a diagonal, 0 below) or a 0 / 255
    checkerboard of single samples."""
    rng = np.random.default_rng(seed)
    out = []
    for p in range(3):
        h, w = geom.plane_shape(p)
        y, x = np.mgrid[0:h, 0:w]
        if kind == "random":
            a = rng.integers(0, 256, (h, w))
        elif kind == "flat":
            a = np.full((h, w), 77 + 50 * p)
        elif kind == "saturated":
            a = np.where(x * h >= y * w, 255, 0)
        else:
            a = ((x + y) & 1) * 255
        out.append(a.astype(np.uint8))
    return out


def inverted(planes):
    """The prediction in inverted phase (255 - source): the largest residuals a P frame can have."""
    return [(255 - np.asarray(a, np.int64)).astype(np.uint8) for a in planes]


def _driver():
    from tests import lossless_oracle
    lib = lossless_oracle.load()
    if lib is None:
        pytest.skip("oracle/_ref/libdaala_ref_lossless.so not built (needs the reference sources)")
    return lib


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("kind", CONTENT)
@pytest.mark.parametrize("inter", [0, 1])
def test_model_matches_reference_driver(size, kind, inter):
    from daala_b200 import lossless
    from daala_b200.frame import Geometry
    from tests import lossless_oracle
    lib = _driver()
    geom = Geometry(*size)
    planes = content(geom, kind, seed=3)
    pred = inverted(planes) if inter else None
    got = lossless.encode_frame(geom, planes, pred)
    want = lossless_oracle.frame(lib, geom, planes, pred)
    for p in range(3):
        assert np.array_equal(got["d"][p], want["d"][p]), ("d", p)
        assert np.array_equal(got["coeffs"][p], want["coeffs"][p]), ("residual", p)
    assert np.array_equal(got["blocks"][..., :3], want["roots"])
    assert not got["blocks"][..., 3].any()


@pytest.mark.parametrize("kind", CONTENT)
@pytest.mark.parametrize("inter", [0, 1])
def test_model_round_trip(kind, inter):
    """What the decoder makes from the residual is the (padded) input: the source in the picture, and for P frames the
    prediction outside it."""
    from daala_b200 import lossless
    from daala_b200.frame import Geometry
    geom = Geometry(200, 130)
    planes = content(geom, kind, seed=5)
    pred = inverted(content(geom, "random", seed=6)) if inter else None
    rec = lossless.decode_frame(geom, lossless.encode_frame(geom, planes, pred)["coeffs"], pred)
    want = lossless.padded_input(geom, planes, pred)
    for p in range(3):
        assert np.array_equal(rec[p].astype(np.int64) - 128, want[p]), p
        if inter:
            ph, pw = geom.pic_h >> (1 if p else 0), geom.pic_w >> (1 if p else 0)
            assert np.array_equal(rec[p][:ph, :pw], planes[p][:ph, :pw])


def test_residuals_fit_int16():
    """The bound DESIGN.md derives: |d - md| <= 16320 (DC included) and |dc0| <= 21420 on 64x64 luma blocks, reached
    (up to the closed form's rounding) by the extreme content."""
    from daala_b200 import lossless
    from daala_b200.frame import Geometry
    b6, b5 = lossless.bounds(6), lossless.bounds(5)
    assert b6 == dict(dc=(-8192, 8128), detail=8160, resid=16320, dc0=(-21420, 21420))
    assert max(b5["resid"], -b5["dc0"][0], b5["dc0"][1]) < max(b6["resid"], -b6["dc0"][0], b6["dc0"][1]) <= 32767
    geom = Geometry(256, 128)
    worst = 0
    for kind in CONTENT:
        planes = content(geom, kind, seed=9)
        for pred in (None, inverted(planes)):
            out = lossless.encode_frame(geom, planes, pred)
            for p in range(3):
                b = b5 if p else b6
                c = out["coeffs"][p]
                n = 32 if p else 64
                ac = c.copy()
                ac[::n, ::n] = 0
                assert np.abs(ac).max() <= b["resid"]
                dc = c[::n, ::n]
                assert (dc >= (b["dc0"][0] if pred is None else -b["resid"])).all()
                assert (dc <= (b["dc0"][1] if pred is None else b["resid"])).all()
                worst = max(worst, int(np.abs(c).max()))
    assert worst >= 16320 - 64   # the inverted checkerboard's finest details reach the bound's order


SRC = r"""
#include <stddef.h>
#include <stdio.h>
#include "daala_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu\n", sizeof(daala_b200_kf_config), offsetof(daala_b200_kf_config, lossless),
         sizeof(daala_b200_kf_io), offsetof(daala_b200_kf_io, ll_coeffs), offsetof(daala_b200_kf_io, ll_blocks),
         offsetof(daala_b200_kf_io, ll_ref_slot_out), sizeof(daala_b200_kf_ll_block));
  return 0;
}
"""


def test_struct_layout(tmp_path):
    from daala_b200 import engine
    (tmp_path / "layout.c").write_text(SRC)
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(tmp_path / "layout.c"), "-o", exe], check=True)
    got = [int(v) for v in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [ctypes.sizeof(engine.Config), engine.Config.lossless.offset, ctypes.sizeof(engine.IO),
                   engine.IO.ll_coeffs.offset, engine.IO.ll_blocks.offset, engine.IO.ll_ref_slot_out.offset, 16]
    assert engine.Config.lossless.offset >= engine.Config.frame_quant.offset + 4   # appended
    assert engine.IO.ll_coeffs.offset > engine.IO.frame_quant.offset


REFUSED = (dict(lossless=2), dict(lossless=-1), dict(dering=1), dict(symbol_stream=1), dict(inter=1, symbol_stream=2),
           dict(inter=1, late_skip=1), dict(inter=1, inter_finish=1), dict(inter=1, frame_quant=1),
           dict(noref_prepass=1), dict(level_chains=1), dict(sb_rows=1))


@pytest.mark.parametrize("kw", REFUSED, ids=lambda kw: ",".join("%s=%d" % i for i in kw.items()))
def test_create_refusals(kw):
    """daala_b200_kf_create refuses these with lossless (before it looks for a device), with a message."""
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    kw = dict(kw)
    kw.setdefault("lossless", 1)
    with pytest.raises(RuntimeError, match="daala_b200_kf_create: lossless is not defined with"):
        engine.KeyframeEngine(Geometry(200, 130), nframes=1, **kw)
