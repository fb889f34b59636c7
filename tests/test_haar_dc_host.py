"""Quantised keyframe DCs (config.haar_dc_quant) without a GPU: the numpy restatement daala_b200/haardc.py against the
reference's own od_compute_dcts, od_quantize_haar_dc_sb and od_quantize_haar_dc_level (tests/haar_dc_oracle.py,
oracle/ref_hooks_haar_dc.c) over extreme content, uniform, random and real encoder block-size maps, partial
superblocks and the encoder's quantizer settings; the C struct layout and the refusals of daala_b200_kf_create."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONTENT = ("random", "flat", "saturated", "checker", "ramp")
SIZES = ((200, 130), (128, 192))


def content(geom, kind, seed=0):
    """Three frame-sized u8 planes: random, flat, saturated (255 above a diagonal, 0 below), a 0 / 255 checkerboard of
    single samples, or a ramp across the frame."""
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
        elif kind == "checker":
            a = ((x + y) & 1) * 255
        else:
            a = (x * 255 // (w - 1) + y * 255 // (h - 1)) // 2
        out.append(a.astype(np.uint8))
    return out


def maps(geom):
    """Uniform 4..64, two random quadtrees and, cropped / tiled to the geometry, a real encoder map of the bench."""
    from daala_b200 import synth
    out = [(m, synth.block_size_map(geom, m)) for m in ("4", "8", "16", "32", "64")]
    out += [("quadtree%d" % s, synth.block_size_map(geom, "mixed", seed=s)) for s in (3, 4)]
    real = np.load(os.path.join(ROOT, "daala_b200", "data", "bench_bsize_4k.npz"))
    bs = real[sorted(real.files)[0]]
    bs = bs.reshape(-1, bs.shape[-2], bs.shape[-1])[0]
    h, w = geom.bsize_shape
    out.append(("encoder", np.ascontiguousarray(bs[:h, :w]).astype(np.uint8)))
    return out


def settings():
    """(quantizer, pvq_qm_q4, pvq_norm_lambda) the reference encoder sets for a keyframe at every SETTINGS_QUANT x
    SETTINGS_CONFIGS point of tests/golden/make_golden.py."""
    s = np.load(os.path.join(ROOT, "tests", "golden", "encoder_settings.npz"))
    return [(int(s["quantizer"][i][c][0]), s["pvq_qm_q4"][i][c][0], float(s["pvq_norm_lambda"][i][c][0]))
            for i in range(s["quantizer"].shape[0]) for c in range(s["quantizer"].shape[1])]


@pytest.fixture(scope="module")
def lib():
    from tests import haar_dc_oracle
    lib = haar_dc_oracle.load()
    if lib is None:
        pytest.skip("needs oracle/_ref/libdaala_ref_haar_dc.so (the reference sources)")
    return lib


@pytest.mark.parametrize("size", SIZES, ids=lambda s: "%dx%d" % s)
def test_model_matches_reference(lib, size):
    """haardc.py equals the reference's DC chain: every reconstructed `d` value and every index, over all content,
    maps and quantizer settings; the set reaches the RDO increment and the xs >= 15 tail of the generic coder."""
    from daala_b200 import haardc
    from daala_b200.frame import Geometry
    from tests import haar_dc_oracle
    geom = Geometry(*size)
    reached = dict(rdo_inc=0, tail=0, symbols=0)
    sets = settings()
    for ki, kind in enumerate(CONTENT):
        planes = content(geom, kind, seed=ki)
        for mi, (name, bs) in enumerate(maps(geom)):
            # every quantizer setting on the random content, a rotating third of them elsewhere
            for si, (q0, q4, lam) in enumerate(sets):
                if kind != "random" and (si + mi) % 3:
                    continue
                want = haar_dc_oracle.frame(lib, geom, planes, bs, q0, q4, lam)
                got = haardc.quantize_frame(geom, want["d_pre"], bs, q0, q4, lam)
                for p in range(3):
                    assert np.array_equal(got["d"][p], want["d_post"][p]), (kind, name, q0, p)
                    assert np.array_equal(got["idx"][p], want["idx"][p]), (kind, name, q0, p)
                    for k in reached:
                        reached[k] += got["stats"][p][k]
    assert reached["rdo_inc"] > 0 and reached["tail"] > 0, reached


def test_index_positions(lib):
    """The index grid holds a value only at a superblock origin or at a child 1..3 origin of a split node, and a 64x64
    map codes one index per superblock and plane."""
    from daala_b200 import haardc, synth
    from daala_b200.frame import Geometry
    from tests import haar_dc_oracle
    geom = Geometry(200, 130)
    planes = content(geom, "random", seed=5)
    q0, q4, lam = settings()[0]
    bs = synth.block_size_map(geom, "64")
    want = haar_dc_oracle.frame(lib, geom, planes, bs, q0, q4, lam)
    for p in range(3):
        idx = want["idx"][p]
        n = 16 >> (1 if p else 0)
        mask = np.zeros(idx.shape, bool)
        mask[::n, ::n] = True
        assert not idx[~mask].any()
        assert idx[mask].any()
        got = haardc.quantize_frame(geom, want["d_pre"], bs, q0, q4, lam)
        assert np.array_equal(got["idx"][p], idx)


SRC = r"""
#include <stddef.h>
#include <stdio.h>
#include "daala_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu\n", sizeof(daala_b200_kf_config), offsetof(daala_b200_kf_config, haar_dc_quant),
         sizeof(daala_b200_kf_io), offsetof(daala_b200_kf_io, dc_index), sizeof(daala_b200_kf_buffers),
         offsetof(daala_b200_kf_buffers, haar_dc));
  return 0;
}
"""


def test_struct_layout(tmp_path):
    from daala_b200 import engine
    (tmp_path / "layout.c").write_text(SRC)
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(tmp_path / "layout.c"), "-o", exe], check=True)
    got = [int(v) for v in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [ctypes.sizeof(engine.Config), engine.Config.haar_dc_quant.offset, ctypes.sizeof(engine.IO),
                   engine.IO.dc_index.offset, ctypes.sizeof(engine.Buffers), engine.Buffers.haar_dc.offset]
    assert engine.Config.haar_dc_quant.offset == engine.Config.lossless.offset + 4   # appended
    assert engine.IO.dc_index.offset > engine.IO.ll_ref_slot_out.offset
    assert engine.Buffers.haar_dc.offset > engine.Buffers.frame_quant.offset


REFUSED = (dict(haar_dc_quant=2), dict(haar_dc_quant=-1), dict(inter=1), dict(lossless=1), dict(sb_row0=0, sb_rows=1))


@pytest.mark.parametrize("kw", REFUSED, ids=lambda k: ",".join("%s=%s" % kv for kv in k.items()))
def test_create_refusals(kw):
    """daala_b200_kf_create refuses these with haar_dc_quant (before it looks for a device), with a message."""
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    kw = dict(kw)
    kw.setdefault("haar_dc_quant", 1)
    with pytest.raises(RuntimeError, match="daala_b200_kf_create: haar_dc_quant is not defined with"):
        engine.KeyframeEngine(Geometry(200, 130), nframes=1, **kw)
