"""The P-frame finishing pass (config.inter_finish; daala_b200_kf_finish, csrc/kf_engine.cu): the host coder's skip and
DC decisions applied to a step's coefficients, the skip maps, deringing over them and the final reconstruction,
against the oracle's frame driver inverse_frame_inter_finish (oracle/inter_finish_driver.inc) fed the numpy restatement
of the patch and the skip map (daala_b200/interfinish.py).  Bit-exact throughout.  The last two tests need no GPU."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from tests import frame_oracle, inter_finish_oracle, oracle_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Q4 = np.full((3, 30), 20, np.uint8)


def _frames(geom, F, seed, mode="mixed"):
    from daala_b200 import synth
    pics = [synth.pad_planes(synth.frame(geom.pic_w, geom.pic_h, f=f, seed=seed + 5 * f)[0], geom) for f in range(F + 1)]
    planes = [np.stack([pics[f + 1][p] for f in range(F)]) for p in range(3)]
    pred = [np.stack([pics[f][p] for f in range(F)]) for p in range(3)]
    bsize = np.stack([synth.block_size_map(geom, mode, seed=seed + f) for f in range(F)])
    return planes, pred, bsize


def _engine(geom, F, q0, **kw):
    from daala_b200 import engine
    return engine.KeyframeEngine(geom, nframes=F, q0=q0, pvq_qm_q4=Q4, inter=1, inter_finish=1, **kw)


def _step(eng, planes, pred, bsize, **kw):
    out = eng.encode(planes, bsize, pred=pred, **kw)
    out = {k: np.array(v) for k, v in out.items()}
    d = [eng.coeff_plane(p) for p in range(3)]
    md = [eng.pred_coeff_plane(p) for p in range(3)]
    return out, d, md


def _sb_of(blocks):
    """Superblock (row, column) of each block record (luma or chroma)."""
    sh = np.where(blocks["pli"] == 0, 6, 5)
    return blocks["y0"].astype(np.int64) >> sh, blocks["x0"].astype(np.int64) >> sh


def _decisions(out, geom, F, seed):
    """Seeded decisions: about 30 % of the blocks skipped, DC = qdc + -2..2 (some skipped blocks keep a non-zero DC),
    levels 0..5; in frame 0 one superblock whose luma is all skipped but one chroma block is coded (forced to level
    0), and one whose only coded luma is a single 4x4 block (filtered).  Returns (ls, ld, cs, cd, levels, special)."""
    rng = np.random.default_rng(seed)
    lb, cb = out["luma_blocks"], out["chroma_blocks"]
    ls = (rng.random(len(lb)) < 0.3).astype(np.uint8)
    cs = (rng.random(len(cb)) < 0.3).astype(np.uint8)
    ld = out["luma_dc"] + rng.integers(-2, 3, len(lb)).astype(np.int32) * (rng.random(len(lb)) < 0.5)
    cd = out["chroma_dc"] + rng.integers(-2, 3, len(cb)).astype(np.int32) * (rng.random(len(cb)) < 0.5)
    ld, cd = ld.astype(np.int32), cd.astype(np.int32)
    levels = rng.integers(0, 6, (F, geom.nvsb, geom.nhsb)).astype(np.uint8)
    ly, lx = _sb_of(lb)
    cy, cx = _sb_of(cb)
    f0 = lb["frame"] == 0
    four = np.nonzero(f0 & (lb["bs"] == 0))[0]
    assert len(four), "the map has no 4x4 luma block"
    one = (int(ly[four[0]]), int(lx[four[0]]))
    chroma_only = next((y, x) for y in range(geom.nvsb) for x in range(geom.nhsb) if (y, x) != one)
    for (sy, sx), keep in ((one, four[0]), (chroma_only, None)):
        sel = f0 & (ly == sy) & (lx == sx)
        ls[sel], ld[sel] = 1, 0
        if keep is not None:
            ls[keep], ld[keep] = 0, out["luma_dc"][keep]
        levels[0, sy, sx] = 3
    csel = np.nonzero((cb["frame"] == 0) & (cy == chroma_only[0]) & (cx == chroma_only[1]))[0]
    cs[csel[0]] = 0
    return ls, ld, cs, cd, levels, dict(one=one, chroma_only=chroma_only)


def _want(geom, F, out, d, md, bsize, q0, dec):
    """Per frame the oracle's (recon planes, applied levels, skip maps) for the decisions dec."""
    from daala_b200 import interfinish
    lib, prefix = inter_finish_oracle.load()
    ls, ld, cs, cd, levels = dec[:5]
    res = []
    for f in range(F):
        dq, bskip = [], []
        for p in range(3):
            blocks, skip, dc = (out["luma_blocks"], ls, ld) if p == 0 else (out["chroma_blocks"], cs, cd)
            dq.append(interfinish.patch(d[p][f], md[p][f], blocks, skip, dc, f, p, q0, Q4))
            bskip.append(interfinish.skip_map(blocks, skip, dc, f, p, geom))
        recs, applied = inter_finish_oracle.finish(lib, prefix, dq, geom, bsize[f], q0, levels[f], bskip)
        assert np.array_equal(applied, np.where(interfinish.coded_superblocks(bskip[0], geom), levels[f], 0))
        res.append((recs, applied, bskip))
    return res


def _check(got, want, F):
    for f in range(F):
        recs, applied, bskip = want[f]
        for p in range(3):
            assert np.array_equal(got["recon%d" % p][f], recs[p]), ("recon", f, p)
            assert np.array_equal(got["bskip%d" % p][f], bskip[p]), ("bskip", f, p)
        assert np.array_equal(got["dering_levels"][f], applied), ("levels", f)


def _copy(r):
    return {k: np.array(v) for k, v in r.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,F", [(200, 130, 2), (1920, 1080, 1)])
def test_finish_identity_is_the_step_reconstruction(w, h, F):
    """skip = 0, dc = qdc, levels 0: the step's own reconstruction, nothing marked skipped."""
    from daala_b200.frame import Geometry
    geom = Geometry(w, h)
    eng = _engine(geom, F, 45)
    planes, pred, bsize = _frames(geom, F, seed=w)
    out, d, md = _step(eng, planes, pred, bsize)
    got = eng.finish(np.zeros(len(out["luma_dc"]), np.uint8), out["luma_dc"],
                     np.zeros(len(out["chroma_dc"]), np.uint8), out["chroma_dc"], np.zeros((F, geom.nvsb, geom.nhsb), np.uint8))
    for p in range(3):
        assert np.array_equal(got["recon%d" % p], out["recon%d" % p]), p
        assert not got["bskip%d" % p].any()
    assert not got["dering_levels"].any()
    # the step's planes are untouched by the pass
    for p in range(3):
        assert np.array_equal(eng.coeff_plane(p), d[p]) and np.array_equal(eng.pred_coeff_plane(p), md[p])
        assert np.array_equal(eng.recon_plane(p), out["recon%d" % p])
    eng.close()


@pytest.mark.gpu
def test_finish_identity_inter_mc():
    from daala_b200.frame import Geometry
    from tests import test_gpu_engine_inter_mc as mc
    geom = Geometry(200, 130)
    F = 2
    refs = mc._pool(geom, 3, seed=7)
    grids = mc._grids(geom, F, seed=3)
    planes, bsize = mc._batch(geom, F, seed=11)
    eng = _engine(geom, F, 45, inter_mc=1)
    out = eng.encode(planes, bsize, refs=refs, ref_slot=np.array([[0, 1], [2, 1]], np.int32), mv_grid=mc._pack(grids))
    out = _copy(out)
    got = eng.finish(np.zeros(len(out["luma_dc"]), np.uint8), out["luma_dc"],
                     np.zeros(len(out["chroma_dc"]), np.uint8), out["chroma_dc"])
    for p in range(3):
        assert np.array_equal(got["recon%d" % p], out["recon%d" % p]), p
    # random decisions on the engine's own prediction
    d = [eng.coeff_plane(p) for p in range(3)]
    md = [eng.pred_coeff_plane(p) for p in range(3)]
    dec = _decisions(out, geom, F, seed=5)
    _check(_copy(eng.finish(*dec[:5])), _want(geom, F, out, d, md, bsize, 45, dec), F)
    eng.close()


@pytest.mark.gpu
def test_finish_all_skipped_is_the_prediction():
    """skip = 1, dc = 0 everywhere: the lapped transform is reversible, so the reconstruction is the prediction;
    every block is skipped and no superblock is deringed whatever its level."""
    from daala_b200.frame import Geometry
    geom = Geometry(328, 200)
    F = 2
    eng = _engine(geom, F, 38)
    planes, pred, bsize = _frames(geom, F, seed=2)
    out, _, _ = _step(eng, planes, pred, bsize)
    rng = np.random.default_rng(1)
    got = eng.finish(np.ones(len(out["luma_dc"]), np.uint8), np.zeros(len(out["luma_dc"]), np.int32),
                     np.ones(len(out["chroma_dc"]), np.uint8), np.zeros(len(out["chroma_dc"]), np.int32),
                     rng.integers(1, 6, (F, geom.nvsb, geom.nhsb)).astype(np.uint8))
    for p in range(3):
        assert np.array_equal(got["recon%d" % p], pred[p]), p
        w4 = geom.plane_shape(p)[1] // 4
        assert got["bskip%d" % p][:, :, :w4].all() and not got["bskip%d" % p][:, :, w4:].any()
    assert not got["dering_levels"].any()
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,F", [(200, 130, 2), (328, 200, 2), (1920, 1080, 1)])
def test_finish_random_decisions_match_oracle(w, h, F):
    from daala_b200.frame import Geometry
    geom = Geometry(w, h)
    q0 = 45
    eng = _engine(geom, F, q0)
    planes, pred, bsize = _frames(geom, F, seed=h)
    out, d, md = _step(eng, planes, pred, bsize)
    dec = _decisions(out, geom, F, seed=w)
    ls, ld, cs = dec[0], dec[1], dec[2]
    assert 0.2 < ls.mean() < 0.4 and (ls.astype(bool) & (ld != 0)).any() and (cs.astype(bool) & (dec[3] != 0)).any()
    got = _copy(eng.finish(*dec[:5]))
    want = _want(geom, F, out, d, md, bsize, q0, dec)
    _check(got, want, F)
    one, chroma_only = dec[5]["one"], dec[5]["chroma_only"]
    assert got["dering_levels"][0][chroma_only] == 0 and got["dering_levels"][0][one] == 3
    assert got["dering_levels"].any()
    eng.close()


@pytest.mark.gpu
def test_finish_repeated_after_one_step():
    """Decisions A, then B, then A again after one step: each matches its oracle and the third run repeats the first
    byte for byte (graph replay)."""
    from daala_b200.frame import Geometry
    geom = Geometry(200, 130)
    F, q0 = 2, 45
    eng = _engine(geom, F, q0)
    planes, pred, bsize = _frames(geom, F, seed=21)
    out, d, md = _step(eng, planes, pred, bsize)
    a, b = _decisions(out, geom, F, seed=1), _decisions(out, geom, F, seed=2)
    first = _copy(eng.finish(*a[:5]))
    _check(first, _want(geom, F, out, d, md, bsize, q0, a), F)
    second = _copy(eng.finish(*b[:5]))
    _check(second, _want(geom, F, out, d, md, bsize, q0, b), F)
    assert any(not np.array_equal(first[k], second[k]) for k in first)
    third = _copy(eng.finish(*a[:5]))
    for k in first:
        assert np.array_equal(first[k], third[k]), k
    eng.close()


@pytest.mark.gpu
def test_dc_resid_is_the_unquantised_dc_residual():
    from daala_b200.frame import Geometry
    from tests import inter_oracle
    geom = Geometry(328, 200)
    F, q0 = 2, 45
    eng = _engine(geom, F, q0)
    planes, pred, bsize = _frames(geom, F, seed=4)
    out, _, _ = _step(eng, planes, pred, bsize)
    ref = oracle_lib.load_ref()
    lib, prefix = (ref, "ref") if ref is not None else (oracle_lib.load_port(), "port")
    for f in range(F):
        want = inter_oracle.inter_chain(lib, prefix, [p[f] for p in planes], [p[f] for p in pred], geom, bsize[f], q0, Q4)
        for p in range(3):
            kind = "luma" if p == 0 else "chroma"
            d = frame_oracle.forward_plane(lib, prefix, planes[p][f], geom, p, bsize[f], 0)
            b = out[kind + "_blocks"]
            sel = (b["pli"] == p) & (b["frame"] == f)
            y, x = b["y0"][sel].astype(np.int64), b["x0"][sel].astype(np.int64)
            assert np.array_equal(out[kind + "_dc_resid"][sel], d[y, x] - want[p]["md"][y, x]), (f, p)
    eng.close()


@pytest.mark.gpu
def test_finish_refusals():
    from daala_b200 import _native, engine
    from daala_b200.frame import Geometry
    geom = Geometry(200, 130)
    F, q0 = 1, 45
    with pytest.raises(RuntimeError, match="inter_finish"):
        engine.KeyframeEngine(geom, nframes=F, q0=q0, pvq_qm_q4=Q4, inter_finish=1)
    planes, pred, bsize = _frames(geom, F, seed=8)
    eng = _engine(geom, F, q0)
    L = eng.L
    dummy = [np.zeros(1 << 16, np.uint8), np.zeros(1 << 16, np.int32)]
    fio = engine.FinishIO()
    fio.luma_skip = fio.chroma_skip = dummy[0].ctypes.data
    fio.luma_dc = fio.chroma_dc = dummy[1].ctypes.data
    assert L.daala_b200_kf_finish(eng.kf, ctypes.byref(fio)) != 0
    assert b"no step" in L.daala_b200_kf_error(eng.kf)
    out, _, _ = _step(eng, planes, pred, bsize)
    before = eng.counts().copy()
    nl, nc = len(out["luma_dc"]), len(out["chroma_dc"])
    good = (np.zeros(nl, np.uint8), out["luma_dc"], np.zeros(nc, np.uint8), out["chroma_dc"])
    ref = _copy(eng.finish(*good))
    for field in ("luma_skip", "chroma_skip", "luma_dc", "chroma_dc"):
        eng.prepare_finish(*good)
        io = engine.FinishIO.from_buffer_copy(eng._fio)
        setattr(io, field, None)
        assert L.daala_b200_kf_finish(eng.kf, ctypes.byref(io)) != 0
        assert b"required" in L.daala_b200_kf_error(eng.kf)
    bad_skip = good[0].copy()
    bad_skip[-1] = 2
    bad_dc = good[3].copy()
    dq_max = max((q0 * int(Q4[p][bs * (bs + 1)])) >> 4 for p in range(3) for bs in range(5))
    bad_dc[0] = (1 << 30) // dq_max + 1
    levels = np.zeros((F, geom.nvsb, geom.nhsb), np.uint8)
    levels[0, -1, -1] = 6
    for args, word in (((bad_skip,) + good[1:], b"skip value"), (good[:3] + (bad_dc,), b"|dc|"),
                       (good + (levels,), b"level")):
        eng.prepare_finish(*args)
        with pytest.raises(_native.CudaError):
            eng.finish_submit()
        assert word in L.daala_b200_kf_error(eng.kf)
    # the boundary itself is accepted
    ok_dc = good[3].copy()
    ok_dc[0] = -((1 << 30) // dq_max)
    eng.finish(*good[:3], ok_dc)
    assert np.array_equal(eng.counts(), before)
    # nothing a refusal left behind changes the next run
    again = _copy(eng.finish(*good))
    for k in ref:
        assert np.array_equal(ref[k], again[k]), k
    eng.close()
    kf = engine.KeyframeEngine(geom, nframes=F, q0=q0, pvq_qm_q4=Q4, inter=1)
    kf.encode(planes, bsize, pred=pred)
    assert L.daala_b200_kf_finish(kf.kf, ctypes.byref(fio)) != 0
    assert b"inter_finish" in L.daala_b200_kf_error(kf.kf)
    kf.close()


@pytest.mark.gpu
def test_inter_finish_off_is_the_inter_engine():
    """inter_finish changes nothing of the step: same launch count, same outputs, with and without the pass."""
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    geom = Geometry(328, 200)
    F = 2
    planes, pred, bsize = _frames(geom, F, seed=13)
    plain = engine.KeyframeEngine(geom, nframes=F, q0=45, pvq_qm_q4=Q4, inter=1)
    off = engine.KeyframeEngine(geom, nframes=F, q0=45, pvq_qm_q4=Q4, inter=1, inter_finish=0)
    on = _engine(geom, F, 45)
    assert plain.launches_per_step() == off.launches_per_step() == on.launches_per_step()
    assert plain.buf.bytes_allocated == off.buf.bytes_allocated < on.buf.bytes_allocated
    want = _copy(plain.encode(planes, bsize, pred=pred))
    for eng in (off, on):
        got = _copy(eng.encode(planes, bsize, pred=pred))
        for k in want:
            if k == "luma_res" or k == "chroma_res":
                continue   # records past a block's last band are not written
            assert np.array_equal(got[k], want[k], equal_nan=k.endswith("skip_diff")), k
        assert ("luma_dc_resid" in got) == (eng is on)
    for e in (plain, off, on):
        e.close()


# ---- no GPU ---------------------------------------------------------------------------------------------------------

def test_finish_driver_port_matches_reference():
    """The new frame driver, plain-C port against the reference build, on seeded coefficient planes and skip maps
    (the reference's od_dering and filters against the port's)."""
    from daala_b200 import synth
    from daala_b200.frame import Geometry
    ref = inter_finish_oracle.load_ref()
    if ref is None:
        pytest.skip("oracle/_ref/libdaala_ref_inter_finish.so not built (needs the reference sources)")
    port = oracle_lib.load_port()
    for w, h, seed in ((200, 130, 1), (328, 200, 2)):
        geom = Geometry(w, h)
        rng = np.random.default_rng(seed)
        planes = synth.pad_planes(synth.frame(w, h, f=3, seed=seed)[0], geom)
        bsize = synth.block_size_map(geom, "mixed", seed=seed)
        dq = [frame_oracle.forward_plane(port, "port", planes[p], geom, p, bsize, 0) for p in range(3)]
        bskip = []
        for p in range(3):
            m = np.zeros((geom.plane_shape(p)[0] // 4, geom.nhsb * 16), np.uint8)
            w4 = geom.plane_shape(p)[1] // 4
            m[:, :w4] = rng.random((m.shape[0], w4)) < 0.6
            bskip.append(m)
        bskip[0][:16, :16] = 1                  # superblock (0, 0): all luma skipped
        bskip[0][16:32, :16] = 1
        bskip[0][20, 5] = 0                     # superblock (1, 0): one coded 4x4 luma unit
        levels = rng.integers(1, 6, (geom.nvsb, geom.nhsb)).astype(np.uint8)
        r_rec, r_lv = inter_finish_oracle.finish(ref, "ref", dq, geom, bsize, 45, levels, bskip)
        p_rec, p_lv = inter_finish_oracle.finish(port, "port", dq, geom, bsize, 45, levels, bskip)
        assert np.array_equal(r_lv, p_lv) and r_lv[0, 0] == 0 and r_lv[1, 0] == levels[1, 0]
        for p in range(3):
            assert np.array_equal(r_rec[p], p_rec[p]), (w, p)
        # deringing did something, and the skip map matters to it
        plain = [frame_oracle.inverse_plane(port, "port", dq[p], geom, p, bsize, 0) for p in range(3)]
        assert any(not np.array_equal(r_rec[p], plain[p]) for p in range(3))
        no_skip = [np.zeros_like(b) for b in bskip]
        n_rec, _ = inter_finish_oracle.finish(ref, "ref", dq, geom, bsize, 45, levels, no_skip)
        assert any(not np.array_equal(r_rec[p], n_rec[p]) for p in range(3))


LAYOUT = r"""
#include <stddef.h>
#include <stdio.h>
#include "daala_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(daala_b200_kf_finish_io),
         offsetof(daala_b200_kf_finish_io, chroma_dc), offsetof(daala_b200_kf_finish_io, dering_level),
         offsetof(daala_b200_kf_finish_io, pixels_out), offsetof(daala_b200_kf_finish_io, bskip_out),
         offsetof(daala_b200_kf_finish_io, dering_level_out), sizeof(daala_b200_kf_config),
         offsetof(daala_b200_kf_config, inter_finish), sizeof(daala_b200_kf_io), offsetof(daala_b200_kf_io, chroma_dc_resid));
  return 0;
}
"""


def test_finish_structs_match_the_header(tmp_path):
    from daala_b200 import engine
    (tmp_path / "layout.c").write_text(LAYOUT)
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(tmp_path / "layout.c"), "-o", exe], check=True)
    got = [int(v) for v in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()]
    F = engine.FinishIO
    assert got == [ctypes.sizeof(F), F.chroma_dc.offset, F.dering_level.offset, F.pixels_out.offset, F.bskip_out.offset,
                   F.dering_level_out.offset, ctypes.sizeof(engine.Config), engine.Config.inter_finish.offset,
                   ctypes.sizeof(engine.IO), engine.IO.chroma_dc_resid.offset]
