"""Reference pictures kept on the device (config.inter_mc with inter_finish; csrc/kf_engine.cu): the finishing pass
stores its reconstruction into the engine's reference-picture pool (daala_b200_kf_finish_io.ref_slot_out,
k_fin_pool_store), a step predicts from the pool as it stands (daala_b200_kf_io.ref_resident) and
daala_b200_kf_pool_load seeds a slot from host or device memory.  A closed loop of P frames against the oracle's own
running pictures, the resident loop against the host round trip, the slot semantics and the refusals.  The first
test needs no GPU."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from tests import inter_mc_oracle
from tests.test_gpu_engine_inter_finish import Q4, _check, _copy, _decisions, _want
from tests.test_gpu_engine_inter_mc import _batch, _grids, _pack, _pool, _same_outputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Q0 = 45


def _engine(geom, F, inter_finish=1, **kw):
    from daala_b200 import engine
    return engine.KeyframeEngine(geom, nframes=F, q0=Q0, pvq_qm_q4=Q4, inter=1, inter_mc=1, inter_finish=inter_finish,
                                 coded_quantizer=Q0, **kw)


def _pools(eng):
    return [eng.pool_plane(p) for p in range(3)]


def _same_pools(a, b):
    return all(np.array_equal(a[p], b[p]) for p in range(3))


def _step_inputs(geom, F, k, seed):
    """Source frames, block sizes and MV grids of step k."""
    planes, bsize = _batch(geom, F, seed=seed + 7 * k)
    return planes, bsize, _grids(geom, F, seed=seed + 100 * k)


def _slots(F, k):
    """GOLD = slot f, PREV = slot F + f; the first step predicts from the keyframe alone."""
    return np.array([[f, f if k == 0 else F + f] for f in range(F)], np.int32)


LAYOUT = r"""
#include <stddef.h>
#include <stdio.h>
#include "daala_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu\n", sizeof(daala_b200_kf_io), offsetof(daala_b200_kf_io, ref_resident),
         sizeof(daala_b200_kf_finish_io), offsetof(daala_b200_kf_finish_io, ref_slot_out));
  return 0;
}
"""


def test_pool_structs_match_the_header(tmp_path):
    from daala_b200 import engine
    (tmp_path / "layout.c").write_text(LAYOUT)
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(tmp_path / "layout.c"), "-o", exe], check=True)
    got = [int(v) for v in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [ctypes.sizeof(engine.IO), engine.IO.ref_resident.offset, ctypes.sizeof(engine.FinishIO),
                   engine.FinishIO.ref_slot_out.offset]


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,F,K", [(328, 200, 2, 4), (1920, 1080, 1, 2)])
def test_closed_loop_matches_oracle(w, h, F, K):
    """F sequences of a keyframe and K P frames, every picture kept in the pool.  Each step's prediction is the
    oracle's on the oracle's own running pictures, each finish is the oracle's finishing pass, and the oracle's
    reconstruction is its next PREV picture; after the last step the pool holds the oracle's pictures."""
    from daala_b200 import engine, synth
    from daala_b200.frame import Geometry
    lib = inter_mc_oracle.load()
    if lib is None:
        pytest.skip("oracle/_ref/libdaala_ref_inter_mc.so not built (needs the reference sources)")
    geom = Geometry(w, h)
    # the GOP's keyframes, from the keyframe engine
    key = engine.KeyframeEngine(geom, nframes=F, q0=Q0, pvq_qm_q4=Q4)
    kpics = [synth.pad_planes(synth.frame(w, h, f=1, seed=w + f)[0], geom) for f in range(F)]
    kplanes = [np.stack([pic[p] for pic in kpics]) for p in range(3)]
    kout = _copy(key.encode(kplanes, np.stack([synth.block_size_map(geom, "mixed", seed=h + f) for f in range(F)])))
    gold = [[kout["recon%d" % p][f] for p in range(3)] for f in range(F)]
    eng = _engine(geom, F, mc_refs=2 * F)
    for f in range(F):
        if f == 0:   # device to device, from the keyframe engine's reconstruction
            eng.pool_load(f, [key.buf.pixels_out[p] + f * int(np.prod(geom.plane_shape(p))) for p in range(3)])
        else:        # from host memory
            eng.pool_load(f, gold[f])
    prev = [list(g) for g in gold]
    for k in range(K):
        planes, bsize, grids = _step_inputs(geom, F, k, seed=w + h)
        slot = _slots(F, k)
        out = _copy(eng.encode(planes, bsize, ref_slot=slot, mv_grid=_pack(grids), resident=True))
        for f in range(F):
            want = inter_mc_oracle.predict(lib, geom, gold[f], prev[f], *grids[f], same=k == 0)
            for p in range(3):
                assert np.array_equal(out["pred%d" % p][f], want[p]), ("prediction", k, f, p)
        d = [eng.coeff_plane(p) for p in range(3)]
        md = [eng.pred_coeff_plane(p) for p in range(3)]
        dec = _decisions(out, geom, F, seed=10 * k + w)
        got = _copy(eng.finish(*dec[:5], ref_slot_out=np.arange(F, 2 * F, dtype=np.int32)))
        want = _want(geom, F, out, d, md, bsize, Q0, dec)
        _check(got, want, F)
        prev = [list(want[f][0]) for f in range(F)]
    pool = _pools(eng)
    for f in range(F):
        for p in range(3):
            assert np.array_equal(pool[p][f], gold[f][p]), ("GOLD", f, p)
            assert np.array_equal(pool[p][F + f], prev[f][p]), ("PREV", f, p)
    key.close()
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("inter_finish", [1, 2])
def test_resident_loop_equals_round_trip(inter_finish):
    """Two engines, identical inputs: one uploads the pictures the previous finish returned, the other keeps them in
    its pool.  Every output of every step and every finish is equal, and so is the pool."""
    from daala_b200.frame import Geometry
    geom = Geometry(200, 130)
    F, K = 2, 3
    gold = _pool(geom, F, seed=17)
    trip, res = _engine(geom, F, inter_finish, mc_refs=2 * F), _engine(geom, F, inter_finish, mc_refs=2 * F)
    for f in range(F):
        res.pool_load(f, [gold[p][f] for p in range(3)])
    refs = [np.concatenate([gold[p], gold[p]]) for p in range(3)]
    for k in range(K):
        planes, bsize, grids = _step_inputs(geom, F, k, seed=3)
        slot = _slots(F, k)
        a = _copy(trip.encode(planes, bsize, refs=refs, ref_slot=slot, mv_grid=_pack(grids)))
        b = _copy(res.encode(planes, bsize, ref_slot=slot, mv_grid=_pack(grids), resident=True))
        _same_outputs(geom, F, b, a, ("pred0", "pred1", "pred2", "luma_dc_resid", "chroma_dc_resid"))
        assert res.h2d_bytes == trip.h2d_bytes - sum(r.nbytes for r in refs)
        dec = _decisions(a, geom, F, seed=k)
        levels = dec[4] if inter_finish == 1 else None
        fa = _copy(trip.finish(*dec[:4], levels))
        fb = _copy(res.finish(*dec[:4], levels, ref_slot_out=np.arange(F, 2 * F, dtype=np.int32)))
        for key in fa:
            assert np.array_equal(fa[key], fb[key]), (k, key)
        assert res.finish_h2d_bytes == trip.finish_h2d_bytes + 4 * F
        refs = [np.concatenate([gold[p], fa["recon%d" % p]]) for p in range(3)]
        pool = _pools(res)
        for p in range(3):
            assert np.array_equal(pool[p], refs[p]), (k, p)
    trip.close()
    res.close()


@pytest.mark.gpu
def test_slot_semantics():
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    geom = Geometry(200, 130)
    F = 2
    eng = _engine(geom, F, mc_refs=5)
    pics = _pool(geom, 5, seed=23)
    for s in range(4):
        eng.pool_load(s, [pics[p][s] for p in range(3)])
    planes, bsize, grids = _step_inputs(geom, F, 1, seed=40)
    slot = np.array([[0, 2], [1, 3]], np.int32)
    out = _copy(eng.encode(planes, bsize, ref_slot=slot, mv_grid=_pack(grids), resident=True))
    a, b = _decisions(out, geom, F, seed=1), _decisions(out, geom, F, seed=2)
    before = _pools(eng)
    # nothing stored: NULL, or every entry -1
    ra = _copy(eng.finish(*a[:5]))
    assert _same_pools(_pools(eng), before)
    assert all(np.array_equal(ra[k], v) for k, v in _copy(eng.finish(*a[:5], ref_slot_out=[-1, -1])).items())
    assert _same_pools(_pools(eng), before)
    # decisions A, then B on one step: the last finish wins
    eng.finish(*a[:5], ref_slot_out=[4, -1])
    rb = _copy(eng.finish(*b[:5], ref_slot_out=[4, -1]))
    assert any(not np.array_equal(ra["recon%d" % p], rb["recon%d" % p]) for p in range(3))
    pool = _pools(eng)
    for p in range(3):
        assert np.array_equal(pool[p][4], rb["recon%d" % p][0]), p
        assert np.array_equal(pool[p][:4], before[p][:4]), p
    # each frame's PREV slot rewritten with the frame itself; a repeated finish reads md, not the pool
    got = _copy(eng.finish(*a[:5], ref_slot_out=[2, 3]))
    again = _copy(eng.finish(*a[:5], ref_slot_out=[2, 3]))
    pool = _pools(eng)
    for p in range(3):
        assert np.array_equal(got["recon%d" % p], ra["recon%d" % p]) and np.array_equal(again["recon%d" % p], ra["recon%d" % p])
        assert np.array_equal(pool[p][2:4], ra["recon%d" % p]), p
        assert np.array_equal(pool[p][:2], before[p][:2]), p
    # the next resident step reads the rewritten slots: as an upload of the same pictures
    planes2, bsize2, grids2 = _step_inputs(geom, F, 2, seed=40)
    nxt = _copy(eng.encode(planes2, bsize2, ref_slot=slot, mv_grid=_pack(grids2), resident=True))
    fresh = _engine(geom, F, mc_refs=5)
    want = _copy(fresh.encode(planes2, bsize2, refs=pool, ref_slot=slot, mv_grid=_pack(grids2)))
    _same_outputs(geom, F, nxt, want, ("pred0", "pred1", "pred2"))
    # after resident steps a host-upload submit works as before and overwrites slots [0, nrefs) only
    up = [pics[p][[3, 2]] for p in range(3)]
    again = _copy(eng.encode(planes2, bsize2, refs=up, ref_slot=np.array([[0, 1], [1, 1]], np.int32),
                             mv_grid=_pack(grids2)))
    want = _copy(fresh.encode(planes2, bsize2, refs=up, ref_slot=np.array([[0, 1], [1, 1]], np.int32),
                              mv_grid=_pack(grids2)))
    _same_outputs(geom, F, again, want, ("pred0", "pred1", "pred2"))
    after = _pools(eng)
    for p in range(3):
        assert np.array_equal(after[p][:2], up[p]) and np.array_equal(after[p][2:], pool[p][2:]), p
    # a pool_load enqueued after a submit does not change that submit's prediction
    eng.stage_inputs(planes, bsize)
    eng.stage_mc(None, slot, _pack(grids), resident=True)
    eng.prepare_io()
    eng.submit()
    eng.pool_load(2, [pics[p][4] for p in range(3)])
    late = _copy(eng.wait())
    want = _copy(fresh.encode(planes, bsize, refs=after, ref_slot=slot, mv_grid=_pack(grids)))
    _same_outputs(geom, F, late, want, ("pred0", "pred1", "pred2"))
    assert np.array_equal(eng.pool_plane(0)[2], pics[0][4])
    assert int(late["counts"][engine.CNT["error"]]) == 0
    fresh.close()
    eng.close()


@pytest.mark.gpu
def test_refusals_before_any_copy():
    from daala_b200 import _native, engine
    from daala_b200.frame import Geometry
    geom = Geometry(200, 130)
    F, R = 2, 4
    pics = _pool(geom, R, seed=5)
    # pool_load
    fin_only = engine.KeyframeEngine(geom, nframes=F, q0=Q0, pvq_qm_q4=Q4, inter=1, inter_finish=1)
    with pytest.raises(_native.CudaError, match="inter_mc"):
        fin_only.pool_load(0, [pics[p][0] for p in range(3)])
    eng = _engine(geom, F, mc_refs=R)
    eng.pool_load(0, [pics[p][0] for p in range(3)])
    eng.pool_load(1, [pics[p][1] for p in range(3)])
    planes, bsize, grids = _step_inputs(geom, F, 0, seed=9)
    slot = np.array([[0, 1], [1, 1]], np.int32)
    out = _copy(eng.encode(planes, bsize, ref_slot=slot, mv_grid=_pack(grids), resident=True))
    pool = _pools(eng)
    staged = [eng.download(eng.buf.pixels[p], (F,) + geom.plane_shape(p), np.uint8) for p in range(3)]
    grid_before = eng.download(eng.buf.mv_grid, (F * (geom.nvsb * 8 + 1) * (geom.nhsb * 8 + 1) * 12,), np.uint8)
    for s, planes_, word in ((-1, [pics[p][2] for p in range(3)], "slot"), (R, [pics[p][2] for p in range(3)], "slot"),
                             (2, [pics[0][2], None, pics[2][2]], "planes")):
        with pytest.raises(_native.CudaError, match=word):
            eng.pool_load(s, planes_)
    # ref_slot_out
    nl, nc = len(out["luma_dc"]), len(out["chroma_dc"])
    good = (np.zeros(nl, np.uint8), out["luma_dc"], np.zeros(nc, np.uint8), out["chroma_dc"])
    ref = _copy(eng.finish(*good))
    for bad, word in (([-2, 3], "outside [-1, mc_refs)"), ([0, R], "outside [-1, mc_refs)"), ([3, 3], "same")):
        eng.prepare_finish(*good, ref_slot_out=np.array(bad, np.int32))
        with pytest.raises(_native.CudaError):
            eng.finish_submit()
        assert word in eng.L.daala_b200_kf_error(eng.kf).decode(), bad
    assert _same_pools(_pools(eng), pool)
    again = _copy(eng.finish(*good))
    for k in ref:
        assert np.array_equal(ref[k], again[k]), k
    # resident submits: the slot of the failed load still holds nothing
    planes2, bsize2, grids2 = _step_inputs(geom, F, 1, seed=9)
    eng.stage_inputs(planes2, bsize2)
    eng.stage_mc(None, slot, _pack(grids2), resident=True)
    eng.prepare_io()
    io = eng._io
    slots = eng._arr("slot", (F, 2), np.int32)
    dummy = eng._arr("dummy", (R,) + geom.plane_shape(0), np.uint8)

    def field(name, value):
        old = getattr(io, name)
        setattr(io, name, value)
        return lambda: setattr(io, name, old)

    def ref_plane(value):
        io.ref_pixels[1] = value
        return lambda: io.ref_pixels.__setitem__(1, None)

    def slot_value(v):
        old = int(slots[1, 0])
        slots[1, 0] = v
        return lambda: slots.__setitem__((1, 0), old)

    cases = [("ref_pixels must be NULL", lambda: ref_plane(dummy.ctypes.data)), ("nrefs must be 0", lambda: field("nrefs", 2)),
             ("outside [0, mc_refs)", lambda: slot_value(R)), ("outside [0, mc_refs)", lambda: slot_value(-1)),
             ("holds no picture", lambda: slot_value(2)), ("ref_resident is 0 or 1", lambda: field("ref_resident", 2))]
    for what, breaker in cases:
        undo = breaker()
        rc = eng.L.daala_b200_kf_submit(eng.kf, ctypes.byref(io))
        msg = eng.L.daala_b200_kf_error(eng.kf).decode()
        undo()
        assert rc != 0 and what in msg, (what, rc, msg)
    eng.wait()
    for p in range(3):
        assert np.array_equal(eng.download(eng.buf.pixels[p], (F,) + geom.plane_shape(p), np.uint8), staged[p])
    assert np.array_equal(eng.download(eng.buf.mv_grid, grid_before.shape, np.uint8), grid_before)
    assert _same_pools(_pools(eng), pool)
    fin_only.encode(planes, bsize, pred=[pics[p][:F] for p in range(3)])
    fin_only.prepare_finish(*[np.zeros(len(fin_only._out["luma_dc"]), np.uint8), fin_only._out["luma_dc"],
                              np.zeros(len(fin_only._out["chroma_dc"]), np.uint8), fin_only._out["chroma_dc"]],
                            ref_slot_out=np.array([0, 1], np.int32))
    with pytest.raises(_native.CudaError):
        fin_only.finish_submit()
    assert b"ref_slot_out needs an engine with inter_mc" in fin_only.L.daala_b200_kf_error(fin_only.kf)
    fin_only.close()
    eng.close()
