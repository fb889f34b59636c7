"""The engine's prediction of P frames from MV grids (config.inter_mc; k_mc_leaves / k_mc_obmc in csrc/mc_kernels.cu)
through the host-buffer C ABI: the prediction against the reference's od_state_mc_predict with two pictures
(inter_mc_oracle.predict), real P frames of the reference encoder against inter_oracle.inter_chain, and the
residual against the host-prediction engine (inter = 1) fed the same prediction."""
import ctypes

import numpy as np
import pytest

from tests import inter_mc_oracle, inter_oracle

pytestmark = [pytest.mark.gpu]

Q4 = np.full((3, 30), 20, np.uint8)
OUTPUTS = ("recon0", "recon1", "recon2", "luma_blocks", "chroma_blocks", "luma_y16", "chroma_y16", "luma_skip_diff",
           "chroma_skip_diff", "chroma_flip", "luma_dc", "chroma_dc")


def _same_outputs(geom, F, got, want, extra=()):
    """Every output array equal; the band records compared where a block has bands (the records past a block's
    last band are not written)."""
    from daala_b200 import engine
    for k in OUTPUTS + tuple(extra):
        assert np.array_equal(got[k], np.asarray(want[k]), equal_nan=k.endswith("skip_diff")), k
    for pli in range(3):
        kind = "luma" if pli == 0 else "chroma"
        for f in range(F):
            assert np.array_equal(engine.band_records(got[kind + "_blocks"], got[kind + "_res"], geom, pli, f),
                                  engine.band_records(np.asarray(want[kind + "_blocks"]), np.asarray(want[kind + "_res"]),
                                                      geom, pli, f)), ("band records", pli, f)


def _ref():
    lib = inter_mc_oracle.load()   # the reference build with the prediction hooks
    if lib is None:
        pytest.skip("oracle/_ref/libdaala_ref_inter_mc.so not built (needs the reference sources)")
    return lib


def _engine(geom, F, q0=45, **kw):
    from daala_b200 import engine
    return engine.KeyframeEngine(geom, nframes=F, q0=q0, pvq_qm_q4=Q4, inter=1, inter_mc=1, **kw)


def _pool(geom, n, seed):
    """n distinct reference pictures (smooth content + noise), per plane [n, h, w]."""
    from daala_b200 import synth
    pics = [synth.pad_planes(synth.frame(geom.pic_w, geom.pic_h, f=3 * k + 1, seed=seed + k)[0], geom) for k in range(n)]
    return [np.stack([p[pl] for p in pics]) for pl in range(3)]


def _batch(geom, F, seed, mode="mixed"):
    from daala_b200 import synth
    src = [synth.pad_planes(synth.frame(geom.pic_w, geom.pic_h, f=f + 2, seed=seed + 50 + f)[0], geom) for f in range(F)]
    planes = [np.stack([s[p] for s in src]) for p in range(3)]
    bsize = np.stack([synth.block_size_map(geom, mode, seed=seed + f) for f in range(F)])
    return planes, bsize


def _grids(geom, F, seed, **kw):
    from daala_b200 import synth
    return [synth.mv_grid(geom, seed=seed + f, **kw) for f in range(F)]


def _pack(grids):
    from daala_b200 import mvgrid
    return mvgrid.pack(*(np.stack([g[i] for g in grids]) for i in range(3)))


def _hook(lib, geom, refs, slot, grid):
    gold, prev = [refs[p][slot[0]] for p in range(3)], [refs[p][slot[1]] for p in range(3)]
    return inter_mc_oracle.predict(lib, geom, gold, prev, *grid, same=slot[0] == slot[1])


def _run(eng, planes, bsize, refs, slot, grids):
    out = eng.encode(planes, bsize, refs=refs, ref_slot=np.asarray(slot, np.int32), mv_grid=_pack(grids))
    return {k: np.array(v) for k, v in out.items()}


def _beyond_model(geom, valid, mv):
    """What k_mc_leaves counts as corner windows past the edge extension, from mvgrid's host leaves."""
    from daala_b200 import mvgrid
    lv = mvgrid.leaves(valid.astype(bool))
    n = 0
    for p in range(3):
        dec = 1 if p else 0
        b = mvgrid.blocks_for(*lv, mv, dec)
        pad, (ph, pw) = 64 >> dec, geom.plane_shape(p)
        size = (1 << b["log_xblk"].astype(np.int64))[:, None]
        x = b["x0"].astype(np.int64)[:, None] + (b["mvx"].astype(np.int64) >> 3)
        y = b["y0"].astype(np.int64)[:, None] + (b["mvy"].astype(np.int64) >> 3)
        n += int(((x - 2 < -pad) | (x + size + 2 > pw - 1 + pad) | (y - 2 < -pad) | (y + size + 2 > ph - 1 + pad)).sum())
    return n


@pytest.mark.parametrize("w,h,shared", [(200, 130, False), (328, 200, False), (328, 200, True), (1920, 1080, False)])
def test_prediction_matches_two_reference_hook(w, h, shared):
    """Random grids with every split level and per-vertex GOLD / PREV, F = 3: distinct slots, or GOLD = PREV."""
    from daala_b200 import engine, mvgrid
    from daala_b200.frame import Geometry
    lib = _ref()
    geom = Geometry(w, h)
    F = 3
    refs = _pool(geom, 4, seed=w + h)
    slot = [[2, 2], [1, 1], [0, 0]] if shared else [[0, 1], [2, 1], [3, 0]]
    grids = _grids(geom, F, seed=w)
    levels = np.bincount(np.concatenate([mvgrid.leaves(g[0].astype(bool))[2] for g in grids]), minlength=4)
    assert (levels > 0).all(), levels   # 8x8 (4x4 chroma) .. 64x64 leaves
    planes, bsize = _batch(geom, F, seed=h)
    eng = _engine(geom, F)
    out = _run(eng, planes, bsize, refs, slot, grids)
    assert int(out["counts"][engine.CNT["mc_bad_ref"]]) == 0 and int(out["counts"][engine.CNT["mc_beyond"]]) == 0
    for f in range(F):
        want = _hook(lib, geom, refs, slot[f], grids[f])
        for p in range(3):
            assert np.array_equal(out["pred%d" % p][f], want[p]), ("prediction", f, p)
    # the residual is the host-prediction engine's on the same prediction, array for array; the prediction costs
    # two launches
    host = engine.KeyframeEngine(geom, nframes=F, q0=45, pvq_qm_q4=Q4, inter=1)
    assert eng.launches_per_step() == host.launches_per_step() + 2
    want = host.encode(planes, bsize, pred=[out["pred%d" % p] for p in range(3)])
    _same_outputs(geom, F, out, want)
    for p in range(3):
        assert np.array_equal(eng.coeff_plane(p), host.coeff_plane(p)), ("quantised plane", p)
        assert np.array_equal(eng.pred_coeff_plane(p), host.pred_coeff_plane(p)), ("md", p)
    host.close()
    eng.close()


@pytest.mark.parametrize("direction", ["left", "right", "up", "down"])
def test_vectors_at_the_edge_extension_limit(direction):
    """Per 1/8-pel phase one frame whose vertices all carry the longest vector that keeps every corner window
    (with the filter's apron) inside the reference's 64 / 32 pixels of edge extension in this direction."""
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    lib = _ref()
    geom = Geometry(200, 130)
    F = 8
    refs = _pool(geom, 2, seed=5)
    axis, sign = {"left": (0, -1), "right": (0, 1), "up": (1, -1), "down": (1, 1)}[direction]
    grids = []
    for ph in range(F):
        valid = _grids(geom, 1, seed=100 + ph)[0][0]
        ref = (np.arange(valid.size).reshape(valid.shape) + ph) % 2
        mv = np.zeros(valid.shape + (2,), np.int32)
        m = sign * (80 * 8) + ph
        while True:   # shorten the vector by whole pixels, same phase, until every window is inside
            mv[..., axis] = m
            if _beyond_model(geom, valid, mv) == 0:
                break
            m -= sign * 8
        mv[..., axis] = m + sign * 8
        assert _beyond_model(geom, valid, mv) > 0   # one pixel further is past the limit
        mv[..., axis] = m
        grids.append((valid, mv, ref.astype(np.uint8)))
    planes, bsize = _batch(geom, F, seed=8)
    eng = _engine(geom, F)
    slot = [[0, 1]] * F
    out = _run(eng, planes, bsize, refs, slot, grids)
    assert int(out["counts"][engine.CNT["mc_beyond"]]) == 0
    for f in range(F):
        want = _hook(lib, geom, refs, slot[f], grids[f])
        for p in range(3):
            assert np.array_equal(out["pred%d" % p][f], want[p]), ("prediction", f, p)
    eng.close()


def test_real_encoder_p_frames():
    """P frames 1-3 of the reference encoder (328x200, complexity 7): the engine, given the captured grids, GOLD /
    PREV pictures and block sizes, predicts what the encoder predicted and codes what inter_chain codes."""
    from daala_b200 import mvgrid
    from daala_b200.frame import Geometry
    from tests.test_gpu_engine_inter import _compare
    lib = _ref()
    geom = Geometry(328, 200)
    caps = inter_mc_oracle.capture_p_frames(lib, geom, 4)
    F = len(caps)
    refs = [np.stack([c[k][p] for c in caps for k in ("gold", "prev")]) for p in range(3)]
    slot = [[2 * f, 2 * f + (0 if c["same"] else 1)] for f, c in enumerate(caps)]
    assert caps[0]["same"] and not caps[2]["same"]   # from the third frame on GOLD is the keyframe, PREV is not
    grids = [(c["valid"], c["mv"], c["ref"]) for c in caps]
    planes = [np.stack([c["src"][p] for c in caps]) for p in range(3)]
    bsize = np.stack([c["bsize"] for c in caps])
    q0 = 45
    eng = _engine(geom, F, q0=q0)
    out = _run(eng, planes, bsize, refs, slot, grids)
    gold_corners = 0
    for f, c in enumerate(caps):
        for p in range(3):
            assert np.array_equal(out["pred%d" % p][f], c["pred"][p]), ("prediction", f, p)
        if not c["same"]:
            for gx, gy in mvgrid.corners(*mvgrid.leaves(c["valid"].astype(bool))):
                gold_corners += int((c["ref"][gy, gx] == 0).sum())
    print("leaf corners on GOLD in the frames with two pictures: %d" % gold_corners)
    coeffs = [eng.coeff_plane(p) for p in range(3)]
    md = [eng.pred_coeff_plane(p) for p in range(3)]
    frames = [(c["src"], c["pred"], c["bsize"]) for c in caps]
    _compare(out, coeffs, md, geom, frames, q0, Q4)
    eng.close()


def test_replay_and_batch_independence():
    """Two submits on one engine with different grids, pools and slot maps each equal a fresh engine; each frame
    of a batch equals the same frame alone."""
    from daala_b200.frame import Geometry
    geom = Geometry(200, 130)
    F = 3
    eng = _engine(geom, F, mc_refs=5)
    runs = []
    for r, (n, slot) in enumerate(((5, [[0, 1], [2, 3], [4, 4]]), (2, [[1, 0], [1, 1], [0, 1]]))):
        refs = _pool(geom, n, seed=31 * r)
        grids = _grids(geom, F, seed=200 + 10 * r)
        planes, bsize = _batch(geom, F, seed=60 + r)
        runs.append((refs, slot, grids, planes, bsize, _run(eng, planes, bsize, refs, slot, grids)))
    eng.close()
    for refs, slot, grids, planes, bsize, got in runs:
        fresh = _engine(geom, F)
        want = _run(fresh, planes, bsize, refs, slot, grids)
        fresh.close()
        _same_outputs(geom, F, got, want, ("pred0", "pred1", "pred2"))
    refs, slot, grids, planes, bsize, got = runs[0]
    for f in range(F):
        one = _engine(geom, 1, mc_refs=5)
        alone = _run(one, [a[f:f + 1] for a in planes], bsize[f:f + 1], refs, [slot[f]], [grids[f]])
        one.close()
        for p in range(3):
            assert np.array_equal(alone["pred%d" % p][0], got["pred%d" % p][f]), ("prediction", f, p)
            assert np.array_equal(alone["recon%d" % p][0], got["recon%d" % p][f]), ("recon", f, p)


def test_refusals_before_any_copy():
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    geom = Geometry(200, 130)
    for kw in (dict(inter=0, inter_mc=1), dict(inter=1, inter_mc=1, mc_refs=-1), dict(inter=1, inter_mc=2)):
        with pytest.raises(RuntimeError, match="daala_b200_kf_create: .*(inter_mc|mc_refs)"):
            engine.KeyframeEngine(geom, nframes=1, q0=45, pvq_qm_q4=Q4, **kw)
    F = 2
    eng = _engine(geom, F, mc_refs=3)
    refs = _pool(geom, 3, seed=1)
    grids = _grids(geom, F, seed=9)
    planes, bsize = _batch(geom, F, seed=4)
    _run(eng, planes, bsize, refs, [[0, 1], [2, 2]], grids)
    before = [eng.download(eng.buf.pixels[p], (F,) + geom.plane_shape(p), np.uint8) for p in range(3)]
    grid_before = eng.download(eng.buf.mv_grid, (F * (geom.nvsb * 8 + 1) * (geom.nhsb * 8 + 1) * 12,), np.uint8)
    # stage another batch, then break one field of the io record at a time
    planes2, bsize2 = _batch(geom, F, seed=5)
    eng.stage_inputs(planes2, bsize2)
    eng.stage_mc(_pool(geom, 3, seed=2), np.array([[0, 1], [1, 2]], np.int32), _pack(_grids(geom, F, seed=10)))
    eng.prepare_io()
    io = eng._io
    pred_dummy = eng._arr("dummy", (F,) + geom.plane_shape(0), np.uint8)
    slots = eng._arr("slot", (F, 2), np.int32)

    def field(name, value):
        old = getattr(io, name)
        setattr(io, name, value)
        return lambda: setattr(io, name, old)

    def plane(name, p, value):
        arr = getattr(io, name)
        old = arr[p]
        arr[p] = value
        return lambda: arr.__setitem__(p, old)

    def slot_value(v):
        old = int(slots[1, 0])
        slots[1, 0] = v
        return lambda: slots.__setitem__((1, 0), old)

    cases = [("mv_grid", lambda: field("mv_grid", None)), ("ref_pixels", lambda: plane("ref_pixels", 1, None)),
             ("ref_slot", lambda: field("ref_slot", None)),
             ("pred_pixels", lambda: plane("pred_pixels", 0, pred_dummy.ctypes.data)),
             ("nrefs", lambda: field("nrefs", 0)), ("nrefs", lambda: field("nrefs", 4)),
             ("ref_slot", lambda: slot_value(3)), ("ref_slot", lambda: slot_value(-1))]
    for what, breaker in cases:
        undo = breaker()
        rc = eng.L.daala_b200_kf_submit(eng.kf, ctypes.byref(io))
        msg = eng.L.daala_b200_kf_error(eng.kf).decode()
        undo()
        assert rc != 0 and what in msg, (what, rc, msg)
    eng.wait()
    for p in range(3):
        assert np.array_equal(eng.download(eng.buf.pixels[p], (F,) + geom.plane_shape(p), np.uint8), before[p])
    assert np.array_equal(eng.download(eng.buf.mv_grid, grid_before.shape, np.uint8), grid_before)
    eng.close()


@pytest.mark.parametrize("fault", ["ref", "vector"])
def test_diagnostics(fault):
    """A used vertex with ref 2, or a vector past the edge extension, in frame 1 of 3: its counter is set, encode
    raises, and frames 0 and 2 still equal the oracle."""
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    lib = _ref()
    geom = Geometry(200, 130)
    F = 3
    refs = _pool(geom, 2, seed=7)
    slot = [[0, 1]] * F
    grids = _grids(geom, F, seed=40)
    valid, mv, ref = (a.copy() for a in grids[1])
    if fault == "ref":
        ref[0, 0] = 2          # a corner of the first 64x64 MV block, used by its leaves
    else:
        mv[0, 0] = (-8 * 70, 0)
    grids[1] = (valid, mv, ref)
    planes, bsize = _batch(geom, F, seed=12)
    eng = _engine(geom, F)
    with pytest.raises(RuntimeError, match="MV grid outside"):
        _run(eng, planes, bsize, refs, slot, grids)
    eng.stage_inputs(planes, bsize)
    eng.stage_mc(refs, np.asarray(slot, np.int32), _pack(grids))
    eng.prepare_io()
    eng.submit()
    out = {k: np.array(v) for k, v in eng.wait().items()}
    key = "mc_bad_ref" if fault == "ref" else "mc_beyond"
    other = "mc_beyond" if fault == "ref" else "mc_bad_ref"
    assert int(out["counts"][engine.CNT[key]]) > 0 and int(out["counts"][engine.CNT[other]]) == 0
    if fault == "vector":
        assert int(out["counts"][engine.CNT[key]]) == _beyond_model(geom, valid, mv)
    coeffs = [eng.coeff_plane(p) for p in range(3)]
    for f in (0, 2):
        want_pred = _hook(lib, geom, refs, slot[f], grids[f])
        for p in range(3):
            assert np.array_equal(out["pred%d" % p][f], want_pred[p]), ("prediction", f, p)
        want = inter_oracle.inter_chain(lib, "ref", [a[f] for a in planes], want_pred, geom, bsize[f], 45, Q4)
        for p in range(3):
            assert np.array_equal(out["recon%d" % p][f], want[p]["recon"]), ("recon", f, p)
            assert np.array_equal(coeffs[p][f], want[p]["dq"]), ("quantised plane", f, p)
    eng.close()
