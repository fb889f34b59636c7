"""B frames in the engine (config.mc_next; k_mc_leaves<true> / k_mc_obmc<true> in csrc/mc_kernels.cu): the prediction
from GOLD / PREV / NEXT with the vertices' second vectors against the reference's od_state_mc_predict with three
pictures (bframe_oracle.predict3), real B frames of the reference encoder, equality with the P-frame engine on P-only
grids, the composition with the finishing pass, symbol stream and late skip, a resident I P B B P B B loop driven by
daala_b200/gop.py against the oracle, and the diagnostics and refusals."""
import ctypes

import numpy as np
import pytest

from tests import bframe_oracle
from tests.test_gpu_engine_inter_finish import _check, _copy, _decisions, _want
from tests.test_gpu_engine_inter_mc import OUTPUTS, Q4, _batch, _pool, _same_outputs

pytestmark = [pytest.mark.gpu]
Q0 = 45


def _ref():
    lib = bframe_oracle.load()
    if lib is None:
        pytest.skip("oracle/_ref/libdaala_ref_bframes.so not built (needs the reference sources)")
    return lib


def _engine(geom, F, mc_next=1, **kw):
    from daala_b200 import engine
    return engine.KeyframeEngine(geom, nframes=F, q0=Q0, pvq_qm_q4=Q4, inter=1, inter_mc=1, mc_next=mc_next, **kw)


def _bgrids(geom, F, seed, **kw):
    from daala_b200 import synth
    return [synth.mv_grid_b(geom, seed=seed + f, **kw) for f in range(F)]


def _pack(grids):
    """(MV_PT_DTYPE grid, mv1 grid) of (valid, mv, mv1, ref) grids."""
    from daala_b200 import mvgrid
    valid, mv, mv1, ref = (np.stack([g[i] for g in grids]) for i in range(4))
    return mvgrid.pack(valid, mv, ref), mv1.astype(np.int32)


def _run(eng, planes, bsize, refs, slot, grids, **kw):
    grid, mv1 = _pack(grids)
    out = eng.encode(planes, bsize, refs=refs, ref_slot=np.asarray(slot, np.int32), mv_grid=grid, mv1_grid=mv1, **kw)
    return {k: np.array(v) for k, v in out.items()}


def _hook(lib, geom, refs, slot, grid):
    """predict3 with the pictures of the pool slots `slot` (GOLD, PREV, NEXT); equal slots share one picture."""
    pics = {}
    g, p, n = (pics.setdefault(int(s), [refs[pl][s] for pl in range(3)]) for s in slot)
    return bframe_oracle.predict3(lib, geom, g, p, n, *grid)


def _beyond_model(geom, valid, mv, mv1, ref):
    """What k_mc_leaves counts as corner windows past the edge extension, with the vector each corner reads."""
    from daala_b200 import mvgrid
    lv = mvgrid.leaves(valid.astype(bool))
    n = 0
    for p in range(3):
        dec = 1 if p else 0
        b = mvgrid.blocks_for(*lv, mv, dec, ref=ref, mv1=mv1)
        pad, (ph, pw) = 64 >> dec, geom.plane_shape(p)
        size = (1 << b["log_xblk"].astype(np.int64))[:, None]
        x = b["x0"].astype(np.int64)[:, None] + (b["mvx"].astype(np.int64) >> 3)
        y = b["y0"].astype(np.int64)[:, None] + (b["mvy"].astype(np.int64) >> 3)
        n += int(((x - 2 < -pad) | (x + size + 2 > pw - 1 + pad) | (y - 2 < -pad) | (y + size + 2 > ph - 1 + pad)).sum())
    return n


@pytest.mark.parametrize("w,h,shared", [(200, 130, False), (200, 130, True), (328, 200, False), (328, 200, True),
                                        (1920, 1080, False)])
def test_prediction_matches_three_reference_hook(w, h, shared):
    """mv_grid_b grids (every split level, refs 0 / 1 / 2 per vertex, mv1 everywhere), F = 3: all slots distinct, or
    NEXT in PREV's slot.  The residual is the host-prediction engine's on the same prediction, array for array."""
    from daala_b200 import engine, mvgrid
    from daala_b200.frame import Geometry
    lib = _ref()
    geom = Geometry(w, h)
    F = 3
    refs = _pool(geom, 6, seed=w + h)
    slot = [[0, 1, 1], [2, 3, 3], [4, 5, 5]] if shared else [[0, 1, 2], [3, 4, 5], [5, 2, 0]]
    grids = _bgrids(geom, F, seed=w + 1)
    levels = np.bincount(np.concatenate([mvgrid.leaves(g[0].astype(bool))[2] for g in grids]), minlength=4)
    assert (levels > 0).all(), levels
    planes, bsize = _batch(geom, F, seed=h)
    eng = _engine(geom, F)
    out = _run(eng, planes, bsize, refs, slot, grids)
    assert int(out["counts"][engine.CNT["mc_bad_ref"]]) == 0 and int(out["counts"][engine.CNT["mc_beyond"]]) == 0
    for f in range(F):
        want = _hook(lib, geom, refs, slot[f], grids[f])
        for p in range(3):
            assert np.array_equal(out["pred%d" % p][f], want[p]), ("prediction", f, p)
    host = engine.KeyframeEngine(geom, nframes=F, q0=Q0, pvq_qm_q4=Q4, inter=1)
    pframe = _engine(geom, F, mc_next=0)
    assert eng.launches_per_step() == pframe.launches_per_step() == host.launches_per_step() + 2
    want = host.encode(planes, bsize, pred=[out["pred%d" % p] for p in range(3)])
    _same_outputs(geom, F, out, want)
    for p in range(3):
        assert np.array_equal(eng.coeff_plane(p), host.coeff_plane(p)), ("quantised plane", p)
        assert np.array_equal(eng.pred_coeff_plane(p), host.pred_coeff_plane(p)), ("md", p)
    for e in (host, pframe, eng):
        e.close()


def test_real_encoder_b_frames():
    """The coded frames after the keyframe of a 7-frame b_frames = 2 sequence (328x200, complexity 7): P3, B1, B2,
    P6 (stale mv1 on its PREV vertices), B4, B5 in one batch.  The engine predicts what the encoder predicted and codes
    what inter_chain codes."""
    from daala_b200.frame import Geometry
    from tests.test_gpu_engine_inter import _compare
    lib = _ref()
    geom = Geometry(328, 200)
    caps = [c for c in bframe_oracle.capture_b_frames(lib, geom, 7, 2) if c["type"] != 0]
    F = len(caps)
    assert [c["type"] for c in caps] == [1, 2, 2, 1, 2, 2]
    v = [c["valid"].astype(bool) for c in caps]
    assert any((c["ref"][m] == 2).any() and (c["ref"][m] == 1).any() for c, m in zip(caps, v) if c["type"] == 2)
    assert any(((c["mv1"] != 0).any(-1) & m & (c["ref"] != 2)).any() for c, m in zip(caps, v) if c["type"] == 1)
    refs = [np.stack([c[k][p] for c in caps for k in ("gold", "prev", "next")]) for p in range(3)]
    slot = [[3 * f, 3 * f + 1, 3 * f + 2] for f in range(F)]
    grids = [(c["valid"], c["mv"], c["mv1"], c["ref"]) for c in caps]
    planes = [np.stack([c["src"][p] for c in caps]) for p in range(3)]
    bsize = np.stack([c["bsize"] for c in caps])
    eng = _engine(geom, F)
    out = _run(eng, planes, bsize, refs, slot, grids)
    for f, c in enumerate(caps):
        for p in range(3):
            assert np.array_equal(out["pred%d" % p][f], c["pred"][p]), ("prediction", c["number"], p)
    coeffs = [eng.coeff_plane(p) for p in range(3)]
    md = [eng.pred_coeff_plane(p) for p in range(3)]
    _compare(out, coeffs, md, geom, [(c["src"], c["pred"], c["bsize"]) for c in caps], Q0, Q4)
    eng.close()


def test_same_results_as_the_p_frame_engine():
    """P-only grids (refs 0 / 1) with arbitrary mv1: every output of an mc_next engine equals the P-frame engine's;
    the extra device memory is the mv1 grid, the NEXT slot table and the larger default pool (3F pictures, not 2F)."""
    from daala_b200.frame import Geometry
    geom = Geometry(328, 200)
    F = 3
    refs = _pool(geom, 4, seed=3)
    slot = [[0, 1], [2, 1], [3, 3]]
    grids = _bgrids(geom, F, seed=70, p_next=0.0, p_gold=0.5)
    assert all(set(np.unique(g[3])) == {0, 1} for g in grids)
    planes, bsize = _batch(geom, F, seed=71)
    b = _engine(geom, F)
    p = _engine(geom, F, mc_next=0)
    got = _run(b, planes, bsize, refs, [s + [s[1]] for s in slot], grids)
    grid, _ = _pack(grids)
    want = {k: np.array(v) for k, v in p.encode(planes, bsize, refs=refs, ref_slot=np.asarray(slot, np.int32),
                                                 mv_grid=grid).items()}
    _same_outputs(geom, F, got, want, ("pred0", "pred1", "pred2", "counts"))
    nv, nh = geom.nvsb * 8 + 1, geom.nhsb * 8 + 1
    px = sum(int(np.prod(geom.plane_shape(q))) for q in range(3))
    assert b.buf.bytes_allocated - p.buf.bytes_allocated == F * nv * nh * 8 + 4 * F + F * px
    assert b.h2d_bytes - p.h2d_bytes == F * nv * nh * 8 + 4 * F
    assert b.buf.mc_refs == 3 * F and p.buf.mc_refs == 2 * F
    assert p.buf.ref_slot_next is None and p.buf.mv1_grid is None
    b.close()
    p.close()


def test_composition_with_finish_stream_and_late_skip():
    """inter_finish = 2, symbol_stream = 2 and late_skip = 1 on an mc_next engine: the step and a stream-order finish
    equal the host-prediction engine with the same options fed the same prediction."""
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    geom = Geometry(328, 200)
    F = 2
    opts = dict(inter_finish=2, symbol_stream=2, late_skip=1, coded_quantizer=Q0)
    refs = _pool(geom, 3, seed=11)
    slot = [[0, 1, 2], [0, 2, 1]]
    grids = _bgrids(geom, F, seed=12)
    planes, bsize = _batch(geom, F, seed=13)
    eng = _engine(geom, F, **opts)
    host = engine.KeyframeEngine(geom, nframes=F, q0=Q0, pvq_qm_q4=Q4, inter=1, **opts)
    got = _run(eng, planes, bsize, refs, slot, grids)
    want = _copy(host.encode(planes, bsize, pred=[got["pred%d" % p] for p in range(3)]))
    _same_outputs(geom, F, got, want, ("luma_dc_resid", "chroma_dc_resid", "luma_late_skip", "chroma_late_skip"))
    idx = got["sym_index"]
    assert np.array_equal(idx, want["sym_index"])
    nb, nbands, nbytes = (int(idx[:, c].sum()) for c in (1, 3, 5))
    for k, n in (("sym_blocks", nb), ("sym_bands", nbands), ("sym_pulses", nbytes), ("sym_dc", nb),
                 ("sym_late_skip", nb)):
        assert np.array_equal(got[k][:n], want[k][:n]), k
    rng = np.random.default_rng(5)
    skip = (rng.random(nb) < 0.3).astype(np.uint8)
    dc = got["sym_dc"]["qdc"][:nb].copy()
    fa = _copy(eng.finish_stream(skip, dc))
    fb = _copy(host.finish_stream(skip, dc))
    for k in fb:
        assert np.array_equal(fa[k], fb[k]), k
    eng.close()
    host.close()


def test_resident_b_frame_loop_matches_oracle():
    """Two sequences of I P B B P B B (b_frames = 2) in coding order from gop.coding_order: the keyframes from the
    keyframe engine into a P engine's pool (slots 4s .. 4s + 3 of sequence s are the reference's four buffers), each P
    frame resident in the P engine with its finish stored in its SELF buffer, each group's B frames as one batch of
    an mc_next engine whose pool is loaded device to device from the P engine's, B finishes storing nothing.  Every
    prediction equals predict3 on the oracle's running pictures, every finish the finishing oracle."""
    from daala_b200 import engine, gop, synth
    from daala_b200.frame import Geometry
    lib = _ref()
    geom = Geometry(328, 200)
    S = 2
    order = gop.coding_order(7, 2)
    assert [f.type for f in order] == [0, 1, 2, 2, 1, 2, 2]
    plane_bytes = [int(np.prod(geom.plane_shape(p))) for p in range(3)]
    # the keyframes
    key = engine.KeyframeEngine(geom, nframes=S, q0=Q0, pvq_qm_q4=Q4)
    src = {(s, n): synth.pad_planes(synth.frame(geom.pic_w, geom.pic_h, f=n, seed=100 * s + n)[0], geom)
           for s in range(S) for n in range(7)}
    kout = _copy(key.encode([np.stack([src[s, 0][p] for s in range(S)]) for p in range(3)],
                            np.stack([synth.block_size_map(geom, "mixed", seed=s) for s in range(S)])))
    pics = {}   # the oracle's running pictures: (sequence, buffer) -> planes
    pe = engine.KeyframeEngine(geom, nframes=S, q0=Q0, pvq_qm_q4=Q4, inter=1, inter_mc=1, inter_finish=1, mc_refs=4 * S)
    be = _engine(geom, 2 * S, inter_finish=1, mc_refs=4 * S)
    for s in range(S):
        self_ = order[0].refs[gop.SELF]
        pe.pool_load(4 * s + self_, [key.buf.pixels_out[p] + s * plane_bytes[p] for p in range(3)])
        pics[s, self_] = [kout["recon%d" % p][s] for p in range(3)]
    k = 1
    step = 0
    while k < len(order):
        P = order[k]
        Bs = order[k + 1:k + 3]
        assert P.type == gop.P_FRAME and all(b.type == gop.B_FRAME for b in Bs)
        # the P frame of each sequence
        grids = [synth.mv_grid_b(geom, seed=200 + 10 * step + s, p_next=0.0, p_gold=0.5) for s in range(S)]
        pgrid, pmv1 = _pack(grids)
        planes = [np.stack([src[s, P.number][p] for s in range(S)]) for p in range(3)]
        bsize = np.stack([synth.block_size_map(geom, "mixed", seed=300 + 10 * step + s) for s in range(S)])
        slot = np.array([[4 * s + P.refs[gop.GOLD], 4 * s + P.refs[gop.PREV]] for s in range(S)], np.int32)
        out = _copy(pe.encode(planes, bsize, ref_slot=slot, mv_grid=pgrid, resident=True))
        for s in range(S):
            want = bframe_oracle.predict3(lib, geom, *(pics[s, P.refs[r]] for r in (gop.GOLD, gop.PREV, gop.NEXT)),
                                            *grids[s])
            for p in range(3):
                assert np.array_equal(out["pred%d" % p][s], want[p]), ("P prediction", P.number, s, p)
        d = [pe.coeff_plane(p) for p in range(3)]
        md = [pe.pred_coeff_plane(p) for p in range(3)]
        dec = _decisions(out, geom, S, seed=step)
        got = _copy(pe.finish(*dec[:5], ref_slot_out=np.array([4 * s + P.refs[gop.SELF] for s in range(S)], np.int32)))
        want = _want(geom, S, out, d, md, bsize, Q0, dec)
        _check(got, want, S)
        for s in range(S):
            pics[s, P.refs[gop.SELF]] = list(want[s][0])
        # the group's B frames: one batch, frame 2s + j is B frame j of sequence s
        for slot_no in range(4 * S):
            pe_filled = any(key_[0] == slot_no // 4 and key_[1] == slot_no % 4 for key_ in pics)
            if pe_filled:
                be.pool_load(slot_no, [pe.buf.ref_pixels[p] + slot_no * plane_bytes[p] for p in range(3)])
        bgr = [synth.mv_grid_b(geom, seed=400 + 10 * step + i) for i in range(2 * S)]
        bplanes = [np.stack([src[s, b.number][p] for s in range(S) for b in Bs]) for p in range(3)]
        bbsize = np.stack([synth.block_size_map(geom, "mixed", seed=500 + 10 * step + i) for i in range(2 * S)])
        bslot = np.array([[4 * s + b.refs[r] for r in (gop.GOLD, gop.PREV, gop.NEXT)] for s in range(S) for b in Bs],
                         np.int32)
        grid, mv1 = _pack(bgr)
        bout = _copy(be.encode(bplanes, bbsize, ref_slot=bslot, mv_grid=grid, mv1_grid=mv1, resident=True))
        i = 0
        for s in range(S):
            for b in Bs:
                want = bframe_oracle.predict3(lib, geom, *(pics[s, b.refs[r]] for r in (gop.GOLD, gop.PREV, gop.NEXT)),
                                                *bgr[i])
                for p in range(3):
                    assert np.array_equal(bout["pred%d" % p][i], want[p]), ("B prediction", b.number, s, p)
                i += 1
        pool_p, pool_b = [pe.pool_plane(p) for p in range(3)], [be.pool_plane(p) for p in range(3)]
        d = [be.coeff_plane(p) for p in range(3)]
        md = [be.pred_coeff_plane(p) for p in range(3)]
        dec = _decisions(bout, geom, 2 * S, seed=50 + step)
        got = _copy(be.finish(*dec[:5], ref_slot_out=np.full(2 * S, -1, np.int32)))
        _check(got, _want(geom, 2 * S, bout, d, md, bbsize, Q0, dec), 2 * S)
        for p in range(3):
            assert np.array_equal(pe.pool_plane(p), pool_p[p]) and np.array_equal(be.pool_plane(p), pool_b[p]), p
        k += 3
        step += 1
    # the P engine's pool holds the oracle's reference pictures
    pool = [pe.pool_plane(p) for p in range(3)]
    for (s, buf), planes in pics.items():
        for p in range(3):
            assert np.array_equal(pool[p][4 * s + buf], planes[p]), (s, buf, p)
    for e in (key, pe, be):
        e.close()


@pytest.mark.parametrize("fault", ["ref3", "next_vector", "stale_prev_vector"])
def test_diagnostics(fault):
    """Frame 1 of 3: a used vertex with ref 3 (counts[19], encode raises), a NEXT vertex whose mv1 reaches past the edge
    extension (counts[20] through mv1, encode raises), or a PREV vertex with such an mv1 (not counted: mv1 is not read
    there).  The other frames equal the oracle."""
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    lib = _ref()
    geom = Geometry(200, 130)
    F = 3
    refs = _pool(geom, 3, seed=7)
    slot = [[0, 1, 2]] * F
    grids = _bgrids(geom, F, seed=40)
    valid, mv, mv1, ref = (a.copy() for a in grids[1])
    if fault == "ref3":
        ref[0, 0] = 3
    else:
        ref[0, 0] = 2 if fault == "next_vector" else 1
        mv[0, 0] = (0, 0)
        mv1[0, 0] = (-8 * 70, 0)
    grids[1] = (valid, mv, mv1, ref)
    planes, bsize = _batch(geom, F, seed=12)
    eng = _engine(geom, F)
    if fault == "stale_prev_vector":
        out = _run(eng, planes, bsize, refs, slot, grids)
        assert int(out["counts"][engine.CNT["mc_beyond"]]) == 0 and int(out["counts"][engine.CNT["mc_bad_ref"]]) == 0
        frames = range(F)
    else:
        with pytest.raises(RuntimeError, match="MV grid outside"):
            _run(eng, planes, bsize, refs, slot, grids)
        out = {k: np.array(v) for k, v in eng._out.items()}
        key = "mc_bad_ref" if fault == "ref3" else "mc_beyond"
        other = "mc_beyond" if fault == "ref3" else "mc_bad_ref"
        assert int(out["counts"][engine.CNT[key]]) > 0 and int(out["counts"][engine.CNT[other]]) == 0
        if fault == "next_vector":
            assert int(out["counts"][engine.CNT[key]]) == _beyond_model(geom, valid, mv, mv1, ref)
        frames = (0, 2)
    for f in frames:
        want = _hook(lib, geom, refs, slot[f], grids[f])
        for p in range(3):
            assert np.array_equal(out["pred%d" % p][f], want[p]), ("prediction", f, p)
    eng.close()


def test_refusals_before_any_copy():
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    geom = Geometry(200, 130)
    for kw in (dict(inter=1, inter_mc=1, mc_next=2), dict(inter=1, inter_mc=0, mc_next=1),
               dict(inter=0, inter_mc=0, mc_next=1)):
        with pytest.raises(RuntimeError, match="daala_b200_kf_create: .*mc_next"):
            engine.KeyframeEngine(geom, nframes=1, q0=Q0, pvq_qm_q4=Q4, **kw)
    F = 2
    eng = _engine(geom, F, mc_refs=5)
    refs = _pool(geom, 3, seed=1)
    planes, bsize = _batch(geom, F, seed=4)
    _run(eng, planes, bsize, refs, [[0, 1, 2], [2, 2, 1]], _bgrids(geom, F, seed=9))
    nv, nh = geom.nvsb * 8 + 1, geom.nhsb * 8 + 1

    def device_state():
        return ([eng.download(eng.buf.pixels[p], (F,) + geom.plane_shape(p), np.uint8) for p in range(3)] +
                [eng.download(eng.buf.mv_grid, (F * nv * nh * 12,), np.uint8),
                 eng.download(eng.buf.mv1_grid, (F * nv * nh * 2,), np.int32),
                 eng.download(eng.buf.ref_slot_next, (F,), np.int32)])

    before = device_state()
    planes2, bsize2 = _batch(geom, F, seed=5)
    eng.stage_inputs(planes2, bsize2)
    grid, mv1 = _pack(_bgrids(geom, F, seed=10))
    eng.stage_mc(_pool(geom, 3, seed=2), np.array([[0, 1, 2], [1, 2, 0]], np.int32), grid, mv1_grid=mv1)
    eng.prepare_io()
    io = eng._io
    nxt = eng._arr("slot_next", (F,), np.int32)

    def field(name, value):
        old = getattr(io, name)
        setattr(io, name, value)
        return lambda: setattr(io, name, old)

    def next_value(v):
        old = int(nxt[1])
        nxt[1] = v
        return lambda: nxt.__setitem__(1, old)

    def resident(v):
        """ref_resident = 1 (no upload) with NEXT slot v; slots 0..2 hold pictures, 3 and 4 do not."""
        saved = [(k, getattr(io, k)) for k in ("ref_resident", "nrefs")] + [("p%d" % p, io.ref_pixels[p]) for p in range(3)]
        io.ref_resident, io.nrefs = 1, 0
        for p in range(3):
            io.ref_pixels[p] = None
        undo_slot = next_value(v)

        def undo():
            undo_slot()
            for k, val in saved:
                if k.startswith("p"):
                    io.ref_pixels[int(k[1])] = val
                else:
                    setattr(io, k, val)
        return undo

    cases = [("mv1_grid", lambda: field("mv1_grid", None)), ("ref_slot_next", lambda: field("ref_slot_next", None)),
             ("ref_slot_next", lambda: next_value(3)), ("ref_slot_next", lambda: next_value(-1)),
             ("ref_slot_next", lambda: resident(5)), ("ref_slot_next", lambda: resident(4))]
    for what, breaker in cases:
        undo = breaker()
        rc = eng.L.daala_b200_kf_submit(eng.kf, ctypes.byref(io))
        msg = eng.L.daala_b200_kf_error(eng.kf).decode()
        undo()
        assert rc != 0 and what in msg, (what, rc, msg)
    eng.wait()
    for a, b in zip(device_state(), before):
        assert np.array_equal(a, b)
    # either B-frame field given to an engine without mc_next
    pe = _engine(geom, F, mc_next=0)
    pe.stage_inputs(planes, bsize)
    pe.stage_mc(refs, np.array([[0, 1], [2, 2]], np.int32), grid)
    pe.prepare_io()
    pin = [pe.download(pe.buf.pixels[p], (F,) + geom.plane_shape(p), np.uint8) for p in range(3)]
    for name, arr in (("mv1_grid", mv1), ("ref_slot_next", nxt)):
        setattr(pe._io, name, arr.ctypes.data)
        rc = pe.L.daala_b200_kf_submit(pe.kf, ctypes.byref(pe._io))
        msg = pe.L.daala_b200_kf_error(pe.kf).decode()
        setattr(pe._io, name, None)
        assert rc != 0 and "mc_next" in msg, (name, msg)
    pe.wait()
    for p in range(3):
        assert np.array_equal(pe.download(pe.buf.pixels[p], (F,) + geom.plane_shape(p), np.uint8), pin[p])
    with pytest.raises(ValueError):
        pe.stage_mc(refs, np.array([[0, 1], [2, 2]], np.int32), grid, mv1_grid=mv1)
    with pytest.raises(ValueError):
        eng.stage_mc(refs, np.array([[0, 1], [2, 2]], np.int32), grid, mv1_grid=mv1)
    pe.close()
    eng.close()
