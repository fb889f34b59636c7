"""Keyframes and P / B frames in one engine batch (config.frame_types = 1) on the GPU.

The mixed engine is compared with the single-kind engines it replaces, frame by frame, exactly: every keyframe with a
keyframe_quant = 1, haar_dc_quant = 1 engine given that frame and record, every P / B frame with the frame_quant = 1
inter engine (inter_mc, mc_next) given that frame, record, pool and grids.  Blocks are compared keyed by (plane, y0,
x0) inside their frame, since the two engines number them differently.  The outputs of the other kind are 0.  Then
the finishing pass (given and searched deringing levels, the P frames' seeded decisions, the keyframes' decisions
ignored), batches of one kind, a GOP on one engine against the two-engine route with pool_load, a 4K batch on the bench
maps, graph replay and the refusals."""
import os

import numpy as np
import pytest

from daala_b200 import engine, gop, mvgrid, synth
from daala_b200.frame import Geometry

pytestmark = [pytest.mark.gpu]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NREFS = 4


def _records(F, seed):
    rng = np.random.default_rng(seed)
    q0 = rng.integers(20, 120, F)
    q4 = rng.integers(12, 28, (F, 3, 30)).astype(np.uint8)
    return engine.frame_quant_records(q0, np.clip(q0 // 4, 1, 63), 0.67 * 0.1 * q0.astype(float) ** 2, q4)


def _real_map(geom, k):
    real = np.load(os.path.join(ROOT, "daala_b200", "data", "bench_bsize_4k.npz"))["bsize_%d" % (k % 4)]
    h, w = geom.bsize_shape
    return np.ascontiguousarray(real[:h, :w])


def _inputs(geom, types, seed):
    """Source planes, block-size maps (random quadtrees and real encoder maps), records, a pool, and per frame the
    (valid, mv, mv1, ref) grid: B frames (type 2 here) read NEXT, P frames GOLD / PREV; keyframes get a grid too, which
    the engine must not read."""
    F = len(types)
    src = [synth.pad_planes(synth.frame(geom.pic_w, geom.pic_h, f=f + 1, seed=seed + f)[0], geom) for f in range(F)]
    planes = [np.stack([s[p] for s in src]) for p in range(3)]
    bsize = np.stack([synth.block_size_map(geom, "mixed", seed=seed + f) if f % 2 else _real_map(geom, f) for f in range(F)])
    pics = [synth.pad_planes(synth.frame(geom.pic_w, geom.pic_h, f=9 + i, seed=seed + 40 + i)[0], geom) for i in range(NREFS)]
    pool = [np.stack([p[pl] for p in pics]) for pl in range(3)]
    grids = []
    for f, t in enumerate(types):
        if t == 2:
            grids.append(synth.mv_grid_b(geom, seed=seed + 60 + f))
        else:
            valid, mv, ref = synth.mv_grid(geom, seed=seed + 60 + f)
            grids.append((valid, mv, np.zeros(mv.shape, np.int32), ref))
    slots = np.array([[f % NREFS, (f + 1) % NREFS, (f + 2) % NREFS] for f in range(F)], np.int32)
    for f, t in enumerate(types):
        if t == 1:
            slots[f] = -1   # a keyframe's slots are neither read nor checked
    return planes, bsize, _records(F, seed), pool, grids, slots


def _pack(grids):
    valid, mv, mv1, ref = (np.stack([g[i] for g in grids]) for i in range(4))
    return mvgrid.pack(valid, mv, ref), mv1.astype(np.int32)


def _mixed(geom, F, inter_finish=1, **kw):
    return engine.KeyframeEngine(geom, nframes=F, q0=999, pvq_qm_q4=np.full((3, 30), 9, np.uint8), inter=1, inter_mc=1,
                                 mc_next=1, mc_refs=8, frame_quant=1, haar_dc_quant=1, inter_finish=inter_finish,
                                 frame_types=1, coded_quantizer=33, **kw)


def _key_engine(geom, dering=0):
    return engine.KeyframeEngine(geom, nframes=1, keyframe_quant=1, haar_dc_quant=1, dering=dering)


def _p_engine(geom, inter_finish=1):
    return engine.KeyframeEngine(geom, nframes=1, inter=1, inter_mc=1, mc_next=1, mc_refs=8, frame_quant=1,
                                 inter_finish=inter_finish)


def _copy(out):
    return {k: np.array(v) for k, v in out.items()}


def _step(eng, planes, bsize, rec, types, pool, grids, slots, resident=False):
    grid, mv1 = _pack(grids)
    out = _copy(eng.encode(planes, bsize, frame_quant=rec, frame_type=np.asarray(types) == 1,
                           refs=None if resident else pool, ref_slot=slots, mv_grid=grid, mv1_grid=mv1,
                           resident=resident))
    out["coeffs"] = [eng.coeff_plane(p).copy() for p in range(3)]
    return out


def _single(eng, planes, bsize, rec, f, pool=None, grids=None, slots=None, levels=None):
    """Frame f of a batch through a one-frame engine."""
    one = [planes[p][f:f + 1] for p in range(3)]
    kw = {}
    if pool is not None:
        grid, mv1 = _pack([grids[f]])
        kw = dict(refs=pool, ref_slot=slots[f:f + 1], mv_grid=grid, mv1_grid=mv1)
    out = _copy(eng.encode(one, bsize[f:f + 1], frame_quant=rec[f:f + 1], dering_levels=levels, **kw))
    out["coeffs"] = [eng.coeff_plane(p).copy() for p in range(3)]
    return out


def _blocks_of(out, kind, f):
    """The blocks of frame f in (plane, y0, x0) order, with their per-block outputs."""
    b = out[kind + "_blocks"]
    sel = np.nonzero(b["frame"] == f)[0]
    sel = sel[np.lexsort((b["x0"][sel], b["y0"][sel], b["pli"][sel]))]
    nb = [1, 4, 7, 9, 9]
    d = {"desc": np.stack([b["x0"][sel], b["y0"][sel], b["bs"][sel], b["pli"][sel]]),
         "res": np.concatenate([out[kind + "_res"][i][:nb[b["bs"][i]]].ravel() for i in sel] + [np.zeros(0, np.int16)]),
         "skip_diff": out[kind + "_skip_diff"][sel]}
    n = np.where(b["bs"][sel] >= 3, 512, 16 << (2 * b["bs"][sel].astype(np.int64)))
    d["pulses"] = np.concatenate([out[kind + "_y16"][b["coef_off"][i]:b["coef_off"][i] + k] for i, k in zip(sel, n)] +
                                 [np.zeros(0, np.int16)])
    for k in ("flip", "dc", "dc_resid"):
        src = {"flip": "chroma_flip", "dc": kind + "_dc", "dc_resid": kind + "_dc_resid"}[k]
        if src in out and (k != "flip" or kind == "chroma"):
            d[k] = out[src][sel]
    return d, sel


def _same_frame(got, gf, want, wf, keys, what):
    for p in range(3):
        assert np.array_equal(got["coeffs"][p][gf], want["coeffs"][p][wf]), (what, "coefficient plane", p)
        assert np.array_equal(got["recon%d" % p][gf], want["recon%d" % p][wf]), (what, "reconstruction", p)
    for kind in ("luma", "chroma"):
        g, _ = _blocks_of(got, kind, gf)
        w, _ = _blocks_of(want, kind, wf)
        assert np.array_equal(g["desc"], w["desc"]), (what, kind, "blocks")
        for k in keys:
            if k in w:
                if k == "skip_diff":
                    np.testing.assert_allclose(g[k], w[k], rtol=1e-5, atol=0, err_msg=str((what, kind, k)))
                else:
                    assert np.array_equal(g[k], w[k]), (what, kind, k)


def _zero_other_kind(out, types):
    for f, t in enumerate(types):
        for kind in ("luma", "chroma"):
            _, sel = _blocks_of(out, kind, f)
            if t == 1:
                for k in ("_dc", "_dc_resid"):
                    assert not out[kind + k][sel].any(), ("keyframe", f, kind + k)
            elif kind == "chroma":
                assert not out["chroma_flip"][sel].any(), ("P frame", f, "chroma_flip")
        for p in range(3):
            if t == 1:
                assert not out["pred%d" % p][f].any(), ("keyframe", f, "pred", p)
            else:
                assert not out["dc_index%d" % p][f].any(), ("P frame", f, "dc_index", p)


def _check_step(geom, types, seed):
    F = len(types)
    planes, bsize, rec, pool, grids, slots = _inputs(geom, types, seed)
    eng = _mixed(geom, F)
    got = _step(eng, planes, bsize, rec, types, pool, grids, slots)
    assert int(got["counts"][engine.CNT["mc_bad_ref"]]) == 0 and int(got["counts"][engine.CNT["mc_beyond"]]) == 0
    key, inter = _key_engine(geom), _p_engine(geom)
    for f, t in enumerate(types):
        if t == 1:
            want = _single(key, planes, bsize, rec, f)
            _same_frame(got, f, want, 0, ("res", "skip_diff", "pulses", "flip"), ("keyframe", f))
            for p in range(3):
                assert np.array_equal(got["dc_index%d" % p][f], want["dc_index%d" % p][0]), ("keyframe", f, "dc_index", p)
        else:
            want = _single(inter, planes, bsize, rec, f, pool, grids, slots)
            _same_frame(got, f, want, 0, ("res", "skip_diff", "pulses", "dc", "dc_resid"), ("P frame", f))
            for p in range(3):
                assert np.array_equal(got["pred%d" % p][f], want["pred%d" % p][0]), ("P frame", f, "prediction", p)
    _zero_other_kind(got, types)
    return eng, got, (planes, bsize, rec, pool, grids, slots), key, inter


@pytest.mark.parametrize("w,h,types", [(200, 130, (1, 0, 2, 1)), (1920, 1080, (0, 1, 0))])
def test_step_matches_single_kind_engines(w, h, types):
    eng, *_ = _check_step(Geometry(w, h), types, seed=w + h)
    eng.close()


def _decisions(out, types, seed):
    """Seeded skip / DC decisions for every block; the keyframes' are garbage, which the pass must ignore."""
    rng = np.random.default_rng(seed)
    res = []
    for kind in ("luma", "chroma"):
        n = len(out[kind + "_blocks"])
        skip = rng.integers(0, 2, n).astype(np.uint8)
        dc = np.where(rng.random(n) < 0.5, out[kind + "_dc"], out[kind + "_dc"] + rng.integers(-2, 3, n)).astype(np.int32)
        res += [skip, dc]
    return res


@pytest.mark.parametrize("inter_finish", [1, 2])
def test_finish_matches_single_kind_engines(inter_finish):
    geom = Geometry(200, 130)
    types = (1, 0, 2, 1)
    planes, bsize, rec, pool, grids, slots = _inputs(geom, types, seed=5)
    eng = _mixed(geom, len(types), inter_finish=inter_finish)
    got = _step(eng, planes, bsize, rec, types, pool, grids, slots)
    ls, ld, cs, cd = _decisions(got, types, seed=11)
    levels = np.random.default_rng(3).integers(0, 6, (len(types), geom.nvsb, geom.nhsb)).astype(np.uint8)
    fin = _copy(eng.finish(ls, ld, cs, cd, dering_levels=levels if inter_finish == 1 else None))
    key = _key_engine(geom, dering=inter_finish)
    inter = _p_engine(geom, inter_finish=inter_finish)
    for f, t in enumerate(types):
        if t == 1:
            want = _single(key, planes, bsize, rec, f, levels=levels[f:f + 1] if inter_finish == 1 else None)
            for p in range(3):
                assert np.array_equal(fin["recon%d" % p][f], want["recon%d" % p][0]), ("keyframe", f, p)
                assert not fin["bskip%d" % p][f].any(), ("keyframe bskip", f, p)
            assert np.array_equal(fin["dering_levels"][f], want["dering_levels"][0]), ("keyframe levels", f)
        else:
            step = _single(inter, planes, bsize, rec, f, pool, grids, slots)
            sl = [np.nonzero(got[k + "_blocks"]["frame"] == f)[0] for k in ("luma", "chroma")]
            for k, s in zip(("luma", "chroma"), sl):
                assert np.array_equal(got[k + "_blocks"][s][["x0", "y0", "bs", "pli"]], step[k + "_blocks"][["x0", "y0", "bs", "pli"]])
            want = _copy(inter.finish(ls[sl[0]], ld[sl[0]], cs[sl[1]], cd[sl[1]],
                                      dering_levels=levels[f:f + 1] if inter_finish == 1 else None))
            for p in range(3):
                assert np.array_equal(fin["recon%d" % p][f], want["recon%d" % p][0]), ("P frame", f, p)
                assert np.array_equal(fin["bskip%d" % p][f], want["bskip%d" % p][0]), ("P frame bskip", f, p)
            assert np.array_equal(fin["dering_levels"][f], want["dering_levels"][0]), ("P frame levels", f)
    eng.close()


@pytest.mark.parametrize("types", [(1, 1, 1), (0, 2, 0)])
def test_batches_of_one_kind(types):
    eng, *_ = _check_step(Geometry(200, 130), types, seed=sum(types) + 17)
    eng.close()


def test_gop_on_one_engine_matches_two_engine_route():
    """I B B P B B P B B I B B P through pipelined_steps(keyframes_inline=True) on one engine, every picture kept in
    its pool with ref_slot_out and read back with resident=True, against a keyframe engine + an inter engine whose pool
    takes each keyframe with pool_load.  Steps shorter than the engine's batch are filled with keyframes that are not
    stored."""
    geom = Geometry(200, 130)
    frames = gop.coding_order(13, 2, keyframe_rate=9)
    steps = gop.pipelined_steps(frames, keyframes_inline=True)
    F = max(len(s) for s in steps)
    src = [synth.pad_planes(synth.frame(geom.pic_w, geom.pic_h, f=i + 1, seed=77 + i)[0], geom) for i in range(13)]
    maps = [synth.block_size_map(geom, "mixed", seed=300 + i) for i in range(13)]
    rec_all = _records(13, seed=9)
    grids = {}
    for fr in frames:
        if fr.type == gop.B_FRAME:
            grids[fr.number] = synth.mv_grid_b(geom, seed=500 + fr.number)
        else:
            v, mv, ref = synth.mv_grid(geom, seed=500 + fr.number)
            grids[fr.number] = (v, mv, np.zeros(mv.shape, np.int32), ref)
    levels = np.zeros((1, geom.nvsb, geom.nhsb), np.uint8)
    one = _mixed(geom, F)
    key = _key_engine(geom, dering=1)
    inter = engine.KeyframeEngine(geom, nframes=F, inter=1, inter_mc=1, mc_next=1, mc_refs=8, frame_quant=1,
                                  inter_finish=1)
    for st in steps:
        nums = [fr.number for fr in st]
        pad = F - len(st)
        idx = nums + [nums[0]] * pad
        types = [1 if fr.type == gop.I_FRAME else 0 for fr in st] + [1] * pad
        slots = np.array([gop.pool_slots(fr) for fr in st] + [[0, 0, 0]] * pad, np.int32)
        out_slot = np.array([fr.refs[gop.SELF] if fr.kept else -1 for fr in st] + [-1] * pad, np.int32)
        planes = [np.stack([src[i][p] for i in idx]) for p in range(3)]
        bsize = np.stack([maps[i] for i in idx])
        rec = rec_all[idx]
        g = [grids[i] for i in idx]
        got = _step(one, planes, bsize, rec, types, None, g, slots, resident=True)
        # the step's own decisions: nothing skipped, the step's DC indices (0 on keyframes, which ignore them)
        ls, cs = (np.zeros(len(got[k + "_blocks"]), np.uint8) for k in ("luma", "chroma"))
        ld, cd = got["luma_dc"], got["chroma_dc"]
        fin = _copy(one.finish(ls, ld, cs, cd, dering_levels=np.zeros((F, geom.nvsb, geom.nhsb), np.uint8),
                               ref_slot_out=out_slot))
        # the two-engine route: the keyframe through the keyframe engine and pool_load, the rest through the inter engine
        for k, fr in enumerate(st):
            if fr.type == gop.I_FRAME:
                want = _single(key, planes, bsize, rec, k, levels=levels)
                for p in range(3):
                    assert np.array_equal(fin["recon%d" % p][k], want["recon%d" % p][0]), ("keyframe", fr.number, p)
                inter.pool_load(int(out_slot[k]), [want["recon%d" % p][0] for p in range(3)])
        rest = [k for k, fr in enumerate(st) if fr.type != gop.I_FRAME]
        if rest:
            ridx = rest + [rest[0]] * (F - len(rest))
            gp, mv1 = _pack([g[k] for k in ridx])
            w = _copy(inter.encode([planes[p][ridx] for p in range(3)], bsize[ridx], frame_quant=rec[ridx],
                                   ref_slot=slots[ridx], mv_grid=gp, mv1_grid=mv1, resident=True))
            wl, wc = (np.zeros(len(w[k + "_blocks"]), np.uint8) for k in ("luma", "chroma"))
            wout = np.array([out_slot[k] for k in rest] + [-1] * (F - len(rest)), np.int32)
            wf = _copy(inter.finish(wl, w["luma_dc"], wc, w["chroma_dc"],
                                    dering_levels=np.zeros((F, geom.nvsb, geom.nhsb), np.uint8), ref_slot_out=wout))
            for j, k in enumerate(rest):
                for p in range(3):
                    assert np.array_equal(fin["recon%d" % p][k], wf["recon%d" % p][j]), ("P/B frame", st[k].number, p)
        for p in range(3):
            assert np.array_equal(one.pool_plane(p)[:4], inter.pool_plane(p)[:4]), ("pool", nums, p)
    one.close()


def test_4k_mixed_batch_on_the_bench_maps():
    geom = Geometry(3840, 2160)
    types = (1, 0, 0)
    planes, _, rec, pool, grids, slots = _inputs(geom, types, seed=4)
    real = np.load(os.path.join(ROOT, "daala_b200", "data", "bench_bsize_4k.npz"))
    bsize = np.stack([np.ascontiguousarray(real["bsize_%d" % f][:geom.bsize_shape[0], :geom.bsize_shape[1]])
                      for f in range(3)])
    eng = _mixed(geom, 3)
    got = _step(eng, planes, bsize, rec, types, pool, grids, slots)
    key, inter = _key_engine(geom), _p_engine(geom)
    want = _single(key, planes, bsize, rec, 0)
    _same_frame(got, 0, want, 0, ("res", "skip_diff", "pulses", "flip"), "4K keyframe")
    for f in (1, 2):
        want = _single(inter, planes, bsize, rec, f, pool, grids, slots)
        _same_frame(got, f, want, 0, ("res", "skip_diff", "pulses", "dc", "dc_resid"), ("4K P frame", f))
    eng.close()


def test_phase_by_phase_equals_the_forked_step():
    """A mixed batch (keyframes, P and B frames, inter_mc, a record per frame) run phase by phase on one stream, the
    forked step as live launches and a graph replay all leave the device state of the submitted step graph: the
    reconstruction, the coefficient planes of the source and of the prediction, the band records, pulses, skip_diff,
    CfL flips and the keyframe DC indices.  The P / B frames' DC indices reach the coefficient planes."""
    from tests.test_gpu_step_fork import _assert_same, _state
    geom = Geometry(200, 130)
    types = (1, 0, 2, 1)
    planes, bsize, rec, pool, grids, slots = _inputs(geom, types, seed=31)
    eng = _mixed(geom, len(types))

    def state():
        st = _state(eng)
        for p in range(3):
            st["pred_coeffs%d" % p] = eng.pred_coeff_plane(p)
            st["dc_index%d" % p] = eng.download(eng.buf.dc_index[p], (eng.F,) + tuple(s >> 2 for s in geom.plane_shape(p)),
                                                np.int32)
        return st

    try:
        got = _step(eng, planes, bsize, rec, types, pool, grids, slots)   # the forked step graph
        forked = state()
        for p in range(3):
            assert np.array_equal(forked["recon%d" % p], got["recon%d" % p])
            assert np.array_equal(forked["dc_index%d" % p], got["dc_index%d" % p])
        assert np.array_equal(forked["chroma_flip"], got["chroma_flip"])
        for ph in (engine.PH_LISTS, engine.PH_FORWARD, engine.PH_PVQ_LUMA, engine.PH_PVQ_CHROMA, engine.PH_INVERSE):
            eng.run_device(ph, False)
        _assert_same(state(), forked, "phase by phase")
        eng.run_device(engine.PH_ALL, False)   # the forked step as live launches
        _assert_same(state(), forked, "live launches")
        eng.run_device(engine.PH_ALL, True)    # and a graph replay
        _assert_same(state(), forked, "graph replay")
    finally:
        eng.close()


def test_replay_is_identical_and_refusals_come_with_messages():
    geom = Geometry(200, 130)
    types = (0, 1, 2)
    planes, bsize, rec, pool, grids, slots = _inputs(geom, types, seed=21)
    eng = _mixed(geom, 3)
    a = _step(eng, planes, bsize, rec, types, pool, grids, slots)
    b = _step(eng, planes, bsize, rec, types, pool, grids, slots)
    for k in a:
        if k == "coeffs":
            assert all(np.array_equal(x, y) for x, y in zip(a[k], b[k]))
        else:
            assert np.array_equal(a[k], b[k], equal_nan=a[k].dtype.kind == "f"), k
    # submit: a missing type, a type other than 0 / 1
    for bad, msg in ((None, "frame_type .* is required"), (np.array([0, 1, 2], np.uint8), "neither 0 nor 1")):
        eng.stage_frame_type(np.array([0, 1, 0]))
        if bad is None:
            eng._ftype = None
        else:
            eng._ftype[...] = bad
        eng.prepare_io()
        with pytest.raises(Exception, match=msg):
            eng.submit()
    eng.close()
    # create: each refusal with its own message
    base = dict(inter=1, inter_mc=1, frame_quant=1, haar_dc_quant=1, inter_finish=1, frame_types=1)
    cases = [(dict(frame_types=2), "frame_types is 0 or 1"),
             (dict(inter=0, inter_mc=0, inter_finish=0), "requires inter = 1"),
             (dict(frame_quant=0), "requires inter = 1, frame_quant = 1"),
             (dict(haar_dc_quant=0), "haar_dc_quant = 1"),
             (dict(inter_finish=0), "inter_finish 1 or 2"),
             (dict(symbol_stream=2), "symbol_stream"),
             (dict(late_skip=1), "late_skip"),
             (dict(lossless=1), "lossless"),
             (dict(dering=1), "dering"),
             (dict(sb_rows=1), "row shard")]
    for over, msg in cases:
        with pytest.raises(RuntimeError, match=msg):
            engine.KeyframeEngine(geom, nframes=2, **{**base, **over})
    # haar_dc_quant stays refused with inter on an engine without frame_types
    with pytest.raises(RuntimeError, match="haar_dc_quant is not defined with inter"):
        engine.KeyframeEngine(geom, nframes=2, inter=1, haar_dc_quant=1)
    # frame_type= on an engine without the mode
    plain = engine.KeyframeEngine(geom, nframes=1, inter=1, frame_quant=1)
    with pytest.raises(ValueError, match="frame_type"):
        plain.encode([planes[p][:1] for p in range(3)], bsize[:1], pred=[planes[p][:1] for p in range(3)],
                     frame_quant=rec[:1], frame_type=np.array([0]))
    plain.close()
