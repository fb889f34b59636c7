"""Per-frame quantizers in one P/B-frame batch (config.frame_quant): one engine whose frames carry different records from
the encoder's own settings (tests/golden/encoder_settings.npz) equals one uniform engine per frame at that frame's
settings in every output, and each frame equals the oracles at its own q0 / pvq_qm_q4 / coded_quantizer /
dering_lambda.  Records equal to the config give the frame_quant = 0 engine's results and launches; refusals happen
before anything is copied."""
import numpy as np
import pytest

from tests import inter_finish_oracle, late_skip_oracle, oracle_lib
from tests.test_gpu_engine_inter_finish import _decisions
from tests.test_gpu_engine_quantizer_range import COARSEST, FINEST, _engine, settings

pytestmark = [pytest.mark.gpu]

# (sweep point, frame column 0 = keyframe settings / 1 = P-frame settings) of each frame: the finest and coarsest
# points, and tables of both columns, all with masking and the HVS matrix (configuration 0), so that q0, coded_quantizer,
# dering_lambda and pvq_qm_q4 all differ between frames while the stream settings agree
POINTS = [(FINEST, 1), (COARSEST, 1), (3, 0), (5, 1)]
MC = dict(inter=1, inter_mc=1, mc_next=1, late_skip=1, symbol_stream=2, inter_finish=2)
PER_BLOCK = ("skip_diff", "dc", "dc_resid")


def _records(points):
    from daala_b200 import engine
    ss = [settings(p, 0, c) for p, c in points]
    return ss, engine.frame_quant_records([s["q0"] for s in ss], [s["cq"] for s in ss],
                                          [s["dering_lambda"] for s in ss], np.stack([s["q4"] for s in ss]))


def _copy(r):
    return {k: np.array(v) for k, v in r.items()}


def _inputs(geom, F, seed):
    from tests.test_gpu_engine_bframes import _bgrids, _pack
    from tests.test_gpu_engine_inter_mc import _batch, _pool
    refs = _pool(geom, 3, seed=seed)
    planes, bsize = _batch(geom, F, seed=seed + 1)
    grid, mv1 = _pack(_bgrids(geom, F, seed=seed + 2))
    slot = np.array([[f % 3, (f + 1) % 3, (f + 2) % 3] for f in range(F)], np.int32)
    return refs, planes, bsize, grid, mv1, slot


def _frame_stream(out, f):
    """Frame f's slices of the stream arrays (block, band, DC and late-skip records, pulse bytes)."""
    i = out["sym_index"][f]
    b0, nb, n0, nn, p0, np_ = (int(v) for v in i)
    return dict(sym_blocks=out["sym_blocks"][b0:b0 + nb], sym_bands=out["sym_bands"][n0:n0 + nn],
                sym_pulses=out["sym_pulses"][p0:p0 + np_], sym_dc=out["sym_dc"][b0:b0 + nb],
                sym_late_skip=out["sym_late_skip"][b0:b0 + nb])


@pytest.mark.parametrize("w,h,F", [(200, 130, 4), (1920, 1080, 2)])
def test_same_as_one_engine_per_frame(w, h, F):
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    geom = Geometry(w, h)
    ss, rec = _records(POINTS[:F])
    assert len({int(r) for r in rec["q0"]}) == F and not all(np.array_equal(rec["pvq_qm_q4"][0], r) for r in rec["pvq_qm_q4"])
    refs, planes, bsize, grid, mv1, slot = _inputs(geom, F, seed=31 + F)
    # the config's per-frame fields are deliberately not those of any frame: a frame_quant engine does not read them
    eng = _engine(geom, F, dict(ss[0], q0=77, cq=20, dering_lambda=1.0, q4=np.full((3, 30), 9, np.uint8)),
                  frame_quant=1, mc_refs=3 + F, **MC)
    try:
        got = _copy(eng.encode(planes, bsize, refs=refs, ref_slot=slot, mv_grid=grid, mv1_grid=mv1, frame_quant=rec))
        gd = [eng.coeff_plane(p) for p in range(3)]
        dec = _decisions(got, geom, F, seed=7)
        fin = _copy(eng.finish(*dec[:4], ref_slot_out=np.arange(3, 3 + F, dtype=np.int32)))
        pool = [eng.pool_plane(p) for p in range(3)]
    finally:
        eng.close()
    for f in range(F):
        one = _engine(geom, 1, ss[f], mc_refs=4, **MC)
        try:
            want = _copy(one.encode([p[f:f + 1] for p in planes], bsize[f:f + 1], refs=refs, ref_slot=slot[f:f + 1],
                                    mv_grid=grid[f:f + 1], mv1_grid=mv1[f:f + 1]))
            wd = [one.coeff_plane(p) for p in range(3)]
            sel = {k: got[k + "_blocks"]["frame"] == f for k in ("luma", "chroma")}
            one_dec = [dec[0][sel["luma"]], dec[1][sel["luma"]], dec[2][sel["chroma"]], dec[3][sel["chroma"]]]
            wfin = _copy(one.finish(*one_dec, ref_slot_out=np.array([3], np.int32)))
            wpool = [one.pool_plane(p) for p in range(3)]
        finally:
            one.close()
        for p in range(3):
            kind = "luma" if p == 0 else "chroma"
            assert np.array_equal(gd[p][f], wd[p][0]), ("quantised plane", f, p)
            assert np.array_equal(got["recon%d" % p][f], want["recon%d" % p][0]), ("step recon", f, p)
            assert np.array_equal(got["pred%d" % p][f], want["pred%d" % p][0]), ("prediction", f, p)
            assert np.array_equal(engine.band_records(got[kind + "_blocks"], got[kind + "_res"], geom, p, f),
                                  engine.band_records(want[kind + "_blocks"], want[kind + "_res"], geom, p, 0)), \
                ("band records", f, p)
            assert np.array_equal(fin["recon%d" % p][f], wfin["recon%d" % p][0]), ("finish recon", f, p)
            assert np.array_equal(fin["bskip%d" % p][f], wfin["bskip%d" % p][0]), ("bskip", f, p)
            assert np.array_equal(pool[p][3 + f], wpool[p][3]), ("pool", f, p)
        for kind in ("luma", "chroma"):
            for k in PER_BLOCK:
                a, b = got["%s_%s" % (kind, k)][sel[kind]], want["%s_%s" % (kind, k)]
                assert np.array_equal(a, b, equal_nan=k == "skip_diff"), (kind, k, f)
            a = got[kind + "_late_skip"][sel[kind]].view(np.float64)
            assert np.array_equal(a, want[kind + "_late_skip"].view(np.float64)), (kind, "late skip", f)
        gs, ws = _frame_stream(got, f), _frame_stream(want, 0)
        for k in gs:
            assert gs[k].tobytes() == ws[k].tobytes(), ("stream", k, f)
        assert np.array_equal(fin["dering_levels"][f], wfin["dering_levels"][0]), ("searched levels", f)


def test_frames_match_oracles_at_their_own_settings():
    """inter = 1 with host prediction, late_skip and the searching finishing pass: each frame against inter_chain,
    the late-skip driver and the searching finishing oracle (level search with the frame's own coded_quantizer and
    dering_lambda) at that frame's settings."""
    from daala_b200.frame import Geometry
    from tests.test_gpu_engine_inter import _compare
    from tests.test_gpu_engine_late_skip import _check_against
    from tests.test_gpu_engine_quantizer_range import _check_finish, _finish_want, _p_frames
    if oracle_lib.load_ref() is None or inter_finish_oracle.load_ref() is None or late_skip_oracle.load_ref() is None:
        pytest.skip("needs the reference build (level search, finishing and late-skip drivers)")
    geom = Geometry(200, 130)
    F = 3
    ss, rec = _records([(FINEST, 1), (COARSEST, 1), (4, 0)])
    planes, pred, bsize = _p_frames(geom, F, seed=71)
    eng = _engine(geom, F, ss[0], inter=1, symbol_stream=2, late_skip=1, inter_finish=2, frame_quant=1)
    try:
        out = _copy(eng.encode(planes, bsize, pred=pred, frame_quant=rec))
        d = [eng.coeff_plane(p) for p in range(3)]
        md = [eng.pred_coeff_plane(p) for p in range(3)]
        frames = [([planes[p][f] for p in range(3)], [pred[p][f] for p in range(3)], bsize[f]) for f in range(F)]
        lib, prefix = late_skip_oracle.load()
        maps = []
        for f, s in enumerate(ss):
            _compare(out, d, md, geom, frames, s["q0"], s["q4"], frame_ids=[f], use_masking=s["masking"], lam=s["lam"],
                     qm=s["qm"], qm_inv=s["qm_inv"])
            maps.append([late_skip_oracle.plane(lib, prefix, planes[p][f], pred[p][f], d[p][f], geom, bsize[f], p, s["q0"],
                                                s["q4"], s["flat"], s["masking"], s["cq"]) for p in range(3)])
        _check_against(out, maps, F, 0)
        dec = _decisions(out, geom, F, seed=72)
        got = _copy(eng.finish(*dec[:4]))
        for f, s in enumerate(ss):
            want = _finish_want(geom, f + 1, s, planes, out, d, md, bsize, dec)[f]
            _check_finish({k: v[f:f + 1] for k, v in got.items()}, [want], 1, ("frame", f))
    finally:
        eng.close()


def test_uniform_records_equal_the_engine_without_them():
    """Records that all equal the config: the same outputs as a frame_quant = 0 engine, and the same launches."""
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    geom = Geometry(328, 200)
    F = 2
    s = settings(5, 0, 1)
    rec = engine.frame_quant_records([s["q0"]] * F, s["cq"], s["dering_lambda"], s["q4"])
    refs, planes, bsize, grid, mv1, slot = _inputs(geom, F, seed=90)
    res = []
    for fq in (0, 1):
        eng = _engine(geom, F, s, frame_quant=fq, **MC)
        try:
            out = _copy(eng.encode(planes, bsize, refs=refs, ref_slot=slot, mv_grid=grid, mv1_grid=mv1,
                                   frame_quant=rec if fq else None))
            dec = _decisions(out, geom, F, seed=91)
            out.update({"fin_" + k: v for k, v in _copy(eng.finish(*dec[:4])).items()})
            out["coeffs"] = [eng.coeff_plane(p) for p in range(3)]
            res.append((out, eng.launches_per_step()))
        finally:
            eng.close()
    (a, na), (b, nb) = res
    assert na == nb
    for k in a:
        if k == "coeffs":
            assert all(np.array_equal(x, y) for x, y in zip(a[k], b[k])), k
        else:
            assert np.array_equal(a[k], b[k], equal_nan=k.endswith("skip_diff")), k


def test_refusals_before_any_copy():
    from daala_b200 import _native, engine
    from daala_b200.frame import Geometry
    geom = Geometry(200, 130)
    s = settings(3, 0, 1)
    for bad in (dict(frame_quant=1), dict(frame_quant=2, inter=1)):
        with pytest.raises(RuntimeError, match="frame_quant is 0 or 1"):
            _engine(geom, 1, s, **bad)
    F = 2
    rec = engine.frame_quant_records([s["q0"]] * F, s["cq"], s["dering_lambda"], s["q4"])
    refs, planes, bsize, grid, mv1, slot = _inputs(geom, F, seed=95)
    eng = _engine(geom, F, s, frame_quant=1, **MC)
    plain = _engine(geom, F, s, **MC)
    try:
        ok = _copy(eng.encode(planes, bsize, refs=refs, ref_slot=slot, mv_grid=grid, mv1_grid=mv1, frame_quant=rec))
        before = [eng.coeff_plane(p) for p in range(3)]
        cases = [(None, "records")]
        for field, value in (("q0", 0), ("q0", 8192), ("coded_quantizer", 0), ("coded_quantizer", 64),
                             ("dering_lambda", -1.0), ("dering_lambda", np.inf), ("dering_lambda", np.nan)):
            r = rec.copy()
            r[field][1] = value
            cases.append((r, field))
        r = rec.copy()
        r["pvq_qm_q4"][1, 2, 29] = 0
        cases.append((r, "pvq_qm_q4"))
        for r, what in cases:
            with pytest.raises(_native.CudaError, match=what):
                eng.encode(planes, bsize, refs=refs, ref_slot=slot, mv_grid=grid, mv1_grid=mv1, frame_quant=r)
            assert all(np.array_equal(eng.coeff_plane(p), before[p]) for p in range(3)), what
        with pytest.raises(_native.CudaError, match="frame_quant needs an engine"):
            plain.encode(planes, bsize, refs=refs, ref_slot=slot, mv_grid=grid, mv1_grid=mv1, frame_quant=rec)
        # the finish limit is the step's: DAALA_B200_KF_FINISH_DC_LIMIT / the largest dc_quant of its records
        _, limit = engine.frame_quant_derive(rec)
        dec = [np.zeros(len(ok["luma_dc"]), np.uint8), ok["luma_dc"].copy(), np.zeros(len(ok["chroma_dc"]), np.uint8),
               ok["chroma_dc"].copy()]
        dec[1][0] = limit
        eng.finish(*dec)
        dec[1][0] = limit + 1
        with pytest.raises(_native.CudaError, match="dc"):
            eng.finish(*dec)
    finally:
        eng.close()
        plain.close()


def test_pipelined_sequence_in_one_engine():
    """One synthetic sequence (b_frames = 2, I P B B P B B P B B) on gop.pipelined_steps: the keyframe from the keyframe
    engine into the pool, then every step (an anchor with the B frames coded before it) as one batch of one mc_next +
    frame_quant engine, P and B frames at their own quantizers, resident pool, anchors stored in their SELF buffer.
    Every prediction equals predict3 on the oracle's running pictures and every finish the finishing oracle at the
    frame's own q0 / pvq_qm_q4."""
    from daala_b200 import engine, gop, interfinish, synth
    from daala_b200.frame import Geometry
    from tests import bframe_oracle
    from tests.test_gpu_engine_bframes import _pack
    lib = bframe_oracle.load()
    if lib is None or inter_finish_oracle.load() is None:
        pytest.skip("needs the reference build with the three-picture prediction hook")
    geom = Geometry(200, 130)
    order = gop.coding_order(10, 2)
    steps = gop.pipelined_steps(order)
    assert [len(s) for s in steps] == [1, 1, 3, 3, 2]
    qs = {gop.P_FRAME: settings(3, 0, 1), gop.B_FRAME: settings(5, 0, 1)}
    F = 3
    src = {n: synth.pad_planes(synth.frame(geom.pic_w, geom.pic_h, f=n, seed=500 + n)[0], geom) for n in range(10)}
    key = engine.KeyframeEngine(geom, nframes=1, q0=qs[gop.P_FRAME]["q0"], pvq_qm_q4=qs[gop.P_FRAME]["q4"])
    eng = _engine(geom, F, qs[gop.P_FRAME], inter=1, inter_mc=1, mc_next=1, inter_finish=1, frame_quant=1, mc_refs=4)
    fin_lib, prefix = inter_finish_oracle.load()
    pics = {}
    try:
        for k, step in enumerate(steps):
            if step[0].type == gop.I_FRAME:
                kout = _copy(key.encode([src[step[0].number][p][None] for p in range(3)],
                                        synth.block_size_map(geom, "mixed", seed=1)[None]))
                eng.pool_load(step[0].refs[gop.SELF], [kout["recon%d" % p][0] for p in range(3)])
                eng.wait()
                pics[step[0].refs[gop.SELF]] = [kout["recon%d" % p][0] for p in range(3)]
                continue
            fr = step + [step[-1]] * (F - len(step))   # a short step repeats its last frame
            ss = [qs[f.type] for f in fr]
            rec = engine.frame_quant_records([s["q0"] for s in ss], [s["cq"] for s in ss],
                                             [s["dering_lambda"] for s in ss], np.stack([s["q4"] for s in ss]))
            grids = [synth.mv_grid_b(geom, seed=600 + 10 * k + i, p_next=0.0 if f.type == gop.P_FRAME else 0.3)
                     for i, f in enumerate(fr)]
            grid, mv1 = _pack(grids)
            bsize = np.stack([synth.block_size_map(geom, "mixed", seed=700 + 10 * k + i) for i in range(F)])
            slot = np.array([gop.pool_slots(f) for f in fr], np.int32)
            out = _copy(eng.encode([np.stack([src[f.number][p] for f in fr]) for p in range(3)], bsize, ref_slot=slot,
                                   mv_grid=grid, mv1_grid=mv1, resident=True, frame_quant=rec))
            for i, f in enumerate(fr):
                want = bframe_oracle.predict3(lib, geom, *(pics[s] for s in slot[i]), *grids[i])
                for p in range(3):
                    assert np.array_equal(out["pred%d" % p][i], want[p]), ("prediction", f.number, p)
            d = [eng.coeff_plane(p) for p in range(3)]
            md = [eng.pred_coeff_plane(p) for p in range(3)]
            dec = _decisions(out, geom, F, seed=800 + k)
            store = np.array([f.refs[gop.SELF] if f.kept and i == 0 else -1 for i, f in enumerate(fr)], np.int32)
            got = _copy(eng.finish(*dec[:5], ref_slot_out=store))
            for i, f in enumerate(fr):
                s = ss[i]
                dq, bskip = [], []
                for p in range(3):
                    blocks, skip, dc = (out["luma_blocks"], dec[0], dec[1]) if p == 0 else (out["chroma_blocks"], dec[2],
                                                                                             dec[3])
                    dq.append(interfinish.patch(d[p][i], md[p][i], blocks, skip, dc, i, p, s["q0"], s["q4"]))
                    bskip.append(interfinish.skip_map(blocks, skip, dc, i, p, geom))
                recs, _ = inter_finish_oracle.finish(fin_lib, prefix, dq, geom, bsize[i], s["q0"], dec[4][i], bskip)
                for p in range(3):
                    assert np.array_equal(got["recon%d" % p][i], recs[p]), ("finish", f.number, p)
                if store[i] >= 0:
                    pics[int(store[i])] = list(recs)
        pool = [eng.pool_plane(p) for p in range(3)]
        for buf, planes in pics.items():
            for p in range(3):
                assert np.array_equal(pool[p][buf], planes[p]), (buf, p)
    finally:
        key.close()
        eng.close()
