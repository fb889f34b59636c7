"""The keyframe and P-frame engines across the encoder's quantizer range, with the settings the reference encoder itself
chooses (tests/golden/encoder_settings.npz, captured through its public API by make_golden.py settings): state.quantizer,
coded_quantizer, the per-plane, per-band pvq_qm_q4 table it interpolates for the quantizer and activity masking,
state.qm / qm_inv (HVS or flat) and dering_lambda.  Every kernel that indexes pvq_qm_q4 sees a table whose entries differ
from band to band and plane to plane, so an index off by one band changes the result.

Sweep: the eight quantizer settings of make_golden.SETTINGS_QUANT (keyframe coded quantizers 4..60, P frames 6..63,
q0 12..8191) times three configurations (masking on / off with the HVS matrix, masking on with the flat matrix).
The first tests need no GPU."""
import math
import os

import numpy as np
import pytest

from tests import frame_oracle, inter_finish_oracle, late_skip_oracle, oracle_lib
from tests.golden import make_golden

HERE = os.path.dirname(os.path.abspath(__file__))
SETTINGS = dict(np.load(os.path.join(HERE, "golden", "encoder_settings.npz")))
NPOINTS, NCONFIGS = len(make_golden.SETTINGS_QUANT), len(make_golden.SETTINGS_CONFIGS)
SWEEP = [(p, c) for p in range(NPOINTS) for c in range(NCONFIGS)]
FINEST, COARSEST = 0, NPOINTS - 1


def settings(point, config, frame):
    """Engine and oracle arguments of one sweep point; frame 0 = the keyframe's settings, 1 = the P frame's."""
    masking, qm = (int(v) for v in SETTINGS["configs"][config])
    name = "hvs" if qm else "flat"
    return dict(q0=int(SETTINGS["quantizer"][point, config, frame]), q4=SETTINGS["pvq_qm_q4"][point, config, frame],
                cq=int(SETTINGS["coded_quantizer"][point, config, frame]), masking=masking, flat=1 - qm,
                qm=SETTINGS["qm_" + name], qm_inv=SETTINGS["qm_inv_" + name],
                lam=float(SETTINGS["pvq_norm_lambda"][point, config, frame]),
                dering_lambda=float(SETTINGS["dering_lambda"][point, config, frame]))


def _engine(geom, F, s, **kw):
    from daala_b200 import engine
    return engine.KeyframeEngine(geom, nframes=F, q0=s["q0"], use_masking=s["masking"], lam=s["lam"], pvq_qm_q4=s["q4"],
                                 qm=s["qm"], qm_inv=s["qm_inv"], coded_quantizer=s["cq"], qm_is_flat=s["flat"],
                                 dering_lambda=s["dering_lambda"], **kw)


def _ids(points):
    return ["q%d-%s" % (make_golden.SETTINGS_QUANT[p], ("hvs-masking", "hvs", "flat-masking")[c]) for p, c in points]


# ---- no GPU -------------------------------------------------------------------------------------------------------

def test_fixture_equals_a_fresh_capture():
    ref = oracle_lib.load_ref()
    if ref is None:
        pytest.skip("needs the reference build")
    assert tuple(SETTINGS["quant"]) == make_golden.SETTINGS_QUANT
    assert [tuple(c) for c in SETTINGS["configs"]] == list(make_golden.SETTINGS_CONFIGS)
    for p, quant in enumerate(make_golden.SETTINGS_QUANT):
        for c, (masking, qm) in enumerate(make_golden.SETTINGS_CONFIGS):
            got = make_golden.capture_settings(ref, quant, masking, qm)
            for k in ("quantizer", "coded_quantizer", "pvq_qm_q4", "pvq_norm_lambda", "dering_lambda"):
                assert np.array_equal(got[k], SETTINGS[k][p, c]), (quant, masking, qm, k)
            for f in range(2):
                assert np.array_equal(got["qm"][f], SETTINGS["qm_hvs" if qm else "qm_flat"])
                assert np.array_equal(got["qm_inv"][f], SETTINGS["qm_inv_hvs" if qm else "qm_inv_flat"])


def test_matrices_are_init_qm_of_the_base_matrices():
    from daala_b200 import pvq
    inp = pvq.qm_inputs()
    for name in ("hvs", "flat"):
        qm, qm_inv = pvq.init_qm(inp["qm8_" + name], inp)
        assert np.array_equal(SETTINGS["qm_" + name], qm) and np.array_equal(SETTINGS["qm_inv_" + name], qm_inv), name
        want = pvq.default_qm(name == "hvs")
        assert np.array_equal(want[0], qm) and np.array_equal(want[1], qm_inv), name
    assert not np.array_equal(SETTINGS["qm_hvs"], SETTINGS["qm_flat"])


def test_quantizers_follow_the_coded_quantizer_map():
    """state.quantizer is the coded quantizer's entry of OD_CODED_QUANTIZER_MAP_Q4, trunc(e^((c - 6.235) * .10989525)
    * 16) (src/quantizer.c); the sweep covers the ends of the range and od_compute_dist's interpolated region."""
    q, cq = SETTINGS["quantizer"], SETTINGS["coded_quantizer"]
    for c in np.unique(cq):
        assert (q[cq == c] == int(math.exp((int(c) - 6.235) * .10989525) * 16)).all(), c
    ref = oracle_lib.load_ref()
    if ref is not None:
        for c in np.unique(cq):
            assert (q[cq == c] == ref.od_codedquantizer_to_quantizer(int(c))).all(), c
    assert (cq[..., 1] > cq[..., 0]).all()                      # the P frame is coarser than its keyframe
    assert q.min() == 12 and q.max() == 8191 and cq.max() == 63
    assert ((cq >= 36) & (cq <= 47)).any()
    # the tables: not constant across bands or planes, and they depend on masking, not on the matrix
    q4 = SETTINGS["pvq_qm_q4"]
    assert (q4.max(axis=-1) > q4.min(axis=-1)).all() and (q4[..., 0, :] != q4[..., 1, :]).any()
    assert np.array_equal(q4[:, 0], q4[:, 2]) and not np.array_equal(q4[:, 0], q4[:, 1])
    assert np.array_equal(q4[..., 0, :, :], q4[..., 1, :, :])   # set on keyframes only


def test_lambdas():
    from daala_b200 import pvq
    assert (SETTINGS["pvq_norm_lambda"] == pvq.PVQ_LAMBDA).all()
    dl = SETTINGS["dering_lambda"]
    assert (dl > 0).all() and (np.diff(dl[:, 0, 0]) > 0).all() and (dl[..., 1] > dl[..., 0]).all()


def test_qm_index_is_the_reference_one():
    """The index of a band's pvq_qm_q4 entry that the kernels and oracle drivers compute by hand,
    bs * (bs + 1) + band - band / 3 (band 0 = DC), is the reference's od_qm_get_index, and the DC quantisers of the
    finishing pass and late skip (interfinish.dc_quant, lateskip.dc_quant) read entry od_qm_get_index(bs, 0)."""
    from daala_b200 import interfinish, lateskip
    ref = oracle_lib.load_ref()
    if ref is None:
        pytest.skip("needs the reference build")
    q4 = SETTINGS["pvq_qm_q4"][COARSEST, 0, 1]
    q0 = int(SETTINGS["quantizer"][COARSEST, 0, 1])
    for bs in range(5):
        for band in range(1 + (1, 4, 7, 9, 9)[bs]):
            assert bs * (bs + 1) + band - band // 3 == ref.od_qm_get_index(bs, band), (bs, band)
        for pli in range(3):
            want = max(1, (q0 * int(q4[pli][ref.od_qm_get_index(bs, 0)])) >> 4)
            assert interfinish.dc_quant(q0, q4, pli, bs) == want
            assert int(lateskip.dc_quant(q0, q4, pli, bs)) == want


# ---- GPU: keyframes -----------------------------------------------------------------------------------------------

def _kf_frames(geom, F, seed, noise=False):
    from daala_b200 import synth
    rng = np.random.default_rng(seed)
    frames = []
    for f in range(F):
        if noise:
            planes = [rng.integers(0, 256, size=geom.plane_shape(p), dtype=np.uint8) for p in range(3)]
        else:
            planes = synth.pad_planes(synth.frame(geom.pic_w, geom.pic_h, f=f + seed)[0], geom)
        frames.append((planes, synth.block_size_map(geom, "mixed", seed=seed + f)))
    return frames


def _run_keyframes(geom, F, point, config, seed, noise=False):
    """Keyframe engine (dering = 2, symbol_stream = 1) at the sweep point's keyframe settings, against keyframe_chain with
    the level search: reconstruction, quantised planes, band records, searched levels and the symbol stream."""
    from daala_b200 import engine, symbols
    from tests.test_gpu_symbol_stream import _assert_matches_reference, _oracle_stream
    from tests.test_gpu_engine import _coding_tables
    ref = oracle_lib.load_ref()
    if ref is None:
        pytest.skip("needs the reference build (the level search of keyframe_chain)")
    s = settings(point, config, 0)
    frames = _kf_frames(geom, F, seed, noise)
    eng = _engine(geom, F, s, dering=2, symbol_stream=1)
    try:
        out = eng.encode([np.stack([fr[0][p] for fr in frames]) for p in range(3)], np.stack([fr[1] for fr in frames]),
                         stream=True)
        out = {k: np.array(v) for k, v in out.items()}
        coeffs = [eng.coeff_plane(p) for p in range(3)]
    finally:
        eng.close()
    _assert_matches_reference(out, F, "keyframes")
    tabs = _coding_tables()
    for f in range(F):
        want = frame_oracle.keyframe_chain(ref, "ref", frames[f][0], geom, frames[f][1], s["q0"], s["q4"], s["masking"],
                                           lam=s["lam"], qm=s["qm"], qm_inv=s["qm_inv"], symbols=True,
                                           dering_search=dict(coded_quantizer=s["cq"], dering_lambda=s["dering_lambda"],
                                                              qm=1 - s["flat"]))
        assert np.array_equal(out["dering_levels"][f], want[0]["dering_levels"]), ("levels", f)
        for pli in range(3):
            kind = "luma" if pli == 0 else "chroma"
            got = engine.band_records(out[kind + "_blocks"], out[kind + "_res"], geom, pli, f)
            assert np.array_equal(got, want[pli]["rec"]), ("band records", f, pli)
            assert np.array_equal(coeffs[pli][f], want[pli]["dq"]), ("quantised plane", f, pli)
            assert np.array_equal(out["recon%d" % pli][f], want[pli]["recon"]), ("recon", f, pli)
        _, parts = _oracle_stream(want, geom, frames[f][1], tabs)
        bad = symbols.stream_equal(out, symbols.concat_frames([parts]), [f], [0])
        assert not bad, ("stream", f, bad[:8])
    return out


def _assert_mostly_uncoded(out):
    """At the coarsest setting nearly every band codes K = 0 (the comparisons before this one hold for them all): in
    each plane kind more than 90 % of the bands."""
    for kind in ("luma", "chroma"):
        nb = np.array([1, 4, 7, 9, 9])[out[kind + "_blocks"]["bs"]]
        k = out[kind + "_res"][..., 3][np.arange(9)[None, :] < nb[:, None]]
        assert (k == 0).mean() > 0.9, (kind, (k == 0).mean())


@pytest.mark.gpu
@pytest.mark.parametrize("point,config", SWEEP, ids=_ids(SWEEP))
def test_keyframes_match_oracle(point, config):
    from daala_b200.frame import Geometry
    out = _run_keyframes(Geometry(200, 130), 1, point, config, seed=3 + point)
    if point == COARSEST:
        _assert_mostly_uncoded(out)


@pytest.mark.gpu
@pytest.mark.parametrize("point", [FINEST + 2, COARSEST - 2])
def test_keyframes_match_oracle_two_frames(point):
    from daala_b200.frame import Geometry
    _run_keyframes(Geometry(328, 200), 2, point, 0, seed=20 + point)


@pytest.mark.gpu
def test_keyframe_wide_pulses_at_the_finest_quantizer():
    """The finest setting on noise: bands with K > 127 occur, and their 16-bit pulses match the oracle's."""
    from daala_b200 import symbols
    from daala_b200.frame import Geometry
    out = _run_keyframes(Geometry(200, 130), 1, FINEST, 0, seed=5, noise=True)
    r = symbols.read_frame(out, 0)
    k = r["bands"][:, 3]
    print("finest keyframe setting (q0 %d) on noise: largest K %d, %d bands with K > 127"
          % (settings(FINEST, 0, 0)["q0"], k.max(), (k > 127).sum()))
    assert (k > 127).any()
    wide = np.nonzero(k > 127)[0]
    assert max(np.abs(r["pulses"][q]).max() for q in wide) > 127


# ---- GPU: P frames ------------------------------------------------------------------------------------------------

def _p_frames(geom, F, seed):
    from tests.test_gpu_engine_inter_finish import _frames
    return _frames(geom, F, seed)


def _finish_want(geom, F, s, planes, out, d, md, bsize, dec):
    """Per frame the oracle's (recon planes, levels, skip maps) of the searching finishing pass for decisions dec[:4]:
    the numpy patch and skip map, the reference's inverse up to the SB-edge postfilter, its level search with the
    encoder's coded quantizer and dering_lambda, then the finishing driver at those levels."""
    from daala_b200 import interfinish
    from tests import test_dering_search as ds
    ref, fin = oracle_lib.load_ref(), inter_finish_oracle.load_ref()
    ls, ld, cs, cd = dec[:4]
    res = []
    for f in range(F):
        dq, bskip = [], []
        for p in range(3):
            blocks, skip, dc = (out["luma_blocks"], ls, ld) if p == 0 else (out["chroma_blocks"], cs, cd)
            dq.append(interfinish.patch(d[p][f], md[p][f], blocks, skip, dc, f, p, s["q0"], s["q4"]))
            bskip.append(np.ascontiguousarray(interfinish.skip_map(blocks, skip, dc, f, p, geom)))
        c = frame_oracle.inverse_plane(ref, "ref", dq[0], geom, 0, bsize[f], 0, lapped_only=True)
        c = np.ascontiguousarray(c, np.int32)
        ref.od_apply_postfilter_frame_sbs(oracle_lib.addr(c), c.shape[1], geom.nhsb, geom.nvsb, 0, 0)
        cdf = np.zeros((11, 6), np.uint16)
        cdf[:] = 32 * np.arange(1, 7, dtype=np.uint16)
        levels, _ = ds.ref_search(ref, np.ascontiguousarray(planes[0][f], np.uint8), c, geom.nhsb, geom.nvsb, s["q0"],
                                  s["masking"], 0, s["dering_lambda"], bskip[0], cdf, qm=1 - s["flat"],
                                  coded_quantizer=s["cq"])
        levels = levels.reshape(geom.nvsb, geom.nhsb)
        recs, applied = inter_finish_oracle.finish(fin, "ref", dq, geom, bsize[f], s["q0"], levels, bskip)
        assert np.array_equal(applied, levels)
        res.append((recs, levels, bskip))
    return res


def _check_finish(got, want, F, what):
    for f in range(F):
        recs, levels, bskip = want[f]
        assert np.array_equal(got["dering_levels"][f], levels), (what, "levels", f, got["dering_levels"][f], levels)
        for p in range(3):
            assert np.array_equal(got["bskip%d" % p][f], bskip[p]), (what, "bskip", f, p)
            assert np.array_equal(got["recon%d" % p][f], recs[p]), (what, "recon", f, p)


def _run_p_frames(geom, F, point, config, seed):
    """P-frame engine (inter = 1, symbol_stream = 2, late_skip = 1, inter_finish = 2) at the sweep point's P-frame
    settings: the residual against inter_chain, the late-skip records against the late-skip driver (also in stream
    order), and a finishing pass with seeded decisions against the searching oracle.  Returns (engine, step)."""
    from daala_b200 import symbols
    from tests.test_gpu_engine_inter import _compare
    from tests.test_gpu_engine_inter_finish import _decisions
    from tests.test_gpu_engine_late_skip import FIELDS, _as_array, _check_against
    if oracle_lib.load_ref() is None or inter_finish_oracle.load_ref() is None or late_skip_oracle.load_ref() is None:
        pytest.skip("needs the reference build (level search, finishing and late-skip drivers)")
    s = settings(point, config, 1)
    planes, pred, bsize = _p_frames(geom, F, seed)
    eng = _engine(geom, F, s, inter=1, symbol_stream=2, late_skip=1, inter_finish=2)
    try:
        out = {k: np.array(v) for k, v in eng.encode(planes, bsize, pred=pred).items()}
        d = [eng.coeff_plane(p) for p in range(3)]
        md = [eng.pred_coeff_plane(p) for p in range(3)]
        frames = [([planes[p][f] for p in range(3)], [pred[p][f] for p in range(3)], bsize[f]) for f in range(F)]
        _compare(out, d, md, geom, frames, s["q0"], s["q4"], use_masking=s["masking"], lam=s["lam"], qm=s["qm"],
                 qm_inv=s["qm_inv"])
        lib, prefix = late_skip_oracle.load()
        maps = [[late_skip_oracle.plane(lib, prefix, planes[p][f], pred[p][f], d[p][f], geom, bsize[f], p, s["q0"], s["q4"],
                                        s["flat"], s["masking"], s["cq"]) for p in range(3)] for f in range(F)]
        _check_against(out, maps, F, s["flat"])
        perm = symbols.stream_to_classic(out)
        classic = np.concatenate([out["luma_late_skip"], out["chroma_late_skip"]])
        assert np.array_equal(_as_array(out["sym_late_skip"][:len(perm)]), _as_array(classic[perm]))
        assert len(FIELDS) == 4
        dec = _decisions(out, geom, F, seed=seed)
        got = {k: np.array(v) for k, v in eng.finish(*dec[:4]).items()}
        _check_finish(got, _finish_want(geom, F, s, planes, out, d, md, bsize, dec), F, "seeded decisions")
    except BaseException:
        eng.close()
        raise
    return eng, s, (planes, pred, bsize, out, d, md)


@pytest.mark.gpu
@pytest.mark.parametrize("point,config", SWEEP, ids=_ids(SWEEP))
def test_p_frames_match_oracle(point, config):
    from daala_b200.frame import Geometry
    eng, _, step = _run_p_frames(Geometry(200, 130), 1, point, config, seed=40 + point)
    eng.close()
    if point == COARSEST:
        _assert_mostly_uncoded(step[3])


@pytest.mark.gpu
@pytest.mark.parametrize("point", [FINEST + 2, COARSEST - 2])
def test_p_frames_match_oracle_two_frames(point):
    from daala_b200.frame import Geometry
    eng, _, _ = _run_p_frames(Geometry(328, 200), 2, point, 2, seed=60 + point)
    eng.close()


def _ctmp_peak(geom, s, dq, bskip, bsize):
    """The largest |sample| of state->ctmp over the three planes for patched coefficient planes dq: the reference's
    inverse and split postfilters, then its superblock-edge postfilter -- what src/encode.c:2703-2705 copies into the
    int16 deringing input state->etmp."""
    ref = oracle_lib.load_ref()
    peak = 0
    for p in range(3):
        c = np.ascontiguousarray(frame_oracle.inverse_plane(ref, "ref", dq[p], geom, p, bsize, 0, lapped_only=True), np.int32)
        x = geom.xdec[p]
        ref.od_apply_postfilter_frame_sbs(oracle_lib.addr(c), c.shape[1], geom.nhsb, geom.nvsb, x, x, s["cq"],
                                          oracle_lib.addr(bskip[p]), bskip[p].shape[1])
        peak = max(peak, int(np.abs(c.astype(np.int64)).max()))
    return peak


def _largest_int16_dc(geom, s, out, d, md, bsize, dec, lst, i, sign, limit):
    """The largest |dc| <= limit of block i of list lst (0 luma, 1 chroma) of frame 0, the other decisions dec[:4]
    fixed, for which every sample of state->ctmp still fits int16 (the bound of the pass's exactness,
    include/daala_b200.h)."""
    from daala_b200 import interfinish
    blocks = out["chroma_blocks"] if lst else out["luma_blocks"]
    b = blocks[i]
    pli, y0, x0 = int(b["pli"]), int(b["y0"]), int(b["x0"])
    dcq = interfinish.dc_quant(s["q0"], s["q4"], pli, int(b["bs"]))
    dq, bskip = [], []
    for p in range(3):
        bl, skip, dc = (out["luma_blocks"], dec[0], dec[1]) if p == 0 else (out["chroma_blocks"], dec[2], dec[3])
        dq.append(interfinish.patch(d[p][0], md[p][0], bl, skip, dc, 0, p, s["q0"], s["q4"]))
        bskip.append(np.ascontiguousarray(interfinish.skip_map(bl, skip, dc, 0, p, geom)))

    def fits(v):
        dq[pli][y0, x0] = int(md[pli][0][y0, x0]) + sign * v * dcq
        return _ctmp_peak(geom, s, dq, bskip, bsize[0]) <= 32767

    lo, hi = abs(int(dec[1 + 2 * lst][i])), limit
    assert fits(lo) and not fits(hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if fits(mid) else (lo, mid)
    return lo


@pytest.mark.gpu
def test_finish_dc_limit_at_the_coarsest_quantizer():
    """The coarsest P-frame setting (q0 8191 and its table).  A DC index of exactly the finishing pass's limit,
    DAALA_B200_KF_FINISH_DC_LIMIT / (the largest DC quantiser of the table, entries od_qm_get_index(bs, 0)), is accepted,
    one more is refused before anything runs.  The pass is exact while state->ctmp fits int16: on the block with the
    largest DC quantiser and on a luma block of the largest size, the largest DC index (either sign) that keeps it there finishes as the
    oracle does, levels searched included."""
    from daala_b200 import _native
    from daala_b200.frame import Geometry
    geom = Geometry(200, 130)
    eng, s, (planes, pred, bsize, out, d, md) = _run_p_frames(geom, 1, COARSEST, 0, seed=80)
    try:
        dq_max = max((s["q0"] * int(s["q4"][p][bs * (bs + 1)])) >> 4 for p in range(3) for bs in range(5))
        limit = (1 << 30) // dq_max
        nl, nc = len(out["luma_dc"]), len(out["chroma_dc"])
        base = (np.zeros(nl, np.uint8), out["luma_dc"].copy(), np.zeros(nc, np.uint8), out["chroma_dc"].copy())
        lb, cb = out["luma_blocks"], out["chroma_blocks"]
        dcq = [np.array([(s["q0"] * int(s["q4"][int(b["pli"])][int(b["bs"]) * (int(b["bs"]) + 1)])) >> 4 for b in blocks])
               for blocks in (lb, cb)]
        lst = 0 if dcq[0].max() >= dcq[1].max() else 1
        i = int(np.argmax(dcq[lst]))
        assert dcq[lst][i] == dq_max
        for sign in (1, -1):
            dec = [a.copy() for a in base]
            dec[1 + 2 * lst][i] = sign * limit
            eng.finish(*dec)
        before = eng.counts().copy()
        dec = [a.copy() for a in base]
        dec[1 + 2 * lst][i] = limit + 1
        eng.prepare_finish(*dec)
        with pytest.raises(_native.CudaError):
            eng.finish_submit()
        assert b"|dc|" in eng.L.daala_b200_kf_error(eng.kf)
        assert np.array_equal(eng.counts(), before)
        big = int(np.argmax(lb["bs"]))
        for blk_list, blk in ((lst, i), (0, big)):
            for sign in (1, -1):
                top = _largest_int16_dc(geom, s, out, d, md, bsize, base, blk_list, blk, sign, limit)
                print("block %d of list %d, sign %+d: largest |dc| with state->ctmp in int16: %d" % (blk, blk_list, sign, top))
                dec = [a.copy() for a in base]
                dec[1 + 2 * blk_list][blk] = sign * top
                got = {k: np.array(v) for k, v in eng.finish(*dec).items()}
                _check_finish(got, _finish_want(geom, 1, s, planes, out, d, md, bsize, dec), 1, ("int16 bound", blk, sign))
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("point", [FINEST, 2, COARSEST])
def test_real_encoder_p_frame(point):
    """The reference encoder's first P frame at the sweep point's quantizer setting (200x130, complexity 7): the engine
    given its motion-vector grid, reference pictures and block sizes predicts what the encoder predicted and, with the
    encoder's own P-frame q0 and pvq_qm_q4, codes what inter_chain codes."""
    from daala_b200.frame import Geometry
    from tests import inter_mc_oracle
    from tests.test_gpu_engine_inter import _compare
    from tests.test_gpu_engine_inter_mc import _ref, _run
    lib = _ref()
    geom = Geometry(200, 130)
    s = settings(point, 0, 1)
    (cap,) = inter_mc_oracle.capture_p_frames(lib, geom, 2, quant=make_golden.SETTINGS_QUANT[point])
    assert cap["same"]
    refs = [np.stack([cap[k][p] for k in ("gold", "prev")]) for p in range(3)]
    eng = _engine(geom, 1, s, inter=1, inter_mc=1)
    try:
        out = _run(eng, [cap["src"][p][None] for p in range(3)], cap["bsize"][None], refs, [[0, 0]],
                   [(cap["valid"], cap["mv"], cap["ref"])])
        for p in range(3):
            assert np.array_equal(out["pred%d" % p][0], cap["pred"][p]), ("prediction", p)
        _compare(out, [eng.coeff_plane(p) for p in range(3)], [eng.pred_coeff_plane(p) for p in range(3)], geom,
                 [(cap["src"], cap["pred"], cap["bsize"])], s["q0"], s["q4"], lam=s["lam"], qm=s["qm"], qm_inv=s["qm_inv"])
    finally:
        eng.close()
