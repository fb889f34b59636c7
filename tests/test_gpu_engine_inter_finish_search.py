"""The P-frame finishing pass with its deringing level search (config.inter_finish = 2; daala_b200_kf_finish,
csrc/kf_engine.cu + csrc/dering_search.cu): the levels of src/encode.c:2708-2811 for a P frame -- every filtered
candidate reads the frame's own skip map, a superblock without a coded luma 4x4 unit is not searched and does not
adapt the CDF, context 0 -- searched inside the pass's CUDA graph and applied there.

Oracle, per frame, composed from reference-bound pieces: the numpy patch and skip map (daala_b200/interfinish.py); the
reference's inverse up to the SB-edge postfilter on the patched luma plane (ctmp); the reference's own search loop
(oracle/ref_hooks_encode.c::oracle_ref_dering_search: od_compute_dist, od_dering, od_encode_cdf_cost / _adapt) on ctmp,
the source luma and the luma skip map, from fresh CDFs; then the frame driver inverse_frame_inter_finish at those
levels.  Bit-exact throughout."""
import numpy as np
import pytest

from tests import frame_oracle, inter_finish_oracle, oracle_lib
from tests import test_dering_search as ds
from tests.test_gpu_engine_inter_finish import Q4, _copy, _decisions, _frames, _step


def _engine(geom, F, q0, inter_finish=2, **kw):
    from daala_b200 import engine
    return engine.KeyframeEngine(geom, nframes=F, q0=q0, pvq_qm_q4=Q4, inter=1, inter_finish=inter_finish,
                                 coded_quantizer=q0, **kw)


def _ref_libs():
    ref, fin = oracle_lib.load_ref(), inter_finish_oracle.load_ref()
    if ref is None or fin is None:
        pytest.skip("needs the reference build (od_compute_dist, od_dering, od_encode_cdf_*, the finishing driver)")
    return ref, fin


def _want(geom, F, planes, out, d, md, bsize, q0, dec, lam, masking=1, qm_is_flat=0):
    """Per frame the oracle's (recon planes, levels, skip maps, coded superblocks) for the decisions dec[:4]."""
    from daala_b200 import interfinish
    ref, fin = _ref_libs()
    a = oracle_lib.addr
    ls, ld, cs, cd = dec[:4]
    res = []
    for f in range(F):
        dq, bskip = [], []
        for p in range(3):
            blocks, skip, dc = (out["luma_blocks"], ls, ld) if p == 0 else (out["chroma_blocks"], cs, cd)
            dq.append(interfinish.patch(d[p][f], md[p][f], blocks, skip, dc, f, p, q0, Q4))
            bskip.append(np.ascontiguousarray(interfinish.skip_map(blocks, skip, dc, f, p, geom)))
        c = frame_oracle.inverse_plane(ref, "ref", dq[0], geom, 0, bsize[f], 0, lapped_only=True)
        c = np.ascontiguousarray(c, np.int32)
        ref.od_apply_postfilter_frame_sbs(a(c), c.shape[1], geom.nhsb, geom.nvsb, 0, 0)
        cdf = np.zeros((11, 6), np.uint16)
        cdf[:] = 32 * np.arange(1, 7, dtype=np.uint16)
        src = np.ascontiguousarray(planes[0][f], np.uint8)
        levels, _ = ds.ref_search(ref, src, c, geom.nhsb, geom.nvsb, q0, masking, 0, lam, bskip[0], cdf,
                                  qm=0 if qm_is_flat else 1)
        levels = levels.reshape(geom.nvsb, geom.nhsb)
        recs, applied = inter_finish_oracle.finish(fin, "ref", dq, geom, bsize[f], q0, levels, bskip)
        assert np.array_equal(applied, levels)     # the search leaves uncoded superblocks at 0 itself
        res.append((recs, levels, bskip, interfinish.coded_superblocks(bskip[0], geom)))
    return res


def _check(got, want, F):
    for f in range(F):
        recs, levels, bskip, _ = want[f]
        assert np.array_equal(got["dering_levels"][f], levels), ("levels", f, got["dering_levels"][f], levels)
        for p in range(3):
            assert np.array_equal(got["bskip%d" % p][f], bskip[p]), ("bskip", f, p)
            assert np.array_equal(got["recon%d" % p][f], recs[p]), ("recon", f, p)


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,F,q0,masking,flat", [
    (200, 130, 2, 30, 1, 0),
    (328, 200, 2, 72, 1, 0),
    (1920, 1080, 1, 72, 1, 0),
    (1920, 1080, 1, 30, 1, 0),
    (328, 200, 2, 30, 0, 0),
    (200, 130, 2, 72, 1, 1),
])
def test_search_random_decisions_match_oracle(w, h, F, q0, masking, flat):
    """Seeded decisions (about 30 % skipped, DC jittered), with a superblock whose luma is all skipped but one chroma
    block is coded (not searched, not adapted: every later decision of the frame depends on that) and one whose only
    coded luma is a single 4x4 block (searched)."""
    from daala_b200.frame import Geometry
    _ref_libs()
    geom = Geometry(w, h)
    eng = _engine(geom, F, q0, use_masking=masking, qm_is_flat=flat)
    planes, pred, bsize = _frames(geom, F, seed=h + q0)
    out, d, md = _step(eng, planes, pred, bsize)
    dec = _decisions(out, geom, F, seed=w + q0)
    got = _copy(eng.finish(*dec[:4]))
    want = _want(geom, F, planes, out, d, md, bsize, q0, dec, eng.dering_lambda, masking, flat)
    _check(got, want, F)
    one, chroma_only = dec[5]["one"], dec[5]["chroma_only"]
    coded0 = want[0][3]
    assert not coded0[chroma_only] and coded0[one]
    assert got["dering_levels"][0][chroma_only] == 0
    if q0 == 72:
        assert got["dering_levels"].any()   # the coarse quantizer rings: some superblock is filtered
    eng.close()


@pytest.mark.gpu
def test_search_all_skipped_is_the_prediction():
    """skip = 1, dc = 0 everywhere: no superblock is coded, so none is searched; levels all 0, and the reconstruction
    is the prediction."""
    from daala_b200.frame import Geometry
    geom = Geometry(328, 200)
    F = 2
    eng = _engine(geom, F, 38)
    planes, pred, bsize = _frames(geom, F, seed=2)
    out, _, _ = _step(eng, planes, pred, bsize)
    nl, nc = len(out["luma_dc"]), len(out["chroma_dc"])
    got = eng.finish(np.ones(nl, np.uint8), np.zeros(nl, np.int32), np.ones(nc, np.uint8), np.zeros(nc, np.int32))
    assert not got["dering_levels"].any()
    for p in range(3):
        assert np.array_equal(got["recon%d" % p], pred[p]), p
        w4 = geom.plane_shape(p)[1] // 4
        assert got["bskip%d" % p][:, :, :w4].all()
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,F,q0", [(328, 200, 2, 72), (1920, 1080, 1, 30)])
def test_search_no_skips_matches_oracle(w, h, F, q0):
    """skip = 0, dc = qdc: all-zero skip maps, every superblock searched with context 0."""
    from daala_b200.frame import Geometry
    _ref_libs()
    geom = Geometry(w, h)
    eng = _engine(geom, F, q0)
    planes, pred, bsize = _frames(geom, F, seed=w)
    out, d, md = _step(eng, planes, pred, bsize)
    nl, nc = len(out["luma_dc"]), len(out["chroma_dc"])
    dec = (np.zeros(nl, np.uint8), out["luma_dc"], np.zeros(nc, np.uint8), out["chroma_dc"])
    got = _copy(eng.finish(*dec))
    want = _want(geom, F, planes, out, d, md, bsize, q0, dec, eng.dering_lambda)
    _check(got, want, F)
    for f in range(F):
        assert want[f][3].all() and not want[f][2][0].any()
    assert got["dering_levels"].any()
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,F,q0", [(328, 200, 2, 72), (1920, 1080, 1, 72)])
def test_search_equals_the_pass_given_the_searched_levels(w, h, F, q0):
    """No reference build: the searching pass equals an inter_finish = 1 pass of a second engine, given the same step,
    the same decisions and the searched levels.  The search's scratch exists only on the searching engine."""
    from daala_b200.frame import Geometry
    geom = Geometry(w, h)
    planes, pred, bsize = _frames(geom, F, seed=h)
    search, given = _engine(geom, F, q0), _engine(geom, F, q0, inter_finish=1)
    assert search.launches_per_step() == given.launches_per_step()
    assert search.buf.bytes_allocated > given.buf.bytes_allocated
    out, _, _ = _step(search, planes, pred, bsize)
    out1, _, _ = _step(given, planes, pred, bsize)
    for k in ("luma_dc", "chroma_dc", "recon0", "recon1", "recon2"):
        assert np.array_equal(out[k], out1[k]), k
    dec = _decisions(out, geom, F, seed=q0)
    got = _copy(search.finish(*dec[:4]))
    assert got["dering_levels"].any()
    ref = _copy(given.finish(*dec[:4], got["dering_levels"]))
    for k in ref:
        assert np.array_equal(got[k], ref[k]), k
    search.close()
    given.close()


@pytest.mark.gpu
def test_search_repeated_after_one_step():
    """Decisions A, then B, then A again after one step: the third pass repeats the first byte for byte (graph replay,
    nothing of the search carried over), and the step's planes and reconstruction are untouched."""
    from daala_b200.frame import Geometry
    geom = Geometry(328, 200)
    F, q0 = 2, 45
    eng = _engine(geom, F, q0)
    planes, pred, bsize = _frames(geom, F, seed=21)
    out, d, md = _step(eng, planes, pred, bsize)
    a, b = _decisions(out, geom, F, seed=1), _decisions(out, geom, F, seed=2)
    first = _copy(eng.finish(*a[:4]))
    second = _copy(eng.finish(*b[:4]))
    assert any(not np.array_equal(first[k], second[k]) for k in first)
    third = _copy(eng.finish(*a[:4]))
    for k in first:
        assert np.array_equal(first[k], third[k]), k
    for p in range(3):
        assert np.array_equal(eng.coeff_plane(p), d[p]) and np.array_equal(eng.pred_coeff_plane(p), md[p])
        assert np.array_equal(eng.recon_plane(p), out["recon%d" % p])
    eng.close()


@pytest.mark.gpu
def test_search_refusals():
    from daala_b200 import _native, engine
    from daala_b200.frame import Geometry
    geom = Geometry(200, 130)
    F, q0 = 1, 45
    with pytest.raises(RuntimeError, match="inter_finish"):
        engine.KeyframeEngine(geom, nframes=F, q0=q0, pvq_qm_q4=Q4, inter_finish=2)
    with pytest.raises(RuntimeError, match="inter_finish is 0, 1 or 2"):
        _engine(geom, F, q0, inter_finish=3)
    planes, pred, bsize = _frames(geom, F, seed=8)
    eng = _engine(geom, F, q0)
    out, _, _ = _step(eng, planes, pred, bsize)
    nl, nc = len(out["luma_dc"]), len(out["chroma_dc"])
    good = (np.zeros(nl, np.uint8), out["luma_dc"], np.zeros(nc, np.uint8), out["chroma_dc"])
    ref = _copy(eng.finish(*good))
    before = eng.counts().copy()
    eng.prepare_finish(*good, np.zeros((F, geom.nvsb, geom.nhsb), np.uint8))
    with pytest.raises(_native.CudaError):
        eng.finish_submit()
    assert b"dering_level must be NULL" in eng.L.daala_b200_kf_error(eng.kf)
    assert np.array_equal(eng.counts(), before)
    # nothing the refusal left behind changes the next pass
    again = _copy(eng.finish(*good))
    for k in ref:
        assert np.array_equal(ref[k], again[k]), k
    eng.close()
