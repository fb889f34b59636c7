"""Lossless frames in the engine (config.lossless; csrc/lossless.cu): keyframes and P frames over extreme content against
the reference's own statics (tests/lossless_oracle.py), real P and B frames of the reference encoder at quantizer 0 with
host and engine-made prediction, the pool slots written through ll_ref_slot_out against the encoder's next PREV picture,
a resident keyframe -> P -> P -> P sequence, and the refusals."""
import ctypes

import numpy as np
import pytest

from tests import bframe_oracle, inter_mc_oracle, lossless_oracle
from tests.test_lossless_host import CONTENT, content, inverted

pytestmark = [pytest.mark.gpu]
SIZES = ((200, 130), (1920, 1080), (3840, 2160))


def _driver():
    lib = lossless_oracle.load()
    if lib is None:
        pytest.skip("oracle/_ref/libdaala_ref_lossless.so not built (needs the reference sources)")
    return lib


def _engine(geom, F, **kw):
    from daala_b200 import engine
    return engine.KeyframeEngine(geom, nframes=F, lossless=1, **kw)


def _copy(out):
    return {k: np.array(v) for k, v in out.items()}


def _check_frame(lib, geom, out, f, planes, pred=None):
    """Frame f of a lossless step against the driver: every residual value, every root sum, and the reconstruction
    equal to the (padded) input."""
    from daala_b200 import lossless
    want = lossless_oracle.frame(lib, geom, planes, pred)
    for p in range(3):
        assert np.array_equal(out["ll_coeffs%d" % p][f].astype(np.int32), want["coeffs"][p]), ("residual", f, p)
        c = lossless.padded_input(geom, planes, pred)[p]
        assert np.array_equal(out["recon%d" % p][f].astype(np.int64) - 128, c), ("reconstruction", f, p)
    assert np.array_equal(out["ll_blocks"][f][..., :3], want["roots"]), ("root sums", f)
    assert not out["ll_blocks"][f][..., 3].any()


@pytest.mark.parametrize("size", SIZES)
def test_keyframes(size):
    from daala_b200.frame import Geometry
    lib = _driver()
    geom = Geometry(*size)
    frames = [content(geom, kind, seed=11) for kind in CONTENT]
    eng = _engine(geom, len(frames))
    assert eng.launches_per_step() == 2
    out = _copy(eng.encode([np.stack([fr[p] for fr in frames]) for p in range(3)], None))
    for f, fr in enumerate(frames):
        _check_frame(lib, geom, out, f, fr)
    eng.close()


@pytest.mark.parametrize("size", SIZES[:2])
def test_p_frames_host_prediction(size):
    """Prediction planes from the host in inverted phase (the largest residuals), so the padding rule and the int16
    bound are both exercised."""
    from daala_b200.frame import Geometry
    lib = _driver()
    geom = Geometry(*size)
    frames = [content(geom, kind, seed=12) for kind in CONTENT]
    preds = [inverted(fr) if k % 2 == 0 else content(geom, "random", seed=40 + k) for k, fr in enumerate(frames)]
    eng = _engine(geom, len(frames), inter=1)
    assert eng.launches_per_step() == 1
    out = _copy(eng.encode([np.stack([fr[p] for fr in frames]) for p in range(3)], None,
                           pred=[np.stack([pr[p] for pr in preds]) for p in range(3)]))
    for f, (fr, pr) in enumerate(zip(frames, preds)):
        _check_frame(lib, geom, out, f, fr, pr)
    eng.close()


def _p_caps(geom, n):
    lib = inter_mc_oracle.load()
    if lib is None:
        pytest.skip("oracle/_ref/libdaala_ref_inter_mc.so not built (needs the reference sources)")
    return inter_mc_oracle.capture_p_frames(lib, geom, n, quant=0)


def test_real_p_frames_host_and_engine_prediction():
    """P frames 1-3 of the reference encoder at quantizer 0 (200x130): with the captured prediction from the host, and
    with the engine predicting from the captured GOLD / PREV pictures and grids.  The pool slot each frame's
    reconstruction goes to (ll_ref_slot_out) equals the encoder's PREV picture of the next frame over the whole padded
    frame."""
    from daala_b200 import mvgrid
    from daala_b200.frame import Geometry
    lib = _driver()
    geom = Geometry(200, 130)
    caps = _p_caps(geom, 5)
    F = len(caps)
    planes = [np.stack([c["src"][p] for c in caps]) for p in range(3)]
    host = _engine(geom, F, inter=1)
    hout = _copy(host.encode(planes, None, pred=[np.stack([c["pred"][p] for c in caps]) for p in range(3)]))
    host.close()
    for f, c in enumerate(caps):
        _check_frame(lib, geom, hout, f, c["src"], c["pred"])
    refs = [np.stack([c[k][p] for c in caps for k in ("gold", "prev")]) for p in range(3)]
    slot = np.asarray([[2 * f, 2 * f + (0 if c["same"] else 1)] for f, c in enumerate(caps)], np.int32)
    grid = mvgrid.pack(*(np.stack([c[k] for c in caps]) for k in ("valid", "mv", "ref")))
    eng = _engine(geom, F, inter=1, inter_mc=1, mc_refs=3 * F)
    assert eng.launches_per_step() == 3
    store = np.arange(2 * F, 3 * F, dtype=np.int32)
    out = _copy(eng.encode(planes, None, refs=refs, ref_slot=slot, mv_grid=grid, ll_ref_slot_out=store))
    pool = [eng.pool_plane(p) for p in range(3)]
    for f, c in enumerate(caps):
        for p in range(3):
            assert np.array_equal(out["pred%d" % p][f], c["pred"][p]), ("prediction", f, p)
            for k in ("ll_coeffs%d" % p, "recon%d" % p):
                assert np.array_equal(out[k][f], hout[k][f]), (k, f)
            if f + 1 < F:
                assert np.array_equal(pool[p][store[f]], caps[f + 1]["prev"][p]), ("pool slot vs next PREV", f, p)
        assert np.array_equal(out["ll_blocks"][f], hout["ll_blocks"][f])
    eng.close()


def test_resident_sequence():
    """Keyframe -> P -> P -> P with every picture on the device: a lossless keyframe engine codes the keyframe, its
    reconstruction is loaded into the pool from device memory, and three one-frame steps each predict from the pool as
    it stands and store their reconstruction for the next."""
    from daala_b200 import mvgrid
    from daala_b200.frame import Geometry
    lib = _driver()
    geom = Geometry(200, 130)
    caps = _p_caps(geom, 4)
    assert all(np.array_equal(caps[0]["gold"][p], caps[0]["prev"][p]) for p in range(3))
    key = _engine(geom, 1)
    kout = _copy(key.encode([a[None] for a in caps[0]["gold"]], None))
    for p in range(3):
        assert np.array_equal(kout["recon%d" % p][0], caps[0]["gold"][p])
    eng = _engine(geom, 1, inter=1, inter_mc=1, mc_refs=3)
    eng.pool_load(0, [key.buf.pixels_out[p] for p in range(3)])
    prev = 0
    for k, c in enumerate(caps):
        grid = mvgrid.pack(*(c[n][None] for n in ("valid", "mv", "ref")))
        nxt = 1 + (k % 2)
        out = _copy(eng.encode([a[None] for a in c["src"]], None, ref_slot=np.asarray([[0, prev]], np.int32),
                               mv_grid=grid, resident=True, ll_ref_slot_out=np.asarray([nxt], np.int32)))
        _check_frame(lib, geom, out, 0, c["src"], c["pred"])
        for p in range(3):
            assert np.array_equal(out["pred%d" % p][0], c["pred"][p]), ("prediction", k, p)
            if k + 1 < len(caps):
                assert np.array_equal(eng.pool_plane(p)[nxt], caps[k + 1]["prev"][p]), ("pool", k, p)
        prev = nxt
    key.close()
    eng.close()


def test_real_b_frames():
    """The coded frames after the keyframe of a 7-frame b_frames = 2 sequence of the reference encoder at quantizer 0
    (P3, B1, B2, P6, B4, B5) in one batch of an mc_next engine: the prediction, every residual and root sum, and the
    reconstruction."""
    from daala_b200 import mvgrid
    from daala_b200.frame import Geometry
    blib = bframe_oracle.load()
    if blib is None:
        pytest.skip("oracle/_ref/libdaala_ref_bframes.so not built (needs the reference sources)")
    lib = _driver()
    geom = Geometry(200, 130)
    allc = bframe_oracle.capture_b_frames(blib, geom, 7, 2, quant=0)
    assert [c["quantizer"] for c in allc] == [0] * len(allc)
    caps = [c for c in allc if c["type"] != 0]
    assert [c["type"] for c in caps] == [1, 2, 2, 1, 2, 2]
    F = len(caps)
    refs = [np.stack([c[k][p] for c in caps for k in ("gold", "prev", "next")]) for p in range(3)]
    slot = np.asarray([[3 * f, 3 * f + 1, 3 * f + 2] for f in range(F)], np.int32)
    grid = mvgrid.pack(*(np.stack([c[k] for c in caps]) for k in ("valid", "mv", "ref")))
    mv1 = np.stack([c["mv1"] for c in caps]).astype(np.int32)
    eng = _engine(geom, F, inter=1, inter_mc=1, mc_next=1)
    out = _copy(eng.encode([np.stack([c["src"][p] for c in caps]) for p in range(3)], None, refs=refs, ref_slot=slot,
                           mv_grid=grid, mv1_grid=mv1))
    for f, c in enumerate(caps):
        for p in range(3):
            assert np.array_equal(out["pred%d" % p][f], c["pred"][p]), ("prediction", c["number"], p)
        _check_frame(lib, geom, out, f, c["src"], c["pred"])
    eng.close()


def test_launches_and_refusals():
    """A lossy engine keeps its launch count; the submit refusals of the lossless fields, each with its message."""
    from daala_b200 import engine, synth
    from daala_b200.frame import Geometry
    geom = Geometry(200, 130)
    q4 = np.full((3, 30), 20, np.uint8)
    a = engine.KeyframeEngine(geom, nframes=1, q0=45, pvq_qm_q4=q4, split_free=1)
    b = engine.KeyframeEngine(geom, nframes=1, q0=45, pvq_qm_q4=q4, split_free=1, lossless=0)
    assert a.launches_per_step() == b.launches_per_step()
    planes = [a_[None] for a_ in content(geom, "random", seed=1)]
    bsize = synth.block_size_map(geom, "mixed", seed=2)[None]
    a.stage_inputs(planes, bsize)
    a.stage_ll_ref_slot_out(None)
    a.prepare_io()
    junk = np.zeros(geom.plane_shape(0), np.int16)
    a._io.ll_coeffs[0] = junk.ctypes.data
    with pytest.raises(engine._native.CudaError, match="need an engine with lossless = 1"):
        a.submit()
    a.close()
    b.close()
    ll = _engine(geom, 2, inter=1)
    pr = [np.stack([p, p]) for p in content(geom, "flat")]
    pl = [np.stack([p, p]) for p in content(geom, "random", seed=3)]
    with pytest.raises(engine._native.CudaError, match="ll_ref_slot_out needs an engine with inter_mc"):
        ll.encode(pl, None, pred=pr, ll_ref_slot_out=np.asarray([0, 1], np.int32))
    ll.close()
    mc = _engine(geom, 2, inter=1, inter_mc=1, mc_refs=3)
    refs = [np.stack([p, p]) for p in content(geom, "random", seed=4)]
    grid = engine.mvgrid.pack(*(np.stack([g[i] for g in (synth.mv_grid(geom, seed=s) for s in (1, 2))]) for i in range(3)))
    slot = np.asarray([[0, 1], [1, 1]], np.int32)
    for store, msg in (([0, 3], "outside \\[-1, mc_refs\\)"), ([-2, 0], "outside \\[-1, mc_refs\\)"),
                       ([2, 2], "two frames name the same ll_ref_slot_out slot")):
        with pytest.raises(engine._native.CudaError, match=msg):
            mc.encode(pl, None, refs=refs, ref_slot=slot, mv_grid=grid, ll_ref_slot_out=np.asarray(store, np.int32))
    out = mc.encode(pl, None, refs=refs, ref_slot=slot, mv_grid=grid, ll_ref_slot_out=np.asarray([2, -1], np.int32))
    for p in range(3):
        assert np.array_equal(mc.pool_plane(p)[2], out["recon%d" % p][0])
    mc.close()
