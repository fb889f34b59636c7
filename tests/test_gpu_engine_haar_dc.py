"""The keyframe engine with haar_dc_quant = 1 on the GPU: the DC chain's index grids and the quantised DCs the step
stores in the coefficient planes equal the reference's own DC chain (tests/haar_dc_oracle.py) at 200x130, 1080p and
4K on multi-frame batches of different content and block sizes, including real encoder maps; a frame coded in a batch
equals the same frame coded alone; submit refuses dc_index on an engine without the mode."""
import os

import numpy as np
import pytest

from daala_b200 import engine, synth
from daala_b200.frame import Geometry

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = ((200, 130), (1920, 1080), (3840, 2160))


def _settings(i, c):
    s = np.load(os.path.join(ROOT, "tests", "golden", "encoder_settings.npz"))
    return int(s["quantizer"][i][c][0]), s["pvq_qm_q4"][i][c][0], float(s["pvq_norm_lambda"][i][c][0])


def _maps(geom, nframes):
    """Frame 0 a random quadtree, frame 1 all 4x4 (every chroma block takes its CfL from four luma 4x4 blocks), frame 2
    a real encoder map where the geometry allows it."""
    out = [synth.block_size_map(geom, "mixed", seed=21), synth.block_size_map(geom, "4")]
    real = np.load(os.path.join(ROOT, "daala_b200", "data", "bench_bsize_4k.npz"))["bsize_1"]
    h, w = geom.bsize_shape
    out.append(np.ascontiguousarray(real[:h, :w]) if real.shape[0] >= h and real.shape[1] >= w
               else synth.block_size_map(geom, "mixed", seed=22))
    return out[:nframes]


def _frames(geom, nframes):
    return [synth.pad_planes(synth.frame(geom.pic_w, geom.pic_h, f=3 + f)[0], geom) for f in range(nframes)]


def _encode(geom, frames, maps, q0, q4, lam, **kw):
    eng = engine.KeyframeEngine(geom, nframes=len(frames), q0=q0, pvq_qm_q4=q4, lam=lam, split_free=1, haar_dc_quant=1,
                                **kw)
    try:
        out = eng.encode([np.stack([fr[p] for fr in frames]) for p in range(3)], np.stack(maps))
        res = {k: np.array(v) for k, v in out.items()}
        res["coeffs"] = [eng.coeff_plane(p) for p in range(3)]
    finally:
        eng.close()
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("size", SIZES, ids=lambda s: "%dx%d" % s)
def test_engine_matches_reference_chain(size):
    from tests import haar_dc_oracle
    lib = haar_dc_oracle.load()
    if lib is None:
        pytest.skip("needs oracle/_ref/libdaala_ref_haar_dc.so")
    geom = Geometry(*size)
    nframes = 3
    frames, maps = _frames(geom, nframes), _maps(geom, nframes)
    q0, q4, lam = _settings(5, 0)
    got = _encode(geom, frames, maps, q0, q4, lam)
    for f in range(nframes):
        want = haar_dc_oracle.frame(lib, geom, frames[f], maps[f], q0, q4, lam)
        for p in range(3):
            assert np.array_equal(got["dc_index%d" % p][f], want["idx"][p]), "indices of frame %d plane %d" % (f, p)
            kind = "luma_blocks" if p == 0 else "chroma_blocks"
            b = got[kind]
            b = b[(b["pli"] == p) & (b["frame"] == f)]
            y, x = b["y0"].astype(np.int64), b["x0"].astype(np.int64)
            assert np.array_equal(got["coeffs"][p][f][y, x], want["d_post"][p][y, x]), \
                "leaf DCs of frame %d plane %d" % (f, p)
    # the same frame alone: the chain and the step see nothing of the other frames
    alone = _encode(geom, frames[1:2], maps[1:2], q0, q4, lam)
    for p in range(3):
        assert np.array_equal(alone["dc_index%d" % p][0], got["dc_index%d" % p][1])
        assert np.array_equal(alone["recon%d" % p][0], got["recon%d" % p][1])
        assert np.array_equal(alone["coeffs"][p][0], got["coeffs"][p][1])


@pytest.mark.gpu
def test_quantised_dcs_change_the_reconstruction():
    """The mode is not a no-op: at a coarse quantizer the reconstruction differs from the unquantised-DC step's, and the
    deringing levels searched on it (dering = 2) come back."""
    geom = Geometry(200, 130)
    frames, maps = _frames(geom, 2), _maps(geom, 2)
    q0, q4, lam = _settings(7, 0)
    got = _encode(geom, frames, maps, q0, q4, lam, dering=2)
    eng = engine.KeyframeEngine(geom, nframes=2, q0=q0, pvq_qm_q4=q4, lam=lam, split_free=1, dering=2)
    try:
        base = eng.encode([np.stack([fr[p] for fr in frames]) for p in range(3)], np.stack(maps))
        assert any(not np.array_equal(base["recon%d" % p], got["recon%d" % p]) for p in range(3))
        assert got["dering_levels"].shape == base["dering_levels"].shape
    finally:
        eng.close()


@pytest.mark.gpu
def test_submit_refuses_dc_index_without_the_mode():
    geom = Geometry(200, 130)
    frames, maps = _frames(geom, 1), _maps(geom, 1)
    eng = engine.KeyframeEngine(geom, nframes=1, q0=45, pvq_qm_q4=np.full((3, 30), 20, np.uint8), split_free=1)
    try:
        eng.stage_inputs([fr[None] for fr in frames[0]], maps[0][None])
        eng.prepare_io()
        grid = np.zeros((1, geom.plane_shape(0)[0] // 4, geom.plane_shape(0)[1] // 4), np.int32)
        eng._io.dc_index[0] = grid.ctypes.data
        with pytest.raises(Exception, match="dc_index needs an engine with haar_dc_quant = 1"):
            eng.submit()
    finally:
        eng.close()


def _oracle_chain(ref, geom, planes, bsize, q0, q4, lam, drv):
    """The pipeline oracle's keyframe chain (frame_oracle.keyframe_chain with the recording hooks) on the DC chain's
    output: the `d` planes the driver quantised (drv["d_post"]: the forward pyramid with every leaf DC final) through
    PVQ (4x4 chroma CfL then reads the quantised luma DCs, as the reference's od_resample_luma_coeffs does), and the
    inverse without the pyramid (haar_dc = 0)."""
    import ctypes
    from daala_b200 import pvq
    from tests import frame_oracle
    from tests.oracle_lib import addr
    qm, qm_inv = pvq.default_qm(True)
    out, luma_q = [], None
    bs = np.ascontiguousarray(bsize, dtype=np.uint8)
    for pli in range(3):
        ph, pw = geom.plane_shape(pli)
        d = np.ascontiguousarray(drv["d_post"][pli], dtype=np.int32).copy()
        stats = np.zeros(5, np.float64)
        rec = np.full((ph // 4, pw // 4, 9, 4), -32768, np.int16)
        yplane = np.zeros((ph, pw), np.int32)
        skip = np.full((ph // 4, pw // 4), np.nan, np.float64)
        flip = np.full((ph // 4, pw // 4), -1, np.int32)
        lp = addr(np.ascontiguousarray(luma_q, dtype=np.int32)) if pli else None
        ref.oracle_ref_pvq_plane_sym(addr(d), None, geom.nhsb, geom.nvsb, geom.xdec[pli], pli, addr(bs), bs.shape[1],
                                     int(q0), 1, 1, ctypes.c_double(lam), addr(np.ascontiguousarray(qm)),
                                     addr(np.ascontiguousarray(qm_inv)), addr(np.ascontiguousarray(q4[pli])),
                                     addr(stats), 1 if pli == 0 else 0, lp, addr(rec), addr(yplane), addr(skip),
                                     addr(flip))
        if pli == 0:
            luma_q = d
        recon = frame_oracle.inverse_plane(ref, "ref", d.copy(), geom, pli, bsize, 0)
        out.append(dict(dq=d, recon=recon, rec=rec, skip_diff=skip, flip=flip))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("size", SIZES, ids=lambda s: "%dx%d" % s)
def test_step_matches_pipeline_oracle_on_quantised_dcs(size):
    """Reconstruction, quantised coefficient planes, every band record, skip_diff and the CfL flips equal the pipeline
    oracle run on the driver's quantised DCs; frame 1 is all 4x4 (CfL of every chroma block from four luma 4x4 DCs)."""
    from tests import haar_dc_oracle, oracle_lib
    lib, ref = haar_dc_oracle.load(), oracle_lib.load_ref()
    if lib is None or ref is None:
        pytest.skip("needs oracle/_ref")
    geom = Geometry(*size)
    frames, maps = _frames(geom, 2), _maps(geom, 2)
    q0, q4, lam = _settings(3, 0)
    got = _encode(geom, frames, maps, q0, q4, lam)
    for f in range(2):
        drv = haar_dc_oracle.frame(lib, geom, frames[f], maps[f], q0, q4, lam)
        want = _oracle_chain(ref, geom, frames[f], maps[f], q0, q4, lam, drv)
        for p in range(3):
            kind = "luma" if p == 0 else "chroma"
            b = got[kind + "_blocks"]
            sel = (b["pli"] == p) & (b["frame"] == f)
            y4, x4 = b["y0"][sel] >> 2, b["x0"][sel] >> 2
            assert np.array_equal(got["recon%d" % p][f], want[p]["recon"]), ("recon", f, p)
            assert np.array_equal(got["coeffs"][p][f], want[p]["dq"]), ("coefficients", f, p)
            assert np.array_equal(engine.band_records(b, got[kind + "_res"], geom, p, f), want[p]["rec"]), ("bands", f, p)
            assert np.array_equal(got[kind + "_skip_diff"][sel], want[p]["skip_diff"][y4, x4]), ("skip_diff", f, p)
            if p:
                assert np.array_equal(got["chroma_flip"][sel], want[p]["flip"][y4, x4]), ("flip", f, p)


@pytest.mark.gpu
@pytest.mark.parametrize("dering", [1, 2])
def test_forked_step_equals_phase_by_phase(dering):
    """With the mode, the forked step graph equals the phase-by-phase path (the chain inside the forward phase), the
    forked step as live launches and a graph replay, bit for bit."""
    import bench
    from tests.test_gpu_step_fork import _assert_same, _state
    geom = Geometry(1920, 1080)
    frames, maps = _frames(geom, 2), _maps(geom, 2)
    q0, q4, lam = _settings(5, 0)
    eng = engine.KeyframeEngine(geom, nframes=2, q0=q0, pvq_qm_q4=q4, lam=lam, dering=dering, split_free=1,
                                coded_quantizer=bench.CODED_Q, dering_lambda=bench.DERING_LAMBDA, haar_dc_quant=1)
    try:
        eng.stage_inputs([np.stack([fr[p] for fr in frames]) for p in range(3)], np.stack(maps))
        if dering == 1:
            eng.stage_dering_levels(np.random.default_rng(5).integers(0, 6, (2, geom.nvsb, geom.nhsb)).astype(np.uint8))
        eng.prepare_io(symbols=True, recon=True)
        eng.submit()
        eng.wait()
        forked = _state(eng)
        for ph in (engine.PH_LISTS, engine.PH_FORWARD, engine.PH_PVQ_LUMA, engine.PH_PVQ_CHROMA, engine.PH_INVERSE):
            eng.run_device(ph, False)
        _assert_same(_state(eng), forked, "phase by phase")
        eng.run_device(engine.PH_ALL, False)
        _assert_same(_state(eng), forked, "live launches")
        eng.run_device(engine.PH_ALL, True)
        _assert_same(_state(eng), forked, "graph replay")
    finally:
        eng.close()


@pytest.mark.gpu
def test_leaf_dcs_equal_the_whole_reference_encoder():
    """On bench.py's four 4K frames the whole reference encoder (OD_SET_QUANT 20, its own block-size decisions) and the
    engine at the encoder's quantizer settings and map leave the same leaf DCs in every plane.  The frames are cropped
    to 3840x2048, whole superblocks: the encoder pads a partial superblock of the picture itself, while the engine
    takes the padded planes as its input."""
    import bench
    from tests import haar_dc_oracle
    lib = haar_dc_oracle.load()
    if lib is None:
        pytest.skip("needs oracle/_ref/libdaala_ref_haar_dc.so")
    geom = Geometry(3840, 2048)
    seed = 12345
    for f in range(4):
        planes, seed = synth.frame(bench.PIC_W, bench.PIC_H, f=f, seed=seed)
        planes = [np.ascontiguousarray(a[:geom.plane_shape(p)[0]]) for p, a in enumerate(planes)]
        want = haar_dc_oracle.encode_keyframe(lib, geom, planes, 20)
        got = _encode(geom, [planes], [want["bsize"]], want["quantizer"], want["pvq_qm_q4"], want["lam"])
        for p in range(3):
            m = haar_dc_oracle.leaf_origins(geom, want["bsize"], p)
            assert np.array_equal(got["coeffs"][p][0][::4, ::4][m], want["d"][p][::4, ::4][m]), ("leaf DCs", f, p)
