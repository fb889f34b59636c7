"""The keyframe step forked into two branches (DAALA_B200_KF_ALL: lists beside the forward transform, the luma
reconstruction beside the chroma stage, CfL read from the luma bands in coding order) computes what the same engine
computes phase by phase on one stream: reconstruction, coefficient planes, band records, pulses, skip_diff, CfL
flips, and a symbol stream that equals the one packed from those outputs.  Synthetic maps: one frame of mixed
sizes (4x4 luma units next to 64x64 blocks, so 32x32 chroma blocks), one of 4x4 units only (every chroma block's
CfL comes from four 4x4 luma blocks)."""
import numpy as np
import pytest

import bench

pytestmark = [pytest.mark.gpu]
Q4 = np.full((3, 30), bench.PVQ_QM_Q4, np.uint8)


def _frames(geom):
    from daala_b200 import synth
    frames = []
    for f, mode in enumerate(("mixed", "4")):
        planes, _ = synth.frame(geom.pic_w, geom.pic_h, f=f, seed=77 + f)
        levels = np.random.default_rng(300 + f).integers(0, 6, size=(geom.nvsb, geom.nhsb)).astype(np.uint8)
        frames.append((synth.pad_planes(planes, geom), synth.block_size_map(geom, mode, seed=40 + f), levels))
    return frames


def _state(eng):
    """Every per-step result the engine keeps on the device."""
    t, b = eng.totals, eng.buf
    nl, nc = int(t.n_luma), int(t.n_chroma)
    st = {"recon%d" % p: eng.recon_plane(p) for p in range(3)}
    st.update({"coeffs%d" % p: eng.coeff_plane(p) for p in range(3)})
    st["luma_res"] = eng.download(b.luma_res, (nl, 9, 4), np.int16)
    st["chroma_res"] = eng.download(b.chroma_res, (nc, 9, 4), np.int16)
    st["luma_y16"] = eng.download(b.luma_y16, (int(t.luma_coefs),), np.int16)
    st["chroma_y16"] = eng.download(b.chroma_y16, (int(t.chroma_coefs),), np.int16)
    st["luma_skip_diff"] = eng.download(b.luma_skip_diff, (nl,), np.float64)
    st["chroma_skip_diff"] = eng.download(b.chroma_skip_diff, (nc,), np.float64)
    st["chroma_flip"] = eng.download(b.chroma_flip, (nc,), np.int32)
    return st


def _assert_same(got, want, what):
    for k in want:
        assert np.array_equal(got[k], want[k]), (what, k, int(np.count_nonzero(got[k] != want[k])))


@pytest.mark.parametrize("size", [(200, 130), (1920, 1080), (3840, 2160)], ids=["200x130", "1080p", "4k"])
@pytest.mark.parametrize("dering", [1, 2])
def test_forked_step_equals_phase_by_phase(size, dering):
    from daala_b200 import engine, symbols
    from daala_b200.frame import Geometry
    geom = Geometry(*size)
    frames = _frames(geom)
    F = len(frames)
    eng = engine.KeyframeEngine(geom, nframes=F, q0=bench.Q0, use_masking=1, pvq_qm_q4=Q4, dering=dering,
                                coded_quantizer=bench.CODED_Q, dering_lambda=bench.DERING_LAMBDA,
                                symbol_stream=1)
    try:
        eng.stage_inputs([np.stack([f[0][p] for f in frames]) for p in range(3)], np.stack([f[1] for f in frames]))
        if dering == 1:
            eng.stage_dering_levels(np.stack([f[2] for f in frames]))
        eng.prepare_io(symbols=True, recon=True, stream=True)
        eng.submit()   # the forked step graph
        out = {k: v.copy() for k, v in eng.wait().items()}
        assert int(out["counts"][engine.CNT["error"]]) == 0
        assert int(out["chroma_res"][..., 3].clip(min=0).sum()) > 0
        bad = symbols.stream_equal(out, symbols.pack_reference(out, F), range(F))
        assert not bad, bad[:8]
        forked = _state(eng)
        for p in range(3):
            assert np.array_equal(forked["recon%d" % p], out["recon%d" % p])
        assert np.array_equal(forked["chroma_flip"], out["chroma_flip"])

        for ph in (engine.PH_LISTS, engine.PH_FORWARD, engine.PH_PVQ_LUMA, engine.PH_PVQ_CHROMA, engine.PH_INVERSE):
            eng.run_device(ph, False)
        _assert_same(_state(eng), forked, "phase by phase")

        eng.run_device(engine.PH_ALL, False)   # the forked step as live launches
        _assert_same(_state(eng), forked, "live launches")
        eng.run_device(engine.PH_ALL, True)    # and a graph replay
        _assert_same(_state(eng), forked, "graph replay")
    finally:
        eng.close()
