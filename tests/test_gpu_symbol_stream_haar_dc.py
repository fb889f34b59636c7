"""The keyframe DC records of the symbol stream (symbol_stream = 1 with haar_dc_quant = 1, io.sym_hdc) on the GPU.

- At 200x130, 1080p and 4K (bench.py's maps and engine options), and on a keyframe_quant batch of every sweep point,
  sym_hdc equals symbols.pack_reference and haardc.stream_records over the engine's own index grids, frame by frame and
  byte for byte, with one record per block record, child 0 first in every (superblock, plane) and every block inside
  its (superblock, plane)'s range.
- At 200x130 and 1080p each frame's records, replayed through the reference's generic_encode, code the bytes of the
  reference's own DC chain (tests/haar_dc_stream_oracle.py).
- Requesting sym_hdc changes no other output; the forked step, the phase-by-phase path and graph replays with new
  inputs write the same records.
- Submit refuses sym_hdc on engines without both modes, below the bound and in unpinned memory, then runs exactly."""
import os

import numpy as np
import pytest

from daala_b200 import engine, haardc, symbols, synth
from daala_b200.frame import Geometry
from tests.test_haar_dc_stream_host import check_structure

pytestmark = [pytest.mark.gpu]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = ((200, 130), (1920, 1080))


def _settings(i, c=0):
    s = np.load(os.path.join(ROOT, "tests", "golden", "encoder_settings.npz"))
    return int(s["quantizer"][i][c][0]), s["pvq_qm_q4"][i][c][0], float(s["pvq_norm_lambda"][i][c][0])


def _frames(geom, n, seed=3):
    """n frames of synthetic content; maps: a random quadtree, all 4x4, a real encoder map (or a second quadtree where
    the geometry is too large for it), all 64x64."""
    real = np.load(os.path.join(ROOT, "daala_b200", "data", "bench_bsize_4k.npz"))["bsize_1"]
    h, w = geom.bsize_shape
    maps = [synth.block_size_map(geom, "mixed", seed=seed), synth.block_size_map(geom, "4"),
            np.ascontiguousarray(real[:h, :w]) if real.shape[0] >= h and real.shape[1] >= w
            else synth.block_size_map(geom, "mixed", seed=seed + 1), synth.block_size_map(geom, "64")]
    planes = [synth.pad_planes(synth.frame(geom.pic_w, geom.pic_h, f=seed + f)[0], geom) for f in range(n)]
    return planes, [maps[f % len(maps)] for f in range(n)]


def _engine(geom, F, setting=5, **kw):
    q0, q4, lam = _settings(setting)
    opts = dict(q0=q0, pvq_qm_q4=q4, lam=lam, split_free=1, symbol_stream=1, haar_dc_quant=1)
    opts.update(kw)
    return engine.KeyframeEngine(geom, nframes=F, **opts)


def _run(eng, planes, maps, **kw):
    out = eng.encode([np.stack([fr[p] for fr in planes]) for p in range(3)], np.stack(maps), **kw)
    return {k: np.array(v) for k, v in out.items()}


def _check_records(out, geom, maps):
    """sym_hdc of every frame against pack_reference and stream_records over the step's grids, and its structure."""
    F = len(maps)
    assert "sym_hdc" in out
    want = symbols.pack_reference(out, F)
    assert symbols.stream_equal(out, want, range(F)) == []
    for f in range(F):
        r = symbols.read_frame(out, f)
        grids = [out["dc_index%d" % p][f] for p in range(3)]
        exp = haardc.stream_records(grids, maps[f], geom)
        assert len(r["hdc"]) == len(r["blocks"]) == out["sym_index"][f][1]
        assert r["hdc"].tobytes() == exp.tobytes(), "frame %d" % f
        check_structure(r["hdc"], maps[f], geom)
        # the records' blocks name the block records of their plane
        assert np.array_equal(r["blocks"]["pli"][r["hdc"]["block"].astype(np.int64)], r["hdc"]["pli"])


@pytest.mark.parametrize("size", SIZES, ids=lambda s: "%dx%d" % s)
def test_records_match_the_grids(size):
    geom = Geometry(*size)
    planes, maps = _frames(geom, 4)
    eng = _engine(geom, 4, dering=2)
    try:
        out = _run(eng, planes, maps)
    finally:
        eng.close()
    _check_records(out, geom, maps)
    assert np.count_nonzero(out["sym_hdc"]["value"][:int(out["sym_index"][:, 1].sum())]) > 0


def test_records_match_the_grids_4k_bench_workload():
    """bench.py's 4K frames, maps and levels with its engine options (dering 1, max_blocks_div 2, use_masking)."""
    import bench
    geom = Geometry(bench.PIC_W, bench.PIC_H)
    hf = bench.make_host_frames(geom, 4)
    eng = engine.KeyframeEngine(geom, nframes=4, q0=bench.Q0, use_masking=1,
                                pvq_qm_q4=np.full((3, 30), bench.PVQ_QM_Q4, np.uint8), dering=1,
                                coded_quantizer=bench.CODED_Q, dering_lambda=bench.DERING_LAMBDA, split_free=1,
                                max_blocks_div=2, symbol_stream=1, haar_dc_quant=1)
    try:
        out = _run(eng, [f[0] for f in hf], [f[1] for f in hf], dering_levels=np.stack([f[2] for f in hf]))
    finally:
        eng.close()
    _check_records(out, geom, [f[1] for f in hf])


def test_keyframe_quant_batch_over_the_sweep():
    """Eight keyframes at the eight sweep points of the encoder's settings in one keyframe_quant batch."""
    from tests.test_gpu_engine_keyframe_quant import ALL, _frames as kq_frames, _mixed, _records
    geom = Geometry(200, 130)
    planes, maps = kq_frames(geom, len(ALL), seed=31)
    eng = _mixed(geom, len(ALL), 0, split_free=1, dering=2, symbol_stream=1, haar_dc_quant=1)
    try:
        out = _run(eng, planes, maps, frame_quant=_records(ALL, 0))
    finally:
        eng.close()
    _check_records(out, geom, maps)


@pytest.mark.parametrize("size", SIZES, ids=lambda s: "%dx%d" % s)
def test_records_code_the_reference_bytes(size):
    from tests import haar_dc_stream_oracle
    lib = haar_dc_stream_oracle.load()
    if lib is None:
        pytest.skip("needs oracle/_ref/libdaala_ref_haar_dc_stream.so")
    geom = Geometry(*size)
    planes, maps = _frames(geom, 4, seed=9)
    for setting in (1, 6):
        q0, q4, lam = _settings(setting)
        eng = _engine(geom, 4, setting)
        try:
            out = _run(eng, planes, maps, symbols=False, dc_grids=False)
        finally:
            eng.close()
        assert "dc_index0" not in out and "luma_blocks" not in out
        for f in range(4):
            rec = symbols.read_frame(out, f)["hdc"]
            want = haar_dc_stream_oracle.frame_bytes(lib, geom, planes[f], maps[f], q0, q4, lam)
            assert haar_dc_stream_oracle.replay(lib, geom, rec) == want, (setting, f)


def _stream_parts(out):
    n = out["sym_index"][:, 1].sum(), out["sym_index"][:, 3].sum(), out["sym_index"][:, 5].sum()
    return dict(sym_index=out["sym_index"], sym_blocks=out["sym_blocks"][:n[0]], sym_bands=out["sym_bands"][:n[1]],
                sym_pulses=out["sym_pulses"][:n[2]])


def test_requesting_records_changes_nothing_else():
    """One engine, one batch, with and without io.sym_hdc: every other output byte-identical."""
    geom = Geometry(1920, 1080)
    planes, maps = _frames(geom, 2, seed=5)
    eng = _engine(geom, 2, dering=2)
    try:
        eng.stage_inputs([np.stack([fr[p] for fr in planes]) for p in range(3)], np.stack(maps))
        outs = []
        for with_hdc in (True, False):
            eng.prepare_io(symbols=True, recon=True, stream=True)
            if not with_hdc:
                eng._io.sym_hdc, eng._io.sym_hdc_cap = None, 0
            eng.submit()
            o = {k: np.array(v) for k, v in eng.wait().items()}
            o["coeffs"] = [eng.coeff_plane(p) for p in range(3)]
            outs.append(o)
    finally:
        eng.close()
    a, b = outs
    for k in [k for k in a if k.startswith(("recon", "dc_index", "luma_", "chroma_", "dering"))]:
        assert np.array_equal(a[k], b[k]), k
    for p in range(3):
        assert np.array_equal(a["coeffs"][p], b["coeffs"][p])
    pa, pb = _stream_parts(a), _stream_parts(b)
    for k in pa:
        assert pa[k].tobytes() == pb[k].tobytes(), k
    _check_records(a, geom, maps)


def _device_records(eng, n):
    return eng.download(eng.buf.sym_hdc, (n,), symbols.HDC_DTYPE)


def _expected_records(eng, geom, maps):
    grids = [eng.download(eng.buf.dc_index[p], (eng.F,) + tuple(s >> 2 for s in geom.plane_shape(p)), np.int32)
             for p in range(3)]
    return np.concatenate([haardc.stream_records([g[f] for g in grids], maps[f], geom) for f in range(eng.F)])


@pytest.mark.parametrize("dering", [1, 2])
def test_forked_phase_by_phase_and_replays_agree(dering):
    """The forked step (submit), the phase-by-phase path, live launches and graph replays write the same records; a
    replay with new inputs writes the new batch's records."""
    geom = Geometry(1920, 1080)
    planes_a, maps_a = _frames(geom, 2, seed=11)
    planes_b, maps_b = _frames(geom, 2, seed=12)
    maps_b = maps_b[::-1]
    eng = _engine(geom, 2, dering=dering)
    try:
        kw = {}
        if dering == 1:
            kw["dering_levels"] = np.random.default_rng(5).integers(0, 6, (2, geom.nvsb, geom.nhsb)).astype(np.uint8)
        out_a = _run(eng, planes_a, maps_a, **kw)
        n_a = int(out_a["sym_index"][:, 1].sum())
        rec_a = out_a["sym_hdc"][:n_a].copy()
        assert _device_records(eng, n_a).tobytes() == rec_a.tobytes()
        stack = lambda pl: [np.stack([fr[p] for fr in pl]) for p in range(3)]
        # batch B replayed through the graph: its own records
        eng.upload(stack(planes_b), np.stack(maps_b))
        eng.run_device(engine.PH_ALL, True)
        want_b = _expected_records(eng, geom, maps_b)
        assert want_b.tobytes() != rec_a.tobytes()
        assert _device_records(eng, len(want_b)).tobytes() == want_b.tobytes(), "graph replay of batch B"
        # batch A again, phase by phase, then as live launches and a replay
        eng.upload(stack(planes_a), np.stack(maps_a))
        for ph in (engine.PH_LISTS, engine.PH_FORWARD, engine.PH_PVQ_LUMA, engine.PH_PVQ_CHROMA, engine.PH_INVERSE):
            eng.run_device(ph, False)
        assert _device_records(eng, n_a).tobytes() == rec_a.tobytes(), "phase by phase"
        eng.upload(stack(planes_b), np.stack(maps_b))
        eng.run_device(engine.PH_ALL, False)
        assert _device_records(eng, len(want_b)).tobytes() == want_b.tobytes(), "live launches of batch B"
        eng.upload(stack(planes_a), np.stack(maps_a))
        eng.run_device(engine.PH_ALL, True)
        assert _device_records(eng, n_a).tobytes() == rec_a.tobytes(), "graph replay of batch A"
    finally:
        eng.close()


def _refused(eng, match):
    with pytest.raises(Exception, match=match):
        eng.submit()


def test_submit_refusals_then_an_exact_submit():
    geom = Geometry(200, 130)
    planes, maps = _frames(geom, 2, seed=13)
    stack = [np.stack([fr[p] for fr in planes]) for p in range(3)]
    # engines without both modes: the stream without haar_dc_quant, haar_dc_quant without the stream
    for kw in (dict(haar_dc_quant=0), dict(symbol_stream=0)):
        eng = _engine(geom, 2, **kw)
        try:
            eng.stage_inputs(stack, np.stack(maps))
            eng.prepare_io(stream=False)
            arr = eng._arr("test_hdc", (int(eng.symbol_bounds().blocks),), symbols.HDC_DTYPE, pinned=True)
            eng._io.sym_hdc, eng._io.sym_hdc_cap = arr.ctypes.data, arr.shape[0]
            _refused(eng, "sym_hdc needs an engine with symbol_stream = 1 and haar_dc_quant = 1")
        finally:
            eng.close()
    eng = _engine(geom, 2)
    try:
        eng.stage_inputs(stack, np.stack(maps))
        eng.prepare_io()
        need = int(eng.symbol_bounds().blocks)
        assert eng._io.sym_hdc_cap == need
        eng._io.sym_hdc_cap = need - 1
        _refused(eng, "sym_hdc must be pinned host memory of at least")
        unpinned = np.zeros(need, symbols.HDC_DTYPE)
        eng._io.sym_hdc, eng._io.sym_hdc_cap = unpinned.ctypes.data, need
        _refused(eng, "sym_hdc must be pinned host memory of at least")
        out = _run(eng, planes, maps)
    finally:
        eng.close()
    _check_records(out, geom, maps)
