"""daala_b200_kf_submit refuses a request before it copies or launches anything, and says why in daala_b200_kf_error.

- A NULL pixels plane on an inter_mc engine with host-uploaded references leaves the reference-picture pool as it was,
  and a following ref_resident step equals the same step on an engine that never saw the refusal.
- A missing dering_level on a dering = 1 engine leaves the last step's block-size map and records on the device, so
  run_device still reproduces that step.
- A NULL bsize, a batch above the block capacity, stream outputs from an engine without symbol_stream, an undersized
  stream buffer and a pageable one each get a message of their own."""
import numpy as np
import pytest

from daala_b200 import _native, engine, symbols
from daala_b200.frame import Geometry
from tests.test_gpu_engine_inter_mc import _batch, _grids, _pack, _pool, _same_outputs
from tests.test_gpu_engine_keyframe_quant import _frames, _levels, _mixed, _records, _run

pytestmark = [pytest.mark.gpu]
GEOM = Geometry(200, 130)


def _refused(eng, pattern):
    with pytest.raises(_native.CudaError, match=pattern) as e:
        eng.submit()
    return str(e.value)


def _pools(eng):
    return [eng.pool_plane(p) for p in range(3)]


def test_refused_upload_leaves_the_pool():
    F = 2
    pics = _pool(GEOM, 2 * F, seed=5)
    planes, bsize = _batch(GEOM, F, seed=9)
    grid = _pack(_grids(GEOM, F, seed=13))
    slot = np.array([[0, 1], [2, 3]], np.int32)   # the resident step's
    engines = [engine.KeyframeEngine(GEOM, nframes=F, q0=45, inter=1, inter_mc=1) for _ in range(2)]
    try:
        for eng in engines:
            for k in range(2 * F):
                eng.pool_load(k, [pics[p][k] for p in range(3)])
        eng = engines[0]
        before = _pools(eng)
        # host references other than the pool's pictures (slots [0, F)), and no third source plane
        eng.stage_frame_type(None)
        eng.stage_inputs(planes, bsize)
        eng.stage_mc([255 - pics[p][:F] for p in range(3)], slot % F, grid)
        eng.stage_frame_quant(None)
        eng.stage_ll_ref_slot_out(None)
        eng.prepare_io()
        eng._io.pixels[2] = None
        _refused(eng, r"pixels\[0\.\.2\] are required")
        after = _pools(eng)
        for p in range(3):
            assert np.array_equal(after[p], before[p]), p
        got, want = (e.encode(planes, bsize, ref_slot=slot, mv_grid=grid, resident=True) for e in engines)
        _same_outputs(GEOM, F, {k: np.array(v) for k, v in got.items()}, {k: np.array(v) for k, v in want.items()})
    finally:
        for eng in engines:
            eng.close()


def test_refused_step_leaves_the_last_inputs():
    F, config = 2, 0
    planes, maps = _frames(GEOM, F, seed=31)
    planes2, maps2 = _frames(GEOM, F, seed=47)
    levels = _levels(GEOM, F, seed=3)
    eng = _mixed(GEOM, F, config, dering=1)
    try:
        first = _run(eng, planes, maps, _records((2, 5), config), levels)
        shape = (F,) + tuple(GEOM.bsize_shape)
        bsize = eng.download(eng.buf.bsize, shape, np.uint8)
        records = eng.download(eng.buf.frame_quant, (F,), engine.FRAME_QUANT_DTYPE)
        # a different map and different records, without the deringing levels
        assert not np.array_equal(np.stack(maps2), bsize)
        eng.stage_inputs([np.stack([fr[p] for fr in planes2]) for p in range(3)], np.stack(maps2))
        eng.stage_dering_levels(levels)
        eng.stage_frame_quant(_records((6, 1), config))
        eng.prepare_io()
        eng._io.dering_level = None
        _refused(eng, "dering_level is required")
        assert np.array_equal(eng.download(eng.buf.bsize, shape, np.uint8), bsize)
        assert eng.download(eng.buf.frame_quant, (F,), engine.FRAME_QUANT_DTYPE).tobytes() == records.tobytes()
        eng.run_device()
        for p in range(3):
            assert np.array_equal(eng.recon_plane(p), first["recon%d" % p]), p
    finally:
        eng.close()


def test_every_refusal_has_its_own_message():
    F = 2
    planes, maps = _frames(GEOM, F, seed=61)
    stacked = [np.stack([fr[p] for fr in planes]) for p in range(3)]
    plain = engine.KeyframeEngine(GEOM, nframes=F, q0=45)
    stream = engine.KeyframeEngine(GEOM, nframes=F, q0=45, symbol_stream=1)
    msgs = []
    try:
        for eng in (plain, stream):
            eng.stage_inputs(stacked, np.stack(maps))

        plain.prepare_io()
        plain._io.bsize = None
        msgs.append(_refused(plain, "bsize is required"))

        plain.prepare_io()
        plain._io.totals.contents.n_luma = plain.buf.max_luma_blocks + 1
        msgs.append(_refused(plain, "more luma or chroma blocks than the engine holds"))
        plain.totals = plain.count_blocks(plain._arr("bsize", (F,) + tuple(GEOM.bsize_shape), np.uint8))

        plain.prepare_io(stream=True)
        plain._io.sym_index = plain._io.sym_blocks = plain._io.sym_bands = None
        msgs.append(_refused(plain, "need an engine with symbol_stream"))

        stream.prepare_io()
        stream._io.sym_pulses_cap -= 1
        msgs.append(_refused(stream, r"sym_pulses must be pinned host memory of at least "
                                     r"daala_b200_kf_symbol_bounds\(\.\.\.\)\.pulse_bytes"))

        stream.prepare_io()
        pageable = np.zeros(int(stream.symbol_bounds().blocks), symbols.BLOCK_DTYPE)
        stream._io.sym_blocks = pageable.ctypes.data
        msgs.append(_refused(stream, r"sym_blocks must be pinned host memory"))
        assert len(set(msgs)) == len(msgs), msgs

        # and the engines still run
        stream.prepare_io()
        stream.submit()
        stream.wait()
    finally:
        plain.close()
        stream.close()
