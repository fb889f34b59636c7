"""The keyframe engine's symbol stream (config.symbol_stream = 1) on the GPU: per frame, in bitstream order, the
blocks, band records and 8/16-bit pulses the device packs equal what daala_b200.symbols.pack_reference builds from
the same submit's classic outputs, and what the oracle alone gives when its records are walked in coding order."""
import ctypes

import numpy as np
import pytest

import bench
from tests import frame_oracle
from tests.test_gpu_engine import _coding_tables, _oracle

pytestmark = [pytest.mark.gpu]
F = 16
DISTINCT = 4
Q4 = np.full((3, 30), bench.PVQ_QM_Q4, np.uint8)


def _engine(geom, nframes, symbol_stream=1, dering=1, q0=bench.Q0, q4=Q4, **kw):
    from daala_b200 import engine
    args = dict(nframes=nframes, q0=q0, use_masking=1, pvq_qm_q4=q4, dering=dering, coded_quantizer=bench.CODED_Q,
                dering_lambda=bench.DERING_LAMBDA, persist_ctas_per_sm=0, max_blocks_div=2, symbol_stream=symbol_stream)
    args.update(kw)
    return engine.KeyframeEngine(geom, **args)


def _stage(eng, frames, levels=True):
    eng.stage_inputs([np.stack([f[0][p] for f in frames]) for p in range(3)], np.stack([f[1] for f in frames]))
    if levels:
        eng.stage_dering_levels(np.stack([f[2] for f in frames]))
    return eng.prepare_io(symbols=True, recon=True, stream=True)


def _copy(out):
    return {k: v.copy() for k, v in out.items()}


def _assert_matches_reference(out, nframes, what=""):
    """The device stream equals pack_reference over the classic outputs of the same submit, frame by frame."""
    from daala_b200 import engine, symbols
    assert int(out["counts"][engine.CNT["error"]]) == 0
    want = symbols.pack_reference(out, nframes)
    bad = symbols.stream_equal(out, want, range(nframes))
    assert not bad, (what, bad[:8])
    # the frames follow each other without gaps
    idx = out["sym_index"]
    for c in (0, 2, 4):
        assert idx[0, c] == 0 and np.array_equal(idx[1:, c], idx[:-1, c] + idx[:-1, c + 1]), (what, c)
    return want


def _oracle_stream(want, geom, bsize, tabs):
    """One frame's stream from the oracle alone (keyframe_chain(..., symbols=True)): its band records, skip_diff
    and flip maps at each block's origin and its raster pulse planes, walked in coding_order."""
    from daala_b200 import symbols
    order = symbols.coding_order(bsize, geom)
    n = len(order)
    res = np.zeros((n, 9, 4), np.int16)
    skip = np.zeros(n)
    flip = np.zeros(n, np.int64)
    ys, y_off = [], np.zeros(n, np.int64)
    total = 0
    for pli in range(3):
        sel = np.nonzero(order["pli"] == pli)[0]
        y4, x4 = order["y0"][sel] >> 2, order["x0"][sel] >> 2
        w = want[pli]
        res[sel] = w["rec"][y4, x4]
        skip[sel] = w["skip_diff"][y4, x4]
        flip[sel] = w["flip"][y4, x4] if pli else 0
        assert not np.isnan(skip[sel]).any()
        for i in sel:   # the block's pulse vector in coding order, from the raster pulse plane
            bs = int(order["bs"][i])
            r, c = tabs[bs]
            ys.append(w["yplane"][order["y0"][i] + r, order["x0"][i] + c])
            y_off[i] = total
            total += len(r)
    y = np.concatenate(ys)
    return order, symbols.pack_blocks(order["x0"], order["y0"], order["bs"], order["pli"], flip, skip, res, y, y_off)


@pytest.fixture(scope="module")
def bench_batch():
    """bench.py's workload (16 x 3840x2160, the reference encoder's maps and deringing levels, q0 72) on an engine
    configured as bench.py configures it, plus symbol_stream = 1; one submit."""
    from daala_b200.frame import Geometry
    geom = Geometry(bench.PIC_W, bench.PIC_H)
    distinct = bench.make_host_frames(geom, DISTINCT, distinct=DISTINCT)
    frames = [distinct[i % DISTINCT] for i in range(F)]
    eng = _engine(geom, F)
    _stage(eng, frames)
    eng.submit()
    out = _copy(eng.wait())
    yield dict(geom=geom, distinct=distinct, frames=frames, eng=eng, out=out)
    eng.close()


def test_bench_batch_stream_matches_classic_outputs(bench_batch):
    """(1) Every frame of the benchmark batch, byte for byte, and the index lengths."""
    from daala_b200 import symbols
    out = bench_batch["out"]
    _assert_matches_reference(out, F, "bench batch")
    for f in range(F):
        t = symbols.read_frame(out, f)
        assert len(t["blocks"]) == int((out["luma_blocks"]["frame"] == f).sum() + (out["chroma_blocks"]["frame"] == f).sum())
    # frames with the same content give the same stream
    for f in range(DISTINCT, F):
        assert not symbols.stream_equal(out, out, [f], [f % DISTINCT])


def test_bench_frame0_stream_matches_oracle(bench_batch):
    """(2) Frame 0 of the benchmark batch against a stream built from the oracle alone."""
    from daala_b200 import symbols
    lib, prefix = _oracle()
    geom = bench_batch["geom"]
    planes, bsize, levels = bench_batch["distinct"][0]
    want = frame_oracle.keyframe_chain(lib, prefix, planes, geom, bsize, bench.Q0, Q4, use_masking=1,
                                       dering_levels=levels, symbols=True)
    _, parts = _oracle_stream(want, geom, bsize, _coding_tables())
    ref = symbols.concat_frames([parts])
    bad = symbols.stream_equal(bench_batch["out"], ref, [0], [0])
    assert not bad, bad


def test_1080p_stream_matches_oracle():
    """(2) A 1920x1080 batch of 2 frames with mixed synthetic maps: every frame against the oracle alone."""
    from daala_b200 import symbols, synth
    from daala_b200.frame import Geometry
    geom = Geometry(1920, 1080)
    lib, prefix = _oracle()
    q0, q4 = 40, np.full((3, 30), 16, np.uint8)
    frames = []
    for f in range(2):
        planes, _ = synth.frame(1920, 1080, f=f)
        frames.append((synth.pad_planes(planes, geom), synth.block_size_map(geom, "mixed", seed=40 + f)))
    eng = _engine(geom, 2, dering=0, q0=q0, q4=q4, max_blocks_div=1)
    try:
        out = eng.encode([np.stack([fr[0][p] for fr in frames]) for p in range(3)], np.stack([fr[1] for fr in frames]),
                         stream=True)
        _assert_matches_reference(out, 2, "1080p")
        tabs = _coding_tables()
        for f in range(2):
            want = frame_oracle.keyframe_chain(lib, prefix, frames[f][0], geom, frames[f][1], q0, q4, 1, symbols=True)
            _, parts = _oracle_stream(want, geom, frames[f][1], tabs)
            bad = symbols.stream_equal(out, symbols.concat_frames([parts]), [f], [0])
            assert not bad, (f, bad)
    finally:
        eng.close()


def test_wide_pulses_at_low_quantizer():
    """(3) q0 = 4 on noise: bands with K >= 128 occur, and their 16-bit pulses are the classic y16 values."""
    from daala_b200 import symbols, synth
    from daala_b200.frame import Geometry
    geom = Geometry(256, 128)
    rng = np.random.default_rng(5)
    planes = [rng.integers(0, 256, size=geom.plane_shape(p), dtype=np.uint8) for p in range(3)]
    bsize = synth.block_size_map(geom, "mixed", seed=9)
    eng = _engine(geom, 1, dering=0, q0=4, q4=np.full((3, 30), 16, np.uint8), max_blocks_div=1)
    try:
        out = eng.encode([p[None] for p in planes], bsize[None], stream=True)
        _assert_matches_reference(out, 1, "q0 4")
        r = symbols.read_frame(out, 0)
        wide = np.nonzero(r["bands"][:, 3] >= 128)[0]
        assert len(wide) > 0, "no band with K >= 128 at q0 = 4 on noise"
        # pulses of the wide bands against the classic y16 of the same blocks
        blocks = r["blocks"]
        for q in wide[:200]:
            i = int(r["band_block"][q])
            name = "luma" if blocks["pli"][i] == 0 else "chroma"
            cb = out[name + "_blocks"]
            j = int(np.nonzero((cb["pli"] == blocks["pli"][i]) & (cb["x0"] == blocks["x0"][i]) &
                               (cb["y0"] == blocks["y0"][i]))[0][0])
            band = int(r["band_no"][q])
            a = int(cb["coef_off"][j]) + symbols.BAND_EDGES[band]
            n = len(r["pulses"][q])
            assert np.array_equal(r["pulses"][q], out[name + "_y16"][a:a + n].astype(np.int32))
            assert np.abs(r["pulses"][q]).max() <= r["bands"][q, 3]
    finally:
        eng.close()


@pytest.mark.parametrize("case", ["200x130", "all4x4", "shard"])
def test_geometries_and_shards(case):
    """(4) A geometry that is not a multiple of 64, an all-4x4 map, and a sharded engine (sb_row0 > 0)."""
    from daala_b200 import symbols, synth
    from daala_b200.frame import Geometry
    size = {"200x130": (200, 130), "all4x4": (256, 192), "shard": (320, 320)}[case]
    geom = Geometry(*size)
    frames = []
    for f in range(3):
        planes, _ = synth.frame(*size, f=f)
        m = synth.block_size_map(geom, "4") if case == "all4x4" else synth.block_size_map(geom, "mixed", seed=20 + f)
        frames.append((synth.pad_planes(planes, geom), m))
    kw = dict(sb_row0=2, sb_rows=2) if case == "shard" else {}
    eng = _engine(geom, 3, dering=0, q0=30, q4=np.full((3, 30), 16, np.uint8), max_blocks_div=1, **kw)
    try:
        out = eng.encode([np.stack([fr[0][p] for fr in frames]) for p in range(3)], np.stack([fr[1] for fr in frames]),
                         stream=True)
        _assert_matches_reference(out, 3, case)
        for f in range(3):
            order = symbols.coding_order(frames[f][1], geom, **({"sb_row0": 2, "sb_rows": 2} if case == "shard" else {}))
            b = symbols.read_frame(out, f)["blocks"]
            assert np.array_equal(b["x0"], order["x0"]) and np.array_equal(b["y0"], order["y0"]), (case, f)
            assert np.array_equal(b["pli"], order["pli"]) and np.array_equal(b["bs"], order["bs"]), (case, f)
    finally:
        eng.close()


def test_two_engines_and_replays_give_identical_streams(bench_batch):
    """(5) Two engines alternating over 6 submits (batches rotated by 0 and 1 frames), and graph replays between
    submits: every stream equals the first one of its batch."""
    from daala_b200 import engine, symbols
    geom, distinct = bench_batch["geom"], bench_batch["distinct"]
    first = bench_batch["out"]
    second = _engine(geom, F)
    try:
        _stage(second, [distinct[(i + 1) % DISTINCT] for i in range(F)])
        slots = [bench_batch["eng"], second]
        _stage(slots[0], bench_batch["frames"])
        ref = [first, None]

        def check(s, what):
            out = slots[s].wait()
            if ref[s] is None:
                _assert_matches_reference(out, F, "second engine")
                ref[s] = _copy(out)
            bad = symbols.stream_equal(out, ref[s], range(F))
            assert not bad, (what, s, bad[:4])

        for i in range(6):   # bench.py's end-to-end loop: submit one engine while the other one's batch runs
            s = i % 2
            if i >= 2:
                check(s, i)
            slots[s].submit()
        for s in range(2):
            check(s, "last")
        for s in range(2):   # graph replays on the uploaded batch, then a submit
            slots[s].time_device(engine.PH_ALL, True, 3)
            slots[s].submit()
            check(s, "after replays")
        # the second engine's frames are the first one's rotated by one
        for f in range(F - 1):
            assert not symbols.stream_equal(ref[1], ref[0], [f], [f + 1])
    finally:
        second.close()


def test_default_engine_is_unchanged():
    """(6) Without symbol_stream the step launches as many kernels as before the stream existed (25 for this
    configuration); with it, 8 more."""
    from daala_b200.frame import Geometry
    geom = Geometry(200, 130)
    counts = []
    for s in (0, 1):
        eng = _engine(geom, 2, symbol_stream=s, dering=0, q4=np.full((3, 30), 20, np.uint8), max_blocks_div=0)
        counts.append(eng.launches_per_step())
        eng.close()
    assert counts == [25, 33]


def test_refusals_before_any_launch():
    """(7) A capacity one below the bound, a buffer that is not pinned, and a stream request to an engine
    without symbol_stream are refused with cudaErrorInvalidValue; a valid submit afterwards is exact."""
    from daala_b200 import _native, engine, synth
    from daala_b200.frame import Geometry
    geom = Geometry(200, 130)
    frames = []
    for f in range(2):
        planes, _ = synth.frame(200, 130, f=f)
        frames.append((synth.pad_planes(planes, geom), synth.block_size_map(geom, "mixed", seed=60 + f)))
    planes = [np.stack([fr[0][p] for fr in frames]) for p in range(3)]
    bsize = np.stack([fr[1] for fr in frames])
    q4 = np.full((3, 30), 16, np.uint8)
    eng = _engine(geom, 2, dering=0, q0=30, q4=q4, max_blocks_div=1)
    plain = _engine(geom, 2, symbol_stream=0, dering=0, q0=30, q4=q4, max_blocks_div=1)
    invalid = 1   # cudaErrorInvalidValue
    try:
        eng.stage_inputs(planes, bsize)
        out = eng.prepare_io(stream=True)
        io = eng._io
        for field in ("sym_index", "sym_blocks", "sym_bands", "sym_pulses"):
            cap = getattr(io, field + "_cap")
            setattr(io, field + "_cap", cap - 1)
            assert eng.L.daala_b200_kf_submit(eng.kf, ctypes.byref(io)) == invalid, field
            setattr(io, field + "_cap", cap)
        for field in ("sym_index", "sym_blocks", "sym_bands", "sym_pulses"):
            ptr = getattr(io, field)
            host = np.zeros(int(getattr(io, field + "_cap")) * 48 + 64, np.uint8)   # ordinary (pageable) memory
            setattr(io, field, host.ctypes.data)
            assert eng.L.daala_b200_kf_submit(eng.kf, ctypes.byref(io)) == invalid, field
            setattr(io, field, ptr)
        plain.stage_inputs(planes, bsize)
        plain.prepare_io(stream=True)
        with pytest.raises(_native.CudaError):
            plain.submit()
        # nothing was launched by the refused calls: the engine's counters are still those of its creation
        assert int(eng.counts()[engine.CNT["n_luma"]]) == 0
        eng.submit()
        out = eng.wait()
        _assert_matches_reference(out, 2, "after refusals")
    finally:
        eng.close()
        plain.close()
