"""The mixed symbol stream (config.symbol_stream = 3 with frame_types = 1) on the GPU.

The mixed stream is pinned to the single-kind streams, which other tests pin to the reference: every keyframe of a
mixed step byte-equal to the stream of a keyframe_quant = 1, haar_dc_quant = 1, symbol_stream = 1 engine given that
frame and record (blocks, bands, pulses, sym_hdc), every P / B frame to that of a frame_quant = 1, symbol_stream = 2
inter engine (blocks, bands, pulses, sym_dc), each frame's other-kind records zero, and the whole stream equal to
symbols.pack_reference(..., frame_type=) of the step's own classic outputs.  Then: the stream changes no other output,
a stream-order finish equals the block-order one, a GOP driven by the stream alone equals the classic route, the
schedule (forked, phase by phase, replays, launch count) and the refusals."""
import os

import numpy as np
import pytest

from daala_b200 import engine, gop, symbols, synth
from daala_b200.frame import Geometry
from tests.test_gpu_engine_frame_types import (ROOT, _copy, _decisions, _inputs, _mixed, _pack, _records, _single,
                                               _step)

pytestmark = [pytest.mark.gpu]
COMMON = ("sym_index", "sym_blocks", "sym_bands", "sym_pulses")


def _key_stream_engine(geom):
    return engine.KeyframeEngine(geom, nframes=1, keyframe_quant=1, haar_dc_quant=1, symbol_stream=1)


def _p_stream_engine(geom):
    return engine.KeyframeEngine(geom, nframes=1, inter=1, inter_mc=1, mc_next=1, mc_refs=8, frame_quant=1,
                                 symbol_stream=2)


def _sub(out, *extra):
    return {k: out[k] for k in COMMON + extra}


def _n_records(out):
    return int(out["sym_index"][:, 1].sum())


def _check_stream(geom, types, seed, bsize=None):
    F = len(types)
    planes, bs, rec, pool, grids, slots = _inputs(geom, types, seed)
    bs = bs if bsize is None else bsize
    eng, key, inter = _mixed(geom, F, symbol_stream=3), _key_stream_engine(geom), _p_stream_engine(geom)
    try:
        got = _step(eng, planes, bs, rec, types, pool, grids, slots)
        assert int(got["counts"][engine.CNT["error"]]) == 0
        assert {"sym_dc", "sym_hdc", "dc_index0", "luma_dc"} <= set(got)
        for f, t in enumerate(types):
            r = symbols.read_frame(got, f)
            if t == 1:
                want = _single(key, planes, bs, rec, f)
                assert "sym_hdc" in want and "sym_dc" not in want
                assert not symbols.stream_equal(_sub(got, "sym_hdc"), want, [f], [0]), ("keyframe", f)
                assert not r["dc"].view(np.uint8).any(), ("keyframe", f, "sym_dc")
                assert np.all((r["hdc"]["bsi"] == 4) | (r["hdc"]["child"] >= 1)), ("keyframe", f)
            else:
                want = _single(inter, planes, bs, rec, f, pool, grids, slots)
                assert "sym_dc" in want and "sym_hdc" not in want
                assert not symbols.stream_equal(_sub(got, "sym_dc"), want, [f], [0]), ("P frame", f)
                assert not r["hdc"].view(np.uint8).any(), ("P frame", f, "sym_hdc")
                assert not r["blocks"]["flip"].any(), ("P frame", f, "flip")
        ref = symbols.pack_reference(got, F, frame_type=np.asarray(types) == 1)
        assert np.array_equal(got["sym_index"], ref["sym_index"])
        assert not symbols.stream_equal(got, ref, range(F))
        # the comparisons saw records of both kinds
        n = _n_records(got)
        if 1 in types:
            assert np.count_nonzero(got["sym_hdc"]["value"][:n]) > 0
        if any(t != 1 for t in types):
            assert np.count_nonzero(got["sym_dc"]["dc_resid"][:n]) > 0
    finally:
        for e in (eng, key, inter):
            e.close()


# types: 1 keyframe, 0 P frame, 2 B frame (frame_type 0, predicted from NEXT with mc_next)
@pytest.mark.parametrize("w,h,types", [(200, 130, (1, 0, 2)), (200, 130, (0, 1, 2, 1)), (200, 130, (1, 1, 1)),
                                       (200, 130, (0, 2, 0)), (1920, 1080, (1, 0, 2)), (1920, 1080, (0, 1, 2, 1))])
def test_stream_equals_the_single_kind_streams(w, h, types):
    _check_stream(Geometry(w, h), types, seed=w + h + len(types))


def test_4k_stream_on_the_bench_maps():
    geom = Geometry(3840, 2160)
    real = np.load(os.path.join(ROOT, "daala_b200", "data", "bench_bsize_4k.npz"))
    bsize = np.stack([np.ascontiguousarray(real["bsize_%d" % f][:geom.bsize_shape[0], :geom.bsize_shape[1]])
                      for f in range(3)])
    _check_stream(geom, (1, 0, 0), seed=4, bsize=bsize)


def test_stream_changes_nothing_else():
    """A symbol_stream = 3 engine and a symbol_stream = 0 engine on the same inputs: every classic output, the
    coefficient planes, and the finishing pass's reconstruction, bskip, levels and pool."""
    geom = Geometry(200, 130)
    types = (1, 0, 2, 1)
    planes, bsize, rec, pool, grids, slots = _inputs(geom, types, seed=23)
    a, b = _mixed(geom, 4, symbol_stream=3), _mixed(geom, 4)
    try:
        ga = _step(a, planes, bsize, rec, types, pool, grids, slots)
        gb = _step(b, planes, bsize, rec, types, pool, grids, slots)
        assert set(gb) < set(ga)
        for k in gb:
            if k == "coeffs":
                assert all(np.array_equal(x, y) for x, y in zip(ga[k], gb[k])), k
            else:
                assert np.array_equal(ga[k], gb[k]), k
        ls, ld, cs, cd = _decisions(gb, types, seed=3)
        levels = np.random.default_rng(8).integers(0, 6, (4, geom.nvsb, geom.nhsb)).astype(np.uint8)
        store = np.array([4, 5, 6, 7], np.int32)
        fa = _copy(a.finish(ls, ld, cs, cd, dering_levels=levels, ref_slot_out=store))
        fb = _copy(b.finish(ls, ld, cs, cd, dering_levels=levels, ref_slot_out=store))
        for k in fb:
            assert np.array_equal(fa[k], fb[k]), ("finish", k)
        for p in range(3):
            assert np.array_equal(a.pool_plane(p), b.pool_plane(p)), ("pool", p)
    finally:
        a.close()
        b.close()


@pytest.mark.parametrize("inter_finish", [1, 2])
def test_stream_order_finish_equals_block_order_finish(inter_finish):
    """The decisions of the classic form mapped through stream_to_classic give the same reconstruction, bskip, levels
    and pool; other valid values in the keyframe entries change nothing."""
    geom = Geometry(200, 130)
    types = (1, 0, 2, 1)
    planes, bsize, rec, pool, grids, slots = _inputs(geom, types, seed=29)
    eng = _mixed(geom, 4, inter_finish=inter_finish, symbol_stream=3)
    try:
        got = _step(eng, planes, bsize, rec, types, pool, grids, slots)
        ls, ld, cs, cd = _decisions(got, types, seed=13)
        levels = None
        if inter_finish == 1:
            levels = np.random.default_rng(2).integers(0, 6, (4, geom.nvsb, geom.nhsb)).astype(np.uint8)
        store = np.array([4, 5, -1, 6], np.int32)
        want = _copy(eng.finish(ls, ld, cs, cd, dering_levels=levels, ref_slot_out=store))
        want_pool = [eng.pool_plane(p) for p in range(3)]
        perm = symbols.stream_to_classic(got)
        skip, dc = np.concatenate([ls, cs])[perm], np.concatenate([ld, cd])[perm]
        # the keyframe entries of the stream, located through the stream's own blocks
        frame = np.repeat(np.arange(4), got["sym_index"][:, 1])
        on_key = np.asarray(types)[frame] == 1
        assert on_key.any() and (~on_key).any()
        rng = np.random.default_rng(17)
        for variant in range(2):
            if variant:
                skip, dc = skip.copy(), dc.copy()
                skip[on_key] = rng.integers(0, 2, int(on_key.sum()))
                dc[on_key] = rng.integers(-50, 51, int(on_key.sum()))
            # a different pool state in between, so the store is seen to rewrite it
            eng.pool_load(4, [np.zeros(geom.plane_shape(p), np.uint8) for p in range(3)])
            fin = _copy(eng.finish_stream(skip, dc, dering_levels=levels, ref_slot_out=store))
            for k in want:
                assert np.array_equal(fin[k], want[k]), (variant, k)
            for p in range(3):
                assert np.array_equal(eng.pool_plane(p), want_pool[p]), (variant, "pool", p)
    finally:
        eng.close()


def test_gop_driven_by_the_stream_alone():
    """I B B P B B P B B I B B P through pipelined_steps(keyframes_inline=True) on one mixed engine with a resident
    pool, outputs limited to the stream (symbols=False, dc_grids=False) and the finishing decisions taken from sym_dc,
    against the same GOP on a classic mixed engine: the step's stream (against pack_reference of the classic outputs),
    reconstruction, finish and pool, step by step."""
    geom = Geometry(200, 130)
    frames = gop.coding_order(13, 2, keyframe_rate=9)
    steps = gop.pipelined_steps(frames, keyframes_inline=True)
    F = max(len(s) for s in steps)
    src = [synth.pad_planes(synth.frame(geom.pic_w, geom.pic_h, f=i + 1, seed=91 + i)[0], geom) for i in range(13)]
    maps = [synth.block_size_map(geom, "mixed", seed=310 + i) for i in range(13)]
    rec_all = _records(13, seed=19)
    grids = {}
    for fr in frames:
        if fr.type == gop.B_FRAME:
            grids[fr.number] = synth.mv_grid_b(geom, seed=520 + fr.number)
        else:
            v, mv, ref = synth.mv_grid(geom, seed=520 + fr.number)
            grids[fr.number] = (v, mv, np.zeros(mv.shape, np.int32), ref)
    lean, classic = _mixed(geom, F, symbol_stream=3), _mixed(geom, F)
    try:
        for st in steps:
            nums = [fr.number for fr in st]
            pad = F - len(st)
            idx = nums + [nums[0]] * pad
            types = [1 if fr.type == gop.I_FRAME else 0 for fr in st] + [1] * pad
            slots = np.array([gop.pool_slots(fr) for fr in st] + [[0, 0, 0]] * pad, np.int32)
            out_slot = np.array([fr.refs[gop.SELF] if fr.kept else -1 for fr in st] + [-1] * pad, np.int32)
            planes = [np.stack([src[i][p] for i in idx]) for p in range(3)]
            bsize = np.stack([maps[i] for i in idx])
            g = [grids[i] for i in idx]
            grid, mv1 = _pack(g)
            kw = dict(frame_quant=rec_all[idx], frame_type=np.asarray(types) == 1, ref_slot=slots, mv_grid=grid,
                      mv1_grid=mv1, resident=True)
            a = _copy(lean.encode(planes, bsize, symbols=False, dc_grids=False, **kw))
            b = _copy(classic.encode(planes, bsize, **kw))
            assert not {"luma_dc", "chroma_dc", "luma_dc_resid", "dc_index0", "luma_blocks"} & set(a), sorted(a)
            assert {"sym_dc", "sym_hdc"} <= set(a)
            assert lean.stream_d2h_bytes() > 0
            ref = symbols.pack_reference(b, F, frame_type=types)
            assert np.array_equal(a["sym_index"], ref["sym_index"]), nums
            assert not symbols.stream_equal(a, ref, range(F)), nums
            for p in range(3):
                assert np.array_equal(a["recon%d" % p], b["recon%d" % p]), ("step recon", nums, p)
            # the step's own decisions: nothing skipped, each block's DC index (0 on keyframes, which ignore them)
            n = _n_records(a)
            fa = _copy(lean.finish_stream(np.zeros(n, np.uint8), a["sym_dc"]["qdc"][:n],
                                          dering_levels=np.zeros((F, geom.nvsb, geom.nhsb), np.uint8),
                                          ref_slot_out=out_slot))
            ls, cs = (np.zeros(len(b[k + "_blocks"]), np.uint8) for k in ("luma", "chroma"))
            fb = _copy(classic.finish(ls, b["luma_dc"], cs, b["chroma_dc"],
                                      dering_levels=np.zeros((F, geom.nvsb, geom.nhsb), np.uint8),
                                      ref_slot_out=out_slot))
            for k in fb:
                assert np.array_equal(fa[k], fb[k]), ("finish", nums, k)
            for p in range(3):
                assert np.array_equal(lean.pool_plane(p), classic.pool_plane(p)), ("pool", nums, p)
    finally:
        lean.close()
        classic.close()


def test_schedule_forked_phase_by_phase_replays_and_launches():
    """The forked step, the phase-by-phase path, live launches and a graph replay write the same keyframe DC records
    (on a device buffer overwritten in between) and device state; two submits give identical outputs; the launch count
    is the stream-less engine's plus the stream's nine kernels."""
    from tests.test_gpu_step_fork import _assert_same, _state
    geom = Geometry(200, 130)
    types = (1, 0, 2, 1)
    planes, bsize, rec, pool, grids, slots = _inputs(geom, types, seed=37)
    eng, plain = _mixed(geom, 4, symbol_stream=3), _mixed(geom, 4)
    try:
        # rank, superblock scan, keyframe DC records, place, three scan kernels, pack, index
        assert eng.launches_per_step() == plain.launches_per_step() + 9
        a = _step(eng, planes, bsize, rec, types, pool, grids, slots)
        b = _step(eng, planes, bsize, rec, types, pool, grids, slots)
        for k in a:
            if k == "coeffs":
                assert all(np.array_equal(x, y) for x, y in zip(a[k], b[k]))
            else:
                assert np.array_equal(a[k], b[k], equal_nan=a[k].dtype.kind == "f"), k
        n = _n_records(a)
        rec_a = a["sym_hdc"][:n].copy()

        def records():
            return eng.download(eng.buf.sym_hdc, (n,), symbols.HDC_DTYPE)

        def poison():
            # pinned, so that the copy has landed when it returns (the engine's stream does not wait for it)
            junk = eng._arr("poison", (n * symbols.HDC_DTYPE.itemsize,), np.uint8, pinned=True)
            junk[...] = 0xA5
            eng._check(eng.L.daala_b200_device_copy(eng.buf.sym_hdc, junk.ctypes.data, junk.nbytes, 0), "poison")

        assert records().tobytes() == rec_a.tobytes()
        forked = _state(eng)
        poison()
        for ph in (engine.PH_LISTS, engine.PH_FORWARD, engine.PH_PVQ_LUMA, engine.PH_PVQ_CHROMA, engine.PH_INVERSE):
            eng.run_device(ph, False)
        _assert_same(_state(eng), forked, "phase by phase")
        assert records().tobytes() == rec_a.tobytes(), "phase by phase"
        for graph in (False, True):
            poison()
            eng.run_device(engine.PH_ALL, graph)
            _assert_same(_state(eng), forked, ("graph" if graph else "live launches"))
            assert records().tobytes() == rec_a.tobytes(), ("graph" if graph else "live launches")
    finally:
        eng.close()
        plain.close()


def _refused(fn, match):
    with pytest.raises(Exception, match=match):
        fn()


def test_refusals_then_an_exact_submit():
    geom = Geometry(200, 130)
    base = dict(inter=1, inter_mc=1, frame_quant=1, haar_dc_quant=1, inter_finish=1)
    # create: 3 without frame_types (on an inter and on a keyframe engine), 1 and 2 with it
    for kw in (dict(base, symbol_stream=3), dict(symbol_stream=3)):
        _refused(lambda: engine.KeyframeEngine(geom, nframes=2, **kw), "symbol_stream .*3 .*frame_types = 1")
    for s in (1, 2):
        _refused(lambda: engine.KeyframeEngine(geom, nframes=2, frame_types=1, symbol_stream=s, **base),
                 "frame_types takes symbol_stream 0 or 3")
    types = (1, 0, 2)
    planes, bsize, rec, pool, grids, slots = _inputs(geom, types, seed=41)
    # stream_skip on a mixed engine without the stream
    plain = _mixed(geom, 3)
    try:
        got = _step(plain, planes, bsize, rec, types, pool, grids, slots)
        n = len(got["luma_blocks"]) + len(got["chroma_blocks"])
        _refused(lambda: plain.finish_stream(np.zeros(n, np.uint8), np.zeros(n, np.int32)),
                 "stream_skip / stream_dc need an engine with symbol_stream = 2 or 3")
    finally:
        plain.close()
    eng = _mixed(geom, 3, symbol_stream=3)
    try:
        grid, mv1 = _pack(grids)
        eng.stage_frame_type(np.asarray(types) == 1)
        eng.stage_inputs(planes, bsize)
        eng.stage_mc(pool, slots, grid, False, mv1)
        eng.stage_frame_quant(rec)
        eng.prepare_io()
        need = int(eng.symbol_bounds().blocks)
        io = eng._io
        for name, dtype in (("sym_hdc", symbols.HDC_DTYPE), ("sym_dc", symbols.DC_DTYPE)):
            ptr = getattr(io, name)
            assert getattr(io, name + "_cap") == need
            setattr(io, name + "_cap", need - 1)
            _refused(eng.submit, "%s must be pinned host memory of at least" % name)
            unpinned = np.zeros(need, dtype)
            setattr(io, name, unpinned.ctypes.data)
            setattr(io, name + "_cap", need)
            _refused(eng.submit, "%s must be pinned host memory of at least" % name)
            setattr(io, name, ptr)
        assert int(eng.counts()[engine.CNT["n_luma"]]) == 0, "a refused submit launched the step"
        eng.submit()
        out = _copy(eng.wait())
        ref = symbols.pack_reference(out, 3, frame_type=np.asarray(types) == 1)
        assert not symbols.stream_equal(out, ref, range(3))
    finally:
        eng.close()
