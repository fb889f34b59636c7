"""The P-frame symbol stream (config.symbol_stream = 2 with inter = 1; csrc/kf_engine.cu): per frame, in bitstream
order, the block records, band records and pulses of the keyframe stream with flip 0, plus one DC record per block
(qdc, in[0] - ref[0]).  Against daala_b200.symbols.pack_reference of the same step's classic outputs, against the oracle
alone (inter_oracle.inter_chain walked in coding order), and on the reference encoder's own P frames.  The finishing
pass takes its decisions in stream order (finish_io.stream_skip / stream_dc) and must then equal the classic-order
finish.  Bit-exact throughout.  The last two tests need no GPU."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from tests import frame_oracle, inter_mc_oracle, inter_oracle
from tests.test_gpu_engine_inter import Q4, _coding_tables, _frames, _oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID = 1   # cudaErrorInvalidValue


def _engine(geom, F, q0=45, **kw):
    from daala_b200 import engine
    args = dict(nframes=F, q0=q0, pvq_qm_q4=Q4, inter=1, symbol_stream=2)
    args.update(kw)
    return engine.KeyframeEngine(geom, **args)


def _stack(frames):
    """(planes, pred, bsize) of a batch from test_gpu_engine_inter._frames' per-frame tuples."""
    return ([np.stack([f[0][p] for f in frames]) for p in range(3)], [np.stack([f[1][p] for f in frames]) for p in range(3)],
            np.stack([f[2] for f in frames]))


def _copy(out):
    return {k: np.array(v) for k, v in out.items()}


def _assert_matches_reference(out, nframes, what=""):
    """The device stream equals pack_reference over the classic outputs of the same submit, DC records included, and
    the frames follow each other without gaps."""
    from daala_b200 import engine, symbols
    assert int(out["counts"][engine.CNT["error"]]) == 0
    want = symbols.pack_reference(out, nframes)
    assert "sym_dc" in want and "sym_dc" in out
    bad = symbols.stream_equal(out, want, range(nframes))
    assert not bad, (what, bad[:8])
    idx = out["sym_index"]
    for c in (0, 2, 4):
        assert idx[0, c] == 0 and np.array_equal(idx[1:, c], idx[:-1, c] + idx[:-1, c + 1]), (what, c)
    assert not out["sym_blocks"]["flip"][:int(idx[:, 1].sum())].any()
    return want


def _oracle_stream(lib, prefix, planes, pred, geom, bsize, q0, tabs):
    """One P frame's stream from the oracle alone: inter_chain's band records, skip_diff, qdc and raster pulse planes
    at each block's origin, walked in coding_order; dc_resid from the oracle's forward planes of source and prediction
    (as test_dc_resid_is_the_unquantised_dc_residual computes it)."""
    from daala_b200 import symbols
    want = inter_oracle.inter_chain(lib, prefix, planes, pred, geom, bsize, q0, Q4)
    order = symbols.coding_order(bsize, geom)
    n = len(order)
    res = np.zeros((n, 9, 4), np.int16)
    skip = np.zeros(n)
    qdc = np.zeros(n, np.int32)
    resid = np.zeros(n, np.int32)
    ys, y_off = [], np.zeros(n, np.int64)
    total = 0
    for pli in range(3):
        sel = np.nonzero(order["pli"] == pli)[0]
        y0, x0 = order["y0"][sel].astype(np.int64), order["x0"][sel].astype(np.int64)
        w = want[pli]
        res[sel] = w["rec"][y0 >> 2, x0 >> 2]
        skip[sel] = w["skip_diff"][y0 >> 2, x0 >> 2]
        qdc[sel] = w["qdc"][y0 >> 2, x0 >> 2]
        d = frame_oracle.forward_plane(lib, prefix, planes[pli], geom, pli, bsize, 0)
        resid[sel] = d[y0, x0] - w["md"][y0, x0]
        assert not np.isnan(skip[sel]).any()
        for i in sel:
            r, c = tabs[int(order["bs"][i])]
            ys.append(w["yplane"][order["y0"][i] + r, order["x0"][i] + c])
            y_off[i] = total
            total += len(r)
    return symbols.pack_blocks(order["x0"], order["y0"], order["bs"], order["pli"], np.zeros(n, np.int64), skip, res,
                               np.concatenate(ys), y_off, qdc, resid)


# ---- the stream against the same step's classic outputs ------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("w,h,F,mode,q0", [(200, 130, 2, "mixed", 45), (328, 200, 3, "mixed", 30), (328, 200, 2, "4", 45),
                                           (328, 200, 2, "64", 45), (1920, 1080, 1, "mixed", 38)])
def test_stream_matches_classic_outputs(w, h, F, mode, q0):
    from daala_b200 import symbols
    from daala_b200.frame import Geometry
    geom = Geometry(w, h)
    frames = _frames(geom, F, mode=mode, seed=w + F)
    planes, pred, bsize = _stack(frames)
    eng = _engine(geom, F, q0)
    out = _copy(eng.encode(planes, bsize, pred=pred, stream=True))
    _assert_matches_reference(out, F, (w, h, mode))
    for f in range(F):
        r = symbols.read_frame(out, f)
        assert len(r["dc"]) == len(r["blocks"]) == int((out["luma_blocks"]["frame"] == f).sum()
                                                       + (out["chroma_blocks"]["frame"] == f).sum())
    # the DC records carry every classic DC index and residual, each once
    perm = symbols.stream_to_classic(out)
    n = int(out["sym_index"][:, 1].sum())
    assert np.array_equal(np.sort(perm), np.arange(n))
    assert np.array_equal(out["sym_dc"]["qdc"][:n], np.concatenate([out["luma_dc"], out["chroma_dc"]])[perm])
    assert np.array_equal(out["sym_dc"]["dc_resid"][:n],
                          np.concatenate([out["luma_dc_resid"], out["chroma_dc_resid"]])[perm])
    assert out["sym_dc"]["qdc"][:n].any() and (out["sym_dc"]["dc_resid"][:n] != out["sym_dc"]["qdc"][:n]).any()
    eng.close()


@pytest.mark.gpu
def test_wide_pulses_at_low_quantizer():
    """q0 = 4 on a noise residual: bands with K > 127 occur and carry 16-bit pulses."""
    from daala_b200 import symbols, synth
    from daala_b200.frame import Geometry
    geom = Geometry(256, 128)
    rng = np.random.default_rng(5)
    planes = [rng.integers(0, 256, size=(2,) + geom.plane_shape(p), dtype=np.uint8) for p in range(3)]
    pred = [rng.integers(0, 256, size=(2,) + geom.plane_shape(p), dtype=np.uint8) for p in range(3)]
    bsize = np.stack([synth.block_size_map(geom, "mixed", seed=9 + f) for f in range(2)])
    eng = _engine(geom, 2, q0=4)
    out = _copy(eng.encode(planes, bsize, pred=pred, stream=True))
    _assert_matches_reference(out, 2, "q0 4")
    wide = 0
    for f in range(2):
        r = symbols.read_frame(out, f)
        wide += int((r["bands"][:, 3] > 127).sum())
    assert wide > 0, "no band with K > 127 at q0 = 4 on noise"
    eng.close()


# ---- against the oracle alone ------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("w,h,F", [(328, 200, 2), (1920, 1080, 1)])
def test_stream_matches_oracle(w, h, F):
    from daala_b200 import symbols
    from daala_b200.frame import Geometry
    geom = Geometry(w, h)
    lib, prefix = _oracle()
    frames = _frames(geom, F, seed=3)
    planes, pred, bsize = _stack(frames)
    eng = _engine(geom, F)
    out = _copy(eng.encode(planes, bsize, pred=pred, stream=True))
    tabs = _coding_tables()
    for f in range(F):
        parts = _oracle_stream(lib, prefix, frames[f][0], frames[f][1], geom, frames[f][2], 45, tabs)
        bad = symbols.stream_equal(out, symbols.concat_frames([parts]), [f], [0])
        assert not bad, (f, bad)
    eng.close()


@pytest.mark.gpu
def test_inter_mc_real_p_frames():
    """The reference encoder's P frames 1-3 (328x200) on an inter_mc engine: the stream equals the oracle's, built from
    the encoder's own source and prediction."""
    from daala_b200 import symbols
    from daala_b200.frame import Geometry
    from tests.test_gpu_engine_inter_mc import _pack
    lib_mc = inter_mc_oracle.load()
    if lib_mc is None:
        pytest.skip("oracle/_ref/libdaala_ref_inter_mc.so not built (needs the reference sources)")
    geom = Geometry(328, 200)
    caps = inter_mc_oracle.capture_p_frames(lib_mc, geom, 4)
    F = len(caps)
    refs = [np.stack([c[k][p] for c in caps for k in ("gold", "prev")]) for p in range(3)]
    slot = np.array([[2 * f, 2 * f + (0 if c["same"] else 1)] for f, c in enumerate(caps)], np.int32)
    grids = [(c["valid"], c["mv"], c["ref"]) for c in caps]
    planes = [np.stack([c["src"][p] for c in caps]) for p in range(3)]
    bsize = np.stack([c["bsize"] for c in caps])
    eng = _engine(geom, F, inter_mc=1)
    out = _copy(eng.encode(planes, bsize, refs=refs, ref_slot=slot, mv_grid=_pack(grids), stream=True))
    _assert_matches_reference(out, F, "inter_mc")
    lib, prefix = _oracle()
    tabs = _coding_tables()
    for f, c in enumerate(caps):
        for p in range(3):
            assert np.array_equal(out["pred%d" % p][f], c["pred"][p]), ("prediction", f, p)
        parts = _oracle_stream(lib, prefix, c["src"], c["pred"], geom, c["bsize"], 45, tabs)
        bad = symbols.stream_equal(out, symbols.concat_frames([parts]), [f], [0])
        assert not bad, (f, bad)
    eng.close()


# ---- the stream changes nothing else -------------------------------------------------------------------------------

@pytest.mark.gpu
def test_stream_changes_nothing_else():
    from daala_b200.frame import Geometry
    from tests.test_gpu_engine_inter_mc import _same_outputs
    geom = Geometry(328, 200)
    F = 2
    planes, pred, bsize = _stack(_frames(geom, F, seed=11))
    plain = _engine(geom, F, symbol_stream=0)
    fin = _engine(geom, F, symbol_stream=0, inter_finish=1)
    eng = _engine(geom, F)
    assert eng.launches_per_step() == plain.launches_per_step() + 8
    assert eng.buf.bytes_allocated > plain.buf.bytes_allocated
    want = _copy(plain.encode(planes, bsize, pred=pred))
    got = _copy(eng.encode(planes, bsize, pred=pred, stream=True))
    _same_outputs(geom, F, got, want)
    # the residual the stream carries is the one an inter_finish engine returns
    resid = _copy(fin.encode(planes, bsize, pred=pred))
    for k in ("luma_dc_resid", "chroma_dc_resid"):
        assert np.array_equal(got[k], resid[k]), k
    for e in (plain, fin, eng):
        e.close()


# ---- the stream-order finish -------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("inter_finish", [1, 2])
def test_stream_order_finish_equals_classic(inter_finish):
    """Seeded decisions, given in classic order and permuted into stream order: reconstruction, skip maps, applied levels
    and pool slots are identical, and the two forms alternate on one engine (one captured graph)."""
    from daala_b200 import symbols
    from daala_b200.frame import Geometry
    from tests.test_gpu_engine_inter_finish import _decisions
    from tests.test_gpu_engine_inter_mc import _batch, _grids, _pack, _pool
    geom = Geometry(328, 200)
    F = 2
    eng = _engine(geom, F, inter_mc=1, mc_refs=2 * F, inter_finish=inter_finish, coded_quantizer=45)
    pics = _pool(geom, F, seed=19)
    for f in range(F):
        eng.pool_load(f, [pics[p][f] for p in range(3)])
    planes, bsize = _batch(geom, F, seed=29)
    slot = np.array([[f, f] for f in range(F)], np.int32)
    out = _copy(eng.encode(planes, bsize, ref_slot=slot, mv_grid=_pack(_grids(geom, F, seed=31)), resident=True,
                           stream=True))
    perm = symbols.stream_to_classic(out)
    for seed in (1, 2):
        ls, ld, cs, cd, levels = _decisions(out, geom, F, seed=seed)[:5]
        levels = levels if inter_finish == 1 else None
        store = np.arange(F, 2 * F, dtype=np.int32)
        classic = _copy(eng.finish(ls, ld, cs, cd, levels, ref_slot_out=store))
        pool_c = [eng.pool_plane(p) for p in range(3)]
        skip, dc = np.concatenate([ls, cs])[perm], np.concatenate([ld, cd])[perm]
        stream = _copy(eng.finish_stream(skip, dc, levels, ref_slot_out=store[::-1].copy()))
        pool_s = [eng.pool_plane(p) for p in range(3)]
        for k in classic:
            assert np.array_equal(classic[k], stream[k]), (seed, k)
        for p in range(3):
            assert np.array_equal(pool_s[p][:F], pool_c[p][:F]), (seed, p)
            assert np.array_equal(pool_s[p][F:], pool_c[p][F:][::-1]), (seed, p)
            assert np.array_equal(pool_s[p][F:][::-1], classic["recon%d" % p]), (seed, p)
        assert eng.finish_h2d_bytes == 5 * len(perm) + (levels.nbytes if levels is not None else 0) + 4 * F
    # the classic form again after a stream-form call
    again = _copy(eng.finish(ls, ld, cs, cd, levels, ref_slot_out=store))
    for k in classic:
        assert np.array_equal(classic[k], again[k]), k
    eng.close()


@pytest.mark.gpu
def test_stream_driven_resident_loop():
    """A keyframe in the pool, then K P frames: one engine reads only the stream and answers in stream order (decisions
    from the DC records), the other reads the classic outputs and gets the same decisions in classic order.  Every
    finish and the final pool are identical."""
    from daala_b200 import symbols
    from daala_b200.frame import Geometry
    from tests.test_gpu_engine_inter_mc import _batch, _grids, _pack, _pool
    geom = Geometry(328, 200)
    F, K = 2, 3
    gold = _pool(geom, F, seed=41)
    engines = [_engine(geom, F, inter_mc=1, mc_refs=2 * F, inter_finish=1, symbol_stream=s) for s in (2, 0)]
    for e in engines:
        for f in range(F):
            e.pool_load(f, [gold[p][f] for p in range(3)])
    rng = np.random.default_rng(8)
    for k in range(K):
        planes, bsize = _batch(geom, F, seed=50 + k)
        slot = np.array([[f, f if k == 0 else F + f] for f in range(F)], np.int32)
        packed = _pack(_grids(geom, F, seed=60 + k))
        st, cl = engines
        st.stage_inputs(planes, bsize)
        st.stage_mc(None, slot, packed, resident=True)
        so = st.prepare_io(symbols=False, recon=False, pred=False)
        assert set(so) == {"counts", "sym_index", "sym_blocks", "sym_bands", "sym_pulses", "sym_dc"}
        st.submit()
        so = _copy(st.wait())
        co = _copy(cl.encode(planes, bsize, ref_slot=slot, mv_grid=packed, resident=True))
        n = int(so["sym_index"][:, 1].sum())
        assert n == len(co["luma_dc"]) + len(co["chroma_dc"])
        qdc = so["sym_dc"]["qdc"][:n]
        skip = (rng.random(n) < 0.3).astype(np.uint8)
        dc = np.where(skip == 1, 0, qdc).astype(np.int32)
        levels = rng.integers(0, 6, (F, geom.nvsb, geom.nhsb)).astype(np.uint8)
        store = np.arange(F, 2 * F, dtype=np.int32)
        a = _copy(st.finish_stream(skip, dc, levels, ref_slot_out=store))
        perm = symbols.stream_to_classic(dict(co, sym_index=so["sym_index"], sym_blocks=so["sym_blocks"]))
        cskip, cdc = np.zeros(n, np.uint8), np.zeros(n, np.int32)
        cskip[perm], cdc[perm] = skip, dc
        nl = len(co["luma_dc"])
        assert np.array_equal(cdc[cskip == 0], np.concatenate([co["luma_dc"], co["chroma_dc"]])[cskip == 0])
        b = _copy(cl.finish(cskip[:nl], cdc[:nl], cskip[nl:], cdc[nl:], levels, ref_slot_out=store))
        for key in a:
            assert np.array_equal(a[key], b[key]), (k, key)
    for p in range(3):
        assert np.array_equal(engines[0].pool_plane(p), engines[1].pool_plane(p)), p
    for e in engines:
        e.close()


# ---- refusals ----------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_create_refusals():
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    geom = Geometry(128, 64)
    for kw in (dict(symbol_stream=2), dict(inter=1, symbol_stream=3), dict(symbol_stream=-1),
               dict(inter=1, symbol_stream=1)):
        with pytest.raises(RuntimeError, match="symbol_stream"):
            engine.KeyframeEngine(geom, nframes=1, q0=45, pvq_qm_q4=Q4, **kw)


@pytest.mark.gpu
def test_submit_refusals():
    """sym_dc from a keyframe stream engine, below its bound, or not pinned: refused before any copy or launch."""
    from daala_b200 import engine, symbols, synth
    from daala_b200.frame import Geometry
    geom = Geometry(200, 130)
    F = 2
    planes, pred, bsize = _stack(_frames(geom, F, seed=5))
    # a keyframe engine with the keyframe stream
    kf = engine.KeyframeEngine(geom, nframes=F, q0=45, pvq_qm_q4=Q4, symbol_stream=1)
    kf.stage_inputs(planes, bsize)
    kf.prepare_io(stream=True)
    b = kf.symbol_bounds()
    dc = engine.Pinned((int(b.blocks),), symbols.DC_DTYPE)
    io = engine.IO.from_buffer_copy(kf._io)
    io.sym_dc, io.sym_dc_cap = dc.ptr, int(b.blocks)
    assert kf.L.daala_b200_kf_submit(kf.kf, ctypes.byref(io)) == INVALID
    assert b"sym_dc" in kf.L.daala_b200_kf_error(kf.kf) and b"symbol_stream = 2" in kf.L.daala_b200_kf_error(kf.kf)
    assert int(kf.counts()[engine.CNT["n_luma"]]) == 0
    dc.free()
    kf.close()
    eng = _engine(geom, F)
    eng.stage_inputs(planes, bsize, pred=pred)
    eng.prepare_io(stream=True)
    io = eng._io
    cap = io.sym_dc_cap
    io.sym_dc_cap = cap - 1
    assert eng.L.daala_b200_kf_submit(eng.kf, ctypes.byref(io)) == INVALID
    io.sym_dc_cap = cap
    ptr = io.sym_dc
    host = np.zeros(int(cap) * 8 + 64, np.uint8)   # pageable memory
    io.sym_dc = host.ctypes.data
    assert eng.L.daala_b200_kf_submit(eng.kf, ctypes.byref(io)) == INVALID
    io.sym_dc = ptr
    assert int(eng.counts()[engine.CNT["n_luma"]]) == 0
    # luma_dc / chroma_dc are optional on a symbol_stream = 2 engine
    lean = engine.IO.from_buffer_copy(io)
    lean.luma_dc = lean.chroma_dc = None
    eng._check(eng.L.daala_b200_kf_submit(eng.kf, ctypes.byref(lean)), "kf_submit")
    lean_out = _copy(eng.wait())
    eng.submit()
    out = _copy(eng.wait())
    _assert_matches_reference(out, F, "after refusals")
    assert not symbols.stream_equal(lean_out, out, range(F))
    eng.close()


@pytest.mark.gpu
def test_finish_refusals():
    """Both forms, the stream form without the stream, half a stream form, a bad skip value or |dc| in the stream form:
    refused before any copy or launch, and the next finish is exact."""
    from daala_b200 import _native, engine, symbols
    from daala_b200.frame import Geometry
    from tests.test_gpu_engine_inter_finish import _decisions
    geom = Geometry(200, 130)
    F, q0 = 2, 45
    planes, pred, bsize = _stack(_frames(geom, F, seed=7))
    eng = _engine(geom, F, q0, inter_finish=1)
    out = _copy(eng.encode(planes, bsize, pred=pred, stream=True))
    perm = symbols.stream_to_classic(out)
    ls, ld, cs, cd, levels = _decisions(out, geom, F, seed=3)[:5]
    skip, dc = np.concatenate([ls, cs])[perm], np.concatenate([ld, cd])[perm]
    ref = _copy(eng.finish_stream(skip, dc, levels))
    before = eng.counts().copy()
    L = eng.L

    def refused(fio, word):
        assert L.daala_b200_kf_finish(eng.kf, ctypes.byref(fio)) == INVALID
        msg = L.daala_b200_kf_error(eng.kf).decode()
        assert word in msg, (word, msg)

    eng.prepare_finish(ls, ld, cs, cd, levels)
    both = engine.FinishIO.from_buffer_copy(eng._fio)
    eng.prepare_finish_stream(skip, dc, levels)
    both.stream_skip, both.stream_dc = eng._fio.stream_skip, eng._fio.stream_dc
    refused(both, "both forms")
    half = engine.FinishIO.from_buffer_copy(eng._fio)
    half.stream_dc = None
    refused(half, "stream_skip and stream_dc are required")
    neither = engine.FinishIO.from_buffer_copy(eng._fio)
    neither.stream_skip = neither.stream_dc = None
    refused(neither, "luma_skip, chroma_skip, luma_dc and chroma_dc are required")
    dq_max = max((q0 * int(Q4[p][bs * (bs + 1)])) >> 4 for p in range(3) for bs in range(5))
    for i in (0, len(skip) - 1):
        bad_skip, bad_dc = skip.copy(), dc.copy()
        bad_skip[i] = 2
        bad_dc[i] = (1 << 30) // dq_max + 1
        eng.prepare_finish_stream(bad_skip, dc, levels)
        with pytest.raises(_native.CudaError, match="skip value"):
            eng.finish_submit()
        eng.prepare_finish_stream(skip, bad_dc, levels)
        with pytest.raises(_native.CudaError, match=r"\|dc\|"):
            eng.finish_submit()
    assert np.array_equal(eng.counts(), before)
    again = _copy(eng.finish_stream(skip, dc, levels))
    for k in ref:
        assert np.array_equal(ref[k], again[k]), k
    eng.close()
    # the stream form on an engine without the stream
    plain = _engine(geom, F, q0, inter_finish=1, symbol_stream=0)
    plain.encode(planes, bsize, pred=pred)
    plain.prepare_finish_stream(skip, dc, levels)
    with pytest.raises(_native.CudaError, match="symbol_stream = 2"):
        plain.finish_submit()
    plain.close()


# ---- replays, engines, copies ------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_replays_engines_and_used_part():
    """Two engines fed the same batch, and graph replays followed by a submit, give identical streams; the copy
    writes only the used part of each host array (buffers 64 entries above their bound, filled with a sentinel)."""
    from daala_b200 import engine, symbols
    from daala_b200.frame import Geometry
    geom = Geometry(328, 200)
    F = 3
    planes, pred, bsize = _stack(_frames(geom, F, seed=21))
    a, b = _engine(geom, F), _engine(geom, F)
    for e in (a, b):
        e.stage_inputs(planes, bsize, pred=pred)
        e.prepare_io(stream=True)
    bd = a.symbol_bounds()
    big = {}
    for k, dt, n, row in (("sym_blocks", symbols.BLOCK_DTYPE, bd.blocks, ()), ("sym_bands", np.int16, bd.bands, (4,)),
                          ("sym_pulses", np.uint8, bd.pulse_bytes, ()), ("sym_dc", symbols.DC_DTYPE, bd.blocks, ())):
        big[k] = engine.Pinned((int(n) + 64,) + row, dt)
        big[k].array.view(np.uint8)[...] = 0xA5
        setattr(a._io, k, big[k].ptr)
        setattr(a._io, k + "_cap", int(n) + 64)
    a.submit()
    b.submit()
    a.wait()
    ra = {k: v.array.copy() for k, v in big.items()}
    ra["sym_index"] = np.array(a._out["sym_index"])
    rb = _copy(b.wait())
    _assert_matches_reference(rb, F)
    assert not symbols.stream_equal(ra, rb, range(F))
    idx = ra["sym_index"]
    used = {"sym_blocks": int(idx[:, 1].sum()), "sym_bands": int(idx[:, 3].sum()), "sym_pulses": int(idx[:, 5].sum()),
            "sym_dc": int(idx[:, 1].sum())}
    for k, n in used.items():
        assert (ra[k][n:].view(np.uint8) == 0xA5).all(), k
    for v in big.values():
        v.free()
    b.time_device(engine.PH_ALL, True, 3)
    b.submit()
    again = _copy(b.wait())
    assert not symbols.stream_equal(again, rb, range(F))
    a.close()
    b.close()


# ---- no GPU ------------------------------------------------------------------------------------------------------

LAYOUT = r"""
#include <stddef.h>
#include <stdio.h>
#include "daala_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(daala_b200_kf_sym_dc), offsetof(daala_b200_kf_sym_dc, dc_resid),
         sizeof(daala_b200_kf_io), offsetof(daala_b200_kf_io, sym_dc), offsetof(daala_b200_kf_io, sym_dc_cap),
         sizeof(daala_b200_kf_finish_io), offsetof(daala_b200_kf_finish_io, ref_slot_out),
         offsetof(daala_b200_kf_finish_io, stream_skip), offsetof(daala_b200_kf_finish_io, stream_dc));
  return 0;
}
"""


def test_stream_structs_match_the_header(tmp_path):
    from daala_b200 import engine, symbols
    (tmp_path / "layout.c").write_text(LAYOUT)
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(tmp_path / "layout.c"), "-o", exe], check=True)
    got = [int(v) for v in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [symbols.DC_DTYPE.itemsize, symbols.DC_DTYPE.fields["dc_resid"][1], ctypes.sizeof(engine.IO),
                   engine.IO.sym_dc.offset, engine.IO.sym_dc_cap.offset, ctypes.sizeof(engine.FinishIO),
                   engine.FinishIO.ref_slot_out.offset, engine.FinishIO.stream_skip.offset,
                   engine.FinishIO.stream_dc.offset]


def _map(geom, f, seed):
    from daala_b200 import synth
    return synth.block_size_map(geom, "mixed", seed=seed + f)


def _classic_outputs(geom, F, seed):
    """Classic outputs of a P-frame step made up on the host: the blocks of seeded maps in a shuffled order, seeded
    band records (K up to 300, so some bands take 16-bit pulses), pulses, skip_diff and DC values."""
    from daala_b200 import pvq, symbols
    rng = np.random.default_rng(seed)
    lists = {"luma": [], "chroma": []}
    for f in range(F):
        o = symbols.coding_order(_map(geom, f, seed), geom)
        for kind, sel in (("luma", o["pli"] == 0), ("chroma", o["pli"] > 0)):
            b = np.zeros(int(sel.sum()), pvq.BLOCK_DTYPE)
            for k in ("x0", "y0", "bs", "pli"):
                b[k] = o[k][sel]
            b["frame"] = f
            lists[kind].append(b)
    out = {}
    for kind in ("luma", "chroma"):
        b = np.concatenate(lists[kind])
        b = b[rng.permutation(len(b))]
        n = np.minimum(16 << (2 * b["bs"].astype(np.int64)), 512)
        b["coef_off"] = np.concatenate([[0], np.cumsum(n)[:-1]])
        res = np.zeros((len(b), 9, 4), np.int16)
        res[:, :, 0] = rng.integers(0, 20, (len(b), 9))
        res[:, :, 1] = rng.integers(-1, 8, (len(b), 9))
        res[:, :, 3] = np.where(rng.random((len(b), 9)) < 0.5, 0, rng.integers(1, 300, (len(b), 9)))
        y16 = rng.integers(-120, 121, int(n.sum())).astype(np.int16)   # fits the 8-bit pulses of K <= 127
        out.update({kind + "_blocks": b, kind + "_res": res, kind + "_y16": y16,
                    kind + "_skip_diff": rng.random(len(b)), kind + "_dc": rng.integers(-50, 50, len(b)).astype(np.int32),
                    kind + "_dc_resid": rng.integers(-900, 900, len(b)).astype(np.int32)})
    out["chroma_flip"] = np.ones(len(out["chroma_blocks"]), np.int32)   # ignored on P frames
    return out


def test_pack_read_round_trip_with_dc():
    """pack_reference / read_frame with DC records, stream_equal's DC comparison, and stream_to_classic."""
    from daala_b200 import symbols
    from daala_b200.frame import Geometry
    geom = Geometry(200, 130)
    F = 3
    out = _classic_outputs(geom, F, seed=4)
    s = symbols.pack_reference(out, F)
    assert s["sym_dc"].dtype == symbols.DC_DTYPE and not s["sym_blocks"]["flip"].any()
    assert not symbols.stream_equal(s, s, range(F))
    perm = symbols.stream_to_classic(dict(out, **s))
    n = len(perm)
    assert np.array_equal(np.sort(perm), np.arange(n))
    classic = {k: np.concatenate([out["luma_" + k], out["chroma_" + k]]) for k in ("blocks", "dc", "dc_resid")}
    for k in ("x0", "y0", "pli", "bs"):
        assert np.array_equal(classic["blocks"][k][perm], s["sym_blocks"][k]), k
    assert np.array_equal(classic["dc"][perm], s["sym_dc"]["qdc"])
    assert np.array_equal(classic["dc_resid"][perm], s["sym_dc"]["dc_resid"])
    for f in range(F):
        r = symbols.read_frame(s, f)
        i0, nb = int(s["sym_index"][f, 0]), int(s["sym_index"][f, 1])
        assert np.array_equal(r["dc"], s["sym_dc"][i0:i0 + nb])
        assert np.array_equal(r["blocks"]["x0"], symbols.coding_order(_map(geom, f, 4), geom)["x0"])
        # every pulse read back is the classic y16 value
        for q in np.nonzero(r["bands"][:, 3] > 0)[0][:50]:
            i = int(perm[i0 + r["band_block"][q]])
            nl = len(out["luma_blocks"])
            kind, j = ("luma", i) if i < nl else ("chroma", i - nl)
            a = int(out[kind + "_blocks"]["coef_off"][j]) + symbols.BAND_EDGES[r["band_no"][q]]
            assert np.array_equal(r["pulses"][q], out[kind + "_y16"][a:a + len(r["pulses"][q])].astype(np.int32))
    assert (s["sym_bands"][:, 3] > 127).any()
    changed = dict(s, sym_dc=s["sym_dc"].copy())
    changed["sym_dc"]["dc_resid"][-1] += 1
    assert [b[1] for b in symbols.stream_equal(changed, s, range(F))] == ["sym_dc"]


