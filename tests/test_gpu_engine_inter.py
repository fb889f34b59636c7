"""The engine's P-frame residual mode (config.inter; csrc/kf_engine.cu) through its host-buffer C ABI against
inter_oracle.inter_chain: every band of every plane quantised against the transformed prediction by the phase
kernels, scalar DC, the inter form of od_init_skipped_coeffs, reconstruction."""
import ctypes

import numpy as np
import pytest

from tests import frame_oracle, inter_oracle, oracle_lib

pytestmark = [pytest.mark.gpu]


def _oracle():
    ref = oracle_lib.load_ref()
    return (ref, "ref") if ref is not None else (oracle_lib.load_port(), "port")


def _coding_tables():
    """Per block size: (rows, cols) of the coded prefix in coding order."""
    from daala_b200 import pvq
    inp = pvq.qm_inputs()
    scans = {m: inp["scan%d" % m].astype(np.int64) for m in (4, 8, 16, 32, 64)}
    tabs = {}
    for bs in range(5):
        n = 4 << bs
        idx = np.arange(n * n).reshape(n, n)
        order = pvq.raster_to_coding_order(idx, scans)[:min(n * n, 512)]
        tabs[bs] = (order // n, order % n)
    return tabs


def _y_plane(blocks, y16, geom, pli, frame, tabs):
    h, w = geom.plane_shape(pli)
    out = np.zeros((h, w), np.int32)
    sel = np.nonzero((blocks["pli"] == pli) & (blocks["frame"] == frame))[0]
    for bs in range(5):
        ids = sel[blocks["bs"][sel] == bs]
        if not len(ids):
            continue
        r, c = tabs[bs]
        off = blocks["coef_off"][ids].astype(np.int64)[:, None] + np.arange(len(r))[None, :]
        out[blocks["y0"][ids].astype(np.int64)[:, None] + r[None, :],
            blocks["x0"][ids].astype(np.int64)[:, None] + c[None, :]] = y16[off]
    return out


def _at_origins(blocks, values, geom, pli, frame, fill, dtype):
    """Per-block values of one plane of one frame at the blocks' origins in 4-sample units (the oracle's layout)."""
    h, w = geom.plane_shape(pli)
    out = np.full((h // 4, w // 4), fill, dtype)
    sel = (blocks["pli"] == pli) & (blocks["frame"] == frame)
    out[blocks["y0"][sel] >> 2, blocks["x0"][sel] >> 2] = values[sel]
    return out


def _compare(out, coeffs, md, geom, frames, q0, q4, frame_ids=None):
    """out / coeffs / md: the engine's results for the batch `frames` = [(planes, pred, bsize)]."""
    from daala_b200 import engine
    lib, prefix = _oracle()
    tabs = _coding_tables()
    wants = []
    for f, (planes, pred, bsize) in enumerate(frames):
        if frame_ids is not None and f not in frame_ids:
            wants.append(None)
            continue
        want = inter_oracle.inter_chain(lib, prefix, planes, pred, geom, bsize, q0, q4)
        wants.append(want)
        for pli in range(3):
            kind = "luma" if pli == 0 else "chroma"
            blocks, res, y16 = out[kind + "_blocks"], out[kind + "_res"], out[kind + "_y16"]
            w = want[pli]
            assert np.array_equal(md[pli][f], w["md"]), ("md", f, pli)
            got = engine.band_records(blocks, res, geom, pli, f)
            bad = np.argwhere(got != w["rec"])
            assert len(bad) == 0, ("band decisions", f, pli, len(bad), bad[:8].tolist(), got[tuple(bad[0][:3])].tolist(),
                                   w["rec"][tuple(bad[0][:3])].tolist())
            assert np.array_equal(_y_plane(blocks, y16, geom, pli, f, tabs), w["yplane"]), ("pulses", f, pli)
            qdc = _at_origins(blocks, out[kind + "_dc"], geom, pli, f, 0, np.int32)
            assert np.array_equal(qdc, w["qdc"]), ("qdc", f, pli)
            sd = _at_origins(blocks, out[kind + "_skip_diff"], geom, pli, f, np.nan, np.float64)
            assert np.array_equal(np.isnan(sd), np.isnan(w["skip_diff"])), ("block origins", f, pli)
            m = ~np.isnan(sd)
            assert np.allclose(sd[m], w["skip_diff"][m], rtol=1e-5, atol=1e-9), ("skip_diff", f, pli)
            assert np.array_equal(coeffs[pli][f], w["dq"]), ("quantised plane", f, pli)
            assert np.array_equal(out["recon%d" % pli][f], w["recon"]), ("recon", f, pli)
        assert not out["chroma_flip"].any()
    return wants


def _check_batch(eng, geom, frames, q0, q4, frame_ids=None):
    planes = [np.stack([f[0][p] for f in frames]) for p in range(3)]
    pred = [np.stack([f[1][p] for f in frames]) for p in range(3)]
    out = eng.encode(planes, np.stack([f[2] for f in frames]), pred=pred)
    out = {k: np.array(v) for k, v in out.items()}
    coeffs = [eng.coeff_plane(p) for p in range(3)]
    md = [eng.pred_coeff_plane(p) for p in range(3)]
    return out, _compare(out, coeffs, md, geom, frames, q0, q4, frame_ids)


def _frames(geom, n, mode="mixed", seed=0, unrelated=()):
    """n frames of (planes, prediction, block sizes): frame f is synthetic frame f + 1 predicted from synthetic
    frame f (a small residual); for f in `unrelated` from a frame of another noise seed and phase instead."""
    from daala_b200 import synth
    pics = []
    s = 12345 + seed
    for f in range(n + 1):
        planes, s = synth.frame(geom.pic_w, geom.pic_h, f=f, seed=s)
        pics.append(synth.pad_planes(planes, geom))
    frames = []
    for f in range(n):
        pred = pics[f]
        if f in unrelated:
            other, _ = synth.frame(geom.pic_w, geom.pic_h, f=40 + 7 * f, seed=999 + f)
            pred = synth.pad_planes(other, geom)
        frames.append((pics[f + 1], pred, synth.block_size_map(geom, mode, seed=70 + f + seed)))
    return frames


def _engine(geom, F, q0, q4, **kw):
    from daala_b200 import engine
    return engine.KeyframeEngine(geom, nframes=F, q0=q0, pvq_qm_q4=q4, inter=1, **kw)


Q4 = np.full((3, 30), 20, np.uint8)


@pytest.mark.parametrize("w,h,q0,F,unrelated", [(200, 130, 45, 1, ()), (384, 256, 38, 2, (1,)), (328, 200, 72, 3, ())])
def test_inter_engine_matches_oracle_on_mixed_maps(w, h, q0, F, unrelated):
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    geom = Geometry(w, h)
    eng = _engine(geom, F, q0, Q4)
    frames = _frames(geom, F, seed=F, unrelated=unrelated)
    out, wants = _check_batch(eng, geom, frames, q0, Q4)
    # the small-residual frames copy the prediction in many bands; the unrelated prediction loses to the
    # no-reference candidates somewhere
    res = out["luma_res"]
    nb = np.array([1, 4, 7, 9, 9])[out["luma_blocks"]["bs"]]
    coded = np.arange(9)[None, :] < nb[:, None]
    assert (res[..., 3][coded] == 0).sum() > 0 and (res[..., 3][coded] > 0).sum() > 0
    if unrelated:
        fr = out["luma_blocks"]["frame"] == unrelated[0]
        assert ((res[..., 1] == -1) & (res[..., 3] > 0) & coded)[fr].any()
    # list bookkeeping: every band of every luma block is an item, and nothing of the chain structure is built
    c = out["counts"]
    assert int(c[engine.CNT["items_l"]:engine.CNT["items_l"] + 3].sum()) == int(nb.sum())
    assert int(c[engine.CNT["total_hi"]]) == 0 and int(c[engine.CNT["n_heads"]]) == 0 and int(c[engine.CNT["n_heads0"]]) == 0
    assert eng.launches_per_step() > 0
    eng.close()


@pytest.mark.parametrize("mode", ["4", "8", "16", "32", "64"])
def test_inter_engine_uniform_maps(mode):
    """Every block size alone; 32 and 64: the uncoded tail of the block is the transformed prediction."""
    from daala_b200.frame import Geometry
    geom = Geometry(192, 128)
    eng = _engine(geom, 2, 45, Q4)
    out, wants = _check_batch(eng, geom, _frames(geom, 2, mode=mode, seed=3, unrelated=(1,)), 45, Q4)
    if mode in ("32", "64"):
        n = int(mode)
        dq, md = wants[0][0]["dq"], wants[0][0]["md"]
        tail = np.ones((n, n), bool)
        r, c = _coding_tables()[{"32": 3, "64": 4}[mode]]
        tail[r, c] = False
        assert tail.sum() == n * n - 512 and np.array_equal(dq[:n, :n][tail], md[:n, :n][tail]) and md[:n, :n][tail].any()
    eng.close()


def test_inter_engine_1080p():
    from daala_b200.frame import Geometry
    geom = Geometry(1920, 1080)
    eng = _engine(geom, 1, 72, Q4)
    _check_batch(eng, geom, _frames(geom, 1, seed=9), 72, Q4)
    eng.close()


def test_inter_engine_edge_content():
    """Prediction equal to the source: no DC index and next to no band is coded (the 16-bit correlation of a vector
    with itself can round below one, and such a band codes a small angle), and where nothing is the reconstruction
    is the inverse of md.  Flat against noise and black against white: the largest residuals 8-bit content has."""
    from daala_b200 import synth
    from daala_b200.frame import Geometry
    geom = Geometry(136, 72)
    rng = np.random.default_rng(4)
    shapes = [geom.plane_shape(p) for p in range(3)]
    src = synth.pad_planes(synth.frame(136, 72, f=5)[0], geom)
    noise = [rng.integers(0, 256, size=s, dtype=np.uint8) for s in shapes]
    flat = [np.full(s, 128, np.uint8) for s in shapes]
    black, white = [np.zeros(s, np.uint8) for s in shapes], [np.full(s, 255, np.uint8) for s in shapes]
    bsize = synth.block_size_map(geom, "mixed", seed=21)
    frames = [(src, src, bsize), (flat, noise, bsize), (noise, flat, synth.block_size_map(geom, "64")),
              (black, white, bsize), (white, black, synth.block_size_map(geom, "8"))]
    eng = _engine(geom, len(frames), 38, Q4)
    out, wants = _check_batch(eng, geom, frames, 38, Q4)
    lib, prefix = _oracle()
    for kind in ("luma", "chroma"):
        f0 = out[kind + "_blocks"]["frame"] == 0
        nb = np.array([1, 4, 7, 9, 9])[out[kind + "_blocks"]["bs"][f0]]
        k = out[kind + "_res"][f0][..., 3][np.arange(9)[None, :] < nb[:, None]]
        assert (k > 0).sum() <= k.size // 500 and not out[kind + "_dc"][f0].any()
        assert out[kind + "_dc"][~f0].any()
    for pli in range(3):
        if not wants[0][pli]["yplane"].any():
            assert np.array_equal(out["recon%d" % pli][0],
                                  frame_oracle.inverse_plane(lib, prefix, wants[0][pli]["md"], geom, pli, bsize, 0))
    eng.close()


def test_inter_engine_batch_independence_and_graph_replay():
    """Frame i of a batch equals the same frame encoded alone; a second submit with other maps and predictions
    on the same engine (the captured graph replayed, the lists rebuilt on the device) is right as well."""
    from daala_b200.frame import Geometry
    geom = Geometry(200, 130)
    q0 = 45
    eng3, eng1 = _engine(geom, 3, q0, Q4), _engine(geom, 1, q0, Q4)
    for seed in (1, 2):   # two submits per engine
        frames = _frames(geom, 3, seed=10 * seed, unrelated=(seed,))
        out, _ = _check_batch(eng3, geom, frames, q0, Q4)
        coeffs = [eng3.coeff_plane(p) for p in range(3)]
        for f in range(3):
            one, _ = _check_batch(eng1, geom, frames[f:f + 1], q0, Q4, frame_ids=())
            for kind in ("luma", "chroma"):
                sel = out[kind + "_blocks"]["frame"] == f
                for key in ("_dc", "_skip_diff"):
                    assert np.array_equal(out[kind + key][sel], one[kind + key]), (kind, key, f)
                # band records: the entries of the bands a block has (the others are never written)
                coded = np.arange(9)[None, :] < np.array([1, 4, 7, 9, 9])[one[kind + "_blocks"]["bs"]][:, None]
                assert np.array_equal(out[kind + "_blocks"]["bs"][sel], one[kind + "_blocks"]["bs"])
                assert np.array_equal(out[kind + "_res"][sel][coded], one[kind + "_res"][coded]), (kind, f)
                offs = out[kind + "_blocks"]["coef_off"][sel]
                n = len(one[kind + "_y16"])
                assert np.array_equal(out[kind + "_y16"][offs[0]:offs[0] + n], one[kind + "_y16"])
            for p in range(3):
                assert np.array_equal(out["recon%d" % p][f], one["recon%d" % p][0])
                assert np.array_equal(coeffs[p][f], eng1.coeff_plane(p)[0])
    eng3.close()
    eng1.close()


def test_inter_engine_device_resident_phases():
    """upload + run_device with the phase flags one after the other gives what the graph gives; the launch
    count of the mode is what launches_per_step says it is made of."""
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    geom = Geometry(200, 130)
    frames = _frames(geom, 2, seed=5)
    eng = _engine(geom, 2, 45, Q4)
    out, _ = _check_batch(eng, geom, frames, 45, Q4)
    want = [eng.coeff_plane(p) for p in range(3)], [eng.recon_plane(p) for p in range(3)]
    eng2 = _engine(geom, 2, 45, Q4)
    eng2.upload([np.stack([f[0][p] for f in frames]) for p in range(3)], np.stack([f[2] for f in frames]),
                pred=[np.stack([f[1][p] for f in frames]) for p in range(3)])
    for ph in (engine.PH_LISTS, engine.PH_FORWARD, engine.PH_PVQ_LUMA, engine.PH_PVQ_CHROMA, engine.PH_INVERSE):
        eng2.run_device(ph, graph=False)
    for p in range(3):
        assert np.array_equal(eng2.coeff_plane(p), want[0][p]) and np.array_equal(eng2.recon_plane(p), want[1][p])
    assert eng2.time_device(engine.PH_PVQ_LUMA, graph=False, reps=2) > 0
    # lists 5, forward 2, per stage gather + finish + 3 phase kernels per chunk, inverse 2
    assert (eng.launches_per_step() - 13) % 3 == 0 and eng.launches_per_step() >= 13 + 3 * 6
    with pytest.raises(ValueError):
        eng2.upload([np.stack([f[0][p] for f in frames]) for p in range(3)], np.stack([f[2] for f in frames]))
    eng.close()
    eng2.close()


def test_inter_engine_refusals():
    from daala_b200 import _native, engine
    from daala_b200.frame import Geometry
    geom = Geometry(128, 64)
    for kw, word in ((dict(dering=1), "dering"), (dict(symbol_stream=1), "symbol_stream"),
                     (dict(noref_prepass=1), "noref_prepass"), (dict(level_chains=1), "level_chains"),
                     (dict(sb_row0=0, sb_rows=1), "shard"), (dict(inter=2), "0 or 1")):
        args = dict(inter=1)
        args.update(kw)
        with pytest.raises(RuntimeError, match=word):
            engine.KeyframeEngine(geom, nframes=1, q0=45, pvq_qm_q4=Q4, **args)
    # a keyframe engine refuses pred=, an inter engine a batch without it
    kf = engine.KeyframeEngine(geom, nframes=1, q0=45, pvq_qm_q4=Q4, split_free=1)
    frames = _frames(geom, 1)
    planes, pred, bsize = ([a[None] for a in frames[0][0]], [a[None] for a in frames[0][1]], frames[0][2][None])
    with pytest.raises(ValueError):
        kf.encode(planes, bsize, pred=pred)
    kf.close()
    eng = _engine(geom, 1, 45, Q4)
    with pytest.raises(ValueError):
        eng.encode(planes, bsize)
    # through the C ABI: NULL prediction planes or DC outputs are refused before anything is copied or launched
    eng.stage_inputs(planes, bsize, pred=pred)
    eng.prepare_io()
    before = eng.counts().copy()
    for field in ("pred_pixels", "luma_dc", "chroma_dc"):
        io = engine.IO.from_buffer_copy(eng._io)
        if field == "pred_pixels":
            io.pred_pixels[1] = None
        else:
            setattr(io, field, None)
        assert eng.L.daala_b200_kf_submit(eng.kf, ctypes.byref(io)) != 0
        assert b"pred_pixels" in eng.L.daala_b200_kf_error(eng.kf)
    eng.wait()
    assert np.array_equal(eng.counts(), before) and int(before[engine.CNT["n_luma"]]) == 0   # no step has run yet
    eng.submit()
    eng.wait()
    assert int(eng.counts()[engine.CNT["n_luma"]]) > 0
    eng.close()


def test_inter_engine_block_capacity_boundary():
    """An all-4x4 map at full capacity: every block is one class-0 item, and block and item lists are filled to
    the last entry.  With max_blocks_div = 2 a batch whose luma block count equals the halved capacity exactly
    passes, and one with three blocks more is refused by submit before anything runs."""
    from daala_b200 import _native, engine
    from daala_b200.frame import Geometry
    from tests.test_gpu_engine import _zorder_map
    geom = Geometry(64, 64)
    F = 2
    nunits = F * geom.bsize_shape[0] * geom.bsize_shape[1]
    eng = _engine(geom, F, 72, Q4)
    out, _ = _check_batch(eng, geom, _frames(geom, F, mode="4", seed=8), 72, Q4)
    assert len(out["luma_blocks"]) == 4 * nunits and int(out["counts"][engine.CNT["items_l"]]) == 4 * nunits
    eng.close()
    eng = _engine(geom, F, 72, Q4, max_blocks_div=2)
    assert eng.buf.max_luma_blocks == nunits * 2 + 64
    # 75 4x4 units, 9 8x8 blocks, 11 16x16 blocks over 128 units: 320 luma blocks; one more unit as 4x4: 323
    maps = _zorder_map(geom, F, [0] * 75 + [1] * 9 + [2] * 11)
    over = _zorder_map(geom, F, [0] * 76 + [1] * 8 + [2] * 11)
    assert eng.count_blocks(maps).n_luma == eng.buf.max_luma_blocks < eng.count_blocks(over).n_luma
    frames = _frames(geom, F, seed=8)
    out, _ = _check_batch(eng, geom, [(f[0], f[1], maps[i]) for i, f in enumerate(frames)], 72, Q4)
    assert int(out["counts"][engine.CNT["error"]]) == 0 and len(out["luma_dc"]) == eng.buf.max_luma_blocks
    with pytest.raises(_native.CudaError):
        eng.encode([np.stack([f[0][p] for f in frames]) for p in range(3)], over,
                   pred=[np.stack([f[1][p] for f in frames]) for p in range(3)])
    eng.close()
