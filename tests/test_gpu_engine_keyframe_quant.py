"""Keyframe batches with a quantizer per frame (config.keyframe_quant = 1) on the GPU.

The settings are the keyframe column of tests/golden/encoder_settings.npz: the eight sweep points (q0 12 to 5890) in the
three stream configurations (masking on / off with the HVS matrix, masking on with the flat matrix).  Each configuration
gets its own engine, because masking, the matrices and pvq_norm_lambda are stream settings.  The engine under test is
created with per-frame config fields far from every record (q0 999, coded quantizer 33, dering_lambda 7, pvq_qm_q4 all
9), so a value baked at create would show.

- Frame by frame, a batch of all eight points equals one keyframe_quant = 0 engine per frame, created at that frame's
  settings, in every output: reconstruction, coefficient planes, band records, the symbol stream (blocks, bands,
  pulses), skip_diff, CfL flips, the DC indices (haar_dc_quant = 1) and the searched deringing levels (dering = 2).
- One mixed batch per oracle: each frame against the pipeline oracle and against the Haar DC frame driver at its own
  settings.
- Nothing is baked at create: batch A then batch B on one engine, live and replayed, equals a fresh engine's B; a
  permuted batch permutes the outputs.
- Uniform records equal the engine without the mode, launches included; the forked graph and the phase-by-phase path
  agree (dering 1 / 2, haar_dc_quant on / off); submit refuses missing and out-of-range records before any copy."""
import os

import numpy as np
import pytest

from daala_b200 import engine, synth
from daala_b200.frame import Geometry
from tests import frame_oracle, haar_dc_oracle, oracle_lib
from tests.test_gpu_engine_quantizer_range import NPOINTS, settings

pytestmark = [pytest.mark.gpu]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIGS = ("hvs-masking", "hvs", "flat-masking")
ALL = tuple(range(NPOINTS))
# the per-frame config fields of the engine under test: none of them is any record's
OFF = dict(q0=999, pvq_qm_q4=np.full((3, 30), 9, np.uint8), coded_quantizer=33, dering_lambda=7.0)
FULL = dict(dering=2, symbol_stream=1, haar_dc_quant=1)


def _records(points, config):
    ss = [settings(p, config, 0) for p in points]
    return engine.frame_quant_records([s["q0"] for s in ss], [s["cq"] for s in ss], [s["dering_lambda"] for s in ss],
                                      np.stack([s["q4"] for s in ss]))


def _stream_kw(config):
    s = settings(0, config, 0)
    return dict(use_masking=s["masking"], lam=s["lam"], qm=s["qm"], qm_inv=s["qm_inv"], qm_is_flat=s["flat"])


def _mixed(geom, F, config, **kw):
    return engine.KeyframeEngine(geom, nframes=F, keyframe_quant=1, **OFF, **_stream_kw(config), **kw)


def _uniform(geom, point, config, F=1, **kw):
    s = settings(point, config, 0)
    return engine.KeyframeEngine(geom, nframes=F, q0=s["q0"], pvq_qm_q4=s["q4"], coded_quantizer=s["cq"],
                                 dering_lambda=s["dering_lambda"], **_stream_kw(config), **kw)


def _real_map(geom, k):
    real = np.load(os.path.join(ROOT, "daala_b200", "data", "bench_bsize_4k.npz"))["bsize_%d" % (k % 4)]
    h, w = geom.bsize_shape
    return np.ascontiguousarray(real[:h, :w])


def _frames(geom, n, seed):
    """n frames: content from the synthetic generator; maps cycle through a random quadtree, a real encoder map (the
    top-left of bench.py's 4K maps) and all 4x4."""
    planes, maps = [], []
    for f in range(n):
        planes.append(synth.pad_planes(synth.frame(geom.pic_w, geom.pic_h, f=seed + f)[0], geom))
        kind = f % 3
        maps.append(synth.block_size_map(geom, "mixed", seed=seed + f) if kind == 0
                    else _real_map(geom, f) if kind == 1 else synth.block_size_map(geom, "4"))
    return planes, maps


def _levels(geom, n, seed):
    return np.random.default_rng(seed).integers(0, 6, size=(n, geom.nvsb, geom.nhsb)).astype(np.uint8)


def _run(eng, planes, maps, records=None, levels=None):
    out = eng.encode([np.stack([fr[p] for fr in planes]) for p in range(3)], np.stack(maps), frame_quant=records,
                     dering_levels=levels, stream=bool(eng.symbol_stream))
    res = {k: np.array(v) for k, v in out.items()}
    res["coeffs"] = [eng.coeff_plane(p) for p in range(3)]
    return res


def _frame(res, geom, f):
    """Every output of frame f of a step, in a form that does not depend on the frame's position in the batch."""
    d = {}
    for p in range(3):
        kind = "luma" if p == 0 else "chroma"
        d["recon%d" % p] = res["recon%d" % p][f]
        d["coeffs%d" % p] = res["coeffs"][p][f]
        d["band records %d" % p] = engine.band_records(res[kind + "_blocks"], res[kind + "_res"], geom, p, f)
        if "dc_index%d" % p in res:
            d["dc_index%d" % p] = res["dc_index%d" % p][f]
    for kind in ("luma", "chroma"):
        b = res[kind + "_blocks"]
        sel = np.nonzero(b["frame"] == f)[0]
        sel = sel[np.lexsort((b["x0"][sel], b["y0"][sel], b["pli"][sel]))]
        d[kind + "_skip_diff"] = res[kind + "_skip_diff"][sel]
        if kind == "chroma":
            d["chroma_flip"] = res["chroma_flip"][sel]
    if "dering_levels" in res:
        d["dering_levels"] = res["dering_levels"][f]
    if "sym_index" in res:
        b0, nb, n0, nn, y0, ny = (int(v) for v in res["sym_index"][f])
        d["sym_blocks"] = np.frombuffer(res["sym_blocks"][b0:b0 + nb].tobytes(), np.uint8)
        d["sym_bands"] = res["sym_bands"][n0:n0 + nn]
        d["sym_pulses"] = res["sym_pulses"][y0:y0 + ny]
    return d


def _assert_same(got, want, what):
    assert set(got) == set(want), (what, sorted(set(got) ^ set(want)))
    for k in want:
        assert got[k].shape == want[k].shape and np.array_equal(got[k], want[k]), (what, k)


def _assert_steps_equal(a, b, geom, F, what):
    for f in range(F):
        _assert_same(_frame(a, geom, f), _frame(b, geom, f), "%s, frame %d" % (what, f))


def _against_uniform(geom, config, points, planes, maps, levels=None, **kw):
    """The keyframe_quant batch of `points`, each frame against a uniform engine at its own point."""
    F = len(points)
    eng = _mixed(geom, F, config, **kw)
    try:
        got = _run(eng, planes, maps, _records(points, config), levels)
    finally:
        eng.close()
    for f, point in enumerate(points):
        ref = _uniform(geom, point, config, **kw)
        try:
            want = _run(ref, planes[f:f + 1], maps[f:f + 1], None, None if levels is None else levels[f:f + 1])
        finally:
            ref.close()
        _assert_same(_frame(got, geom, f), _frame(want, geom, 0), "%s, frame %d at point %d" % (CONFIGS[config], f, point))
    return got


@pytest.mark.parametrize("config", range(3), ids=CONFIGS)
@pytest.mark.parametrize("size", ((200, 130), (1920, 1080)), ids=lambda s: "%dx%d" % s)
def test_each_frame_equals_its_uniform_engine(size, config):
    geom = Geometry(*size)
    planes, maps = _frames(geom, NPOINTS, seed=7 + config)
    got = _against_uniform(geom, config, ALL, planes, maps, **FULL)
    # the sweep's ends: the finest point codes pulses in every frame kind, the coarsest almost none
    k = got["luma_res"][..., 3]
    assert k[got["luma_blocks"]["frame"] == 0].max() > 0
    assert k[got["luma_blocks"]["frame"] == NPOINTS - 1].sum() < k[got["luma_blocks"]["frame"] == 0].sum()


def test_4k_two_points_on_bench_maps():
    """bench.py's 4K maps and deringing levels, two frames at different points, bench.py's engine options (dering 1,
    max_blocks_div 2) with the DC chain and the symbol stream."""
    import bench
    geom = Geometry(bench.PIC_W, bench.PIC_H)
    frames = bench.make_host_frames(geom, 2)
    planes, maps = [fr[0] for fr in frames], [fr[1] for fr in frames]
    levels = np.stack([fr[2] for fr in frames])
    _against_uniform(geom, 0, (1, 6), planes, maps, levels, dering=1, max_blocks_div=2, symbol_stream=1,
                     haar_dc_quant=1)


def test_mixed_batch_matches_pipeline_oracle():
    """Each frame of a mixed batch against the reference pipeline (keyframe_chain with its level search) at the
    frame's own settings."""
    ref = oracle_lib.load_ref()
    if ref is None:
        pytest.skip("needs the reference build (the level search of keyframe_chain)")
    geom, config, points = Geometry(200, 130), 0, (0, 3, 7)
    planes, maps = _frames(geom, len(points), seed=31)
    eng = _mixed(geom, len(points), config, dering=2)
    try:
        got = _run(eng, planes, maps, _records(points, config))
    finally:
        eng.close()
    for f, point in enumerate(points):
        s = settings(point, config, 0)
        want = frame_oracle.keyframe_chain(ref, "ref", planes[f], geom, maps[f], s["q0"], s["q4"], s["masking"],
                                           lam=s["lam"], qm=s["qm"], qm_inv=s["qm_inv"],
                                           dering_search=dict(coded_quantizer=s["cq"], dering_lambda=s["dering_lambda"],
                                                              qm=1 - s["flat"]))
        assert np.array_equal(got["dering_levels"][f], want[0]["dering_levels"]), ("levels", f)
        for p in range(3):
            kind = "luma" if p == 0 else "chroma"
            assert np.array_equal(engine.band_records(got[kind + "_blocks"], got[kind + "_res"], geom, p, f),
                                  want[p]["rec"]), ("band records", f, p)
            assert np.array_equal(got["coeffs"][p][f], want[p]["dq"]), ("quantised plane", f, p)
            assert np.array_equal(got["recon%d" % p][f], want[p]["recon"]), ("recon", f, p)


def test_mixed_batch_matches_haar_dc_driver():
    """Each frame's DC indices and leaf DCs against the reference's DC chain at the frame's own settings."""
    lib = haar_dc_oracle.load()
    if lib is None:
        pytest.skip("needs oracle/_ref/libdaala_ref_haar_dc.so")
    geom, config, points = Geometry(200, 130), 1, (1, 5, 7)
    planes, maps = _frames(geom, len(points), seed=41)
    eng = _mixed(geom, len(points), config, haar_dc_quant=1)
    try:
        got = _run(eng, planes, maps, _records(points, config))
    finally:
        eng.close()
    for f, point in enumerate(points):
        s = settings(point, config, 0)
        want = haar_dc_oracle.frame(lib, geom, planes[f], maps[f], s["q0"], s["q4"], s["lam"])
        for p in range(3):
            assert np.array_equal(got["dc_index%d" % p][f], want["idx"][p]), ("indices", f, p)
            b = got["luma_blocks" if p == 0 else "chroma_blocks"]
            b = b[(b["pli"] == p) & (b["frame"] == f)]
            y, x = b["y0"].astype(np.int64), b["x0"].astype(np.int64)
            assert np.array_equal(got["coeffs"][p][f][y, x], want["d_post"][p][y, x]), ("leaf DCs", f, p)


def _device_step(eng, planes, maps, records, graph, levels=None):
    """One step through upload + run_device (live launches or the graph), outputs read from the device."""
    eng.upload([np.stack([fr[p] for fr in planes]) for p in range(3)], np.stack(maps), frame_quant=records)
    eng.run_device(graph=graph)
    return dict(recon=[eng.recon_plane(p) for p in range(3)], coeffs=[eng.coeff_plane(p) for p in range(3)])


def test_nothing_baked_at_create():
    """Batch A, then batch B with other records, on one engine: B equals a fresh engine's B, through submit and
    through live launches and graph replays; a permuted batch permutes the outputs with the records."""
    geom, config = Geometry(200, 130), 2
    F = 4
    planes, maps = _frames(geom, F, seed=51)
    ra, rb = _records((0, 2, 4, 6), config), _records((7, 5, 3, 1), config)
    fresh = _mixed(geom, F, config, **FULL)
    try:
        want_b = _run(fresh, planes, maps, rb)
    finally:
        fresh.close()
    eng = _mixed(geom, F, config, **FULL)
    try:
        _run(eng, planes, maps, ra)
        got_b = _run(eng, planes, maps, rb)
        _assert_steps_equal(got_b, want_b, geom, F, "submit A then B")
        for graph in (False, True, True):   # live, the graph's capture, a replay
            _device_step(eng, planes, maps, ra, graph)
            dev = _device_step(eng, planes, maps, rb, graph)
            for p in range(3):
                assert np.array_equal(dev["recon"][p], want_b["recon%d" % p]), ("run_device", graph, p)
                assert np.array_equal(dev["coeffs"][p], want_b["coeffs"][p]), ("run_device", graph, p)
        perm = [2, 0, 3, 1]
        got_p = _run(eng, [planes[i] for i in perm], [maps[i] for i in perm], rb[perm])
    finally:
        eng.close()
    for f, i in enumerate(perm):
        _assert_same(_frame(got_p, geom, f), _frame(want_b, geom, i), "permuted frame %d (was %d)" % (f, i))


@pytest.mark.parametrize("point", (0, 4, 7))
def test_uniform_records_run_as_the_engine_without_the_mode(point):
    """Records that all equal the config: the outputs of the engine without the mode, and the same kernel launches (both
    read their quantizers from per-frame records)."""
    geom, config, F = Geometry(200, 130), 0, 3
    planes, maps = _frames(geom, F, seed=61 + point)
    base = _uniform(geom, point, config, F=F, **FULL)
    try:
        want = _run(base, planes, maps)
        n_base = base.launches_per_step()
    finally:
        base.close()
    s = settings(point, config, 0)
    eng = engine.KeyframeEngine(geom, nframes=F, keyframe_quant=1, q0=s["q0"], pvq_qm_q4=s["q4"], coded_quantizer=s["cq"],
                                dering_lambda=s["dering_lambda"], **_stream_kw(config), **FULL)
    try:
        got = _run(eng, planes, maps, _records((point,) * F, config))
        assert eng.launches_per_step() == n_base
    finally:
        eng.close()
    _assert_steps_equal(got, want, geom, F, "uniform records")


SCHEDULES = [dict(dering=d, haar_dc_quant=h) for d in (1, 2) for h in (0, 1)]


@pytest.mark.parametrize("opts", SCHEDULES, ids=lambda o: "dering%d-hdc%d" % (o["dering"], o["haar_dc_quant"]))
def test_schedules_agree(opts):
    """The forked graph against the phase-by-phase path on the device, with each dering and DC option."""
    geom, config, points = Geometry(200, 130), 0, (0, 4, 7)
    F = len(points)
    planes, maps = _frames(geom, F, seed=71)
    rec = _records(points, config)
    levels = _levels(geom, F, 72) if opts["dering"] == 1 else None
    eng = _mixed(geom, F, config, **opts)
    try:
        want = _run(eng, planes, maps, rec, levels)
        # the phase-by-phase path (each phase enqueued on its own) on the inputs the submit left on the device
        eng.run_device(phases=engine.PH_LISTS | engine.PH_FORWARD, graph=False)
        eng.run_device(phases=engine.PH_PVQ_LUMA, graph=False)
        eng.run_device(phases=engine.PH_PVQ_CHROMA | engine.PH_INVERSE, graph=False)
        phased = [eng.recon_plane(p) for p in range(3)], [eng.coeff_plane(p) for p in range(3)]
    finally:
        eng.close()
    for p in range(3):
        assert np.array_equal(phased[0][p], want["recon%d" % p]), ("phase by phase", p)
        assert np.array_equal(phased[1][p], want["coeffs"][p]), ("phase by phase", p)


def test_submit_refusals_before_any_copy():
    geom, config, F = Geometry(200, 130), 0, 2
    planes, maps = _frames(geom, F, seed=81)
    eng = _mixed(geom, F, config)
    try:
        _run(eng, planes, maps, _records((2, 5), config))
        before = [eng.coeff_plane(p) for p in range(3)]
        other = [np.stack([np.full_like(fr[p], 77) for fr in planes]) for p in range(3)]
        bad = []
        r = _records((2, 5), config); r["q0"][1] = 0; bad.append((r, "q0 is outside"))
        r = _records((2, 5), config); r["q0"][0] = engine.MAX_Q0 + 1; bad.append((r, "q0 is outside"))
        r = _records((2, 5), config); r["coded_quantizer"][1] = 64; bad.append((r, "coded_quantizer is outside"))
        r = _records((2, 5), config); r["dering_lambda"][0] = np.nan; bad.append((r, "dering_lambda"))
        r = _records((2, 5), config); r["pvq_qm_q4"][1, 2, 20] = 0; bad.append((r, "pvq_qm_q4 entry is 0"))
        for rec, why in [(None, "the records .* are required")] + bad:
            with pytest.raises(Exception, match=why):
                eng.encode(other, np.stack(maps), frame_quant=rec)
            for p in range(3):
                assert np.array_equal(eng.coeff_plane(p), before[p]), (why, p)
        with pytest.raises(Exception, match="q0 is outside"):
            eng.upload(other, np.stack(maps), frame_quant=bad[0][0])
    finally:
        eng.close()
    # records on an engine with neither mode
    plain = _uniform(geom, 2, config, F=F)
    try:
        with pytest.raises(Exception, match="needs an engine with frame_quant = 1 or keyframe_quant = 1"):
            _run(plain, planes, maps, _records((2, 5), config))
    finally:
        plain.close()
