#!/usr/bin/env python
"""The P-frame finishing pass (inter_finish=1, daala_b200_kf_finish) on bench_engine_inter.py's workload: 16 synthetic
3840x2160 4:2:0 frames, the shipped block-size maps of the reference encoder, q0 72, the prediction of frame f =
synthetic frame f - 1.  One step, then the pass with seeded decisions: 30 % of the blocks skipped with DC 0 (the late
skip's form, so they are skipped in bskip too), the others keep the step's qdc; deringing levels from the same
shipped maps bench.py uses.  Frame 0 of the pass is checked against the oracle's frame driver before anything is timed.

Times (host clock around enqueues that end in a stream synchronise, --reps calls per round):
  finish_ms           the whole call: H2D of the decisions and levels, the pass's graph, D2H of the reconstruction,
                      the three skip maps and the applied levels;
  finish_no_d2h_ms    the same without the D2H (outputs not requested);
and, for comparison, the step's PH_INVERSE phase alone (daala_b200_kf_time_device, CUDA events).  Needs a CUDA
device; prints one JSON line.

--search: the pass with its deringing level search (inter_finish=2) on the same frames, decisions and quantizer
(coded_quantizer and dering_lambda of bench.py), no levels given.  Frame 0 is checked first against the oracle
composed from the reference's pieces (patch and skip map, the reference's inverse to the SB-edge postfilter, its own
search loop oracle_ref_dering_search, then inverse_frame_inter_finish at the searched levels); this needs the
reference build.  finish_ms / finish_no_d2h_ms are then those of the searching pass, and
given_levels_finish_ms / given_levels_finish_no_d2h_ms those of the inter_finish=1 pass on a second engine given the
searched levels, timed in alternating rounds; search_ms is the difference of the two no-D2H medians.  The line also
counts the superblocks searched (coded) and the histogram of the levels.

    python tools/bench_engine_inter_finish.py [--rounds 3] [--reps 10] [--frames 16] [--search]
"""
import argparse
import ctypes
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def finish_records(eng):
    """Two copies of the engine's prepared finish record: with every output, and with none (no D2H)."""
    from daala_b200 import engine
    full = engine.FinishIO.from_buffer_copy(eng._fio)
    bare = engine.FinishIO.from_buffer_copy(eng._fio)
    for p in range(3):
        bare.pixels_out[p] = bare.bskip_out[p] = None
    bare.dering_level_out = None
    return full, bare


def timed(eng, fio, reps):
    """Milliseconds per daala_b200_kf_finish call: host clock around `reps` enqueues ending in a stream synchronise."""
    eng.wait()
    t0 = time.perf_counter()
    for _ in range(reps):
        eng._check(eng.L.daala_b200_kf_finish(eng.kf, ctypes.byref(fio)), "kf_finish")
    eng.wait()
    return (time.perf_counter() - t0) * 1e3 / reps


def search_oracle(geom, planes, out, d, md, bsize, q4, dec, lam, frame):
    """Levels, reconstruction and skip maps of one frame of the searching pass, from the reference's pieces."""
    import numpy as np
    import bench
    from daala_b200 import interfinish
    from tests import frame_oracle, inter_finish_oracle, oracle_lib
    from tests.oracle_lib import addr
    ref, fin = oracle_lib.load_ref(), inter_finish_oracle.load_ref()
    if ref is None or fin is None:
        sys.exit("bench_engine_inter_finish.py --search checks frame 0 against the reference build (oracle/_ref), "
                 "which is missing")
    dq, bskip = [], []
    for p in range(3):
        blocks, skip, dc = (out["luma_blocks"], dec[0], dec[1]) if p == 0 else (out["chroma_blocks"], dec[2], dec[3])
        dq.append(interfinish.patch(d[p], md[p], blocks, skip, dc, frame, p, bench.Q0, q4))
        bskip.append(np.ascontiguousarray(interfinish.skip_map(blocks, skip, dc, frame, p, geom)))
    c = np.ascontiguousarray(frame_oracle.inverse_plane(ref, "ref", dq[0], geom, 0, bsize[frame], 0, lapped_only=True),
                             np.int32)
    ref.od_apply_postfilter_frame_sbs(addr(c), c.shape[1], geom.nhsb, geom.nvsb, 0, 0)
    src = np.ascontiguousarray(planes[0][frame], np.uint8)
    cdf = np.zeros((11, 6), np.uint16)
    cdf[:] = 32 * np.arange(1, 7, dtype=np.uint16)   # fresh per frame, src/state.c:573-574
    levels = np.zeros(geom.nvsb * geom.nhsb, np.uint8)
    f = ref.oracle_ref_dering_search
    f.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p] + [ctypes.c_int] * 7 + [
        ctypes.c_double, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    r = f(addr(src), src.shape[1], addr(c), geom.nhsb, geom.nvsb, bench.Q0, bench.CODED_Q, 1, 1, 0, lam,
          addr(bskip[0]), bskip[0].shape[1], addr(cdf), 128, addr(levels), None)
    assert r == 0
    levels = levels.reshape(geom.nvsb, geom.nhsb)
    recs, applied = inter_finish_oracle.finish(fin, "ref", dq, geom, bsize[frame], bench.Q0, levels, bskip)
    return levels, applied, recs, bskip


def search(args, given, geom, planes, pred, bsize, q4, out, dec):
    """--search: the inter_finish=2 pass against the inter_finish=1 pass of `given` (same step) at the searched levels."""
    import numpy as np
    import bench
    from daala_b200 import engine, interfinish
    F = args.frames
    eng = engine.KeyframeEngine(geom, nframes=F, q0=bench.Q0, use_masking=1, pvq_qm_q4=q4, max_blocks_div=2, inter=1,
                                inter_finish=2, coded_quantizer=bench.CODED_Q, dering_lambda=bench.DERING_LAMBDA)
    out2 = {k: np.array(v) for k, v in eng.encode(planes, bsize, pred=pred).items()}
    assert all(np.array_equal(out2[k], out[k]) for k in ("luma_dc", "chroma_dc")), "the two engines' steps differ"
    got = {k: np.array(v) for k, v in eng.finish(*dec).items()}
    levels = got["dering_levels"]

    # parity of frame 0 before timing
    d = [eng.coeff_plane(p)[0] for p in range(3)]
    md = [eng.pred_coeff_plane(p)[0] for p in range(3)]
    want, applied, recs, bskip = search_oracle(geom, planes, out2, d, md, bsize, q4, dec, eng.dering_lambda, 0)
    mism = int(np.count_nonzero(levels[0] != want)) + int(np.count_nonzero(applied != want))
    for p in range(3):
        mism += int(np.count_nonzero(got["recon%d" % p][0] != recs[p]))
        mism += int(np.count_nonzero(got["bskip%d" % p][0] != bskip[p]))
    if mism:
        sys.exit("bench_engine_inter_finish.py --search: frame 0 of the pass differs from the oracle (%d mismatches)" % mism)
    # the pass without the search, given the searched levels, makes the same outputs (all frames)
    ref = {k: np.array(v) for k, v in given.finish(*dec, levels).items()}
    same = int(sum(np.count_nonzero(ref[k] != got[k]) for k in got))

    eng.prepare_finish(*dec)
    s_full, s_bare = finish_records(eng)
    given.prepare_finish(*dec, levels)
    g_full, g_bare = finish_records(given)
    timed(eng, s_full, args.reps)
    timed(given, g_full, args.reps)
    rounds = {"finish_ms": [], "finish_no_d2h_ms": [], "given_levels_finish_ms": [], "given_levels_finish_no_d2h_ms": []}
    for _ in range(args.rounds):
        rounds["finish_ms"].append(timed(eng, s_full, args.reps))
        rounds["given_levels_finish_ms"].append(timed(given, g_full, args.reps))
        rounds["finish_no_d2h_ms"].append(timed(eng, s_bare, args.reps))
        rounds["given_levels_finish_no_d2h_ms"].append(timed(given, g_bare, args.reps))

    coded = np.stack([interfinish.coded_superblocks(got["bskip0"][f], geom) for f in range(F)])
    res = {"workload": "%d synthetic 3840x2160 4:2:0 frames, reference block sizes, q0 %d, coded_quantizer %d, "
                       "prediction of frame f = synthetic frame f - 1; 30 %% of the blocks skipped with DC 0, the others "
                       "DC = qdc; deringing levels searched in the pass (inter_finish=2)" % (F, bench.Q0, bench.CODED_Q),
           "gpu": bench.gpu_identity(0), "reps_per_round": args.reps, "rounds": args.rounds,
           "parity_checked": "frame 0 against the reference's search loop and inverse_frame_inter_finish: levels, "
                             "reconstruction, skip maps",
           "oracle_mismatches_frame0": mism,
           "given_levels_mismatches": same,
           "superblocks": int(levels.size),
           "superblocks_searched": int(np.count_nonzero(coded)),
           "level_histogram": np.bincount(levels.ravel(), minlength=6).tolist(),
           "level_histogram_searched": np.bincount(levels[coded].ravel(), minlength=6).tolist(),
           "search_scratch_bytes": int(eng.buf.bytes_allocated - given.buf.bytes_allocated)}
    for k, v in rounds.items():
        res[k] = round(statistics.median(v), 4)
        res[k + "_rounds"] = [round(x, 4) for x in v]
    res["search_ms"] = round(res["finish_no_d2h_ms"] - res["given_levels_finish_no_d2h_ms"], 4)
    eng.close()
    given.close()
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--search", action="store_true", help="time the pass with its level search (inter_finish=2)")
    args = ap.parse_args()
    import numpy as np
    import bench
    from daala_b200 import _native, engine, interfinish
    from daala_b200.frame import Geometry
    from tests import inter_finish_oracle
    if _native.lib().daala_b200_device_count() < 1:
        sys.exit("bench_engine_inter_finish.py needs a CUDA device: nothing is measured without one")

    geom = Geometry(bench.PIC_W, bench.PIC_H)
    F = args.frames
    q4 = np.full((3, 30), bench.PVQ_QM_Q4, np.uint8)
    hf = bench.make_host_frames(geom, F)
    planes = [np.stack([f[0][p] for f in hf]) for p in range(3)]
    pred = [np.roll(planes[p], 1, axis=0) for p in range(3)]
    bsize = np.stack([f[1] for f in hf])
    levels = np.stack([f[2] for f in hf])
    eng = engine.KeyframeEngine(geom, nframes=F, q0=bench.Q0, use_masking=1, pvq_qm_q4=q4, max_blocks_div=2, inter=1,
                                inter_finish=1)
    out = {k: np.array(v) for k, v in eng.encode(planes, bsize, pred=pred).items()}
    rng = np.random.default_rng(30)
    ls = (rng.random(len(out["luma_dc"])) < 0.3).astype(np.uint8)
    cs = (rng.random(len(out["chroma_dc"])) < 0.3).astype(np.uint8)
    dec = (ls, np.where(ls == 1, 0, out["luma_dc"]).astype(np.int32), cs,
           np.where(cs == 1, 0, out["chroma_dc"]).astype(np.int32), levels)
    if args.search:
        return search(args, eng, geom, planes, pred, bsize, q4, out, dec[:4])
    got = {k: np.array(v) for k, v in eng.finish(*dec).items()}

    # parity of frame 0 before timing
    lib, prefix = inter_finish_oracle.load()
    dq, bskip = [], []
    for p in range(3):
        blocks, skip, dc = (out["luma_blocks"], dec[0], dec[1]) if p == 0 else (out["chroma_blocks"], dec[2], dec[3])
        dq.append(interfinish.patch(eng.coeff_plane(p)[0], eng.pred_coeff_plane(p)[0], blocks, skip, dc, 0, p, bench.Q0, q4))
        bskip.append(interfinish.skip_map(blocks, skip, dc, 0, p, geom))
    recs, applied = inter_finish_oracle.finish(lib, prefix, dq, geom, bsize[0], bench.Q0, levels[0], bskip)
    mism = int(np.count_nonzero(got["dering_levels"][0] != applied))
    for p in range(3):
        mism += int(np.count_nonzero(got["recon%d" % p][0] != recs[p]))
        mism += int(np.count_nonzero(got["bskip%d" % p][0] != bskip[p]))
    if mism:
        sys.exit("bench_engine_inter_finish.py: frame 0 of the pass differs from the oracle (%d mismatches)" % mism)

    eng.prepare_finish(*dec)
    full, bare = finish_records(eng)

    timed(eng, full, args.reps)
    rounds = {"finish_ms": [], "finish_no_d2h_ms": []}
    for _ in range(args.rounds):
        rounds["finish_ms"].append(timed(eng, full, args.reps))
        rounds["finish_no_d2h_ms"].append(timed(eng, bare, args.reps))
    eng.time_device(engine.PH_INVERSE, False, 1)
    inverse_ms = eng.time_device(engine.PH_INVERSE, False, args.reps) / args.reps
    eng.time_device(engine.PH_ALL, True, 1)   # leave the planes consistent

    nl, nc = len(ls), len(cs)
    res = {"workload": "%d synthetic 3840x2160 4:2:0 frames, reference block sizes, q0 %d, prediction of frame f = "
                       "synthetic frame f - 1; 30 %% of the blocks skipped with DC 0, the others DC = qdc, the shipped "
                       "deringing levels"
                       % (F, bench.Q0),
           "gpu": bench.gpu_identity(0), "reps_per_round": args.reps, "rounds": args.rounds,
           "parity_checked": "frame 0 against the oracle's inverse_frame_inter_finish (%s): reconstruction, skip maps, "
                             "applied levels" % prefix,
           "skipped_in_bskip": [float(got["bskip%d" % p][:, :, :geom.plane_shape(p)[1] // 4].mean()) for p in range(3)],
           "superblocks_deringed": int(np.count_nonzero(got["dering_levels"])),
           "superblocks_forced_to_0": int(np.count_nonzero(levels) - np.count_nonzero(got["dering_levels"])),
           "h2d_bytes": 5 * (nl + nc) + int(levels.nbytes),
           "d2h_bytes": int(sum(got[k].nbytes for k in got)),
           "step_inverse_phase_ms": round(inverse_ms, 4)}
    for k, v in rounds.items():
        res[k] = round(statistics.median(v), 4)
        res[k + "_rounds"] = [round(x, 4) for x in v]
    eng.close()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
