#!/usr/bin/env python
"""The engine's lossless step (lossless=1, quantizer 0): 16 synthetic 3840x2160 4:2:0 frames (bench.py's content)
coded as keyframes, then as P frames predicted by the engine (inter_mc) from seeded synthetic MV grids and a pool of 2F
pictures, as tools/bench_engine_inter_mc.py builds them.  Before timing, frame 0 of each is checked against the
reference's own statics (the quantizer-0 frame driver of oracle/lossless.mk): every residual value, every root sum, the
reconstruction; the P frame's prediction also against od_state_mc_predict (oracle/inter_mc.mk).  The two engines are
then timed in alternating rounds (CUDA events, inputs resident in HBM, one graph replay per step).  Reported per
engine: ms per step, launches, and the step's algorithmic bytes (every input read once, every output written once,
the prediction written and read once) over its time against the 3.35 TB/s of the H100 SXM data sheet, with the card's
name and power limit.  Needs a CUDA device; prints one JSON line.

    python tools/bench_engine_lossless.py [--rounds 3] [--steps 10] [--warmup 3] [--frames 16]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def _check(lib, geom, out, planes, pred, what):
    """Frame 0 of `out` against the driver; exits on the first difference."""
    import numpy as np
    from daala_b200 import lossless
    from tests import lossless_oracle
    want = lossless_oracle.frame(lib, geom, planes, pred)
    c = lossless.padded_input(geom, planes, pred)
    bad = sum(int(np.count_nonzero(out["ll_coeffs%d" % p][0].astype(np.int32) != want["coeffs"][p])) +
              int(np.count_nonzero(out["recon%d" % p][0].astype(np.int64) - 128 != c[p])) for p in range(3))
    bad += int(np.count_nonzero(out["ll_blocks"][0][..., :3] != want["roots"]))
    if bad:
        sys.exit("bench_engine_lossless.py: %s frame 0 differs from the reference driver in %d values" % (what, bad))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10, help="steps per round and engine (at least 10)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--frames", type=int, default=16)
    args = ap.parse_args()
    args.steps = max(args.steps, 10)
    import numpy as np
    import bench
    from daala_b200 import _native, engine, mvgrid, synth
    from daala_b200.frame import Geometry
    from tests import inter_mc_oracle, lossless_oracle
    if _native.lib().daala_b200_device_count() < 1:
        sys.exit("bench_engine_lossless.py needs a CUDA device: nothing is measured without one")
    lib, mclib = lossless_oracle.load(), inter_mc_oracle.load()
    if lib is None or mclib is None:
        sys.exit("bench_engine_lossless.py: frame 0 is checked against oracle/_ref/libdaala_ref_lossless.so and "
                 "libdaala_ref_inter_mc.so, which are not built")

    geom = Geometry(bench.PIC_W, bench.PIC_H)
    F = args.frames
    hf = bench.make_host_frames(geom, F)
    planes = [np.stack([f[0][p] for f in hf]) for p in range(3)]
    # pool: slot f = synthetic frame f - 1 (PREV of frame f), slot F + f = frame f - 2 (GOLD of frame f)
    refs = [np.concatenate([np.roll(planes[p], 1, axis=0), np.roll(planes[p], 2, axis=0)]) for p in range(3)]
    slot = np.array([[F + f, f] for f in range(F)], np.int32)
    grids = [synth.mv_grid(geom, seed=1000 + f) for f in range(F)]
    packed = mvgrid.pack(*(np.stack([g[i] for g in grids]) for i in range(3)))

    key = engine.KeyframeEngine(geom, nframes=F, lossless=1)
    out = key.encode(planes, None)
    _check(lib, geom, out, [planes[p][0] for p in range(3)], None, "keyframe")
    mc = engine.KeyframeEngine(geom, nframes=F, lossless=1, inter=1, inter_mc=1)
    out = mc.encode(planes, None, refs=refs, ref_slot=slot, mv_grid=packed)
    pred0 = [np.array(out["pred%d" % p][0]) for p in range(3)]
    want = inter_mc_oracle.predict(mclib, geom, [refs[p][slot[0, 0]] for p in range(3)],
                                   [refs[p][slot[0, 1]] for p in range(3)], *grids[0])
    if any(not np.array_equal(pred0[p], want[p]) for p in range(3)):
        sys.exit("bench_engine_lossless.py: frame 0's prediction differs from od_state_mc_predict")
    _check(lib, geom, out, [planes[p][0] for p in range(3)], pred0, "P")
    cnt = out["counts"]
    if int(cnt[engine.CNT["mc_bad_ref"]]) or int(cnt[engine.CNT["mc_beyond"]]):
        sys.exit("bench_engine_lossless.py: the synthetic grids left the reference's definition")

    px = sum(int(np.prod(geom.plane_shape(p))) for p in range(3))
    rec = geom.nvsb * geom.nhsb * 3 * 16
    # keyframes: u8 in, int16 residual and u8 reconstruction out, the records; P frames: also the two reference
    # pictures and the grid read, the prediction written and read
    alg = {"keyframe": F * (px + 2 * px + px + rec),
           "p_inter_mc": F * (px + 2 * px + px + rec + 2 * px + 2 * px + packed[0].nbytes)}
    engines = {"keyframe": key, "p_inter_mc": mc}
    for eng in engines.values():
        eng.time_device(engine.PH_ALL, True, max(args.warmup, 1))
    rounds = {name: [] for name in engines}
    for _ in range(args.rounds):
        for name, eng in engines.items():
            rounds[name].append(eng.time_device(engine.PH_ALL, True, args.steps) / args.steps)
    res = {"workload": "%d synthetic 3840x2160 4:2:0 frames per step at quantizer 0 (lossless); P frames: seeded MV "
                       "grids, GOLD / PREV per vertex from a pool of %d pictures" % (F, 2 * F),
           "gpu": bench.gpu_identity(0), "steps_per_round": args.steps, "rounds": args.rounds,
           "parity_checked": "frame 0 of both engines: residual, root sums and reconstruction against the reference's "
                             "quantizer-0 driver; the P frame's prediction against od_state_mc_predict"}
    for name, eng in engines.items():
        ms = statistics.median(rounds[name])
        res[name] = {"ms_per_step": round(ms, 4), "ms_per_step_rounds": [round(v, 4) for v in rounds[name]],
                     "launches_per_step": eng.launches_per_step(), "algorithmic_bytes_per_step": alg[name],
                     "gb_per_s": round(alg[name] / (ms * 1e-3) / 1e9, 1),
                     "share_of_3_35_tb_per_s": round(alg[name] / HBM_BYTES_PER_S / (ms * 1e-3), 4),
                     "device_bytes": int(eng.buf.bytes_allocated)}
        eng.close()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
