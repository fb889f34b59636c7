#!/usr/bin/env python
"""Cost of the late-skip distortions (late_skip = 1) in the P-frame engine on the workload of
tools/bench_engine_inter.py: 16 synthetic 3840x2160 4:2:0 frames, the shipped block-size maps of the reference encoder,
q0 72, the prediction of frame f = synthetic frame f - 1, HVS distortion with activity masking.  Two engines with the
P-frame symbol stream (symbol_stream = 2), late_skip 0 and 1, live in one process and are timed in alternating rounds
(CUDA events on the engine's stream, inputs resident in HBM, one graph replay per step).  Reports the step time of
both, the extra device memory and the extra D2H bytes of the records in block order and in stream order.  Frame 0's
records are checked against the oracle before anything is timed.  Needs a CUDA device; prints one JSON line.

    python tools/bench_engine_late_skip.py [--rounds 5] [--steps 10] [--warmup 3] [--frames 16]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

CODED_Q = 72   # state->coded_quantizer (od_compute_dist's scale)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10, help="steps per round and engine (at least 10)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--frames", type=int, default=16)
    args = ap.parse_args()
    args.steps = max(args.steps, 10)
    import numpy as np
    import bench
    from daala_b200 import _native, engine, symbols
    from daala_b200.frame import Geometry
    from tests import late_skip_oracle
    if _native.lib().daala_b200_device_count() < 1:
        sys.exit("bench_engine_late_skip.py needs a CUDA device: nothing is measured without one")

    geom = Geometry(bench.PIC_W, bench.PIC_H)
    F = args.frames
    q4 = np.full((3, 30), bench.PVQ_QM_Q4, np.uint8)
    hf = bench.make_host_frames(geom, F)
    planes = [np.stack([f[0][p] for f in hf]) for p in range(3)]
    pred = [np.roll(planes[p], 1, axis=0) for p in range(3)]
    bsize = np.stack([f[1] for f in hf])
    common = dict(nframes=F, q0=bench.Q0, use_masking=1, pvq_qm_q4=q4, max_blocks_div=2, inter=1, symbol_stream=2,
                  coded_quantizer=CODED_Q)
    engines = {"late_skip_0": engine.KeyframeEngine(geom, **common),
               "late_skip_1": engine.KeyframeEngine(geom, late_skip=1, **common)}
    outs = {name: eng.encode(planes, bsize, pred=pred) for name, eng in engines.items()}

    # parity of frame 0's records before timing
    lib, prefix = late_skip_oracle.load()
    eng, out = engines["late_skip_1"], outs["late_skip_1"]
    mism = 0
    for p in range(3):
        kind = "luma" if p == 0 else "chroma"
        b = out[kind + "_blocks"]
        sel = (b["pli"] == p) & (b["frame"] == 0)
        want = late_skip_oracle.plane(lib, prefix, planes[p][0], pred[p][0], eng.coeff_plane(p)[0], geom, bsize[0], p,
                                      bench.Q0, q4, 0, 1, CODED_Q)[b["y0"][sel] >> 2, b["x0"][sel] >> 2]
        rec = out[kind + "_late_skip"][sel]
        got = np.stack([rec[f] for f in symbols.LATE_SKIP_DTYPE.names], axis=-1)
        mism += int(np.count_nonzero(~np.isclose(got, want, rtol=1e-12, atol=0)))
    if mism:
        sys.exit("bench_engine_late_skip.py: frame 0's late-skip records differ from the oracle (%d values)" % mism)
    nblocks = int(len(out["luma_blocks"]) + len(out["chroma_blocks"]))
    used = int(out["sym_index"][:, 1].sum())

    for e in engines.values():
        e.time_device(engine.PH_ALL, True, max(args.warmup, 1))
    rounds = {name: [] for name in engines}
    for _ in range(args.rounds):
        for name, e in engines.items():
            rounds[name].append(e.time_device(engine.PH_ALL, True, args.steps) / args.steps)
    res = {"workload": "%d synthetic 3840x2160 4:2:0 P frames per step (prediction of frame f = synthetic frame f - 1), "
                       "block sizes decided by the reference encoder, q0 %d, coded_quantizer %d, HVS distortion with "
                       "activity masking, symbol_stream 2" % (F, bench.Q0, CODED_Q),
           "gpu": bench.gpu_identity(0), "steps_per_round": args.steps, "rounds": args.rounds,
           "parity_checked": "frame 0's late-skip records against the oracle (%s), rtol 1e-12" % prefix,
           "blocks": nblocks, "blocks_with_late_skip": int((out["luma_blocks"]["bs"] > 0).sum()
                                                          + (out["chroma_blocks"]["bs"] > 0).sum()),
           "extra_d2h_bytes_block_order": nblocks * symbols.LATE_SKIP_DTYPE.itemsize,
           "extra_d2h_bytes_stream_order": used * symbols.LATE_SKIP_DTYPE.itemsize}
    for name, e in engines.items():
        ms = statistics.median(rounds[name])
        res[name] = {"ms_per_step": round(ms, 4), "ms_per_step_rounds": [round(v, 4) for v in rounds[name]],
                     "launches_per_step": e.launches_per_step(), "device_bytes": int(e.buf.bytes_allocated)}
    res["late_skip_cost_ms_per_step"] = round(res["late_skip_1"]["ms_per_step"] - res["late_skip_0"]["ms_per_step"], 4)
    res["extra_device_bytes"] = res["late_skip_1"]["device_bytes"] - res["late_skip_0"]["device_bytes"]
    for e in engines.values():
        e.close()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
