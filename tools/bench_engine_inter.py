#!/usr/bin/env python
"""The engine's P-frame residual mode (inter=1) against its keyframe mode on bench.py's workload: 16 synthetic
3840x2160 4:2:0 frames, the shipped block-size maps of the reference encoder, q0 72; the prediction of frame f is
synthetic frame f - 1 (frame 0: the last frame of the cycle).  The two engines live in one process and are timed
in alternating rounds (CUDA events on the engine's stream, inputs resident in HBM, one graph replay per step),
then phase by phase through daala_b200_kf_time_device.  Frame 0 of the inter batch is checked against the oracle
before anything is timed.  Needs a CUDA device; prints one JSON line.

    python tools/bench_engine_inter.py [--rounds 3] [--steps 10] [--warmup 3] [--frames 16]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


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
    from daala_b200 import _native, engine
    from daala_b200.frame import Geometry
    from tests import inter_oracle, oracle_lib
    if _native.lib().daala_b200_device_count() < 1:
        sys.exit("bench_engine_inter.py needs a CUDA device: nothing is measured without one")

    geom = Geometry(bench.PIC_W, bench.PIC_H)
    F = args.frames
    q4 = np.full((3, 30), bench.PVQ_QM_Q4, np.uint8)
    hf = bench.make_host_frames(geom, F)
    planes = [np.stack([f[0][p] for f in hf]) for p in range(3)]
    pred = [np.roll(planes[p], 1, axis=0) for p in range(3)]
    bsize = np.stack([f[1] for f in hf])
    common = dict(nframes=F, q0=bench.Q0, use_masking=1, pvq_qm_q4=q4, max_blocks_div=2)
    engines = {"keyframe": engine.KeyframeEngine(geom, **common),
               "inter": engine.KeyframeEngine(geom, inter=1, **common)}
    outs = {}
    for name, eng in engines.items():
        outs[name] = eng.encode(planes, bsize, pred=pred if name == "inter" else None)

    # parity of frame 0 before timing
    ref = oracle_lib.load_ref()
    lib, prefix = (ref, "ref") if ref is not None else (oracle_lib.load_port(), "port")
    want = inter_oracle.inter_chain(lib, prefix, [planes[p][0] for p in range(3)], [pred[p][0] for p in range(3)], geom,
                                    bsize[0], bench.Q0, q4, 1)
    out = outs["inter"]
    mism = 0
    for p in range(3):
        kind = "luma" if p == 0 else "chroma"
        b = out[kind + "_blocks"]
        sel = (b["pli"] == p) & (b["frame"] == 0)
        mism += int(np.count_nonzero(out["recon%d" % p][0] != want[p]["recon"]))
        mism += int(np.count_nonzero(engine.band_records(b, out[kind + "_res"], geom, p, 0) != want[p]["rec"]))
        mism += int(np.count_nonzero(out[kind + "_dc"][sel] != want[p]["qdc"][b["y0"][sel] >> 2, b["x0"][sel] >> 2]))
        mism += int(np.count_nonzero(engines["inter"].coeff_plane(p)[0] != want[p]["dq"]))
    if mism:
        sys.exit("bench_engine_inter.py: frame 0 of the inter batch differs from the oracle (%d mismatches)" % mism)

    cnt = {name: outs[name]["counts"].copy() for name in engines}
    items = {name: {"luma": [int(v) for v in c[engine.CNT["items_l"]:engine.CNT["items_l"] + 3]],
                    "chroma": [int(v) for v in c[engine.CNT["items_c"]:engine.CNT["items_c"] + 3]],
                    "luma_chain_items": int(c[engine.CNT["total_hi"]])} for name, c in cnt.items()}
    pulses = {name: int(o["luma_res"][..., 3].clip(min=0).sum()) + int(o["chroma_res"][..., 3].clip(min=0).sum())
              for name, o in outs.items()}

    for eng in engines.values():
        eng.time_device(engine.PH_ALL, True, max(args.warmup, 1))
    rounds = {name: [] for name in engines}
    for _ in range(args.rounds):
        for name, eng in engines.items():
            rounds[name].append(eng.time_device(engine.PH_ALL, True, args.steps) / args.steps)
    phases = {}
    for name, eng in engines.items():
        ph = {}
        for label, flag in (("work_lists", engine.PH_LISTS), ("forward", engine.PH_FORWARD), ("pvq_luma", engine.PH_PVQ_LUMA),
                            ("pvq_chroma", engine.PH_PVQ_CHROMA), ("inverse", engine.PH_INVERSE),
                            ("pvq_luma_band_kernels_alone", engine.PH_PVQ_LUMA | engine.PH_SEARCH_ONLY),
                            ("pvq_chroma_band_kernels_alone", engine.PH_PVQ_CHROMA | engine.PH_SEARCH_ONLY)):
            eng.time_device(flag, False, 1)
            ph[label] = round(eng.time_device(flag, False, args.steps) / args.steps, 4)
        eng.time_device(engine.PH_ALL, True, 1)   # leave the planes consistent
        phases[name] = ph

    px = geom.luma_pixels * F
    res = {"workload": "%d synthetic 3840x2160 4:2:0 frames per step, block sizes decided by the reference encoder, q0 %d, "
                       "no deringing; inter: prediction of frame f = synthetic frame f - 1" % (F, bench.Q0),
           "gpu": bench.gpu_identity(0), "steps_per_round": args.steps, "rounds": args.rounds,
           "parity_checked": "frame 0 of the inter batch against the oracle (%s): reconstruction, quantised planes, "
                             "band decisions, DC indices" % prefix}
    for name, eng in engines.items():
        ms = statistics.median(rounds[name])
        res[name] = {"ms_per_step": round(ms, 4), "ms_per_step_rounds": [round(v, 4) for v in rounds[name]],
                     "mpixels_per_s": round(px / (ms * 1e-3) / 1e6, 1), "phases_ms": phases[name],
                     "items_per_class": items[name], "pulses": pulses[name], "launches_per_step": eng.launches_per_step(),
                     "device_bytes": int(eng.buf.bytes_allocated)}
        eng.close()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
