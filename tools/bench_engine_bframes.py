#!/usr/bin/env python
"""The engine's B-frame prediction (inter_mc=1, mc_next=1) against the P-frame engine (mc_next=0) on
bench_engine_inter.py's workload: 16 synthetic 3840x2160 4:2:0 frames, the shipped block-size maps, q0 72.  Each frame
predicts from a seeded synth.mv_grid_b grid (every split level, about half the vertices on NEXT with their mv1, the
others on GOLD / PREV) and three pictures of a pool of 3F.  The P-frame engine runs the same grids with NEXT folded
onto PREV (ref 1, mv = mv1): the same OBMC work minus the third picture.  Frame 0's prediction is checked against the
reference's od_state_mc_predict with three pictures (the hook library of oracle/bframes.mk) before timing.  The two
engines are timed in alternating rounds (CUDA events, inputs resident in HBM, one graph replay per step; medians over
rounds).  With --profile the OBMC and leaf kernels of both engines alone are timed by torch.profiler in a run of their
own.  Also reported: H2D bytes per step, leaves per step, launches, device bytes, and the GPU with its power limit.
Needs a CUDA device; prints one JSON line.

    python tools/bench_engine_bframes.py [--rounds 5] [--steps 10] [--warmup 3] [--frames 16] [--profile]
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
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10, help="steps per round and engine (at least 10)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--profile", action="store_true", help="only the torch.profiler run of the prediction kernels")
    args = ap.parse_args()
    args.steps = max(args.steps, 10)
    import numpy as np
    import bench
    from daala_b200 import _native, engine, mvgrid, synth
    from daala_b200.frame import Geometry
    from tests import bframe_oracle
    if _native.lib().daala_b200_device_count() < 1:
        sys.exit("bench_engine_bframes.py needs a CUDA device: nothing is measured without one")

    geom = Geometry(bench.PIC_W, bench.PIC_H)
    F = args.frames
    q4 = np.full((3, 30), bench.PVQ_QM_Q4, np.uint8)
    hf = bench.make_host_frames(geom, F)
    planes = [np.stack([f[0][p] for f in hf]) for p in range(3)]
    bsize = np.stack([f[1] for f in hf])
    # pool: slot f = frame f - 1 (PREV of frame f), F + f = frame f + 1 (NEXT), 2F + f = frame f - 2 (GOLD)
    refs = [np.concatenate([np.roll(planes[p], 1, axis=0), np.roll(planes[p], -1, axis=0), np.roll(planes[p], 2, axis=0)])
            for p in range(3)]
    slot = np.array([[2 * F + f, f, F + f] for f in range(F)], np.int32)
    grids = [synth.mv_grid_b(geom, seed=3000 + f, p_next=0.5, p_gold=0.3) for f in range(F)]
    valid, mv, mv1, ref = (np.stack([g[i] for g in grids]) for i in range(4))
    packed = mvgrid.pack(valid, mv, ref)
    next_share = float((ref[valid.astype(bool)] == 2).mean())
    # NEXT folded onto PREV: the P-frame engine reads PREV with the vector the B engine reads NEXT with
    folded = mvgrid.pack(valid, mvgrid.vectors(mv, ref, mv1), np.where(ref == 2, 1, ref))
    leaves = sum(len(mvgrid.leaves(g[0].astype(bool))[0]) for g in grids)
    common = dict(nframes=F, q0=bench.Q0, use_masking=1, pvq_qm_q4=q4, max_blocks_div=2, inter=1, inter_mc=1)
    b = engine.KeyframeEngine(geom, mc_next=1, **common)
    out = b.encode(planes, bsize, refs=refs, ref_slot=slot, mv_grid=packed, mv1_grid=mv1.astype(np.int32))
    pred0 = [np.array(out["pred%d" % p][0]) for p in range(3)]
    cnt = np.array(out["counts"])
    p = engine.KeyframeEngine(geom, mc_next=0, mc_refs=3 * F, **common)
    p.encode(planes, bsize, refs=refs, ref_slot=slot[:, :2], mv_grid=folded)
    engines = {"mc_next": b, "p_frame_folded": p}

    if args.profile:
        import torch
        from torch.profiler import ProfilerActivity, profile
        kern = {}
        for name, eng in engines.items():
            for _ in range(max(args.warmup, 1)):
                eng.run_device(engine.PH_ALL, graph=False)
            eng.wait()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.steps):
                    eng.run_device(engine.PH_ALL, graph=False)
                eng.wait()
                torch.cuda.synchronize()
            kern[name] = {}
            for e in prof.key_averages():
                for tag in ("k_mc_obmc", "k_mc_leaves"):
                    if tag in e.key:
                        kern[name][tag] = round(e.device_time_total / 1e3 / args.steps, 4)   # ms per step
        for eng in engines.values():
            eng.close()
        print(json.dumps({"profile": "torch.profiler, %d steps without the graph" % args.steps,
                          "gpu": bench.gpu_identity(0), "kernel_ms_per_step": kern}), flush=True)
        return

    lib = bframe_oracle.load()
    if lib is None:
        sys.exit("bench_engine_bframes.py: the prediction is checked against oracle/_ref/libdaala_ref_bframes.so, "
                 "which is not built")
    want = bframe_oracle.predict3(lib, geom, *([refs[q][slot[0, k]] for q in range(3)] for k in range(3)),
                                    *grids[0])
    mism = sum(int(np.count_nonzero(pred0[q] != want[q])) for q in range(3))
    if mism:
        sys.exit("bench_engine_bframes.py: frame 0's prediction differs from od_state_mc_predict (%d pixels)" % mism)
    if int(cnt[engine.CNT["mc_bad_ref"]]) or int(cnt[engine.CNT["mc_beyond"]]):
        sys.exit("bench_engine_bframes.py: the synthetic grids left the reference's definition")
    for eng in engines.values():
        eng.time_device(engine.PH_ALL, True, max(args.warmup, 1))
    rounds = {name: [] for name in engines}
    for _ in range(args.rounds):
        for name, eng in engines.items():
            rounds[name].append(eng.time_device(engine.PH_ALL, True, args.steps) / args.steps)
    res = {"workload": "%d synthetic 3840x2160 4:2:0 frames per step, shipped block-size maps, q0 %d; mv_grid_b grids "
                       "(%.2f of the valid vertices on NEXT), pool of %d pictures; the P-frame engine on the same grids "
                       "with NEXT folded onto PREV" % (F, bench.Q0, next_share, 3 * F),
           "gpu": bench.gpu_identity(0), "steps_per_round": args.steps, "rounds": args.rounds,
           "parity_checked": "frame 0's prediction against the reference's od_state_mc_predict with three pictures",
           "leaves_per_step": leaves}
    for name, eng in engines.items():
        res[name] = {"ms_per_step": round(statistics.median(rounds[name]), 4),
                     "ms_per_step_rounds": [round(v, 4) for v in rounds[name]], "h2d_bytes_per_step": eng.h2d_bytes,
                     "launches_per_step": eng.launches_per_step(), "device_bytes": int(eng.buf.bytes_allocated)}
        eng.close()
    res["third_picture_ms"] = round(res["mc_next"]["ms_per_step"] - res["p_frame_folded"]["ms_per_step"], 4)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
