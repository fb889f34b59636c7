#!/usr/bin/env python
"""The engine's P-frame prediction from MV grids (inter_mc=1) against the host-prediction inter mode (inter=1) on
bench_engine_inter.py's workload: 16 synthetic 3840x2160 4:2:0 frames, the shipped block-size maps, q0 72.  Each
frame predicts from a seeded synthetic MV grid (every split level, GOLD / PREV mixed per vertex, vectors within
OD_UMV_CLAMP) and two pictures of a pool of 2F; the inter engine is fed the inter_mc engine's prediction, so both
code the same residual.  Frame 0's prediction is checked against the reference's od_state_mc_predict (the hook library
of oracle/inter_mc.mk) before timing.  The two engines are timed in alternating rounds (CUDA events, inputs resident in HBM, one graph
replay per step), then their forward phase (for inter_mc: OBMC + both transforms).  With --profile the OBMC and
leaf kernels alone are timed by torch.profiler in a run of their own.  Also reported: H2D bytes per step, leaves
per step, the OBMC kernel's algorithmic bytes against 3.35 TB/s, and the C od_state_mc_predict of one frame on
one host core.  Needs a CUDA device; prints one JSON line.

    python tools/bench_engine_inter_mc.py [--rounds 3] [--steps 10] [--warmup 3] [--frames 16] [--profile]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
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
    from tests import inter_mc_oracle
    if _native.lib().daala_b200_device_count() < 1:
        sys.exit("bench_engine_inter_mc.py needs a CUDA device: nothing is measured without one")

    geom = Geometry(bench.PIC_W, bench.PIC_H)
    F = args.frames
    q4 = np.full((3, 30), bench.PVQ_QM_Q4, np.uint8)
    hf = bench.make_host_frames(geom, F)
    planes = [np.stack([f[0][p] for f in hf]) for p in range(3)]
    bsize = np.stack([f[1] for f in hf])
    # pool: slot f = synthetic frame f - 1 (PREV of frame f), slot F + f = frame f - 2 (GOLD of frame f)
    refs = [np.concatenate([np.roll(planes[p], 1, axis=0), np.roll(planes[p], 2, axis=0)]) for p in range(3)]
    slot = np.array([[F + f, f] for f in range(F)], np.int32)
    grids = [synth.mv_grid(geom, seed=1000 + f) for f in range(F)]
    packed = mvgrid.pack(*(np.stack([g[i] for g in grids]) for i in range(3)))
    leaves = sum(len(mvgrid.leaves(g[0].astype(bool))[0]) for g in grids)
    common = dict(nframes=F, q0=bench.Q0, use_masking=1, pvq_qm_q4=q4, max_blocks_div=2)
    mc = engine.KeyframeEngine(geom, inter=1, inter_mc=1, **common)
    out = mc.encode(planes, bsize, refs=refs, ref_slot=slot, mv_grid=packed)
    pred = [np.array(out["pred%d" % p]) for p in range(3)]

    if args.profile:
        import torch
        from torch.profiler import ProfilerActivity, profile
        for _ in range(max(args.warmup, 1)):
            mc.run_device(engine.PH_ALL, graph=False)
        mc.wait()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                mc.run_device(engine.PH_ALL, graph=False)
            mc.wait()
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            for tag in ("k_mc_obmc", "k_mc_leaves"):
                if tag in e.key:
                    kern[tag] = round(e.device_time_total / 1e3 / args.steps, 4)   # ms per step
        px = sum(int(np.prod(geom.plane_shape(p))) for p in range(3))
        # the prediction written once, each frame's two pictures and its grid read once
        alg = F * (px + 2 * px + packed[0].nbytes)
        res = {"profile": "torch.profiler, %d steps without the graph" % args.steps, "gpu": bench.gpu_identity(0),
               "kernel_ms_per_step": kern, "obmc_algorithmic_bytes": alg}
        if "k_mc_obmc" in kern:
            res["obmc_gb_per_s"] = round(alg / (kern["k_mc_obmc"] * 1e-3) / 1e9, 1)
            res["obmc_share_of_3_35_tb_per_s"] = round(alg / HBM_BYTES_PER_S / (kern["k_mc_obmc"] * 1e-3), 4)
        mc.close()
        print(json.dumps(res), flush=True)
        return

    ref = inter_mc_oracle.load()
    if ref is None:
        sys.exit("bench_engine_inter_mc.py: the prediction is checked against oracle/_ref/libdaala_ref_inter_mc.so, "
                 "which is not built")
    want, host_s = inter_mc_oracle.predict(ref, geom, [refs[p][slot[0, 0]] for p in range(3)],
                                           [refs[p][slot[0, 1]] for p in range(3)], *grids[0], timed=True)
    mism = sum(int(np.count_nonzero(pred[p][0] != want[p])) for p in range(3))
    if mism:
        sys.exit("bench_engine_inter_mc.py: frame 0's prediction differs from od_state_mc_predict (%d pixels)" % mism)
    cnt = out["counts"]
    if int(cnt[engine.CNT["mc_bad_ref"]]) or int(cnt[engine.CNT["mc_beyond"]]):
        sys.exit("bench_engine_inter_mc.py: the synthetic grids left the reference's definition")
    mc_h2d = mc.h2d_bytes
    host = engine.KeyframeEngine(geom, inter=1, **common)
    host.encode(planes, bsize, pred=pred)
    host_h2d = host.h2d_bytes
    engines = {"inter": host, "inter_mc": mc}
    for eng in engines.values():
        eng.time_device(engine.PH_ALL, True, max(args.warmup, 1))
    rounds = {name: [] for name in engines}
    for _ in range(args.rounds):
        for name, eng in engines.items():
            rounds[name].append(eng.time_device(engine.PH_ALL, True, args.steps) / args.steps)
    fwd = {}
    for name, eng in engines.items():
        eng.time_device(engine.PH_LISTS | engine.PH_FORWARD, False, 1)
        fwd[name] = round(eng.time_device(engine.PH_FORWARD, False, args.steps) / args.steps, 4)
        eng.time_device(engine.PH_ALL, True, 1)
    res = {"workload": "%d synthetic 3840x2160 4:2:0 frames per step, shipped block-size maps, q0 %d; seeded MV grids, "
                       "GOLD / PREV per vertex from a pool of %d pictures" % (F, bench.Q0, 2 * F),
           "gpu": bench.gpu_identity(0), "steps_per_round": args.steps, "rounds": args.rounds,
           "parity_checked": "frame 0's prediction against the reference's od_state_mc_predict",
           "leaves_per_step": leaves, "host_od_state_mc_predict_ms_one_frame_one_core": round(host_s * 1e3, 2)}
    for name, eng in engines.items():
        ms = statistics.median(rounds[name])
        res[name] = {"ms_per_step": round(ms, 4), "ms_per_step_rounds": [round(v, 4) for v in rounds[name]],
                     "forward_ms": fwd[name], "h2d_bytes_per_step": mc_h2d if name == "inter_mc" else host_h2d,
                     "launches_per_step": eng.launches_per_step(), "device_bytes": int(eng.buf.bytes_allocated)}
        eng.close()
    res["forward_difference_ms"] = round(fwd["inter_mc"] - fwd["inter"], 4)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
