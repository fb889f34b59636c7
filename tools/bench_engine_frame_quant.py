#!/usr/bin/env python
"""Per-frame quantizers (config.frame_quant) on the P/B-frame engine.

(a) Overhead: bench_engine_bframes.py's workload (16 synthetic 3840x2160 4:2:0 frames, the shipped block-size maps,
    mv_grid_b grids, three pictures each from a pool of 3F) on an mc_next engine with late_skip, symbol_stream = 2 and
    the searching finishing pass, once with frame_quant = 1 and every record at q0 72, once with frame_quant = 0 at q0
    72.  Step time (CUDA events, one graph replay per step, inputs resident) and finishing-pass time (host clock around
    finish + wait, decisions = the step's own) in alternating rounds; medians.  The outputs of the two engines are
    compared first.
(b) One sequence: frames of one synthetic 3840x2160 sequence with b_frames = 2.  The pipelined schedule of gop.py puts
    a P frame and the two B frames coded before it, at the encoder's P and B quantizers, in one frame_quant engine of 3
    frames; without per-frame quantizers the same frames need a P engine (1 frame) and a B engine (2 frames), one step
    each.  Device time per coded frame of the step (CUDA events, graph replay) for both.
Needs a CUDA device; prints one JSON line with the GPU and its power limit.

    python tools/bench_engine_frame_quant.py [--rounds 5] [--steps 10] [--warmup 3] [--frames 16]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--frames", type=int, default=16)
    args = ap.parse_args()
    import numpy as np
    import bench
    from daala_b200 import _native, engine, mvgrid, synth
    from daala_b200.frame import Geometry
    if _native.lib().daala_b200_device_count() < 1:
        sys.exit("bench_engine_frame_quant.py needs a CUDA device: nothing is measured without one")
    geom = Geometry(bench.PIC_W, bench.PIC_H)
    F = args.frames
    q0, q4 = bench.Q0, np.full((3, 30), bench.PVQ_QM_Q4, np.uint8)
    cq = 30
    hf = bench.make_host_frames(geom, F)
    planes = [np.stack([f[0][p] for f in hf]) for p in range(3)]
    bsize = np.stack([f[1] for f in hf])
    refs = [np.concatenate([np.roll(planes[p], 1, axis=0), np.roll(planes[p], -1, axis=0), np.roll(planes[p], 2, axis=0)])
            for p in range(3)]
    slot = np.array([[2 * F + f, f, F + f] for f in range(F)], np.int32)
    grids = [synth.mv_grid_b(geom, seed=3000 + f, p_next=0.5, p_gold=0.3) for f in range(F)]
    valid, mv, mv1, ref = (np.stack([g[i] for g in grids]) for i in range(4))
    grid, mv1 = mvgrid.pack(valid, mv, ref), mv1.astype(np.int32)
    opts = dict(q0=q0, use_masking=1, pvq_qm_q4=q4, coded_quantizer=cq, max_blocks_div=2, inter=1, inter_mc=1,
                mc_next=1, late_skip=1, symbol_stream=2, inter_finish=2)
    rec = engine.frame_quant_records([q0] * F, cq, None, q4)

    # (a)
    engines, outs = {}, {}
    for name, fq in (("frame_quant", 1), ("uniform", 0)):
        eng = engine.KeyframeEngine(geom, nframes=F, frame_quant=fq, **opts)
        out = eng.encode(planes, bsize, refs=refs, ref_slot=slot, mv_grid=grid, mv1_grid=mv1,
                         frame_quant=rec if fq else None)
        outs[name] = {k: np.array(v) for k, v in out.items()}
        dec = (np.zeros(len(out["luma_dc"]), np.uint8), outs[name]["luma_dc"], np.zeros(len(out["chroma_dc"]), np.uint8),
               outs[name]["chroma_dc"])
        fin = eng.finish(*dec)
        outs[name].update({"fin_" + k: np.array(v) for k, v in fin.items()})
        engines[name] = (eng, dec)
    same = all(np.array_equal(outs["frame_quant"][k], outs["uniform"][k], equal_nan=k.endswith("skip_diff"))
               for k in outs["uniform"])
    if not same:
        sys.exit("bench_engine_frame_quant.py: frame_quant = 1 with uniform records differs from frame_quant = 0")
    for eng, _ in engines.values():
        eng.time_device(engine.PH_ALL, True, max(args.warmup, 1))
    step = {n: [] for n in engines}
    fin = {n: [] for n in engines}
    for _ in range(args.rounds):
        for name, (eng, dec) in engines.items():
            step[name].append(eng.time_device(engine.PH_ALL, True, args.steps) / args.steps)
            eng.prepare_finish(*dec)
            eng.finish_submit()
            eng.wait()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                eng.finish_submit()
            eng.wait()
            fin[name].append((time.perf_counter() - t0) * 1e3 / args.steps)
    res = {"gpu": bench.gpu_identity(0), "rounds": args.rounds, "steps_per_round": args.steps,
           "a_workload": "%d synthetic 3840x2160 4:2:0 frames, shipped block-size maps, mv_grid_b grids, q0 %d, "
                         "late_skip, symbol_stream 2, inter_finish 2" % (F, q0),
           "a_outputs_equal": same}
    for name, (eng, _) in engines.items():
        res["a_" + name] = {"step_ms": round(statistics.median(step[name]), 4),
                            "step_ms_rounds": [round(v, 4) for v in step[name]],
                            "finish_ms": round(statistics.median(fin[name]), 4),
                            "finish_ms_rounds": [round(v, 4) for v in fin[name]],
                            "launches_per_step": eng.launches_per_step(), "h2d_bytes_per_step": eng.h2d_bytes}
        eng.close()

    # (b): slot 0 GOLD, 1 PREV (the previous anchor), 2 NEXT (this interval's end)
    rq = dict(P=(72, 30), B=(114, 38))
    kinds = ["P", "B", "B"]
    prefs = [np.stack([planes[p][0], planes[p][1], planes[p][2]]) for p in range(3)]
    g3 = [synth.mv_grid_b(geom, seed=4000 + i, p_next=0.0 if kinds[i] == "P" else 0.5) for i in range(3)]
    v3, m3, m13, r3 = (np.stack([g[i] for g in g3]) for i in range(4))
    pk3, m13 = mvgrid.pack(v3, m3, r3), m13.astype(np.int32)
    sl3 = np.array([[0, 1, 1], [0, 0, 1], [0, 0, 1]], np.int32)
    common = dict(use_masking=1, pvq_qm_q4=q4, max_blocks_div=2, inter=1, inter_mc=1, mc_next=1, late_skip=1,
                  symbol_stream=2)
    one = engine.KeyframeEngine(geom, nframes=3, q0=rq["P"][0], coded_quantizer=rq["P"][1], frame_quant=1, **common)
    one.encode([planes[p][3:6] for p in range(3)], bsize[3:6], refs=prefs, ref_slot=sl3, mv_grid=pk3, mv1_grid=m13,
               frame_quant=engine.frame_quant_records([rq[k][0] for k in kinds], [rq[k][1] for k in kinds], None, q4))
    pe = engine.KeyframeEngine(geom, nframes=1, q0=rq["P"][0], coded_quantizer=rq["P"][1], **common)
    pe.encode([planes[p][3:4] for p in range(3)], bsize[3:4], refs=prefs, ref_slot=sl3[:1], mv_grid=pk3[:1],
              mv1_grid=m13[:1])
    be = engine.KeyframeEngine(geom, nframes=2, q0=rq["B"][0], coded_quantizer=rq["B"][1], **common)
    be.encode([planes[p][4:6] for p in range(3)], bsize[4:6], refs=prefs, ref_slot=sl3[1:], mv_grid=pk3[1:],
              mv1_grid=m13[1:])
    for e in (one, pe, be):
        e.time_device(engine.PH_ALL, True, max(args.warmup, 1))
    piped, two = [], []
    for _ in range(args.rounds):
        piped.append(one.time_device(engine.PH_ALL, True, args.steps) / args.steps / 3)
        two.append((pe.time_device(engine.PH_ALL, True, args.steps) + be.time_device(engine.PH_ALL, True, args.steps))
                   / args.steps / 3)
    res["b_workload"] = ("one 3840x2160 sequence, b_frames 2: a P frame (q0 %d) and two B frames (q0 %d); pipelined: "
                         "one frame_quant engine of 3 frames, one step; two engines: P engine (1 frame) + B engine "
                         "(2 frames), one step each" % (rq["P"][0], rq["B"][0]))
    res["b_pipelined_ms_per_frame"] = round(statistics.median(piped), 4)
    res["b_pipelined_rounds"] = [round(v, 4) for v in piped]
    res["b_two_engines_ms_per_frame"] = round(statistics.median(two), 4)
    res["b_two_engines_rounds"] = [round(v, 4) for v in two]
    for e in (one, pe, be):
        e.close()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
