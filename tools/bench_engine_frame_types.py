#!/usr/bin/env python
"""One engine for keyframes and P frames (config.frame_types = 1) against the two-engine route, on 16-frame 3840x2160
4:2:0 steps: synthetic frames, the shipped block-size maps (daala_b200/data/bench_bsize_4k.npz, cycled), seeded MV
grids and per-frame records, inputs and reference pool resident on the device.

  mixed       one engine (inter, inter_mc, frame_quant, haar_dc_quant, inter_finish = 1, frame_types): a step of
              1 keyframe + 15 P frames, then its finishing pass, which stores all 16 reconstructions in the pool;
  two_engine  a keyframe engine step of 1 frame (keyframe_quant, haar_dc_quant), an inter engine step + finishing pass
              of the 15 P frames (inter, inter_mc, frame_quant, inter_finish = 1), and the pool_load of the keyframe's
              reconstruction into the inter engine's pool, device to device.
Both routes run alternately, --rounds rounds of --steps iterations each; an iteration's time is the host clock around
it ending in a stream synchronise (device-resident inputs: no H2D of pictures).  Also the step graph alone (CUDA events
around --steps replays, daala_b200_kf_time_device) of an all-P batch on the mixed engine against the plain frame_quant
inter engine: the cost of carrying the mode.  Reports bytes_allocated of every engine and the card's name and power
limit.  Needs a CUDA device; prints one JSON line.

--stream measures the mixed symbol stream (symbol_stream = 3) instead, on the same 1 keyframe + 15 P frame step: the
step graph's device time on the mixed engine with symbol_stream 0 and 3 (CUDA events around --steps replays,
daala_b200_kf_time_device, the two engines alternated over --rounds rounds, same inputs and pool contents), and the
step's D2H bytes of the stream route (encode(..., symbols=False, dc_grids=False): reconstruction, prediction, counters
and the used part of the stream with its DC and keyframe DC records) against the classic route (the same outputs with
the block-order arrays and the DC index grids in place of the stream).

    python tools/bench_engine_frame_types.py [--rounds 3] [--steps 5] [--stream]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, check=True)
        return r.stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def main():
    import numpy as np
    from daala_b200 import engine, mvgrid, synth
    from daala_b200.frame import Geometry
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--stream", action="store_true", help="the mixed symbol stream (symbol_stream = 3) instead")
    args = ap.parse_args()
    geom, F = Geometry(3840, 2160), 16
    real = np.load(os.path.join(ROOT, "daala_b200", "data", "bench_bsize_4k.npz"))
    bsize = np.stack([real["bsize_%d" % (f % 4)] for f in range(F)]).astype(np.uint8)
    pic = synth.pad_planes(synth.frame(geom.pic_w, geom.pic_h, f=1, seed=3)[0], geom)
    planes = [np.stack([pic[p]] * F) for p in range(3)]
    pool = [np.stack([pic[p]] * 2) for p in range(3)]
    grids = [synth.mv_grid(geom, seed=10 + f) for f in range(F)]
    grid = mvgrid.pack(*(np.stack([g[i] for g in grids]) for i in range(3)))
    q0 = np.array([40] + [60] * (F - 1))
    rec = engine.frame_quant_records(q0, q0 // 4, 0.67 * 0.1 * q0.astype(float) ** 2, np.full((F, 3, 30), 20, np.uint8))
    levels = np.ones((F, geom.nvsb, geom.nhsb), np.uint8)
    types = np.array([1] + [0] * (F - 1), np.uint8)
    slot = np.zeros((F, 2), np.int32)
    slot[:, 1] = 1
    if args.stream:
        print(json.dumps(stream_result(args, geom, planes, bsize, pool, grid, rec, types, slot)))
        return

    def finish_inputs(eng, out):
        return (np.zeros(len(out["luma_blocks"]), np.uint8), np.array(out["luma_dc"]),
                np.zeros(len(out["chroma_blocks"]), np.uint8), np.array(out["chroma_dc"]))

    mixed = engine.KeyframeEngine(geom, nframes=F, inter=1, inter_mc=1, mc_refs=F + 2, frame_quant=1, haar_dc_quant=1,
                                  inter_finish=1, frame_types=1)
    out = mixed.encode(planes, bsize, frame_quant=rec, frame_type=types, refs=pool, ref_slot=slot, mv_grid=grid)
    mixed.prepare_finish(*finish_inputs(mixed, out), dering_levels=levels,
                         ref_slot_out=np.arange(2, F + 2, dtype=np.int32))
    key = engine.KeyframeEngine(geom, nframes=1, keyframe_quant=1, haar_dc_quant=1)
    key.encode([p[:1] for p in planes], bsize[:1], frame_quant=rec[:1])
    inter = engine.KeyframeEngine(geom, nframes=F - 1, inter=1, inter_mc=1, mc_refs=F + 2, frame_quant=1, inter_finish=1)
    out = inter.encode([p[1:] for p in planes], bsize[1:], frame_quant=rec[1:], refs=pool, ref_slot=slot[1:],
                       mv_grid=grid[1:])
    inter.prepare_finish(*finish_inputs(inter, out), dering_levels=levels[1:],
                         ref_slot_out=np.arange(3, F + 2, dtype=np.int32))
    key_planes = [key.buf.pixels_out[p] for p in range(3)]

    def run_mixed():
        mixed.run_device()
        mixed.finish_submit()
        mixed.wait()

    def run_two():
        key.run_device()
        key.wait()
        inter.pool_load(2, key_planes)
        inter.run_device()
        inter.finish_submit()
        inter.wait()

    routes = {"mixed": run_mixed, "two_engine": run_two}
    for fn in routes.values():
        fn()
    times = {k: [] for k in routes}
    for _ in range(args.rounds):
        for k, fn in routes.items():
            t0 = time.perf_counter()
            for _ in range(args.steps):
                fn()
            times[k].append((time.perf_counter() - t0) * 1e3 / args.steps)
    result = {"metric": "frame_types_route_ms_per_16_frames", "card": card(), "geometry": "3840x2160", "frames": F,
              "route_ms": {k: {"median": statistics.median(v), "all": v} for k, v in times.items()},
              "bytes_allocated": {"mixed": mixed.buf.bytes_allocated, "keyframe_engine": key.buf.bytes_allocated,
                                  "inter_engine_15": inter.buf.bytes_allocated,
                                  "two_engine": key.buf.bytes_allocated + inter.buf.bytes_allocated},
              "launches_per_step": {"mixed": mixed.launches_per_step(), "keyframe_engine": key.launches_per_step(),
                                    "inter_engine_15": inter.launches_per_step()}}
    key.close()
    inter.close()
    # the cost of carrying the mode: an all-P step graph on the mixed engine and on the plain frame_quant engine
    plain = engine.KeyframeEngine(geom, nframes=F, inter=1, inter_mc=1, mc_refs=F + 2, frame_quant=1, inter_finish=1)
    plain.encode(planes, bsize, frame_quant=rec, refs=pool, ref_slot=slot, mv_grid=grid)
    mixed.encode(planes, bsize, frame_quant=rec, frame_type=np.zeros(F, np.uint8), refs=pool, ref_slot=slot, mv_grid=grid)
    step = {"mixed_all_p": [], "frame_quant_engine": []}
    for _ in range(args.rounds):
        for k, eng in (("mixed_all_p", mixed), ("frame_quant_engine", plain)):
            step[k].append(eng.time_device(reps=args.steps) / args.steps)
    result["all_p_step_graph_ms"] = {k: {"median": statistics.median(v), "all": v} for k, v in step.items()}
    result["bytes_allocated"]["frame_quant_engine"] = plain.buf.bytes_allocated
    plain.close()
    mixed.close()
    print(json.dumps(result))


def stream_result(args, geom, planes, bsize, pool, grid, rec, types, slot):
    """--stream: the step graph with and without the mixed stream, and the step's D2H bytes by route."""
    from daala_b200 import engine
    F = len(types)
    engines = {s: engine.KeyframeEngine(geom, nframes=F, inter=1, inter_mc=1, mc_refs=F + 2, frame_quant=1,
                                        haar_dc_quant=1, inter_finish=1, frame_types=1, symbol_stream=s) for s in (0, 3)}
    kw = dict(frame_quant=rec, frame_type=types, refs=pool, ref_slot=slot, mv_grid=grid)
    try:
        engines[0].encode(planes, bsize, **kw)
        classic = engines[0].d2h_bytes
        out = engines[3].encode(planes, bsize, symbols=False, dc_grids=False, **kw)
        fixed, stream = engines[3].d2h_bytes, engines[3].stream_d2h_bytes()
        blocks = int(out["sym_index"][:, 1].sum())
        step = {"symbol_stream_0": [], "symbol_stream_3": []}
        for s, eng in engines.items():
            eng.time_device(reps=1)   # warm-up of the graph as it is timed
        for _ in range(args.rounds):
            for s, eng in engines.items():
                step["symbol_stream_%d" % s].append(eng.time_device(reps=args.steps) / args.steps)
        med = {k: statistics.median(v) for k, v in step.items()}
        return {"metric": "frame_types_stream", "card": card(), "geometry": "%dx%d" % (geom.pic_w, geom.pic_h),
                "frames": F, "keyframes": int(types.sum()),
                "step_graph_ms": {k: {"median": med[k], "all": v} for k, v in step.items()},
                "stream_cost_ms": med["symbol_stream_3"] - med["symbol_stream_0"],
                "d2h_bytes": {"classic_route": classic, "stream_route": fixed + stream,
                              "stream_route_stream_part": stream, "stream_route_other_part": fixed},
                "stream_blocks": blocks,
                "launches_per_step": {k: e.launches_per_step() for k, e in (("symbol_stream_0", engines[0]),
                                                                             ("symbol_stream_3", engines[3]))}}
    finally:
        for eng in engines.values():
            eng.close()


if __name__ == "__main__":
    main()
