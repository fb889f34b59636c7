"""What the keyframe engine's symbol stream (config.symbol_stream = 1) costs and saves on the benchmark workload.

The workload is bench.py's (16 x 3840x2160 per batch, the reference encoder's block-size maps and deringing
levels, q0 72, max_blocks_div = 2, dering = 1), built with bench.py's own helpers.  In one
process, alternating the two configurations round by round, it measures:
  - the device step time (graph replay, CUDA events on the engine's stream) with symbol_stream 0 and 1;
  - end-to-end Mpixels/s through two double-buffered engines (submit one batch while the other one runs, as
    bench.py's e2e loop does) for (a) reconstruction + the classic symbol arrays and (b) reconstruction + the
    symbol stream;
  - the bytes copied device -> host per step in (a) and (b).
With --haar-dc both configurations quantise the keyframe DCs (haar_dc_quant = 1): (a) returns the classic arrays and
the DC index grids, (b) the stream with its keyframe DC records (sym_hdc) and no grids; the device step of (b) also
times the DC record kernel alone (k_sym_hdc, torch.profiler).
Prints the GPU's name and power limit with the numbers, and one JSON line at the end.

    python tools/bench_symbol_stream.py [--steps 10] [--rounds 3] [--haar-dc]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--haar-dc", action="store_true")
    args = ap.parse_args()

    import numpy as np
    import torch
    import bench
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    assert torch.cuda.is_available(), "needs a CUDA device"

    gpu = bench.gpu_identity(0)
    print("GPU: %s, power limit %s W" % (gpu["name"], gpu["power_limit_w"]), flush=True)
    geom = Geometry(bench.PIC_W, bench.PIC_H)
    F = 16
    q4 = np.full((3, 30), bench.PVQ_QM_Q4, np.uint8)

    def make(stream, rotate):
        hf = bench.make_host_frames(geom, F, rotate=rotate)
        eng = engine.KeyframeEngine(geom, nframes=F, q0=bench.Q0, use_masking=1, pvq_qm_q4=q4, dering=1,
                                    coded_quantizer=bench.CODED_Q, dering_lambda=bench.DERING_LAMBDA, persist_ctas_per_sm=0,
                                    max_blocks_div=2, symbol_stream=stream, haar_dc_quant=int(args.haar_dc))
        eng.stage_inputs([np.stack([f[0][p] for f in hf]) for p in range(3)], np.stack([f[1] for f in hf]))
        eng.stage_dering_levels(np.stack([f[2] for f in hf]))
        eng.prepare_io(symbols=not stream, recon=True, stream=bool(stream), dc_grids=not stream)
        return eng

    # (a): two engines without the stream, classic symbols; (b): two with the stream, no classic symbols
    cfg = {"a": [make(0, 0), make(0, 1)], "b": [make(1, 0), make(1, 1)]}
    for engs in cfg.values():
        for e in engs:
            e.submit()
        for e in engs:
            out = e.wait()
            assert int(out["counts"][engine.CNT["error"]]) == 0

    def d2h(e):
        return e.d2h_bytes + (e.stream_d2h_bytes() if e.symbol_stream else 0)

    def e2e(engs, steps):
        for i in range(steps):
            e = engs[i % 2]
            if i >= 2:
                e.wait()
            e.submit()
        for e in engs:
            e.wait()

    px = geom.luma_pixels * F
    dev = {"a": [], "b": []}
    rate = {"a": [], "b": []}
    for e in cfg["a"] + cfg["b"]:
        e.time_device(engine.PH_ALL, True, 3)
    for r in range(args.rounds):
        for k in ("a", "b"):
            dev[k].append(cfg[k][0].time_device(engine.PH_ALL, True, args.steps) / args.steps)
        for k in ("a", "b"):
            e2e(cfg[k], 4)
            t0 = time.perf_counter()
            e2e(cfg[k], args.steps)
            rate[k].append(px * args.steps / (time.perf_counter() - t0) / 1e6)
        print("round %d: step ms  symbol_stream 0: %.3f  1: %.3f | e2e Mpixels/s  (a) classic: %.1f  (b) stream: %.1f"
              % (r, dev["a"][-1], dev["b"][-1], rate["a"][-1], rate["b"][-1]), flush=True)
    bytes_a, bytes_b = d2h(cfg["a"][0]), d2h(cfg["b"][0])
    res = {
        "gpu": gpu, "frames_per_step": F, "steps": args.steps, "rounds": args.rounds, "haar_dc_quant": int(args.haar_dc),
        "device_step_ms": {"symbol_stream_0": [round(v, 3) for v in dev["a"]],
                           "symbol_stream_1": [round(v, 3) for v in dev["b"]],
                           "stream_extra_ms_median": round(statistics.median(dev["b"]) - statistics.median(dev["a"]), 3)},
        "e2e_mpixels_s": {"a_recon_classic": [round(v, 1) for v in rate["a"]],
                          "b_recon_stream": [round(v, 1) for v in rate["b"]]},
        "d2h_bytes_per_step": {"a_recon_classic": int(bytes_a), "b_recon_stream": int(bytes_b)},
        "launches_per_step": {"symbol_stream_0": cfg["a"][0].launches_per_step(),
                              "symbol_stream_1": cfg["b"][0].launches_per_step()},
    }
    out = cfg["b"][0].wait()
    idx = out["sym_index"]
    lb = cfg["a"][0].wait()
    nk = int((lb["luma_res"][..., 3] > 0).sum() + (lb["chroma_res"][..., 3] > 0).sum())
    res["stream_per_step"] = {"blocks": int(idx[:, 1].sum()), "bands": int(idx[:, 3].sum()),
                              "pulse_bytes": int(idx[:, 5].sum()), "bands_with_k_gt_0": nk}
    if args.haar_dc:
        res["stream_per_step"]["hdc_records"] = int(idx[:, 1].sum())
        res["k_sym_hdc_us"] = kernel_us(cfg["b"][0], "k_sym_hdc")
    print(json.dumps(res), flush=True)
    for engs in cfg.values():
        for e in engs:
            e.close()


def kernel_us(eng, name, reps=5):
    """Mean device time of the kernels whose name contains `name` over `reps` graph replays (torch.profiler)."""
    from torch.profiler import ProfilerActivity, profile
    from daala_b200 import engine
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            eng.run_device(engine.PH_ALL, True)
        eng.wait()
    us = [e.device_time_total for e in prof.key_averages() if name in e.key]
    return round(sum(us) / reps, 2) if us else None


if __name__ == "__main__":
    main()
