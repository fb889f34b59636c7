#!/usr/bin/env python
"""The keyframe step with quantised DCs (haar_dc_quant = 1) against the default step (unquantised DCs): bench.py's 16
synthetic 3840x2160 4:2:0 frames with the reference encoder's block-size maps, quantizer 72, deringing levels given.
Two engines, timed in alternating rounds (CUDA events on the engine's stream, inputs resident in HBM, one graph replay
per step).  Reported: ms per step of each; the DC chain's own device time and its place in the step (the median node
timeline of tools/profile_step.py under torch.profiler: start and end of k_haar_dc against the luma chain kernel
k_pvq_persist and the luma finishing scatter that waits for it); the index grids' D2H bytes per step; the card's
name and power limit.  Needs a CUDA device; prints one JSON line.

    python tools/bench_engine_haar_dc.py [--rounds 3] [--steps 10] [--reps 10]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=10, help="steps traced for the node timeline")
    args = ap.parse_args()
    import numpy as np
    import torch
    import bench
    import profile_step
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    if not torch.cuda.is_available():
        sys.exit("bench_engine_haar_dc.py needs a CUDA device: nothing is measured without one")
    torch.cuda.init()
    geom = Geometry(bench.PIC_W, bench.PIC_H)
    F = 16
    q4 = np.full((3, 30), bench.PVQ_QM_Q4, np.uint8)
    hf = bench.make_host_frames(geom, F)
    engines, d2h = {}, {}
    for mode in (0, 1):
        eng = engine.KeyframeEngine(geom, nframes=F, q0=bench.Q0, use_masking=1, pvq_qm_q4=q4, dering=1,
                                    coded_quantizer=bench.CODED_Q, dering_lambda=bench.DERING_LAMBDA,
                                    max_blocks_div=2, haar_dc_quant=mode)
        eng.stage_inputs([np.stack([f[0][p] for f in hf]) for p in range(3)], np.stack([f[1] for f in hf]))
        eng.stage_dering_levels(np.stack([f[2] for f in hf]))
        eng.prepare_io(symbols=True, recon=True)
        eng.submit()
        out = eng.wait()
        assert int(out["counts"][engine.CNT["error"]]) == 0
        d2h[mode] = int(sum(out["dc_index%d" % p].nbytes for p in range(3))) if mode else 0
        eng.time_device(engine.PH_ALL, True, 3)
        engines[mode] = eng
    ms = {0: [], 1: []}
    for _ in range(args.rounds):
        for mode in (0, 1):
            ms[mode].append(engines[mode].time_device(engine.PH_ALL, True, args.steps) / args.steps)
    tl = profile_step.summarise(profile_step.trace_steps(lambda: engines[1].run_device(engine.PH_ALL, True), args.reps))
    base = profile_step.summarise(profile_step.trace_steps(lambda: engines[0].run_device(engine.PH_ALL, True),
                                                           args.reps))
    for eng in engines.values():
        eng.close()

    def node(s, prefix):
        return next((r for r in s["nodes"] if r["node"].startswith(prefix)), None)

    chain = node(tl, "daala_b200::haar_dc::k_haar_dc") or node(tl, "k_haar_dc")
    persist = node(tl, "daala_b200::kf::k_pvq_persist") or node(tl, "k_pvq_persist")
    scatter = node(tl, "daala_b200::kf::k_finish_scatter<false, true>") or node(tl, "k_finish_scatter<false, true>")
    m0, m1 = statistics.median(ms[0]), statistics.median(ms[1])
    res = dict(gpu=bench.gpu_identity(torch.cuda.current_device()), frames=F, size="%dx%d" % (bench.PIC_W, bench.PIC_H),
               quantizer=bench.Q0, ms_per_step_default=[round(v, 3) for v in ms[0]],
               ms_per_step_haar_dc=[round(v, 3) for v in ms[1]], median_default=round(m0, 3),
               median_haar_dc=round(m1, 3), cost_pct=round(100 * (m1 - m0) / m0, 2),
               chain=chain, luma_chain_kernel=persist, luma_scatter=scatter,
               chain_inside_luma_chain_kernel=bool(chain and persist and chain["end_ms"] <= persist["end_ms"]),
               span_ms=dict(default=base["span_ms"], haar_dc=tl["span_ms"]), dc_index_d2h_bytes=d2h[1],
               timeline=tl["nodes"])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
