#!/usr/bin/env python
"""Per-kernel device time of the keyframe engine's inverse phase (PH_INVERSE: iDCT + lapped postfilter,
SB-edge postfilter, deringing, u8 store) on the workload bench.py measures, under torch.profiler with CUDA
activities.

The workload is built with bench.py's own helpers and constants (16 frames of 3840x2160 4:2:0, the reference
encoder's block-size maps and deringing levels, q0 72, max_blocks_div 2, split_free 1).  One full step runs first
so that the inverse phase has its inputs, then PH_INVERSE is launched `--reps` times without a graph under the
profiler, then PH_ALL once more in a trace of its own.  For every kernel of the phase the script prints its mean
device time per step, the bytes it has to move (computed from the plane shapes: every sample read and written
once, the deringing apron and the direction map not counted) and that over the H100 SXM data sheet's 3.35 TB/s.
The GPU's name and power limit are printed in the same output.

    python tools/profile_inverse.py [--dering 1|2] [--reps 20] [--out DIR]
"""
import argparse
import collections
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402

PEAK_GBS = 3350.0   # H100 SXM data sheet, HBM3


def kernel_table(events, dering_launches):
    """{label: total device ns} of the traced kernels.  k_dering_sb is split by its position in the step: the level
    search's passes (luma) come first, then the final application to planes 0, 1, 2."""
    tot = collections.OrderedDict()
    order = []
    for e in sorted(events, key=lambda e: e.start_ns()):
        name = e.name()
        short = name.split("(")[0].split("<")[0].split("::")[-1].replace("void ", "").strip()
        order.append((short, e.duration_ns()))
    nder = 0
    for short, ns in order:
        label = short
        if short == "k_dering_sb":
            k = nder % dering_launches
            nder += 1
            search = dering_launches - 3
            label = "k_dering_sb search pass %d (luma)" % (k + 1) if k < search else "k_dering_sb plane %d" % (k - search)
        tot[label] = tot.get(label, 0) + ns
    return tot


def profile(fn):
    import torch
    from torch.profiler import ProfilerActivity
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    from torch.autograd import DeviceType
    return [e for e in prof.profiler.kineto_results.events() if e.device_type() == DeviceType.CUDA
            and "memset" not in e.name().lower() and "memcpy" not in e.name().lower()]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dering", type=int, default=1, choices=[1, 2])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the result as JSON to OUT/profile_inverse_dering<N>.json")
    args = ap.parse_args()
    bench.DERING = args.dering

    import numpy as np
    import torch
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    assert torch.cuda.is_available(), "profile_inverse.py needs a CUDA device"
    torch.cuda.init()

    geom = Geometry(bench.PIC_W, bench.PIC_H)
    F = 16
    q4 = np.full((3, 30), bench.PVQ_QM_Q4, np.uint8)
    hf = bench.make_host_frames(geom, F)
    eng = engine.KeyframeEngine(geom, nframes=F, q0=bench.Q0, use_masking=1, pvq_qm_q4=q4, dering=args.dering,
                                coded_quantizer=bench.CODED_Q, dering_lambda=bench.DERING_LAMBDA, persist_ctas_per_sm=0,
                                split_free=1, level_chains=0, noref_prepass=0, max_blocks_div=2)
    eng.stage_inputs([np.stack([f[0][p] for f in hf]) for p in range(3)], np.stack([f[1] for f in hf]))
    if args.dering == 1:
        eng.stage_dering_levels(np.stack([f[2] for f in hf]))
    eng.prepare_io(symbols=True, recon=True)
    eng.submit()
    out = eng.wait()
    assert int(out["counts"][engine.CNT["error"]]) == 0
    eng.time_device(engine.PH_ALL, False, 2)
    eng.time_device(engine.PH_INVERSE, False, 3)
    ev_ms = eng.time_device(engine.PH_INVERSE, False, args.reps) / args.reps

    dering_launches = 3 + (5 if args.dering == 2 else 0)
    inv = kernel_table(profile(lambda: eng.time_device(engine.PH_INVERSE, False, args.reps)), dering_launches)
    full = kernel_table(profile(lambda: eng.time_device(engine.PH_ALL, False, 1)), dering_launches)
    gpu = bench.gpu_identity(torch.cuda.current_device())
    eng.close()

    # bytes each kernel has to move per step
    samples = [F * geom.plane_shape(p)[0] * geom.plane_shape(p)[1] for p in range(3)]
    nsb = F * geom.nhsb * geom.nvsb
    dering_u8 = "k_i16_to_u8" not in inv     # the deringing kernel stores the u8 reconstruction itself
    need = {"k_inverse_sb": 8 * sum(samples), "k_sb_postfilter_store": 6 * sum(samples),
            "k_i16_to_u8": 3 * sum(samples), "k_dering_thresholds": 9 * nsb}
    for p in range(3):
        need["k_dering_sb plane %d" % p] = (2 + (1 if dering_u8 else 2)) * samples[p]
    for k in range(5):
        need["k_dering_sb search pass %d (luma)" % (k + 1)] = 4 * samples[0]

    rows = []
    for label, ns in inv.items():
        ms = ns / 1e6 / args.reps
        b = need.get(label)
        rows.append(dict(kernel=label, ms_per_step=round(ms, 4), bytes_per_step=b,
                         hbm_frac=None if b is None else round(b / (ms * 1e-3) / 1e9 / PEAK_GBS, 3)))
    sum_ms = sum(r["ms_per_step"] for r in rows)
    print("GPU: %s, power limit %s W, max SM clock %s MHz" % (gpu["name"], gpu["power_limit_w"], gpu["sm_max_mhz"]))
    print("PH_INVERSE, dering=%d, %d frames 3840x2160, %d reps: %.3f ms per step by CUDA events (graph off), "
          "%.3f ms summed kernel time" % (args.dering, F, args.reps, ev_ms, sum_ms))
    print("%-36s %10s %14s %9s" % ("kernel", "ms/step", "bytes/step", "of 3.35TB/s"))
    for r in rows:
        print("%-36s %10.4f %14s %9s" % (r["kernel"], r["ms_per_step"], "-" if r["bytes_per_step"] is None else
                                         "%d" % r["bytes_per_step"], "-" if r["hbm_frac"] is None else "%.3f" % r["hbm_frac"]))
    print("PH_ALL, one step (kernels of the inverse phase):")
    for label in inv:
        if label in full:
            print("  %-34s %10.4f" % (label, full[label] / 1e6))
    print("  %-34s %10.4f" % ("all kernels of the step", sum(full.values()) / 1e6))
    res = dict(gpu=gpu, dering=args.dering, reps=args.reps, inverse_event_ms=round(ev_ms, 4), kernels=rows,
               ph_all_ms={k: round(v / 1e6, 4) for k, v in full.items()})
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "profile_inverse_dering%d.json" % args.dering), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
