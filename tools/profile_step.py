#!/usr/bin/env python
"""Where one keyframe step goes: every kernel and memset node of the step graph, with its device time and its
start / end offset within the step, and the idle gaps between nodes, under torch.profiler with CUDA activities.

The workload is bench.py's (built with its own helpers and constants): 16 frames of 3840x2160 4:2:0, the reference
encoder's block-size maps and deringing levels, q0 72, max_blocks_div 2, symbol stream on.  After one
end-to-end pass and a few warm-up steps, `--reps` replays of the whole-step graph run under the profiler, each
followed by a device synchronise and a short host pause, so that the trace falls apart into one segment per step.
The same is done with live launches (no graph) unless --graph-only is given.  Per node the script reports the
median over the steps of its duration and of its start and end offset from the first node of the step; a name
that occurs more than once in a step (both k_finish_scatter, both k_begin_pvq, the memsets) is numbered in order
of its start.  The idle time of a step is its span minus the union of its nodes' intervals; the largest gaps are
listed with the nodes around them.  The GPU's name and power limit go into the same output.

    python tools/profile_step.py [--dering 1|2] [--reps 20] [--out DIR] [--graph-only]

Writes OUT/profile_step_dering<N>.json and prints the tables.
"""
import argparse
import collections
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402

STEP_GAP_NS = 2_000_000    # a host pause of 5 ms separates two steps; no gap inside a step comes near 2 ms


def short_name(name):
    """`void k_gather<1>(Stage)` -> `k_gather<1>`; memsets keep the profiler's name."""
    if "memset" in name.lower():
        return "memset"
    return name.split("(")[0].replace("void ", "").strip()


def trace_steps(fn, reps):
    """Runs fn() `reps` times under the profiler, synchronising and pausing after each, and returns one list of
    (name, start_ns, end_ns) per step, sorted by start."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
            torch.cuda.synchronize()
            time.sleep(0.005)
    ev = sorted(((short_name(e.name()), e.start_ns(), e.start_ns() + e.duration_ns())
                 for e in prof.profiler.kineto_results.events()
                 if e.device_type() == DeviceType.CUDA and "memcpy" not in e.name().lower()), key=lambda t: t[1])
    steps, cur, end = [], [], None
    for t in ev:
        if cur and t[1] - end > STEP_GAP_NS:
            steps.append(cur)
            cur = []
        cur.append(t)
        end = t[2] if end is None or not cur[:-1] else max(end, t[2])
    if cur:
        steps.append(cur)
    return steps


def summarise(steps):
    """Median per numbered node of (duration, start offset, end offset), median span / busy / idle of a step,
    and the largest idle gaps of the median-span step."""
    per = collections.OrderedDict()
    spans, busys = [], []
    for st in steps:
        t0 = st[0][1]
        seen = collections.Counter()
        for name, s, e in st:
            seen[name] += 1
            label = name if seen[name] == 1 else "%s #%d" % (name, seen[name])
            per.setdefault(label, []).append((e - s, s - t0, e - t0))
        span = max(e for _, _, e in st) - t0
        busy, cs, ce = 0, None, None
        for _, s, e in st:
            if ce is None or s > ce:
                if ce is not None:
                    busy += ce - cs
                cs, ce = s, e
            else:
                ce = max(ce, e)
        busy += ce - cs
        spans.append(span)
        busys.append(busy)
    # numbered labels of names that occur once per step lose nothing; a name seen twice gets "#1" for the first
    counts = collections.Counter(l.split(" #")[0] for l in per)
    rows = []
    for label, v in per.items():
        base = label.split(" #")[0]
        shown = label if " #" in label or counts[base] == 1 else label + " #1"
        rows.append(dict(node=shown, ms=round(statistics.median(x[0] for x in v) / 1e6, 4),
                         start_ms=round(statistics.median(x[1] for x in v) / 1e6, 4),
                         end_ms=round(statistics.median(x[2] for x in v) / 1e6, 4), steps=len(v)))
    rows.sort(key=lambda r: r["start_ms"])
    mid = sorted(range(len(steps)), key=lambda i: spans[i])[len(steps) // 2]
    st = steps[mid]
    t0 = st[0][1]
    gaps, ce, prev = [], None, None
    for name, s, e in st:
        if ce is not None and s > ce:
            gaps.append(dict(after=prev, before=name, at_ms=round((ce - t0) / 1e6, 4), gap_us=round((s - ce) / 1e3, 2)))
        if ce is None or e > ce:
            ce, prev = e, name
    gaps.sort(key=lambda g: -g["gap_us"])
    return dict(steps=len(steps), span_ms=round(statistics.median(spans) / 1e6, 4),
                busy_ms=round(statistics.median(busys) / 1e6, 4),
                idle_ms=round(statistics.median(s - b for s, b in zip(spans, busys)) / 1e6, 4),
                gaps_total=len(gaps), largest_gaps=gaps[:15], nodes=rows)


def print_summary(title, s):
    print("%s: %d steps, span %.3f ms, busy (union of nodes) %.3f ms, idle %.3f ms in %d gaps"
          % (title, s["steps"], s["span_ms"], s["busy_ms"], s["idle_ms"], s["gaps_total"]))
    print("  %-44s %9s %9s %9s" % ("node", "ms", "start", "end"))
    for r in s["nodes"]:
        print("  %-44s %9.4f %9.4f %9.4f" % (r["node"][:44], r["ms"], r["start_ms"], r["end_ms"]))
    print("  largest idle gaps (median-span step):")
    for g in s["largest_gaps"]:
        print("    %8.2f us at %8.4f ms  %s -> %s" % (g["gap_us"], g["at_ms"], g["after"], g["before"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dering", type=int, default=1, choices=[1, 2])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="write the result as JSON to OUT/profile_step_dering<N>.json")
    ap.add_argument("--graph-only", action="store_true", help="skip the live-launch (no graph) trace")
    args = ap.parse_args()
    bench.DERING = args.dering

    import numpy as np
    import torch
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    assert torch.cuda.is_available(), "profile_step.py needs a CUDA device"
    torch.cuda.init()

    geom = Geometry(bench.PIC_W, bench.PIC_H)
    F = 16
    q4 = np.full((3, 30), bench.PVQ_QM_Q4, np.uint8)
    hf = bench.make_host_frames(geom, F)
    eng = engine.KeyframeEngine(geom, nframes=F, q0=bench.Q0, use_masking=1, pvq_qm_q4=q4, dering=args.dering,
                                coded_quantizer=bench.CODED_Q, dering_lambda=bench.DERING_LAMBDA, persist_ctas_per_sm=0,
                                max_blocks_div=2)
    eng.stage_inputs([np.stack([f[0][p] for f in hf]) for p in range(3)], np.stack([f[1] for f in hf]))
    if args.dering == 1:
        eng.stage_dering_levels(np.stack([f[2] for f in hf]))
    eng.prepare_io(symbols=True, recon=True)
    eng.submit()
    out = eng.wait()
    assert int(out["counts"][engine.CNT["error"]]) == 0
    eng.time_device(engine.PH_ALL, True, 3)
    ev_ms = eng.time_device(engine.PH_ALL, True, args.reps) / args.reps

    res = dict(gpu=bench.gpu_identity(torch.cuda.current_device()), dering=args.dering, frames=F,
               size="%dx%d" % (bench.PIC_W, bench.PIC_H), reps=args.reps, launches_per_step=eng.launches_per_step(),
               graph_step_event_ms=round(ev_ms, 4))
    res["graph"] = summarise(trace_steps(lambda: eng.run_device(engine.PH_ALL, True), args.reps))
    if not args.graph_only:
        eng.time_device(engine.PH_ALL, False, 2)
        res["live"] = summarise(trace_steps(lambda: eng.run_device(engine.PH_ALL, False), args.reps))
    eng.close()

    g = res["gpu"]
    print("GPU: %s, power limit %s W, max SM clock %s MHz" % (g["name"], g["power_limit_w"], g["sm_max_mhz"]))
    print("dering=%d, %d frames %s, %d kernel launches per step; graph replay %.3f ms per step by CUDA events "
          "(profiler off)" % (args.dering, F, res["size"], res["launches_per_step"], ev_ms))
    print_summary("graph replays", res["graph"])
    if "live" in res:
        print_summary("live launches", res["live"])
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "profile_step_dering%d.json" % args.dering), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
