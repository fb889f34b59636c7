"""Timeline of the luma chain kernel k_pvq_persist<intra> on bench.py's workload.

Builds a copy of the library whose chain kernel records every item it runs (kf_engine.cu compiled with
-DDAALA_B200_CHAIN_TRACE, in a temporary directory; the in-tree library and its kernel are untouched), runs
bench.py's keyframe batch (same maps, quantizer and frames) through the engine, and reports from the records of
one luma stage:
  * warps busy over time, in bins of 1 % of the kernel's span;
  * the idle tail: from the moment the first warp runs out of items until the kernel's last item ends;
  * the mean duration of an item per band class while every warp is still working;
  * per band, when its last chain started and when its last item ended.

Needs a GPU and a prior build() (the other objects of the library are linked from daala_b200/_obj).

    python tools/chain_timeline.py [--json out.json] [--ctas-per-sm 0] [--split-free 1]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

REC = np.dtype([("t0", "<u8"), ("t1", "<u8"), ("item", "<u4"), ("cta", "<u4"), ("sm", "<u2"), ("bs", "u1"),
                ("kind", "u1"), ("pad", "<u4")])
KINDS = ("band-0 slot", "chain head", "free item", "chain successor")
TRACE_N = 240   # kf_engine.cu kTraceN


def build_traced(tmp):
    from daala_b200 import build as b
    b.build()
    objs = []
    for s in sorted(f for f in os.listdir(b.CSRC) if f.endswith(".cu")):
        if s == "kf_engine.cu":
            o = os.path.join(tmp, "kf_engine_trace.o")
            subprocess.run([b.NVCC] + b.FLAGS + ["-DDAALA_B200_CHAIN_TRACE", "-c", os.path.join(b.CSRC, s), "-o", o],
                           check=True)
            objs.append(o)
        else:
            objs.append(os.path.join(b.OBJ, s[:-3] + ".o"))
    lib = os.path.join(tmp, "libdaala_b200.so")
    subprocess.run([b.NVCC, "-shared", "-o", lib] + objs + b.ARCH, check=True)
    return lib


def analyse(r, nwarps):
    t_lo = int(r["t0"].min())
    t0 = (r["t0"] - t_lo) / 1e6   # ms from the kernel's first item
    t1 = (r["t1"] - t_lo) / 1e6
    span = float(t1.max())
    # warps busy, per 1 % of the span
    edges = np.linspace(0.0, span, 101)
    busy = []
    for a, b in zip(edges[:-1], edges[1:]):
        busy.append(float(np.clip(np.minimum(t1, b) - np.maximum(t0, a), 0, None).sum() / (b - a)))
    # the first warp to go idle: the smallest "last item end" over the warps
    last_end = np.full(int(r["cta"].max()) + 1, -1.0)
    np.maximum.at(last_end, r["cta"], t1)
    first_idle = float(last_end[last_end >= 0].min())
    band = (r["item"] & 15).astype(np.int64)
    cls = np.where(band < 3, 0, np.where(band < 6, 1, 2))
    loaded = t1 <= first_idle
    dur = (t1 - t0) * 1e3   # us
    per_class = {}
    for c, name in enumerate(("n<=16", "n=32", "n=128")):
        sel = (cls == c) & loaded
        per_class[name] = {"items": int(sel.sum()), "mean_us": float(dur[sel].mean()) if sel.any() else None}
    per_band = {}
    for bnd in range(9):
        sel = band == bnd
        if not sel.any():
            continue
        starts = sel & ((r["kind"] == 1) | (r["kind"] == 0))
        per_band[str(bnd)] = {"items": int(sel.sum()), "last_start_ms": float(t0[starts].max()) if starts.any() else None,
                              "last_end_ms": float(t1[sel].max())}
    return {
        "items": int(len(r)), "warps_seen": int((last_end >= 0).sum()), "warps": nwarps,
        "span_ms": span, "first_warp_idle_ms": first_idle, "idle_tail_ms": span - first_idle,
        "idle_tail_frac": (span - first_idle) / span,
        "busy_warps_per_pct": [round(x, 1) for x in busy],
        "items_by_kind": {k: int((r["kind"] == i).sum()) for i, k in enumerate(KINDS)},
        "mean_item_us_loaded": per_class, "per_band": per_band,
    }


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--json", help="write the report here as well")
    ap.add_argument("--ctas-per-sm", type=int, default=0)
    ap.add_argument("--split-free", type=int, default=1)
    ap.add_argument("--runs", type=int, default=3, help="luma stages to run; the last one is reported")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        lib = build_traced(tmp)
        from daala_b200 import _native
        _native.LIB_PATH = lib
        import bench
        from daala_b200 import engine
        from daala_b200.frame import Geometry
        L = _native.lib()
        L.daala_b200_kf_chain_trace.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_void_p),
                                                ctypes.POINTER(ctypes.c_int)]
        geom = Geometry(bench.PIC_W, bench.PIC_H)
        hf = bench.make_host_frames(geom, 16)
        q4 = np.full((3, 30), bench.PVQ_QM_Q4, np.uint8)
        eng = engine.KeyframeEngine(geom, nframes=16, q0=bench.Q0, use_masking=1, pvq_qm_q4=q4,
                                    persist_ctas_per_sm=args.ctas_per_sm, split_free=args.split_free, max_blocks_div=2)
        eng.upload([np.stack([f[0][p] for f in hf]) for p in range(3)], np.stack([f[1] for f in hf]))
        eng.run_device(engine.PH_ALL, graph=False)
        for _ in range(args.runs):
            eng.run_device(engine.PH_PVQ_LUMA | engine.PH_SEARCH_ONLY, graph=False)
        ptr, cap = ctypes.c_void_p(), ctypes.c_int()
        if L.daala_b200_kf_chain_trace(eng.kf, ctypes.byref(ptr), ctypes.byref(cap)) != 0:
            raise RuntimeError("daala_b200_kf_chain_trace failed")
        n = int(eng.download(eng.buf.counts, (256,), np.int32)[TRACE_N])
        if n > cap.value:
            raise RuntimeError("trace overflow: %d items, %d records" % (n, cap.value))
        r = eng.download(ptr.value, (n,), REC)
        import torch
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        rep = analyse(r, sms * (args.ctas_per_sm or 32))
        rep["gpu"] = torch.cuda.get_device_name(0)
        try:
            rep["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                                capture_output=True, text=True).stdout.strip()
        except OSError:
            rep["power_limit"] = None
        eng.close()
    print(json.dumps(rep))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(rep, f, indent=1)


if __name__ == "__main__":
    main()
