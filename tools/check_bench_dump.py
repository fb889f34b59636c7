"""Checks what `bench.py --dump-outputs DIR` wrote against the oracle.

bench.py checks one frame before it times anything; its dump holds a seeded sample of what the LAST timed step
left on the device for all frames of the batch.  This script rebuilds that batch (bench.make_host_frames, first
engine, default options: reference block sizes and deringing levels, q0 72), runs the oracle once per distinct
frame (the reference build when oracle/_ref is present, else the plain-C port), lays the oracle's results out as
the full arrays bench.dump_outputs samples -- planes [F, h, w], per-band results [blocks, 9, 4] in (frame, plane,
y, x) block order -- takes the same positions with bench._sample and the same seeds, and counts the values that
differ.  Band slots a block does not have (bands >= its band count) are not outputs and are not compared.

Prints one JSON line with the mismatches per array; exits 1 if there are any.

    python tools/check_bench_dump.py DIR [--frames 16]
"""
import argparse
import json
import multiprocessing
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402
from tests import frame_oracle, oracle_lib  # noqa: E402

_JOB = {}


def _oracle():
    ref = oracle_lib.load_ref()
    return (ref, "ref") if ref is not None else (oracle_lib.load_port(), "port")


def _run(k):
    lib, prefix = _oracle()
    planes, bsize, levels = _JOB["frames"][k]
    q4 = np.full((3, 30), bench.PVQ_QM_Q4, np.uint8)
    out = frame_oracle.keyframe_chain(lib, prefix, planes, _JOB["geom"], bsize, bench.Q0, q4, use_masking=1,
                                      dering_levels=levels if bench.DERING == 1 else None)
    return [dict(recon=o["recon"], dq=o["dq"], rec=o["rec"]) for o in out]


def expected(geom, nframes, workers):
    """The full arrays bench.dump_outputs samples, from the oracle; band results with a mask of the used slots."""
    distinct = bench.make_host_frames(geom, 4, distinct=4)
    _JOB.update(geom=geom, frames=distinct)
    if workers > 1:
        with multiprocessing.get_context("fork").Pool(min(workers, len(distinct))) as pool:
            want = pool.map(_run, range(len(distinct)), chunksize=1)
    else:
        want = [_run(k) for k in range(len(distinct))]
    # batch frame i holds distinct frame i % 4 (make_host_frames, rotation 0 = the first engine)
    frame_of = [i % len(distinct) for i in range(nframes)]
    full = {}
    for p in range(3):
        full["recon%d" % p] = np.stack([want[k][p]["recon"] for k in frame_of])
        full["coeffs%d" % p] = np.stack([want[k][p]["dq"] for k in frame_of])
    for name, planes in (("luma", (0,)), ("chroma", (1, 2))):
        res = []
        for k in frame_of:
            for p in planes:
                rec = want[k][p]["rec"]
                origin = rec[:, :, 0, 0] != -32768           # band 0 exists in every block: the block origins
                res.append(rec[origin])                          # row-major = sorted by (y0, x0)
        res = np.concatenate(res)
        full[name + "_band_results"] = (res, np.broadcast_to((res[:, :, :1] != -32768), res.shape))
    return full


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("dir", help="the --dump-outputs directory of a bench.py run")
    ap.add_argument("--frames", type=int, default=16, help="bench.py --frames of that run")
    args = ap.parse_args()
    from daala_b200.frame import Geometry
    geom = Geometry(bench.PIC_W, bench.PIC_H)
    _, prefix = _oracle()
    full = expected(geom, args.frames, bench.usable_cores()[0])
    seeds = {"recon%d" % p: (10 + p, np.float32) for p in range(3)}
    seeds.update({"coeffs%d" % p: (20 + p, np.float64) for p in range(3)})
    seeds.update(luma_band_results=(30, np.float32), chroma_band_results=(31, np.float32))
    report = {"against": prefix, "frames": args.frames, "mismatches": {}, "compared": {}}
    total = 0
    for name, (seed, dtype) in seeds.items():
        got = np.load(os.path.join(args.dir, name + ".npy"))
        want = full[name]
        used = None
        if isinstance(want, tuple):
            want, used = want
            used = bench._sample(np.ascontiguousarray(used), seed)
        want = bench._sample(want, seed).astype(dtype)
        if got.shape != want.shape:
            report["mismatches"][name] = "shape %s, expected %s" % (got.shape, want.shape)
            total += 1
            continue
        diff = got != want
        if used is not None:
            diff &= used
        n = int(diff.sum())
        report["mismatches"][name] = n
        report["compared"][name] = int(got.size if used is None else used.sum())
        total += n
    report["total_mismatches"] = total
    print(json.dumps(report))
    sys.exit(1 if total else 0)


if __name__ == "__main__":
    main()
