#!/usr/bin/env python
"""Reference pictures kept on the device (inter_mc with inter_finish: finish_io.ref_slot_out, io.ref_resident) against
the host round trip, on bench_engine_inter_finish.py's workload: 16 synthetic 3840x2160 4:2:0 frames, the shipped
block-size maps and deringing levels, q0 72.  The 16 frames of a step are 16 independent sequences in a pool of
mc_refs = 32 pictures: slot f holds sequence f's GOLD picture and slot 16 + f its PREV picture.  Every step codes the
same source frames with seeded MV grids (synth.mv_grid, GOLD / PREV mixed per vertex) and applies seeded decisions
(30 % of the blocks skipped with DC 0, the others keep the first step's qdc) in the finishing pass, whose
reconstruction becomes each sequence's next PREV picture.

Two loops of steps (submit, wait for the step's outputs, finish), run alternately in one process:
  round_trip         the finish copies its reconstruction to the host, straight into the pinned host pool's PREV
                     slots, and the next submit uploads the whole 32-picture pool;
  resident           the submit reads the pool on the device (ref_resident), the finish stores its reconstruction
                     into slots 16..31 (ref_slot_out) and still copies it to the host (pixels_out);
  resident_no_recon  the same without pixels_out.
These three request the same step outputs (block records, band records, pulses, DC indices, the prediction) and no
skip maps or levels from the finish.  Two more loops copy neither the reconstruction nor the prediction, so that the
difference between them is the P-frame symbol stream's alone:
  classic_no_pred    resident_no_recon without the prediction planes (prepare_io(pred=False));
  stream             an engine with symbol_stream = 2: the step returns only the stream (index, block, band, pulse and
                     DC records, the used part of each) and the finish takes the same decisions in stream order
                     (finish_io.stream_skip / stream_dc).  Before timing: after 3 steps the round trip's and the resident loop's outputs
and pools must be identical, and, when oracle/_ref was built, frame 0 of the first step is checked against the oracle
(prediction against od_state_mc_predict, reconstruction against inverse_frame_inter_finish).  The stream loop's first
step must equal symbols.pack_reference of the resident loop's classic outputs of the same step, and after 3 steps its
pool must equal the resident loop's.

Reports per-step wall time (host clock around --steps steps ending in a stream synchronise, --rounds rounds), the H2D
and D2H bytes of a step, the device time of the step graph with symbol_stream 0 and 2 (CUDA events around --steps graph
replays, --rounds alternating rounds: their difference is the stream kernels' cost), and the card's name and power
limit.  --profile: a run of its own that times
k_fin_pool_store with torch.profiler over --steps resident steps and sets its bytes (read + write of every stored
plane) against the 3.35 TB/s of the H100 SXM data sheet.  Needs a CUDA device; prints one JSON line.

    python tools/bench_engine_pool.py [--rounds 3] [--steps 5] [--frames 16] [--profile]
"""
import argparse
import ctypes
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


class Loop:
    """One engine and the C records of one loop: a submit record (resident or uploading the host pool) and a finish
    record (storing into the pool slots, or copying the reconstruction into the host pool's PREV slots)."""

    def __init__(self, eng, geom, F, planes, bsize, slot, packed, pool, mode):
        import numpy as np
        self.eng, self.F, self.mode = eng, F, mode
        eng.stage_inputs(planes, bsize)
        resident = mode != "round_trip"
        eng.stage_mc(None if resident else pool, slot, packed, resident=resident)
        lean = mode in ("classic_no_pred", "stream")
        self.out = eng.prepare_io(symbols=mode != "stream", recon=False, pred=not lean)
        self.io = eng._io
        self.h2d, self.d2h = eng.h2d_bytes, eng.d2h_bytes
        self.px = [int(np.prod(geom.plane_shape(p))) for p in range(3)]
        # the host pool of the round trip is the engine's pinned upload buffer itself
        self.host_pool = [eng._arr("ref%d" % p, (2 * F,) + geom.plane_shape(p), np.uint8) for p in range(3)] \
            if not resident else None

    def set_decisions(self, dec):
        import numpy as np
        from daala_b200 import engine
        eng, F = self.eng, self.F
        store = None if self.mode == "round_trip" else np.arange(F, 2 * F, dtype=np.int32)
        if self.mode == "stream":   # dec: (skip, dc, levels) in stream order
            eng.prepare_finish_stream(*dec, ref_slot_out=store)
        else:
            eng.prepare_finish(*dec, ref_slot_out=store)
        fio = engine.FinishIO.from_buffer_copy(eng._fio)
        for p in range(3):
            fio.bskip_out[p] = None
            if self.mode == "round_trip":
                fio.pixels_out[p] = self.host_pool[p].ctypes.data + F * self.px[p]
            elif self.mode != "resident":
                fio.pixels_out[p] = None
        fio.dering_level_out = None
        self.fio = fio
        self.recon = [eng._fout["recon%d" % p] for p in range(3)] if self.mode == "resident" else None
        self.finish_h2d = eng.finish_h2d_bytes
        self.finish_d2h = sum(self.px) * F if self.mode in ("round_trip", "resident") else 0

    def step(self):
        eng = self.eng
        eng._check(eng.L.daala_b200_kf_submit(eng.kf, ctypes.byref(self.io)), "kf_submit")
        eng.wait()   # the host coder reads the step's outputs before it decides
        eng._check(eng.L.daala_b200_kf_finish(eng.kf, ctypes.byref(self.fio)), "kf_finish")

    def timed(self, steps):
        self.eng.wait()
        t0 = time.perf_counter()
        for _ in range(steps):
            self.step()
        self.eng.wait()
        return (time.perf_counter() - t0) * 1e3 / steps

    def pool(self):
        import numpy as np
        if self.host_pool is not None:
            self.eng.wait()
            return [np.array(a) for a in self.host_pool]
        return [self.eng.pool_plane(p) for p in range(3)]


def oracle_check(geom, loop, gold, prev, grid, bsize, q4, dec, q0):
    """Frame 0 of the first step against the oracle; None when oracle/_ref is missing, else the mismatch count."""
    import numpy as np
    from daala_b200 import interfinish
    from tests import inter_finish_oracle, inter_mc_oracle
    ref = inter_mc_oracle.load()
    fin = inter_finish_oracle.load_ref()
    if ref is None or fin is None:
        return None
    eng, out = loop.eng, loop.out
    want = inter_mc_oracle.predict(ref, geom, gold, prev, *grid)
    mism = sum(int(np.count_nonzero(out["pred%d" % p][0] != want[p])) for p in range(3))
    dq, bskip = [], []
    for p in range(3):
        blocks, skip, dc = (out["luma_blocks"], dec[0], dec[1]) if p == 0 else (out["chroma_blocks"], dec[2], dec[3])
        dq.append(interfinish.patch(eng.coeff_plane(p)[0], eng.pred_coeff_plane(p)[0], blocks, skip, dc, 0, p, q0, q4))
        bskip.append(interfinish.skip_map(blocks, skip, dc, 0, p, geom))
    recs, _ = inter_finish_oracle.finish(fin, "ref", dq, geom, bsize[0], q0, dec[4][0], bskip)
    got = [loop.pool()[p][loop.F] for p in range(3)]   # sequence 0's new PREV picture
    return mism + sum(int(np.count_nonzero(got[p] != recs[p])) for p in range(3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5, help="steps per round and loop")
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--profile", action="store_true", help="only the torch.profiler run of k_fin_pool_store")
    args = ap.parse_args()
    import numpy as np
    import bench
    from daala_b200 import _native, engine, mvgrid, symbols, synth
    from daala_b200.frame import Geometry
    if _native.lib().daala_b200_device_count() < 1:
        sys.exit("bench_engine_pool.py needs a CUDA device: nothing is measured without one")

    geom = Geometry(bench.PIC_W, bench.PIC_H)
    F = args.frames
    q4 = np.full((3, 30), bench.PVQ_QM_Q4, np.uint8)
    hf = bench.make_host_frames(geom, F)
    planes = [np.stack([f[0][p] for f in hf]) for p in range(3)]
    bsize = np.stack([f[1] for f in hf])
    levels = np.stack([f[2] for f in hf])
    # sequence f: GOLD = synthetic frame f - 1, PREV at the start = frame f - 2
    pool0 = [np.concatenate([np.roll(planes[p], 1, axis=0), np.roll(planes[p], 2, axis=0)]) for p in range(3)]
    slot = np.array([[f, F + f] for f in range(F)], np.int32)
    grids = [synth.mv_grid(geom, seed=2000 + f) for f in range(F)]
    packed = mvgrid.pack(*(np.stack([g[i] for g in grids]) for i in range(3)))
    common = dict(nframes=F, q0=bench.Q0, use_masking=1, pvq_qm_q4=q4, max_blocks_div=2, inter=1, inter_mc=1,
                  mc_refs=2 * F, inter_finish=1)

    res_eng = engine.KeyframeEngine(geom, **common)
    for s in range(2 * F):
        res_eng.pool_load(s, [pool0[p][s] for p in range(3)])
    res = Loop(res_eng, geom, F, planes, bsize, slot, packed, None, "resident")
    # decisions from the first step's outputs (the same block lists every step: the maps do not change)
    res_eng._check(res_eng.L.daala_b200_kf_submit(res_eng.kf, ctypes.byref(res.io)), "kf_submit")
    out = res_eng.wait()
    if int(out["counts"][engine.CNT["error"]]) or int(out["counts"][engine.CNT["mc_bad_ref"]]) or \
            int(out["counts"][engine.CNT["mc_beyond"]]):
        sys.exit("bench_engine_pool.py: the step left the engine's capacity or the reference's MV definition")
    rng = np.random.default_rng(30)
    ls = (rng.random(len(out["luma_dc"])) < 0.3).astype(np.uint8)
    cs = (rng.random(len(out["chroma_dc"])) < 0.3).astype(np.uint8)
    dec = (ls, np.where(ls == 1, 0, out["luma_dc"]).astype(np.int32), cs,
           np.where(cs == 1, 0, out["chroma_dc"]).astype(np.int32), levels)
    res.set_decisions(dec)

    if args.profile:
        import torch
        from torch.profiler import ProfilerActivity, profile
        res_eng._check(res_eng.L.daala_b200_kf_finish(res_eng.kf, ctypes.byref(res.fio)), "kf_finish")
        res.timed(1)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            res.timed(args.steps)
            torch.cuda.synchronize()
        ms = {}
        for e in prof.key_averages():
            for tag in ("k_fin_pool_store", "k_fin_patch", "k_dering_sb"):
                if tag in e.key:
                    ms[tag] = ms.get(tag, 0.0) + e.device_time_total / 1e3 / args.steps   # ms per step
        alg = 2 * F * sum(res.px)   # every plane of every frame read once and written once
        line = {"profile": "torch.profiler, %d resident steps" % args.steps, "gpu": bench.gpu_identity(0),
                "kernel_ms_per_step": {k: round(v, 4) for k, v in ms.items()}, "pool_store_bytes": alg}
        if ms.get("k_fin_pool_store"):
            t = ms["k_fin_pool_store"] * 1e-3
            line["pool_store_gb_per_s"] = round(alg / t / 1e9, 1)
            line["pool_store_share_of_3_35_tb_per_s"] = round(alg / HBM_BYTES_PER_S / t, 4)
        res_eng.close()
        print(json.dumps(line), flush=True)
        return

    # the first step again from the same pool, now with its decisions, so that both loops start alike
    for s in range(2 * F):
        res_eng.pool_load(s, [pool0[p][s] for p in range(3)])
    trip_eng = engine.KeyframeEngine(geom, **common)
    trip = Loop(trip_eng, geom, F, planes, bsize, slot, packed, pool0, "round_trip")
    trip.set_decisions(dec)
    bare = Loop(res_eng, geom, F, planes, bsize, slot, packed, None, "resident_no_recon")
    bare.set_decisions(dec)
    lean = Loop(res_eng, geom, F, planes, bsize, slot, packed, None, "classic_no_pred")
    lean.set_decisions(dec)
    # the stream loop: its own engine and pool; a first submit gives the stream order the decisions are permuted into
    st_eng = engine.KeyframeEngine(geom, symbol_stream=2, **common)
    for s in range(2 * F):
        st_eng.pool_load(s, [pool0[p][s] for p in range(3)])
    stream = Loop(st_eng, geom, F, planes, bsize, slot, packed, None, "stream")
    st_eng._check(st_eng.L.daala_b200_kf_submit(st_eng.kf, ctypes.byref(stream.io)), "kf_submit")
    sout = st_eng.wait()
    perm = symbols.stream_to_classic(dict(out, sym_index=np.array(sout["sym_index"]), sym_blocks=np.array(sout["sym_blocks"])))
    stream.set_decisions((np.concatenate([dec[0], dec[2]])[perm], np.concatenate([dec[1], dec[3]])[perm], dec[4]))

    # parity: frame 0 of the first step against the oracle, then 3 steps of both loops equal
    res.step()
    trip.step()
    stream.step()
    res_eng.wait()
    st_eng.wait()
    bad = symbols.stream_equal(stream.out, symbols.pack_reference(res.out, F), range(F))
    if bad:
        sys.exit("bench_engine_pool.py: the stream differs from the classic outputs of the same step: %s" % (bad[:4],))
    mism = oracle_check(geom, res, [pool0[p][0] for p in range(3)], [pool0[p][F] for p in range(3)], grids[0], bsize,
                        q4, dec, bench.Q0)
    if mism:
        sys.exit("bench_engine_pool.py: frame 0 of the first step differs from the oracle (%d mismatches)" % mism)
    for _ in range(2):
        res.step()
        trip.step()
        stream.step()
    res_eng.wait()
    trip_eng.wait()
    diff = 0
    for k in res.out:
        a, b = np.asarray(res.out[k]), np.asarray(trip.out[k])
        if k in ("luma_res", "chroma_res"):
            continue   # records past a block's last band are not written; the block records and pulses cover them
        diff += int(np.count_nonzero((a != b) & ~(np.isnan(a) & np.isnan(b)) if a.dtype.kind == "f" else a != b))
    rp, tp = res.pool(), trip.pool()
    diff += sum(int(np.count_nonzero(rp[p] != tp[p])) for p in range(3))
    diff += sum(int(np.count_nonzero(res.recon[p] != tp[p][F:])) for p in range(3))
    sp = stream.pool()
    diff += sum(int(np.count_nonzero(rp[p] != sp[p])) for p in range(3))
    if diff:
        sys.exit("bench_engine_pool.py: after 3 steps the resident and stream loops differ from the round trip (%d values)"
                 % diff)
    stream.d2h += st_eng.stream_d2h_bytes()   # the used part of the stream arrays (the same every step)

    loops = {"round_trip": trip, "resident": res, "resident_no_recon": bare, "classic_no_pred": lean, "stream": stream}
    for lp in loops.values():
        lp.timed(1)
    rounds = {name: [] for name in loops}
    for _ in range(args.rounds):
        for name, lp in loops.items():
            rounds[name].append(lp.timed(args.steps))
    # the step graph alone, symbol_stream 0 against 2, on the same inputs and pool
    graph = {"symbol_stream_0": [], "symbol_stream_2": []}
    for e in (res_eng, st_eng):
        e.time_device(engine.PH_ALL, True, 1)
    for _ in range(args.rounds):
        graph["symbol_stream_0"].append(res_eng.time_device(engine.PH_ALL, True, args.steps) / args.steps)
        graph["symbol_stream_2"].append(st_eng.time_device(engine.PH_ALL, True, args.steps) / args.steps)
    line = {"workload": "%d independent sequences of synthetic 3840x2160 4:2:0 frames, shipped block-size maps and "
                        "deringing levels, q0 %d, mc_refs %d (GOLD slot f, PREV slot %d + f), seeded MV grids, 30 %% of "
                        "the blocks skipped with DC 0; a step = submit, wait, finish" % (F, bench.Q0, 2 * F, F),
            "gpu": bench.gpu_identity(0), "steps_per_round": args.steps, "rounds": args.rounds,
            "parity_checked": ("frame 0 of the first step against od_state_mc_predict and inverse_frame_inter_finish "
                               "(reference build)" if mism is not None else "oracle/_ref not built: frame 0 not checked")
                              + "; 3 steps of the round trip and the resident loop: outputs and pools identical; the "
                                "stream loop's first stream equals pack_reference of the resident loop's outputs, its "
                                "pool after 3 steps the resident loop's"}
    for name, lp in loops.items():
        line[name] = {"ms_per_step": round(statistics.median(rounds[name]), 3),
                      "ms_per_step_rounds": [round(v, 3) for v in rounds[name]],
                      "h2d_bytes_per_step": int(lp.h2d + lp.finish_h2d),
                      "d2h_bytes_per_step": int(lp.d2h + lp.finish_d2h)}
    line["h2d_saved_bytes_per_step"] = line["round_trip"]["h2d_bytes_per_step"] - line["resident"]["h2d_bytes_per_step"]
    line["stream_d2h_saved_bytes_per_step"] = (line["classic_no_pred"]["d2h_bytes_per_step"]
                                               - line["stream"]["d2h_bytes_per_step"])
    line["step_graph_ms"] = {k: {"median": round(statistics.median(v), 3), "rounds": [round(x, 3) for x in v]}
                             for k, v in graph.items()}
    line["stream_kernels_ms_per_step"] = round(statistics.median(graph["symbol_stream_2"])
                                               - statistics.median(graph["symbol_stream_0"]), 3)
    trip_eng.close()
    res_eng.close()
    st_eng.close()
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
