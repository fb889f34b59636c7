#!/usr/bin/env python
"""Keyframe batches with a quantizer per frame (keyframe_quant = 1) against the default keyframe step: bench.py's 16
synthetic 3840x2160 4:2:0 frames with the reference encoder's block-size maps and deringing levels (dering = 1,
max_blocks_div = 2).  Arms, each its own engine, timed in alternating rounds (CUDA events on the
engine's stream, inputs resident in HBM, one graph replay per step):

  default       bench.py's engine: q0 72, flat pvq_qm_q4 16
  uniform       keyframe_quant = 1, every record at bench.py's q0 72 settings
  mixed         keyframe_quant = 1, the 16 frames spread over the eight keyframe settings of
                tests/golden/encoder_settings.npz (HVS matrix, masking on), two frames per point
  hdc_default   the default engine with haar_dc_quant = 1
  hdc_mixed     the mixed arm with haar_dc_quant = 1

Before timing, the uniform arm's outputs (reconstruction, coefficient planes, band records, skip_diff, CfL flips) must
equal the default arm's.  Reported: ms per step of each round per arm, median, min and max; the cost of each mode
against its base arm; the card's name and power limit.  Needs a CUDA device; prints one JSON line.

    python tools/bench_engine_keyframe_quant.py [--rounds 5] [--steps 10]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

ARMS = ("default", "uniform", "mixed", "hdc_default", "hdc_mixed")
OUTPUTS = ("recon0", "recon1", "recon2", "luma_res", "chroma_res", "luma_skip_diff", "chroma_skip_diff", "chroma_flip")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    import numpy as np
    import torch
    import bench
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    if not torch.cuda.is_available():
        sys.exit("bench_engine_keyframe_quant.py needs a CUDA device: nothing is measured without one")
    torch.cuda.init()
    geom = Geometry(bench.PIC_W, bench.PIC_H)
    F = 16
    q4 = np.full((3, 30), bench.PVQ_QM_Q4, np.uint8)
    hf = bench.make_host_frames(geom, F)
    st = np.load(os.path.join(ROOT, "tests", "golden", "encoder_settings.npz"))
    npoints = st["quantizer"].shape[0]
    pts = [f % npoints for f in range(F)]
    mixed = engine.frame_quant_records([int(st["quantizer"][p, 0, 0]) for p in pts],
                                       [int(st["coded_quantizer"][p, 0, 0]) for p in pts],
                                       [float(st["dering_lambda"][p, 0, 0]) for p in pts],
                                       np.stack([st["pvq_qm_q4"][p, 0, 0] for p in pts]))
    uniform = engine.frame_quant_records([bench.Q0] * F, bench.CODED_Q, bench.DERING_LAMBDA, q4)
    records = dict(default=None, uniform=uniform, mixed=mixed, hdc_default=None, hdc_mixed=mixed)
    engines, outs = {}, {}
    for arm in ARMS:
        eng = engine.KeyframeEngine(geom, nframes=F, q0=bench.Q0, use_masking=1, pvq_qm_q4=q4, dering=1,
                                    coded_quantizer=bench.CODED_Q, dering_lambda=bench.DERING_LAMBDA,
                                    max_blocks_div=2, keyframe_quant=int(records[arm] is not None),
                                    haar_dc_quant=int(arm.startswith("hdc")))
        eng.stage_inputs([np.stack([f[0][p] for f in hf]) for p in range(3)], np.stack([f[1] for f in hf]))
        eng.stage_dering_levels(np.stack([f[2] for f in hf]))
        eng.stage_frame_quant(records[arm])
        eng.prepare_io(symbols=True, recon=True)
        eng.submit()
        out = eng.wait()
        assert int(out["counts"][engine.CNT["error"]]) == 0
        outs[arm] = {k: np.array(out[k]) for k in OUTPUTS}
        outs[arm]["coeffs"] = [eng.coeff_plane(p) for p in range(3)]
        eng.time_device(engine.PH_ALL, True, 3)
        engines[arm] = eng
    for k in OUTPUTS:
        assert np.array_equal(outs["uniform"][k], outs["default"][k]), "uniform records: %s differs" % k
    for p in range(3):
        assert np.array_equal(outs["uniform"]["coeffs"][p], outs["default"]["coeffs"][p]), "uniform: coeffs %d" % p
    assert not np.array_equal(outs["mixed"]["recon0"], outs["default"]["recon0"])
    launches = {arm: engines[arm].launches_per_step() for arm in ARMS}
    ms = {arm: [] for arm in ARMS}
    for _ in range(args.rounds):
        for arm in ARMS:
            ms[arm].append(engines[arm].time_device(engine.PH_ALL, True, args.steps) / args.steps)
    for eng in engines.values():
        eng.close()
    med = {arm: statistics.median(v) for arm, v in ms.items()}

    def cost(a, b):
        return round(100 * (med[a] - med[b]) / med[b], 2)

    res = dict(gpu=bench.gpu_identity(torch.cuda.current_device()), frames=F,
               size="%dx%d" % (bench.PIC_W, bench.PIC_H), mixed_q0=[int(v) for v in mixed["q0"]],
               uniform_equals_default=True, launches_per_step=launches,
               ms_per_step={arm: [round(v, 3) for v in ms[arm]] for arm in ARMS},
               median={arm: round(med[arm], 3) for arm in ARMS},
               spread={arm: [round(min(ms[arm]), 3), round(max(ms[arm]), 3)] for arm in ARMS},
               cost_pct=dict(uniform=cost("uniform", "default"), mixed=cost("mixed", "default"),
                             hdc_mixed=cost("hdc_mixed", "hdc_default")))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
