#!/usr/bin/env python
"""Throughput of the motion-compensation / motion-estimation kernels on a 1080p inter-frame workload
(BASELINE.json config 3's building blocks; not the headline bench): whole-frame OBMC prediction from a random
MV grid (od_state_mc_predict = k_obmc_blocks per plane), the OBMC-based cost of every MV-grid block
(od_mv_est_calc_sads' inner operation = daala_b200_mv_est_sad), and half-pel BMA candidate costs
(od_mv_est_bma_sad = daala_b200_mv_bma_sad, 9 candidates around every 16x16 block).  Prints one JSON line with
times (CUDA events), rates and the fraction of the measured copy bandwidth the algorithmic bytes of SURVEY.md
8(d) (K_obmc, K_sad) correspond to."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from daala_b200 import mc, mvgrid, synth          # noqa: E402
from daala_b200.frame import Geometry              # noqa: E402


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    pic_w, pic_h, reps = 1920, 1080, 20
    geom = Geometry(pic_w, pic_h)
    W, H = geom.frame_w, geom.frame_h
    cur, _ = synth.frame(pic_w, pic_h, f=1)
    prev, _ = synth.frame(pic_w, pic_h, f=0)
    cur, prev = synth.pad_planes(cur, geom), synth.pad_planes(prev, geom)
    rng = np.random.default_rng(5)
    nv, nh = H // 8, W // 8
    valid, mv = random_mv_grid(rng, nv, nh)
    vx, vy, l, oc, s = mvgrid.leaves(valid)
    dev_cur = [torch.from_numpy(c).cuda() for c in cur]
    refs = [mc.PaddedPlane(prev[p], pad=mc.OD_BUFFER_PADDING >> (1 if p else 0)) for p in range(3)]
    dsts = [torch.zeros_like(c) for c in dev_cur]
    blocks = [mvgrid.blocks_for(vx, vy, l, oc, s, mv, xdec=1 if p else 0) for p in range(3)]
    dblocks = [mc.to_device(b) for b in blocks]
    nblk = len(vx)

    def obmc():
        for p in range(3):
            mc.predict_blocks(refs[p], dsts[p], dblocks[p], nblk)
    ms_obmc = timed(obmc, reps)
    # K_obmc: <= 4 (n+5)^2 read + n^2 written per block and plane
    n = (8 << l).astype(np.int64)
    bytes_obmc = int(sum(((4 * ((n >> d) + 5) ** 2 + (n >> d) ** 2).sum()) for d in (0, 1, 1)))

    b3 = np.ascontiguousarray(np.stack(blocks, axis=1))
    d_b3 = mc.to_device(b3)
    out = torch.empty(nblk, dtype=torch.int32, device="cuda")
    ms_est = timed(lambda: mc.est_sad(dev_cur, refs, pic_w, pic_h, d_b3, nblk, out=out), reps)
    bytes_est = bytes_obmc + int(sum((((n >> d) ** 2).sum()) for d in (0, 1, 1)))   # + the current block

    # BMA: 9 half-pel candidates around every 16x16 block
    gx, gy = np.meshgrid(np.arange(0, pic_w, 16), np.arange(0, pic_h, 16))
    cand = [(dx, dy) for dy in (-1, 0, 1) for dx in (-1, 0, 1)]
    jobs = np.zeros(gx.size * 9, mc.BMA_JOB_DTYPE)
    jobs["bx"] = np.repeat(gx.ravel(), 9)
    jobs["by"] = np.repeat(gy.ravel(), 9)
    base = rng.integers(-40, 41, size=(gx.size, 2))
    jobs["mvx"] = (np.repeat(base[:, 0], 9) + np.tile([c[0] for c in cand], gx.size))
    jobs["mvy"] = (np.repeat(base[:, 1], 9) + np.tile([c[1] for c in cand], gx.size))
    jobs["log_mvb_sz"] = 1
    d_jobs = mc.to_device(jobs)
    out2 = torch.empty(len(jobs), dtype=torch.int32, device="cuda")
    ms_bma = timed(lambda: mc.bma_sad(dev_cur, refs, pic_w, pic_h, d_jobs, len(jobs), out=out2), reps)
    bytes_bma = len(jobs) * sum(2 * m * m + (m + 5) ** 2 for m in (16, 8, 8))      # K_sad with fused interpolation

    peak = 3350.0    # GB/s, H100 SXM data sheet (HBM3); not a measured peak
    px = pic_w * pic_h
    print(json.dumps({
        "workload": "1920x1080 4:2:0 inter-frame building blocks, random MV grid (%d OBMC blocks: %s per level 8..64)" % (
            nblk, np.bincount(l, minlength=4).tolist()),
        "obmc_frame": {"ms": round(ms_obmc, 4), "mpixels_per_s": round(px / ms_obmc / 1e3, 1),
                       "algorithmic_gbs": round(bytes_obmc / ms_obmc / 1e6, 1), "frac_of_copy_peak": round(bytes_obmc / ms_obmc / 1e6 / peak, 4)},
        "mv_est_sad_all_blocks": {"ms": round(ms_est, 4), "blocks_per_s": round(nblk / ms_est * 1e3),
                                  "algorithmic_gbs": round(bytes_est / ms_est / 1e6, 1),
                                  "frac_of_copy_peak": round(bytes_est / ms_est / 1e6 / peak, 4)},
        "bma_sad_9_candidates_per_16x16": {"ms": round(ms_bma, 4), "candidates_per_s": round(len(jobs) / ms_bma * 1e3),
                                           "algorithmic_gbs": round(bytes_bma / ms_bma / 1e6, 1),
                                           "frac_of_copy_peak": round(bytes_bma / ms_bma / 1e6 / peak, 4)},
        "peak_gbs": peak}))


def random_mv_grid(rng, nv, nh, max_mv=96):
    """Hierarchically consistent validity flags (a vertex is valid only inside a split block) + random MVs in
    1/8 pel, partly full-pel and partly shared between neighbours."""
    valid = np.zeros((nv + 1, nh + 1), bool)
    valid[::8, ::8] = True

    def split(vx, vy, l):
        if l == 0:
            return
        h = (1 << l) >> 1
        if rng.random() < 0.6:
            valid[vy + h, vx + h] = True
            for dx, dy in ((h, 0), (0, h), (2 * h, h), (h, 2 * h)):
                if rng.random() < 0.7:
                    valid[vy + dy, vx + dx] = True
            for dx, dy in ((0, 0), (h, 0), (0, h), (h, h)):
                split(vx + dx, vy + dy, l - 1)

    for vy in range(0, nv, 8):
        for vx in range(0, nh, 8):
            split(vx, vy, 3)
    mv = rng.integers(-max_mv, max_mv + 1, size=(nv + 1, nh + 1, 2)).astype(np.int32)
    mv[::2, ::2] = (mv[::2, ::2] // 8) * 8
    return valid, mv


if __name__ == "__main__":
    main()
