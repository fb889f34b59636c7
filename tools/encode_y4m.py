"""Y4M in -> keyframe engine (GPU) -> reconstructed Y4M out + symbol statistics: the data path of
`encoder_example -v <quant> -k 1` (all-intra) without the entropy coder.  Needs an H100.

  python tools/encode_y4m.py in.y4m recon.y4m [--q0 72] [--batch 16] [--bsize 3] [--dering 2]

Block sizes: a uniform map (--bsize: 0..3 = 4x4..32x32) -- the block-size RDO is the reference encoder's; maps it
decided can be passed with --bsize-npz (an array [frames, nvsb*8, nhsb*8])."""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from daala_b200 import engine, synth, y4m          # noqa: E402
from daala_b200.frame import Geometry              # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("src")
    ap.add_argument("dst")
    ap.add_argument("--q0", type=int, default=72, help="state->quantizer")
    ap.add_argument("--coded-quantizer", type=int, default=20)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--bsize", type=int, default=3)
    ap.add_argument("--bsize-npz", default=None)
    ap.add_argument("--dering", type=int, default=2, help="0 off, 2 = search + apply")
    ap.add_argument("--max-frames", type=int, default=None)
    args = ap.parse_args()
    hdr, frames = y4m.read_frames(args.src, args.max_frames)
    if not frames:
        raise SystemExit("no frames in %s" % args.src)
    geom = Geometry(hdr["width"], hdr["height"])
    maps = np.load(args.bsize_npz) if args.bsize_npz else None
    F = min(args.batch, len(frames))
    q4 = np.full((3, 30), 16, np.uint8)
    eng = engine.KeyframeEngine(geom, nframes=F, q0=args.q0, pvq_qm_q4=q4, split_free=1, dering=args.dering,
                                coded_quantizer=args.coded_quantizer)
    out_frames, pulses, blocks = [], 0, 0
    for i in range(0, len(frames), F):
        chunk = frames[i:i + F]
        n = len(chunk)
        chunk = chunk + [chunk[-1]] * (F - n)                    # the engine's batch size is fixed
        padded = [synth.pad_planes(pl, geom) for pl in chunk]
        planes = [np.stack([f[p] for f in padded]) for p in range(3)]
        if maps is not None:
            bs = np.stack([maps[min(i + k, len(maps) - 1)] for k in range(F)]).astype(np.uint8)
        else:
            bs = np.full((F,) + tuple(geom.bsize_shape), args.bsize, np.uint8)
        out = eng.encode(planes, bs)
        for k in range(n):
            out_frames.append([out["recon%d" % p][k][:(hdr["height"] + (p > 0)) >> (p > 0),
                                                     :(hdr["width"] + (p > 0)) >> (p > 0)].copy() for p in range(3)])
        pulses += int(out["luma_res"][..., 3].clip(min=0).sum()) + int(out["chroma_res"][..., 3].clip(min=0).sum())
        blocks += int(eng.totals.n_luma) + int(eng.totals.n_chroma)
    eng.close()
    y4m.write_frames(args.dst, out_frames, fps=hdr["fps"], aspect=hdr["aspect"], chroma=hdr["chroma"])
    mse = np.mean([(a[0].astype(np.float64) - b[0]) ** 2 for a, b in zip(frames, out_frames)])
    print("%d frames %dx%d, %d blocks, %d pulses, luma PSNR %.2f dB -> %s" % (
        len(out_frames), hdr["width"], hdr["height"], blocks, pulses, 10 * np.log10(255.0 ** 2 / max(mse, 1e-12)), args.dst))


if __name__ == "__main__":
    main()
