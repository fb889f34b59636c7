"""Y4M in -> keyframe engine (GPU) -> reconstructed Y4M out + symbol statistics: the data path of
`encoder_example -v <quant> -k 1` (all-intra) without the entropy coder.  Needs an H100.

  python tools/encode_y4m.py in.y4m recon.y4m [--q0 72] [--batch 16] [--bsize 3] [--dering 2] [--symbols DIR]
                            [--haar-dc]

The engine runs with its symbol stream (daala_b200/symbols.py): per frame, in bitstream order, the block records,
band records and 8/16-bit pulses a host entropy coder reads; the statistics come from it, and --symbols DIR writes
each frame's part as DIR/frame_NNNNNN.npz (blocks, bands, pulses).  --haar-dc quantises the keyframe DCs as the
reference does (haar_dc_quant = 1), so the reconstruction is the one a decoder makes, and adds each frame's DC records
(hdc, symbols.HDC_DTYPE: one per block record, in coding order) to the stream and to the --symbols files.

Block sizes: a uniform map (--bsize: 0..3 = 4x4..32x32) -- the block-size RDO is the reference encoder's; maps it
decided can be passed with --bsize-npz (an array [frames, nvsb*8, nhsb*8])."""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from daala_b200 import engine, symbols, synth, y4m  # noqa: E402
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
    ap.add_argument("--symbols", default=None, help="directory for one symbol stream file per frame")
    ap.add_argument("--haar-dc", action="store_true", help="quantise the keyframe DCs (haar_dc_quant = 1) and stream "
                    "their records")
    args = ap.parse_args()
    hdr, frames = y4m.read_frames(args.src, args.max_frames)
    if not frames:
        raise SystemExit("no frames in %s" % args.src)
    geom = Geometry(hdr["width"], hdr["height"])
    maps = np.load(args.bsize_npz) if args.bsize_npz else None
    F = min(args.batch, len(frames))
    q4 = np.full((3, 30), 16, np.uint8)
    eng = engine.KeyframeEngine(geom, nframes=F, q0=args.q0, pvq_qm_q4=q4, dering=args.dering,
                                coded_quantizer=args.coded_quantizer, symbol_stream=1,
                                haar_dc_quant=int(args.haar_dc))
    if args.symbols:
        os.makedirs(args.symbols, exist_ok=True)
    out_frames, pulses, blocks, nonzero, sym_bytes = [], 0, 0, 0, 0
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
        out = eng.encode(planes, bs, symbols=False, stream=True, dc_grids=False)
        for k in range(n):
            out_frames.append([out["recon%d" % p][k][:(hdr["height"] + (p > 0)) >> (p > 0),
                                                     :(hdr["width"] + (p > 0)) >> (p > 0)].copy() for p in range(3)])
        for k in range(n):
            fr = symbols.read_frame(out, k)
            blocks += len(fr["blocks"])
            pulses += int(fr["bands"][:, 3].clip(min=0).sum())
            nonzero += sum(int(np.count_nonzero(v)) for v in fr["pulses"])
            b0, nb, n0, nn, y0, ny = (int(v) for v in out["sym_index"][k])
            sym_bytes += nb * symbols.BLOCK_DTYPE.itemsize + nn * 8 + ny
            extra = {}
            if args.haar_dc:
                sym_bytes += nb * symbols.HDC_DTYPE.itemsize
                extra["hdc"] = fr["hdc"]
            if args.symbols:
                np.savez(os.path.join(args.symbols, "frame_%06d.npz" % (i + k)), blocks=fr["blocks"],
                         bands=fr["bands"], pulses=out["sym_pulses"][y0:y0 + ny], **extra)
    eng.close()
    y4m.write_frames(args.dst, out_frames, fps=hdr["fps"], aspect=hdr["aspect"], chroma=hdr["chroma"])
    mse = np.mean([(a[0].astype(np.float64) - b[0]) ** 2 for a, b in zip(frames, out_frames)])
    print("%d frames %dx%d, %d blocks, %d pulses (sum of K), %d non-zero pulse values, %d symbol stream bytes, "
          "luma PSNR %.2f dB -> %s" % (len(out_frames), hdr["width"], hdr["height"], blocks, pulses, nonzero, sym_bytes,
                                      10 * np.log10(255.0 ** 2 / max(mse, 1e-12)), args.dst))


if __name__ == "__main__":
    main()
