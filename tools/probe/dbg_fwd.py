import os, sys, zlib, numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from daala_b200 import synth
from daala_b200.frame import FrameBuffers, Geometry
from tests import frame_oracle, oracle_lib
size=(200,130); mode="mixed"; haar=1
geom = Geometry(*size)
planes, _ = synth.frame(size[0], size[1], f=1)
planes = synth.pad_planes(planes, geom)
bsize = synth.block_size_map(geom, mode, seed=zlib.crc32(repr((mode, size)).encode()) & 0xffff)
lib = oracle_lib.load_port()
for tma in ((False,) if len(sys.argv) > 1 else (True, False)):
    fb = FrameBuffers(geom); fb.haar_dc = haar
    fb.upload(planes, bsize); fb.forward(tma=tma); torch.cuda.synchronize()
    for pli in range(3):
        d_gpu = fb.coeffs[pli][0].cpu().numpy()
        d_cpu = frame_oracle.forward_plane(lib, "port", planes[pli], geom, pli, bsize, haar)
        bad = d_gpu != d_cpu
        print("tma", tma, "plane", pli, "mismatches", int(bad.sum()))
        if bad.any():
            ys, xs = np.nonzero(bad)
            u = sorted(set(zip((ys//4).tolist(), (xs//4).tolist())))
            print(" 4x4 units (y,x):", u[:40], len(u))
            sh = 1 if pli else 0
            for (y,x) in u[:6]:
                print("  unit", y, x, "bsize", bsize[(y*4<<sh)//8, (x*4<<sh)//8])
print(bsize)
