#!/bin/bash
# tiny end-to-end run of tools/encode_y4m.py on an H100 (synthetic 3-frame 200x130 clip)
set -e
python - <<'PY'
import sys; sys.path.insert(0, '.')
from daala_b200 import synth, y4m
frames, seed = [], 1
for f in range(3):
    planes, seed = synth.frame(200, 130, f=f, seed=seed)
    frames.append(planes)
y4m.write_frames('gpurun_out/y4m_in.y4m', frames)
PY
python tools/encode_y4m.py gpurun_out/y4m_in.y4m gpurun_out/y4m_out.y4m --batch 2 --dering 2 --bsize 2
python tools/encode_y4m.py gpurun_out/y4m_in.y4m gpurun_out/y4m_out0.y4m --batch 3 --dering 0 --bsize 1 --q0 38
ls -la gpurun_out/y4m_out.y4m gpurun_out/y4m_out0.y4m
