"""HotPath with the work lists built on the device (daala_b200/lists_torch.py) against the numpy-built
lists: identical planes.  The tensor-op construction is also verified on CPU tensors
(tests/test_host_logic.py)."""
import os

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]


def test_device_built_lists_give_the_same_planes():
    import torch
    from daala_b200 import synth
    from daala_b200.frame import Geometry
    from daala_b200.pipeline import HotPath
    geom = Geometry(384, 256)
    q4 = np.full((3, 30), 20, np.uint8)
    frames = []
    for f in range(2):
        planes, _ = synth.frame(384, 256, f=30 + f)
        frames.append((synth.pad_planes(planes, geom), synth.block_size_map(geom, "mixed", seed=60 + f)))
    outs = []
    for device_lists in (False, True):
        hp = HotPath(geom, nframes=2, q0=45, is_keyframe=1, pvq_qm_q4=q4, keyframe_prediction=True)
        for f, (planes, bsize) in enumerate(frames):
            hp.fb.upload(planes, bsize, frame=f)
        hp.set_block_sizes([b for _, b in frames], device_lists=device_lists)
        hp.run()
        torch.cuda.synchronize()
        outs.append([t.clone() for t in hp.fb.coeffs + hp.fb.pixels_out])
        assert int(sum(b.res_k.sum().item() for b in hp.pvq_batches())) > 0
    for a, b in zip(*outs):
        assert torch.equal(a, b)
