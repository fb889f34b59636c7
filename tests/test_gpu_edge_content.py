"""Edge-case pictures (SURVEY.md 8(d): flat-128, pure noise; plus saturated black / white) through the
device keyframe chain against the oracle: same kernels as the other tests, new inputs."""
import os

import numpy as np
import pytest

from tests import frame_oracle, oracle_lib

pytestmark = [pytest.mark.gpu]


@pytest.mark.parametrize("content", ["flat128", "noise", "black", "white"])
def test_edge_content_keyframe_chain_matches_oracle(content):
    import torch
    from daala_b200 import pvq, synth
    from daala_b200.frame import Geometry
    from daala_b200.pipeline import HotPath
    ref = oracle_lib.load_ref()
    lib, prefix = (ref, "ref") if ref is not None else (oracle_lib.load_port(), "port")
    geom = Geometry(200, 136)
    rng = np.random.default_rng(3)
    planes = []
    for pli in range(3):
        h, w = (136, 200) if pli == 0 else (68, 100)
        value = {"flat128": 128, "black": 0, "white": 255}.get(content)
        planes.append(np.full((h, w), value, np.uint8) if value is not None
                      else rng.integers(0, 256, size=(h, w), dtype=np.uint8))
    planes = synth.pad_planes(planes, geom)
    bsize = synth.block_size_map(geom, "mixed", seed=8)
    q4 = np.full((3, 30), 16, np.uint8)
    hp = HotPath(geom, q0=30, is_keyframe=1, pvq_qm_q4=q4, keyframe_prediction=True)
    hp.fb.upload(planes, bsize)
    hp.set_block_sizes([bsize])
    hp.run()
    torch.cuda.synchronize()
    qm, qm_inv = pvq.default_qm(True)
    luma_q = None
    for pli in range(3):
        d = frame_oracle.forward_plane(lib, prefix, planes[pli], geom, pli, bsize, 1)
        dq, _ = frame_oracle.pvq_plane_pred(lib, prefix, d, geom, pli, bsize, 30, 1, 0.147, qm, qm_inv, q4,
                                            luma_d=luma_q)
        if pli == 0:
            luma_q = dq
        assert np.array_equal(hp.fb.coeffs[pli][0].cpu().numpy(), dq), pli
        rec = frame_oracle.inverse_plane(lib, prefix, dq, geom, pli, bsize, 1)
        assert np.array_equal(hp.fb.pixels_out[pli][0].cpu().numpy(), rec), pli


def test_real_encoder_block_sizes_match_recorded_reference_checksums():
    """The golden picture with the block-size map the whole reference encoder decided
    (tests/golden/reference_vectors.npz: real_bsize) -- plane CRCs recorded from the reference build."""
    import torch
    from daala_b200.pipeline import HotPath
    from tests.golden import make_golden
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_vectors.npz"))
    want = dict(zip(gold["real_keys"].tolist(), gold["real_crc"].tolist()))
    F = make_golden.FRAME
    geom, planes, _, _ = make_golden.frame_inputs()
    bsize = np.ascontiguousarray(gold["real_bsize"])
    q4 = np.full((3, 30), F["q4"], np.uint8)
    hp = HotPath(geom, q0=F["q0"], is_keyframe=1, pvq_qm_q4=q4, keyframe_prediction=True)
    hp.fb.upload(planes, bsize)
    hp.set_block_sizes([bsize])
    hp.fb.forward()
    torch.cuda.synchronize()
    for pli in range(3):
        assert make_golden.crc(hp.fb.coeffs[pli][0].cpu().numpy()) == want["fwd_p%d" % pli], pli
    hp.run()
    torch.cuda.synchronize()
    for pli in range(3):
        assert make_golden.crc(hp.fb.coeffs[pli][0].cpu().numpy()) == want["pred_p%d" % pli], pli
        assert make_golden.crc(hp.fb.pixels_out[pli][0].cpu().numpy()) == want["inv_p%d" % pli], pli
