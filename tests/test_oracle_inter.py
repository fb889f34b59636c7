"""inter_oracle.inter_chain (the non-key-frame residual chain the engine's inter mode is checked against): pinned
to the reference's recorded plane checksums (tests/golden/reference_vectors.npz, the inter rows), to the
reference build itself where oracle/_ref exists, and its derived DC index to the scalar quantiser's rule."""
import os

import numpy as np
import pytest

from tests import frame_oracle, inter_oracle
from tests.golden import make_golden

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_vectors.npz")
F = make_golden.FRAME


def _golden_chain(lib, prefix, gold):
    geom, planes, prev, bsize = make_golden.frame_inputs()
    q4 = np.full((3, 30), F["q4"], np.uint8)
    return geom, bsize, q4, inter_oracle.inter_chain(lib, prefix, planes, prev, geom, bsize, F["q0"], q4, 1, F["lam"],
                                                     gold["qm"], gold["qm_inv"])


def test_inter_chain_matches_recorded_reference_plane_checksums(port):
    gold = np.load(PATH)
    want = dict(zip(gold["frame_keys"].tolist(), gold["frame_crc"].tolist()))
    geom, bsize, q4, got = _golden_chain(port, "port", gold)
    for pli in range(3):
        assert make_golden.crc(got[pli]["dq"]) == want["pvq_p%d_k0" % pli]
        assert make_golden.crc(got[pli]["recon"]) == want["inv_p%d_k0" % pli]


def test_inter_chain_dc_index_follows_the_scalar_quantiser(port):
    """qdc is derived from the quantised plane; here the other way round: the non-keyframe DC rule of the
    encoder applied to the unquantised DC and the prediction's gives the same index, block by block."""
    gold = np.load(PATH)
    geom, bsize, q4, got = _golden_chain(port, "port", gold)
    _, planes, _, _ = make_golden.frame_inputs()
    nonzero = 0
    for pli in range(3):
        g = got[pli]
        d = frame_oracle.forward_plane(port, "port", planes[pli], geom, pli, bsize, 0)
        ys, xs = np.nonzero(~np.isnan(g["skip_diff"]))
        nb = (g["rec"][ys, xs, :, 0] != -32768).sum(axis=1)
        assert set(nb.tolist()) <= {1, 4, 7, 9}
        for y, x, n in zip(ys.tolist(), xs.tolist(), nb.tolist()):
            bs = {1: 0, 4: 1, 7: 2}.get(n)
            if bs is None:   # 32x32 or 64x64: the map tells
                bs = max(int(bsize[(y * 4 << geom.xdec[pli]) >> 3, (x * 4 << geom.xdec[pli]) >> 3]), geom.xdec[pli]) - geom.xdec[pli]
            dcq = max((F["q0"] * int(q4[pli][bs * (bs + 1)])) >> 4, 1)
            diff = int(d[4 * y, 4 * x]) - int(g["md"][4 * y, 4 * x])
            if abs(diff) < dcq * 141 // 256:
                q = 0
            else:
                half = ((dcq + 1) >> 1) - 1
                q = int((diff + (-half if diff < 0 else half)) / dcq)   # C division truncates
            assert q == g["qdc"][y, x], (pli, y, x)
            nonzero += q != 0
    assert nonzero > 20


def test_inter_chain_with_the_source_as_prediction_codes_next_to_nothing(port):
    gold = np.load(PATH)
    geom, planes, _, bsize = make_golden.frame_inputs()
    q4 = np.full((3, 30), F["q4"], np.uint8)
    got = inter_oracle.inter_chain(port, "port", planes, planes, geom, bsize, F["q0"], q4, 1, F["lam"], gold["qm"],
                                   gold["qm_inv"])
    # nearly nothing: in 16-bit arithmetic the correlation of a vector with itself can round below one, and such a
    # band codes a small angle with a pulse or two
    for g in got:
        k = g["rec"][..., 3][g["rec"][..., 3] != -32768]
        assert not g["qdc"].any() and (k > 0).sum() <= len(k) // 500
        assert (g["dq"] != g["md"]).sum() <= 16 * (k > 0).sum()


def test_inter_chain_port_matches_reference_build(port, ref):
    from daala_b200 import synth
    from daala_b200.frame import Geometry
    geom = Geometry(328, 200)
    q4 = np.full((3, 30), 20, np.uint8)
    cur = synth.pad_planes(synth.frame(328, 200, f=4)[0], geom)
    for prev, seed in ((synth.frame(328, 200, f=3)[0], 3), (synth.frame(328, 200, f=31, seed=99)[0], 4)):
        pred = synth.pad_planes(prev, geom)
        bsize = synth.block_size_map(geom, "mixed", seed=seed)
        a = inter_oracle.inter_chain(port, "port", cur, pred, geom, bsize, 72, q4)
        b = inter_oracle.inter_chain(ref, "ref", cur, pred, geom, bsize, 72, q4)
        for pli in range(3):
            for k in ("md", "dq", "recon", "rec", "yplane", "qdc"):
                assert np.array_equal(a[pli][k], b[pli][k]), (pli, k)
            assert np.array_equal(a[pli]["skip_diff"], b[pli]["skip_diff"], equal_nan=True), pli
