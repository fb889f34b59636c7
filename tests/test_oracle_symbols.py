"""Pins the oracle's per-block symbol recording (oracle/pipeline_driver.inc, pvq_plane_sym, reached through
frame_oracle.keyframe_chain(..., symbols=True)): each block's skip_diff and keyframe CfL flip, which the host
entropy coder reads besides the band records.  The port and the reference build agree bit for bit, the
per-block skip_diff adds up to the driver's stats[4] in block order, and single blocks agree with the
block-level oracle (tests/pvq_oracle.block)."""
import os

import numpy as np
import pytest

from tests import frame_oracle, pvq_oracle
from tests.oracle_lib import addr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Q0 = 72
Q4 = np.full((3, 30), 16, np.uint8)


def _case(kind):
    """(geom, padded planes, bsize) of one keyframe: a seeded mixed quadtree, all 4x4, or the top two
    superblock rows of a map the whole reference encoder decided (daala_b200/data/bench_bsize_4k.npz)."""
    from daala_b200 import synth
    from daala_b200.frame import Geometry
    geom = Geometry(3840, 128) if kind == "real" else Geometry(328, 200)
    planes, _ = synth.frame(geom.pic_w, geom.pic_h, f=1, seed=777)
    if kind == "real":
        real = np.load(os.path.join(ROOT, "daala_b200", "data", "bench_bsize_4k.npz"))
        bsize = np.ascontiguousarray(real["bsize_2"][:geom.bsize_shape[0]])
    else:
        bsize = synth.block_size_map(geom, kind, seed=31)
    return geom, synth.pad_planes(planes, geom), bsize


def _blocks_in_order(geom, pli, bsize):
    """(y0, x0, bs) of every leaf block of a plane in the order the driver codes them (superblocks in
    raster order, quadtree order inside: pvq_recurse)."""
    xdec = geom.xdec[pli]
    out = []

    def rec(bx, by, bsi):
        obs = int(bsize[(by << bsi) >> 1, (bx << bsi) >> 1])
        bs = max(obs, xdec)
        if bs == bsi:
            sh = 2 + bs - xdec
            out.append((by << sh, bx << sh, bs - xdec))
            return
        for dy, dx in ((0, 0), (0, 1), (1, 0), (1, 1)):
            rec(2 * bx + dx, 2 * by + dy, bsi - 1)

    for sby in range(geom.nvsb):
        for sbx in range(geom.nhsb):
            rec(sbx, sby, 4)
    return out


def _check_maps(geom, bsize, got):
    """Every block origin carries a value and nothing else does; flips only on chroma."""
    for pli in range(3):
        origin = np.zeros(got[pli]["flip"].shape, bool)
        for y0, x0, _ in _blocks_in_order(geom, pli, bsize):
            origin[y0 >> 2, x0 >> 2] = True
        assert np.array_equal(~np.isnan(got[pli]["skip_diff"]), origin), pli
        assert np.array_equal(got[pli]["flip"] >= 0, origin), pli
        assert set(np.unique(got[pli]["flip"][origin]).tolist()) <= {0, 1}, pli
    assert not got[0]["flip"][got[0]["flip"] >= 0].any()


@pytest.mark.parametrize("kind", ["mixed", "4", "real"])
def test_symbol_maps_port_matches_reference(port, ref, kind):
    geom, planes, bsize = _case(kind)
    got = {}
    for lib, prefix in ((ref, "ref"), (port, "port")):
        got[prefix] = frame_oracle.keyframe_chain(lib, prefix, planes, geom, bsize, Q0, Q4, symbols=True)
    _check_maps(geom, bsize, got["ref"])
    for pli in range(3):
        a, b = got["ref"][pli], got["port"][pli]
        # bit for bit, NaN (no block) included
        assert a["skip_diff"].tobytes() == b["skip_diff"].tobytes(), ("skip_diff", kind, pli)
        assert np.array_equal(a["flip"], b["flip"]), ("flip", kind, pli)
        assert np.array_equal(a["rec"], b["rec"]) and np.array_equal(a["dq"], b["dq"]), (kind, pli)
    # the maps carry information: chroma blocks with and without the CfL sign flip on every plane
    for pli in (1, 2):
        f = got["ref"][pli]["flip"]
        assert (f == 1).sum() > 0 and (f == 0).sum() > 0, (kind, pli)


@pytest.mark.parametrize("kind", ["mixed", "4", "real"])
def test_symbol_maps_sum_to_stats_and_keep_results(port, kind):
    """symbols=True adds the maps and changes nothing else; the per-block skip_diff summed in the driver's
    block order is bit-identical to its accumulated stats[4]."""
    from tests import oracle_lib
    lib = oracle_lib.load_ref()
    lib, prefix = (lib, "ref") if lib is not None else (port, "port")
    geom, planes, bsize = _case(kind)
    want = frame_oracle.keyframe_chain(lib, prefix, planes, geom, bsize, Q0, Q4)
    got = frame_oracle.keyframe_chain(lib, prefix, planes, geom, bsize, Q0, Q4, symbols=True)
    _check_maps(geom, bsize, got)
    for pli in range(3):
        for k in ("dq", "recon", "rec", "yplane", "stats"):
            assert np.array_equal(got[pli][k], want[pli][k]), (k, pli)
        assert "skip_diff" not in want[pli] and "flip" not in want[pli]
        s = 0.0
        for y0, x0, _ in _blocks_in_order(geom, pli, bsize):
            s += got[pli]["skip_diff"][y0 >> 2, x0 >> 2]
        assert s == got[pli]["stats"][4], (pli, s, got[pli]["stats"][4])
    assert sum(int((got[p]["flip"] == 1).sum()) for p in (1, 2)) > 0


def _prediction(port, geom, pli, bsize, dq, y0, x0, bs):
    """The block's predictor in raster order, as the driver forms it: od_hv_intra_pred from the quantised luma
    neighbours, or CfL from the quantised luma plane (the port's restatements of both)."""
    n = 4 << bs
    pred = np.zeros((n, n), np.int32)
    if pli == 0:
        port.port_hv_intra_pred(addr(pred), addr(np.ascontiguousarray(dq[0], np.int32)), dq[0].shape[1], x0 >> 2,
                                y0 >> 2, addr(np.ascontiguousarray(bsize, np.uint8)), bsize.shape[1], bs)
    else:
        luma = np.ascontiguousarray(dq[0], np.int32)
        lw = luma.shape[1]
        port.port_resample_luma_coeffs_420(addr(pred), n, addr(luma, (2 * y0) * lw + 2 * x0), lw, bs,
                                           int(bsize[y0 >> 2, x0 >> 2] == 0))
    return pred


@pytest.mark.parametrize("kind", ["mixed", "real"])
def test_symbol_maps_match_block_oracle(port, kind):
    """A few blocks per plane (flipped and unflipped chroma among them) through the block-level oracle: the
    forward coefficients and the predictor in coding order, the band loop and CfL flip of od_pvq_encode."""
    from daala_b200 import pvq
    geom, planes, bsize = _case(kind)
    got = frame_oracle.keyframe_chain(port, "port", planes, geom, bsize, Q0, Q4, symbols=True)
    dq = [got[p]["dq"] for p in range(3)]
    qm, qm_inv = pvq.default_qm(True)
    rng = np.random.default_rng(5)
    checked_flips = set()
    for pli in range(3):
        d = frame_oracle.forward_plane(port, "port", planes[pli], geom, pli, bsize, 1)
        blocks = _blocks_in_order(geom, pli, bsize)
        pick = list(rng.choice(len(blocks), size=6, replace=False))
        if pli:
            # make sure both flip values are among the checked blocks
            for v in (0, 1):
                idx = [i for i, (y0, x0, _) in enumerate(blocks) if got[pli]["flip"][y0 >> 2, x0 >> 2] == v]
                pick.append(idx[len(idx) // 2])
        for i in pick:
            y0, x0, bs = blocks[i]
            n = 4 << bs
            dvec = pvq_oracle.coding_order(port, "port", np.ascontiguousarray(d, np.int32), x0, y0, n)
            pred = _prediction(port, geom, pli, bsize, dq, y0, x0, bs)
            pvec = pvq_oracle.coding_order(port, "port", pred, 0, 0, n)
            o = pvq_oracle.block(port, "port", dvec, pvec, bs, pli, geom.xdec[pli], Q0, 1, 1, pvq.PVQ_LAMBDA, qm, qm_inv, Q4)
            assert got[pli]["skip_diff"][y0 >> 2, x0 >> 2] == o["skip_diff"], (kind, pli, y0, x0, bs)
            assert got[pli]["flip"][y0 >> 2, x0 >> 2] == o["flip"], (kind, pli, y0, x0, bs)
            # the same block's band records: the predictor above is the one the driver used
            for band, r in enumerate(o["bands"]):
                assert got[pli]["rec"][y0 >> 2, x0 >> 2, band].tolist() == [r["gain"], r["itheta"], r["max_theta"],
                                                                             r["k"]], (kind, pli, y0, x0, band)
            if pli:
                checked_flips.add(o["flip"])
    assert checked_flips == {0, 1}
