"""The symbol stream's host side (daala_b200/symbols.py) without a GPU: pack_reference followed by the reader
round-trips synthetic records, and coding_order lists the leaf blocks the oracle codes, in the order its
quadtree recursion visits them."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from daala_b200 import pvq, symbols, synth
from daala_b200.frame import Geometry
from tests import oracle_lib
from tests.oracle_lib import addr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _classic(geom, maps, seed):
    """Synthetic classic engine outputs for frames with block-size maps `maps`: the blocks of each frame (luma
    list, then chroma) in a shuffled order, random band records covering K = 0, 127, 128, noref and reference
    bands, pulses with |y| <= K."""
    rng = np.random.default_rng(seed)
    lists = {"luma": [], "chroma": []}
    for f, m in enumerate(maps):
        o = symbols.coding_order(m, geom)
        for name, sel in (("luma", o["pli"] == 0), ("chroma", o["pli"] > 0)):
            b = np.zeros(int(sel.sum()), pvq.BLOCK_DTYPE)
            for k in ("x0", "y0", "bs", "pli"):
                b[k] = o[k][sel]
            b["frame"] = f
            b["xdec"] = 0 if name == "luma" else 1
            lists[name].append(b[rng.permutation(len(b))])
    out = {}
    for name, parts in lists.items():
        b = np.concatenate(parts)
        length = np.minimum(16 << (2 * b["bs"].astype(np.int64)), 512)
        b["coef_off"] = np.concatenate([[0], np.cumsum(length)[:-1]])
        n = len(b)
        res = np.zeros((n, 9, 4), np.int16)
        k = rng.choice([0, 0, 1, 5, 127, 128, 300], size=(n, 9))
        res[..., 0] = rng.integers(0, 20, size=(n, 9))
        res[..., 1] = np.where(rng.random((n, 9)) < 0.5, -1, rng.integers(0, 8, size=(n, 9)))
        res[..., 2] = rng.integers(0, 10, size=(n, 9))
        res[..., 3] = k
        y16 = np.zeros(int(length.sum()), np.int16)
        kk = np.zeros(len(y16), np.int64)
        for i in range(n):   # each coefficient gets the K of its band
            for band in range(symbols.NBANDS[b["bs"][i]]):
                a, e = symbols.BAND_EDGES[band], symbols.BAND_EDGES[band + 1]
                kk[b["coef_off"][i] + a:b["coef_off"][i] + e] = k[i, band]
        y16[:] = (rng.integers(-(1 << 15), 1 << 15, size=len(y16)) % (2 * kk + 1)) - kk
        out[name + "_blocks"] = b
        out[name + "_res"] = res
        out[name + "_y16"] = y16
        out[name + "_skip_diff"] = rng.standard_normal(n)
    out["chroma_flip"] = rng.integers(0, 2, size=len(out["chroma_blocks"])).astype(np.int32)
    return out


def _maps(geom, modes):
    return [synth.block_size_map(geom, "mixed", seed=3 + i) if m == "mixed" else synth.block_size_map(geom, m)
            for i, m in enumerate(modes)]


@pytest.mark.parametrize("size,modes", [((128, 128), ("mixed", "4", "mixed")), ((200, 130), ("mixed", "4")),
                                        ((320, 192), ("16", "mixed", "64"))])
def test_pack_reference_round_trips(size, modes):
    geom = Geometry(*size)
    maps = _maps(geom, modes)
    out = _classic(geom, maps, seed=sum(size))
    st = symbols.pack_reference(out, len(maps))
    seen_k = set()
    for f, m in enumerate(maps):
        r = symbols.read_frame(st, f)
        order = symbols.coding_order(m, geom)
        blocks = r["blocks"]
        assert np.array_equal(blocks["x0"], order["x0"]) and np.array_equal(blocks["y0"], order["y0"])
        assert np.array_equal(blocks["pli"], order["pli"]) and np.array_equal(blocks["bs"], order["bs"])
        for i in range(len(blocks)):
            name = "luma" if blocks["pli"][i] == 0 else "chroma"
            cb = out[name + "_blocks"]
            j = np.nonzero((cb["frame"] == f) & (cb["pli"] == blocks["pli"][i]) & (cb["x0"] == blocks["x0"][i]) &
                           (cb["y0"] == blocks["y0"][i]))[0]
            assert len(j) == 1
            j = int(j[0])
            assert blocks["skip_diff"][i] == out[name + "_skip_diff"][j]
            assert blocks["flip"][i] == (out["chroma_flip"][j] if name == "chroma" else 0)
            sel = np.nonzero(r["band_block"] == i)[0]
            nb = symbols.NBANDS[blocks["bs"][i]]
            assert len(sel) == nb
            assert np.array_equal(r["bands"][sel], out[name + "_res"][j, :nb])
            for band, q in zip(range(nb), sel):
                k, itheta = int(r["bands"][q, 3]), int(r["bands"][q, 1])
                a = int(cb["coef_off"][j]) + symbols.BAND_EDGES[band]
                n = symbols.BAND_EDGES[band + 1] - symbols.BAND_EDGES[band] - (itheta != -1)
                want = out[name + "_y16"][a:a + n] if k > 0 else np.zeros(0, np.int16)
                assert np.array_equal(r["pulses"][q], want.astype(np.int32)), (f, i, band, k)
                seen_k.add((min(k, 128), itheta == -1))
    assert {(127, True), (127, False), (128, True), (128, False), (0, True)} <= seen_k


def test_pulse_widths():
    """K <= 127: one signed byte per value; K >= 128: two bytes, little-endian."""
    bands = np.array([[1, -1, 0, 127], [1, 2, 3, 128]], np.int16)
    res = np.zeros((1, 9, 4), np.int16)
    res[0, :1] = bands[:1]
    y = np.zeros(16, np.int32)
    y[1:16] = np.arange(15) - 7
    y[1] = -127
    b, n, p = symbols.pack_blocks([0], [0], [0], [0], [0], [0.5], res, y, [0])
    assert len(p) == 15 and p[0] == 0x81 and p.view(np.int8)[1] == -6
    res[0, 0] = bands[1]
    y[1] = -300
    b, n, p = symbols.pack_blocks([0], [0], [0], [0], [0], [0.5], res, y, [0])
    assert len(p) == 28 and p[:2].view(np.int16)[0] == -300


# --- coding order against the oracle's recursion --------------------------------------------------------------
@pytest.fixture(scope="module")
def visits(tmp_path_factory):
    """tests/oracle_visits.c built against the oracle's C port: oracle/pipeline_driver.inc with every block visit
    recorded."""
    port = oracle_lib.load_port()
    assert port is not None
    so = str(tmp_path_factory.mktemp("visits") / "liboracle_visits.so")
    oracle = os.path.join(ROOT, "oracle")
    subprocess.run(["gcc", "-shared", "-fPIC", "-O2", "-w", "-I", oracle, os.path.join(ROOT, "tests", "oracle_visits.c"),
                    os.path.join(oracle, "libdaala_port.so"), "-Wl,-rpath," + oracle, "-o", so], check=True)
    lib = ctypes.CDLL(so)
    lib.oracle_visits.restype = ctypes.c_long
    return lib, port


def _oracle_plane(visits, geom, bsize, pli):
    """(visit order [(x0, y0, n)], band-record origins {(y4, x4)}) of one plane of a zero-coefficient frame."""
    lib, port = visits
    h, w = geom.plane_shape(pli)
    qm, qm_inv = pvq.default_qm(True)
    q4 = np.full(30, 16, np.uint8)
    bs = np.ascontiguousarray(bsize, np.uint8)
    luma = np.zeros(geom.plane_shape(0), np.int32)
    d = np.zeros((h, w), np.int32)
    cap = h * w // 16
    rec_out = np.zeros((cap, 3), np.int32)
    n = lib.oracle_visits(addr(d), h, geom.nhsb, geom.nvsb, geom.xdec[pli], pli, addr(bs), bs.shape[1], 60, addr(qm),
                          addr(qm_inv), addr(q4), addr(luma) if pli else None, addr(rec_out), ctypes.c_long(cap))
    assert 0 < n <= cap
    rec = np.full((h // 4, w // 4, 9, 4), -32768, np.int16)
    d = np.zeros((h, w), np.int32)
    stats = np.zeros(5, np.float64)
    port.oracle_port_pvq_plane_rec(addr(d), None, geom.nhsb, geom.nvsb, geom.xdec[pli], pli, addr(bs), bs.shape[1], 60,
                                   1, 1, ctypes.c_double(0.147), addr(qm), addr(qm_inv), addr(q4), addr(stats),
                                   1 if pli == 0 else 0, addr(luma) if pli else None, addr(rec), None)
    origins = {tuple(v) for v in np.argwhere(rec[:, :, 0, 0] != -32768).tolist()}
    return rec_out[:n], origins


def _check_order(visits, geom, bsize):
    order = symbols.coding_order(bsize, geom)
    for pli in range(3):
        o = order[order["pli"] == pli]
        seq, origins = _oracle_plane(visits, geom, bsize, pli)
        assert len(seq) == len(o) == len(origins), pli
        assert np.array_equal(seq[:, 0], o["x0"]) and np.array_equal(seq[:, 1], o["y0"]), pli
        assert np.array_equal(seq[:, 2], 4 << o["bs"].astype(np.int32)), pli
        assert origins == set(zip((o["y0"] >> 2).tolist(), (o["x0"] >> 2).tolist())), pli
    # superblocks in raster order, planes 0, 1, 2 inside each
    sb = np.where(order["pli"] > 0, 5, 6)
    key = (order["y0"].astype(np.int64) >> sb) * geom.nhsb + (order["x0"].astype(np.int64) >> sb)
    k2 = key * 3 + order["pli"]
    assert np.all(np.diff(k2) >= 0)


@pytest.mark.parametrize("mode,size", [("mixed", (200, 130)), ("4", (128, 64)), ("mixed", (640, 384)),
                                       ("64", (192, 128))])
def test_coding_order_matches_oracle_recursion(visits, mode, size):
    geom = Geometry(*size)
    _check_order(visits, geom, _maps(geom, (mode,))[0])


@pytest.mark.parametrize("frame", [0, 3])
def test_coding_order_matches_oracle_on_encoder_maps(visits, frame):
    """The reference encoder's own block-size decisions for a 3840x2160 frame (the benchmark's maps)."""
    real = np.load(os.path.join(ROOT, "daala_b200", "data", "bench_bsize_4k.npz"))
    geom = Geometry(3840, 2160)
    bsize = np.ascontiguousarray(real["bsize_%d" % frame][:geom.bsize_shape[0]])
    assert (bsize == 0).any() and (bsize >= 3).any()
    _check_order(visits, geom, bsize)
