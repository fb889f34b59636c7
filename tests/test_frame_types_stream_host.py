"""The mixed symbol stream (symbol_stream = 3 with frame_types = 1) without a GPU: on seeded synthetic classic outputs
of a mixed step, symbols.pack_reference(..., frame_type=) gives each keyframe the keyframe stream (CfL flips, the
keyframe DC records) and each P / B frame the P-frame stream (DC records), each with the other kind's records zero;
read_frame reads it back; no keyframe DC record is all zero, which is what tells the two kinds apart in sym_hdc."""
import numpy as np
import pytest

from daala_b200 import haardc, symbols, synth
from daala_b200.frame import Geometry
from tests.test_symbol_stream import _classic

CASES = [((200, 130), (1, 0, 0, 1)), ((320, 192), (0, 1, 0, 1)), ((128, 128), (1, 1)), ((200, 130), (0, 0, 0))]


def _mixed_outputs(geom, types, seed):
    """_classic outputs with what a mixed step adds: DC indices and residuals (0 on keyframe blocks), index grids (0 on
    P / B frames) and CfL flips 0 on P / B frames."""
    rng = np.random.default_rng(seed)
    maps = [synth.block_size_map(geom, "mixed", seed=seed + f) for f in range(len(types))]
    out = _classic(geom, maps, seed)
    key = np.asarray(types, bool)
    for kind in ("luma", "chroma"):
        on_p = ~key[out[kind + "_blocks"]["frame"].astype(np.int64)]
        n = len(on_p)
        out[kind + "_dc"] = np.where(on_p, rng.integers(-40, 41, n), 0).astype(np.int32)
        out[kind + "_dc_resid"] = np.where(on_p, rng.integers(-900, 901, n), 0).astype(np.int32)
    out["chroma_flip"][~key[out["chroma_blocks"]["frame"].astype(np.int64)]] = 0
    for p in range(3):
        h, w = geom.plane_shape(p)
        g = rng.integers(-30, 31, (len(types), h >> 2, w >> 2)).astype(np.int32)
        g[~key] = 0
        out["dc_index%d" % p] = g
    return out, maps


def _only(out, kind_keys):
    return {k: v for k, v in out.items() if k in kind_keys}


@pytest.mark.parametrize("size,types", CASES, ids=lambda v: "x".join(map(str, v)))
def test_mixed_reference_is_the_single_kind_streams_frame_by_frame(size, types):
    geom = Geometry(*size)
    F = len(types)
    out, maps = _mixed_outputs(geom, types, seed=sum(size) + F)
    mixed = symbols.pack_reference(out, F, frame_type=types)
    assert {"sym_dc", "sym_hdc"} <= set(mixed)
    keys = [f for f in range(F) if types[f]]
    pfs = [f for f in range(F) if not types[f]]
    # the keyframe-only outputs (no DC arrays: the keyframe path with the index grids) and the P-only outputs
    kout = {k: v for k, v in out.items() if not k.endswith(("_dc", "_dc_resid"))}
    pout = {k: v for k, v in out.items() if not k.startswith("dc_index")}
    common = ("sym_index", "sym_blocks", "sym_bands", "sym_pulses")
    if keys:
        want = symbols.pack_reference(kout, keys)
        assert "sym_hdc" in want and "sym_dc" not in want
        assert not symbols.stream_equal(_only(mixed, common + ("sym_hdc",)), want, keys, range(len(keys)))
    if pfs:
        want = symbols.pack_reference(pout, pfs)
        assert "sym_dc" in want and "sym_hdc" not in want
        assert not symbols.stream_equal(_only(mixed, common + ("sym_dc",)), want, pfs, range(len(pfs)))
    nonzero = {"flip": 0, "dc": 0, "hdc": 0}
    for f, m in enumerate(maps):
        r = symbols.read_frame(mixed, f)
        order = symbols.coding_order(m, geom)
        for k in ("x0", "y0", "pli", "bs"):
            assert np.array_equal(r["blocks"][k], order[k]), (f, k)
        assert len(r["dc"]) == len(r["hdc"]) == len(order)
        if types[f]:
            assert not r["dc"].view(np.uint8).any(), ("keyframe", f, "sym_dc")
            assert np.all((r["hdc"]["bsi"] == 4) | (r["hdc"]["child"] >= 1)), ("keyframe", f)
            nonzero["flip"] += int(np.count_nonzero(r["blocks"]["flip"]))
            nonzero["hdc"] += int(np.count_nonzero(r["hdc"]["value"]))
        else:
            assert not r["hdc"].view(np.uint8).any(), ("P frame", f, "sym_hdc")
            assert not r["blocks"]["flip"].any(), ("P frame", f, "flip")
            nonzero["dc"] += int(np.count_nonzero(r["dc"]["qdc"]))
    # the records compared are not trivially zero
    for k, v in nonzero.items():
        assert v > 0 or (k == "dc" and not pfs) or (k != "dc" and not keys), k


@pytest.mark.parametrize("size", [(200, 130), (1920, 1080)], ids=lambda s: "%dx%d" % s)
def test_no_keyframe_dc_record_is_all_zero(size):
    """Every record stream_records makes has bsi = 4 (the superblock DC) or child >= 1, whatever the indices: an
    all-zero record marks a P / B frame's block in the mixed stream."""
    geom = Geometry(*size)
    rng = np.random.default_rng(size[0])
    maps = [synth.block_size_map(geom, m) for m in ("4", "8", "16", "32", "64")]
    maps += [synth.block_size_map(geom, "mixed", seed=s) for s in range(3)]
    for bs in maps:
        idx = [np.zeros(tuple(s >> 2 for s in geom.plane_shape(p)), np.int32) for p in range(3)]
        for variant in (idx, [rng.integers(-5, 6, g.shape).astype(np.int32) for g in idx]):
            rec = haardc.stream_records(variant, bs, geom)
            assert len(rec) == len(symbols.coding_order(bs, geom))
            assert np.all((rec["bsi"] == 4) | (rec["child"] >= 1))
