"""The late-skip distortions of a P-frame step (config.late_skip = 1; csrc/late_skip.cu): per block the four
od_compute_dist values od_block_encode's late skip can ask for (include/daala_b200.h, daala_b200_kf_late_skip), against
the oracle's plane driver (oracle/late_skip_driver.inc: c_orig taken from the forward transform's prefiltered plane,
candidates inverted with the reference's leaf iDCT) fed the step's coded coefficient planes.  Bit-exact with flat
quantisation matrices; 1e-12 relative with the HVS metric (pow of the CUDA math library).  The decisions taken from the
records drive the finishing pass.  The last tests need no GPU."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from tests import late_skip_oracle, oracle_lib
from tests.test_gpu_engine_inter import Q4, _frames

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID = 1   # cudaErrorInvalidValue
FIELDS = ("dist_skip", "noskip_coded_dc0", "noskip_coded_dcq", "noskip_pred_dcq")


def _stack(frames):
    return ([np.stack([f[0][p] for f in frames]) for p in range(3)], [np.stack([f[1][p] for f in frames]) for p in range(3)],
            np.stack([f[2] for f in frames]))


def _copy(out):
    return {k: np.array(v) for k, v in out.items()}


def _engine(geom, F, q0, flat=0, masking=1, cq=40, **kw):
    from daala_b200 import engine
    return engine.KeyframeEngine(geom, nframes=F, q0=q0, pvq_qm_q4=Q4, inter=1, late_skip=1, use_masking=masking,
                                 qm_is_flat=flat, coded_quantizer=cq, **kw)


def _as_array(recs):
    return np.stack([recs[f] for f in FIELDS], axis=-1)


def _oracle_maps(geom, F, planes, pred, coded, bsize, q0, flat, masking, cq):
    """[F][3] oracle maps [h/4, w/4, 4]."""
    lib, prefix = late_skip_oracle.load()
    return [[late_skip_oracle.plane(lib, prefix, planes[p][f], pred[p][f], coded[p][f], geom, bsize[f], p, q0, Q4, flat,
                                    masking, cq) for p in range(3)] for f in range(F)]


def _check_against(out, maps, F, flat):
    """Every block record of the step equals the oracle's entry at the block's origin (zero for bs = 0)."""
    seen = {0: 0, 1: 0}
    for kind in ("luma", "chroma"):
        b = out[kind + "_blocks"]
        got = _as_array(out[kind + "_late_skip"])
        want = np.zeros_like(got)
        for f in range(F):
            for p in (0,) if kind == "luma" else (1, 2):
                sel = (b["frame"] == f) & (b["pli"] == p)
                want[sel] = maps[f][p][b["y0"][sel] >> 2, b["x0"][sel] >> 2]
        assert not got[b["bs"] == 0].any() and not want[b["bs"] == 0].any()
        big = b["bs"] > 0
        assert (got[big] > 0).any()
        if flat:
            assert np.array_equal(got, want), kind
        else:
            assert np.allclose(got, want, rtol=1e-12, atol=0), (kind, np.abs(got - want).max())
        seen[kind == "chroma"] += int(big.sum())
    return seen


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,q0,flat,masking", [(200, 130, 30, 0, 1), (200, 130, 72, 1, 1), (328, 200, 30, 1, 0),
                                                 (328, 200, 72, 0, 0), (1920, 1080, 30, 0, 1), (1920, 1080, 72, 1, 0)])
def test_records_match_oracle(w, h, q0, flat, masking):
    from daala_b200.frame import Geometry
    geom = Geometry(w, h)
    F = 2 if w < 1000 else 1
    planes, pred, bsize = _stack(_frames(geom, F, seed=w + q0))
    eng = _engine(geom, F, q0, flat, masking, cq=q0 + 10)
    out = _copy(eng.encode(planes, bsize, pred=pred))
    coded = [eng.coeff_plane(p) for p in range(3)]
    # the maps have every class: 32x32 / 64x64 luma tails, 8x8 chroma, 4x4 blocks without a late skip
    lb, cb = out["luma_blocks"], out["chroma_blocks"]
    assert {0, 3, 4} <= set(lb["bs"].tolist()) and {0, 1} <= set(cb["bs"].tolist())
    _check_against(out, _oracle_maps(geom, F, planes, pred, coded, bsize, q0, flat, masking, q0 + 10), F, flat)
    eng.close()


@pytest.mark.gpu
def test_records_match_oracle_inter_mc():
    """The engine's own prediction (inter_mc): the oracle gets the prediction planes the step made."""
    from daala_b200.frame import Geometry
    from tests import test_gpu_engine_inter_mc as mc
    geom = Geometry(200, 130)
    F = 2
    refs = mc._pool(geom, 3, seed=7)
    planes, bsize = mc._batch(geom, F, seed=11)
    eng = _engine(geom, F, 45, inter_mc=1)
    out = _copy(eng.encode(planes, bsize, refs=refs, ref_slot=np.array([[0, 1], [2, 1]], np.int32),
                           mv_grid=mc._pack(mc._grids(geom, F, seed=3))))
    pred = [out["pred%d" % p] for p in range(3)]
    coded = [eng.coeff_plane(p) for p in range(3)]
    _check_against(out, _oracle_maps(geom, F, planes, pred, coded, bsize, 45, 0, 1, 40), F, 0)
    eng.close()


def _q1(out, kind, q0):
    from daala_b200 import lateskip
    b = out[kind + "_blocks"]
    return lateskip.q1(out[kind + "_dc_resid"], lateskip.dc_quant(q0, Q4, b["pli"], b["bs"]))


@pytest.mark.gpu
def test_decisions_close_the_loop():
    """Seeded rates and lambda: the late-skip decisions from the engine's records equal those from the oracle's, records
    obey the candidate rule where q1 = 0, and the finishing pass fed the decisions equals the oracle's reconstruction."""
    from daala_b200 import lateskip
    from daala_b200.frame import Geometry
    from tests.test_gpu_engine_inter_finish import _check, _want
    geom = Geometry(328, 200)
    F, q0 = 2, 45
    planes, pred, bsize = _stack(_frames(geom, F, seed=3))
    for p in range(3):   # the top half predicted exactly: DC residuals 0 there, so both q1 = 0 and q1 != 0 occur
        h2 = planes[p].shape[1] // 2
        pred[p][:, :h2] = planes[p][:, :h2]
    eng = _engine(geom, F, q0, inter_finish=1)
    out = _copy(eng.encode(planes, bsize, pred=pred))
    d = [eng.coeff_plane(p) for p in range(3)]
    md = [eng.pred_coeff_plane(p) for p in range(3)]
    maps = _oracle_maps(geom, F, planes, pred, d, bsize, q0, 0, 1, 40)
    _check_against(out, maps, F, 0)
    rng = np.random.default_rng(17)
    dec = {}
    for kind in ("luma", "chroma"):
        b, rec = out[kind + "_blocks"], out[kind + "_late_skip"]
        q1 = _q1(out, kind, q0)
        zero = (q1 == 0) & (b["bs"] > 0)
        assert zero.any() and (q1 != 0).any()
        # the candidate rule where od_rdo_quant can only return 0
        assert np.array_equal(rec["noskip_pred_dcq"][zero], rec["dist_skip"][zero])
        assert np.array_equal(rec["noskip_coded_dc0"][zero], rec["noskip_coded_dcq"][zero])
        assert not _as_array(rec)[b["bs"] == 0].any()
        n = len(b)
        pvq_skip = rng.random(n) < 0.3
        dc = np.where(rng.random(n) < 0.5, q1, 0).astype(np.int32)
        r_noskip = rng.integers(8, 800, n)
        r_skip = rng.integers(1, 40, n)
        spread = np.abs(rec["noskip_coded_dcq"] - rec["dist_skip"]) / np.maximum(1, r_noskip - r_skip)
        lam = float(np.median(spread[b["bs"] > 0]))
        skip, dcs = np.zeros(n, np.uint8), np.zeros(n, np.int32)
        nlate = 0
        for i in range(n):
            skip[i], dcs[i] = pvq_skip[i], dc[i]
            if b["bs"][i] == 0:
                continue
            p = int(b["pli"][i])
            want_rec = maps[int(b["frame"][i])][p][b["y0"][i] >> 2, b["x0"][i] >> 2]
            orec = {f: want_rec[k] for k, f in enumerate(FIELDS)}
            late = lateskip.decide(rec[i], pvq_skip[i], dc[i], r_noskip[i], r_skip[i], lam)
            assert late == lateskip.decide(orec, pvq_skip[i], dc[i], r_noskip[i], r_skip[i], lam), (kind, i)
            if late:
                skip[i], dcs[i] = 1, 0
                nlate += 1
        assert 0 < nlate < n
        dec[kind] = (skip, dcs)
    levels = rng.integers(0, 6, (F, geom.nvsb, geom.nhsb)).astype(np.uint8)
    got = _copy(eng.finish(dec["luma"][0], dec["luma"][1], dec["chroma"][0], dec["chroma"][1], levels))
    _check(got, _want(geom, F, out, d, md, bsize, q0, dec["luma"] + dec["chroma"] + (levels,)), F)
    eng.close()


@pytest.mark.gpu
def test_stream_order_resident_sequence():
    """symbol_stream = 2: sym_late_skip is the block-order records permuted by the stream's slot order, over a
    resident-pool sequence of two steps; only the used part is counted in the stream's D2H."""
    from daala_b200 import symbols
    from daala_b200.frame import Geometry
    from tests.test_gpu_engine_inter_mc import _batch, _grids, _pack, _pool
    geom = Geometry(328, 200)
    F = 2
    eng = _engine(geom, F, 45, inter_mc=1, mc_refs=2 * F, inter_finish=1, symbol_stream=2)
    gold = _pool(geom, F, seed=41)
    for f in range(F):
        eng.pool_load(f, [gold[p][f] for p in range(3)])
    for k in range(2):
        planes, bsize = _batch(geom, F, seed=50 + k)
        slot = np.array([[f, f if k == 0 else F + f] for f in range(F)], np.int32)
        out = _copy(eng.encode(planes, bsize, ref_slot=slot, mv_grid=_pack(_grids(geom, F, seed=60 + k)), resident=True))
        perm = symbols.stream_to_classic(out)
        classic = np.concatenate([out["luma_late_skip"], out["chroma_late_skip"]])
        n = len(perm)
        assert np.array_equal(_as_array(out["sym_late_skip"][:n]), _as_array(classic[perm])), k
        assert (_as_array(classic) > 0).any()
        nb = int(out["sym_index"][:, 1].sum())
        assert eng.stream_d2h_bytes() >= nb * (symbols.DC_DTYPE.itemsize + symbols.LATE_SKIP_DTYPE.itemsize)
        skip = np.zeros(len(out["luma_dc"]), np.uint8), np.zeros(len(out["chroma_dc"]), np.uint8)
        eng.finish(skip[0], out["luma_dc"], skip[1], out["chroma_dc"], ref_slot_out=np.arange(F, 2 * F, dtype=np.int32))
    eng.close()


@pytest.mark.gpu
def test_late_skip_zero_changes_nothing():
    """late_skip = 0 is the engine without the field: same launches, bytes and outputs; late_skip = 1 adds its launches
    and leaves every other output as it was."""
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    geom = Geometry(200, 130)
    F = 2
    planes, pred, bsize = _stack(_frames(geom, F, seed=9))
    base = dict(nframes=F, q0=45, pvq_qm_q4=Q4, inter=1, symbol_stream=2, inter_finish=1)
    engines = [engine.KeyframeEngine(geom, **base), engine.KeyframeEngine(geom, late_skip=0, **base),
               engine.KeyframeEngine(geom, late_skip=1, **base)]
    outs = [_copy(e.encode(planes, bsize, pred=pred)) for e in engines]
    assert engines[0].launches_per_step() == engines[1].launches_per_step()
    assert engines[2].launches_per_step() == engines[0].launches_per_step() + 5
    assert engines[0].buf.bytes_allocated == engines[1].buf.bytes_allocated < engines[2].buf.bytes_allocated
    idx = outs[0]["sym_index"]
    used = dict(sym_blocks=int(idx[:, 1].sum()), sym_dc=int(idx[:, 1].sum()), sym_bands=int(idx[:, 3].sum()),
                sym_pulses=int(idx[:, 5].sum()))   # the stream buffers' tails are not written
    for k in outs[0]:
        n = used.get(k)
        for o in outs[1:]:
            assert np.array_equal(outs[0][k][:n], o[k][:n]), k
    assert set(outs[2]) - set(outs[0]) == {"luma_late_skip", "chroma_late_skip", "sym_late_skip"}
    for p in range(3):
        assert np.array_equal(engines[0].coeff_plane(p), engines[2].coeff_plane(p))
    for e in engines:
        e.close()


@pytest.mark.gpu
def test_refusals():
    from daala_b200 import engine, symbols
    from daala_b200.frame import Geometry
    geom = Geometry(200, 130)
    F = 2
    for kw in (dict(late_skip=1), dict(inter=1, late_skip=2), dict(inter=1, late_skip=-1)):
        with pytest.raises(RuntimeError, match="late_skip"):
            engine.KeyframeEngine(geom, nframes=F, q0=45, pvq_qm_q4=Q4, **kw)
    planes, pred, bsize = _stack(_frames(geom, F, seed=5))
    recs = engine.Pinned((4096,), symbols.LATE_SKIP_DTYPE)

    def refused(eng, io, words):
        assert eng.L.daala_b200_kf_submit(eng.kf, ctypes.byref(io)) == INVALID
        msg = eng.L.daala_b200_kf_error(eng.kf)
        assert all(w in msg for w in words), msg
        assert int(eng.counts()[engine.CNT["n_luma"]]) == 0   # nothing was launched

    # an engine without late_skip: block order and stream order
    plain = engine.KeyframeEngine(geom, nframes=F, q0=45, pvq_qm_q4=Q4, inter=1, symbol_stream=2)
    plain.stage_inputs(planes, bsize, pred=pred)
    plain.prepare_io()
    for field in ("luma_late_skip", "chroma_late_skip", "sym_late_skip"):
        io = engine.IO.from_buffer_copy(plain._io)
        setattr(io, field, recs.ptr)
        io.sym_late_skip_cap = 4096
        refused(plain, io, [b"late_skip = 1"])
    plain.close()
    # sym_late_skip without symbol_stream = 2
    eng = _engine(geom, F, 45)
    eng.stage_inputs(planes, bsize, pred=pred)
    eng.prepare_io()
    io = engine.IO.from_buffer_copy(eng._io)
    io.sym_late_skip, io.sym_late_skip_cap = recs.ptr, 4096
    refused(eng, io, [b"sym_late_skip", b"symbol_stream = 2"])
    eng.close()
    # below the bound, and pageable memory
    eng = _engine(geom, F, 45, symbol_stream=2)
    eng.stage_inputs(planes, bsize, pred=pred)
    eng.prepare_io()
    io = eng._io
    cap = io.sym_late_skip_cap
    io.sym_late_skip_cap = cap - 1
    refused(eng, io, [b"sym_late_skip", b"pinned"])
    io.sym_late_skip_cap = cap
    ptr = io.sym_late_skip
    host = np.zeros(int(cap) * 32 + 64, np.uint8)
    io.sym_late_skip = host.ctypes.data
    refused(eng, io, [b"sym_late_skip", b"pinned"])
    io.sym_late_skip = ptr
    eng.submit()
    out = _copy(eng.wait())
    assert (_as_array(out["luma_late_skip"]) > 0).any()
    eng.close()
    recs.free()


# ---- no GPU ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("flat,masking", [(1, 1), (0, 1), (0, 0)])
def test_oracle_driver_port_matches_reference(flat, masking):
    """The late-skip driver bound to the port equals the one bound to the reference build (bit for bit: the port's
    od_compute_dist is the reference's operation order on the same libm), on a coded plane of the inter oracle."""
    from daala_b200 import synth
    from daala_b200.frame import Geometry
    from tests import inter_oracle
    ref = late_skip_oracle.load_ref()
    if ref is None:
        pytest.skip("needs the reference build")
    port = oracle_lib.load_port()
    geom = Geometry(200, 130)
    planes, pred, bsize = _frames(geom, 1, seed=4)[0]
    coded = inter_oracle.inter_chain(port, "port", planes, pred, geom, bsize, 45, Q4)
    for p in range(3):
        a = late_skip_oracle.plane(ref, "ref", planes[p], pred[p], coded[p]["dq"], geom, bsize, p, 45, Q4, flat, masking, 40)
        b = late_skip_oracle.plane(port, "port", planes[p], pred[p], coded[p]["dq"], geom, bsize, p, 45, Q4, flat, masking,
                                   40)
        assert np.array_equal(a, b), p
        assert (a[..., 0] > 0).any()


SRC = r"""
#include <stddef.h>
#include <stdio.h>
#include "daala_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(daala_b200_kf_late_skip),
         offsetof(daala_b200_kf_late_skip, noskip_pred_dcq), sizeof(daala_b200_kf_config),
         offsetof(daala_b200_kf_config, late_skip), sizeof(daala_b200_kf_io), offsetof(daala_b200_kf_io, luma_late_skip),
         offsetof(daala_b200_kf_io, sym_late_skip), offsetof(daala_b200_kf_io, sym_late_skip_cap));
  return 0;
}
"""


def test_late_skip_structs_match_the_header(tmp_path):
    from daala_b200 import engine, symbols
    (tmp_path / "layout.c").write_text(SRC)
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(tmp_path / "layout.c"), "-o", exe], check=True)
    got = [int(v) for v in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [symbols.LATE_SKIP_DTYPE.itemsize, symbols.LATE_SKIP_DTYPE.fields["noskip_pred_dcq"][1],
                   ctypes.sizeof(engine.Config), engine.Config.late_skip.offset, ctypes.sizeof(engine.IO),
                   engine.IO.luma_late_skip.offset, engine.IO.sym_late_skip.offset, engine.IO.sym_late_skip_cap.offset]


def test_candidate_rule():
    """lateskip.q1 is OD_DIV_R0 (C division), and the field chosen per (pvq_skip, dc) pair."""
    from daala_b200 import lateskip
    x = np.array([-7, -6, -5, -1, 0, 1, 5, 6, 7, 100, -100])
    assert lateskip.q1(x, 4).tolist() == [int((v + (-1 if v < 0 else 1)) / 4) for v in x]
    assert lateskip.field(0, 0) == "noskip_coded_dc0" and lateskip.field(0, 3) == "noskip_coded_dcq"
    assert lateskip.field(1, -2) == "noskip_pred_dcq" and lateskip.field(1, 0) is None
    rec = dict(dist_skip=100.0, noskip_coded_dc0=90.0, noskip_coded_dcq=200.0, noskip_pred_dcq=50.0)
    assert not lateskip.decide(rec, 0, 0, 10, 10, 1.0) and lateskip.decide(rec, 0, 1, 10, 10, 1.0)
    assert lateskip.decide(rec, 0, 0, 30, 10, 1.0) and not lateskip.decide(rec, 1, 0, 1000, 0, 1.0)
    assert lateskip.dc_quant(45, Q4, 0, 4).tolist() == max(1, (45 * 20) >> 4)
