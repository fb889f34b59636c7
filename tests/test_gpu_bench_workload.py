"""The workload bench.py measures, checked whole against the oracle: 16 frames of 3840x2160 per batch, the
reference encoder's block-size maps and deringing levels, q0 72, the engine configured exactly as bench.py
configures it (max_blocks_div = 2, dering = 1).  Every frame, every plane and every output the
host reads is compared -- reconstruction, band records, pulses, quantised coefficient planes, per-block
skip_diff and CfL flip -- after the first submit, after the bench's timing sequence, and across two engines
used alternately.  The batch cycles 4 distinct frames, so the oracle runs once per distinct frame."""
import numpy as np
import pytest

import bench
from tests import frame_oracle
from tests.test_gpu_engine import _coding_tables, _oracle, _y_plane

pytestmark = [pytest.mark.gpu]
F = 16
DISTINCT = 4
Q4 = np.full((3, 30), bench.PVQ_QM_Q4, np.uint8)
SKIP_RTOL = 1e-9


def _geom():
    from daala_b200.frame import Geometry
    return Geometry(bench.PIC_W, bench.PIC_H)


def _engine(geom, nframes=F, dering=1):
    """A keyframe engine with bench.py's keyword arguments (reference block sizes, default options)."""
    from daala_b200 import engine
    return engine.KeyframeEngine(geom, nframes=nframes, q0=bench.Q0, use_masking=1, pvq_qm_q4=Q4, dering=dering,
                                 coded_quantizer=bench.CODED_Q, dering_lambda=bench.DERING_LAMBDA,
                                 persist_ctas_per_sm=0, max_blocks_div=2)


def _stage(eng, hf, dering_levels=True):
    eng.stage_inputs([np.stack([f[0][p] for f in hf]) for p in range(3)], np.stack([f[1] for f in hf]))
    if dering_levels:
        eng.stage_dering_levels(np.stack([f[2] for f in hf]))
    return eng.prepare_io(symbols=True, recon=True)


_JOB = {}


def _oracle_job(job):
    """One distinct frame through the oracle (runs in a forked worker, or inline): ("levels", k) with the bench's
    deringing levels and every symbol recorded, ("search", k) with the reference's deringing level search."""
    kind, k = job
    lib, prefix = _oracle()
    planes, bsize, levels = _JOB["frames"][k]
    geom = _JOB["geom"]
    if kind == "levels":
        return frame_oracle.keyframe_chain(lib, prefix, planes, geom, bsize, bench.Q0, Q4, use_masking=1,
                                           dering_levels=levels, symbols=True)
    out = frame_oracle.keyframe_chain(lib, prefix, planes, geom, bsize, bench.Q0, Q4, use_masking=1, record=False,
                                      dering_search=dict(coded_quantizer=bench.CODED_Q,
                                                         dering_lambda=bench.DERING_LAMBDA))
    return dict(levels=out[0]["dering_levels"], recon=[o["recon"] for o in out])


@pytest.fixture(scope="module")
def workload():
    """The distinct host frames and their oracle results, computed once for the module."""
    geom = _geom()
    frames = bench.make_host_frames(geom, DISTINCT, distinct=DISTINCT)
    _, prefix = _oracle()
    jobs = [("levels", k) for k in range(DISTINCT)]
    if prefix == "ref":
        jobs += [("search", k) for k in range(DISTINCT)]
    _JOB.update(geom=geom, frames=frames)
    cores = bench.usable_cores()[0]
    if cores > 1:
        import multiprocessing
        with multiprocessing.get_context("fork").Pool(min(cores, len(jobs))) as pool:
            res = pool.map(_oracle_job, jobs, chunksize=1)
    else:
        res = [_oracle_job(j) for j in jobs]
    want = res[:DISTINCT]
    search = res[DISTINCT:] if prefix == "ref" else None
    return dict(geom=geom, frames=frames, want=want, search=search, prefix=prefix, tabs=_coding_tables())


def _batch(workload, rotate):
    """bench.make_host_frames(geom, F, rotate=rotate) without synthesising the frames again: the distinct frames
    cycled from frame `rotate` on."""
    return [workload["frames"][(i + rotate) % DISTINCT] for i in range(F)]


def _order(blocks, sel):
    return sel[np.lexsort((blocks["x0"][sel], blocks["y0"][sel], blocks["pli"][sel]))]


def _segments(y16, blocks, order):
    """The pulse vectors of the blocks `order`, concatenated in that order."""
    length = np.minimum(16 << (2 * blocks["bs"][order].astype(np.int64)), 512)
    start = blocks["coef_off"][order].astype(np.int64)
    first = np.concatenate([[0], np.cumsum(length)[:-1]])
    idx = np.repeat(start - first, length) + np.arange(int(length.sum()))
    return y16[idx]


def _canon(out, f):
    """One frame of an engine's host outputs in an order that does not depend on how the device lists were
    built: per plane group the blocks sorted by (pli, y0, x0) with their band records, pulses, skip_diff and
    flip, and the three reconstructed planes.  Copies (the engine reuses its host buffers)."""
    c = {}
    for name in ("luma", "chroma"):
        b = out[name + "_blocks"]
        o = _order(b, np.nonzero(b["frame"] == f)[0])
        c[name + "_key"] = np.stack([b["pli"][o], b["y0"][o], b["x0"][o], b["bs"][o]], 1).astype(np.int32)
        c[name + "_res"] = out[name + "_res"][o].copy()
        c[name + "_pulses"] = _segments(out[name + "_y16"], b, o).copy()
        c[name + "_skip_diff"] = out[name + "_skip_diff"][o].copy()
    c["chroma_flip"] = out["chroma_flip"][_order(out["chroma_blocks"],
                                                  np.nonzero(out["chroma_blocks"]["frame"] == f)[0])].copy()
    for p in range(3):
        c["recon%d" % p] = out["recon%d" % p][f].copy()
    return c


def _assert_canon_equal(a, b, what):
    for k in a:
        assert a[k].dtype == b[k].dtype and a[k].tobytes() == b[k].tobytes(), (what, k)


def _check_frame(out, coeffs, f, want, geom, tabs):
    """Every output of frame f against the oracle's results `want` for its content."""
    from daala_b200 import engine
    for pli in range(3):
        name = "luma" if pli == 0 else "chroma"
        blocks, res = out[name + "_blocks"], out[name + "_res"]
        w = want[pli]
        assert np.array_equal(out["recon%d" % pli][f], w["recon"]), ("recon", f, pli)
        got = engine.band_records(blocks, res, geom, pli, f)
        bad = np.argwhere(got != w["rec"])
        assert len(bad) == 0, ("band records", f, pli, len(bad), bad[:8].tolist())
        assert np.array_equal(_y_plane(blocks, out[name + "_y16"], geom, pli, f, tabs), w["yplane"]), ("pulses", f, pli)
        assert np.array_equal(coeffs[pli][f], w["dq"]), ("quantised plane", f, pli)
        sel = np.nonzero((blocks["pli"] == pli) & (blocks["frame"] == f))[0]
        y4, x4 = blocks["y0"][sel] >> 2, blocks["x0"][sel] >> 2
        # one device block per oracle block origin
        assert len(sel) == int((~np.isnan(w["skip_diff"])).sum()), ("block count", f, pli)
        sd_dev, sd_ref = out[name + "_skip_diff"][sel], w["skip_diff"][y4, x4]
        assert not np.isnan(sd_ref).any(), ("block origins", f, pli)
        not_exact = int((sd_dev != sd_ref).sum())
        rel = np.abs(sd_dev - sd_ref) / np.maximum(np.abs(sd_ref), 1.0)
        assert rel.max(initial=0.0) <= SKIP_RTOL, ("skip_diff", f, pli, "max rel %.3g" % rel.max(initial=0.0), "not bit-identical",
                                                  not_exact)
        assert not_exact == 0, ("skip_diff within %g but not bit-identical" % SKIP_RTOL, f, pli, not_exact)
        if pli:
            flip = out["chroma_flip"][sel]
            bad = int((flip != w["flip"][y4, x4]).sum())
            assert bad == 0, ("chroma flip", f, pli, bad)


def _coeffs(eng):
    return [eng.coeff_plane(p) for p in range(3)]


@pytest.fixture(scope="module")
def first_pass(workload):
    """One submit / wait of the bench's first batch (rotation 0) on an engine configured as bench.py does; the
    engine then plays bench.py's first slot in the tests below."""
    from daala_b200 import engine
    geom = workload["geom"]
    hf = _batch(workload, 0)
    eng = _engine(geom)
    out = _stage(eng, hf)
    eng.submit()
    out = eng.wait()
    assert int(out["counts"][engine.CNT["error"]]) == 0
    canon = [_canon(out, f) for f in range(F)]
    coeffs = _coeffs(eng)
    yield dict(eng=eng, out=out, canon=canon, coeffs=coeffs)
    eng.close()


def test_every_frame_of_a_bench_batch_matches_oracle(workload, first_pass):
    """(a) All 16 frames, all planes: reconstruction, band records, pulses, quantised planes, skip_diff, flip."""
    out, coeffs = first_pass["out"], first_pass["coeffs"]
    flips = 0
    for f in range(F):
        want = workload["want"][f % DISTINCT]
        _check_frame(out, coeffs, f, want, workload["geom"], workload["tabs"])
        flips += int(out["chroma_flip"][out["chroma_blocks"]["frame"] == f].sum())
    assert flips > 0


def test_output_does_not_depend_on_position_in_batch(first_pass):
    """(b) Frames f, f+4, f+8, f+12 carry the same input: identical symbols, pulses, skip_diff, flip and planes."""
    canon, coeffs = first_pass["canon"], first_pass["coeffs"]
    for f in range(DISTINCT):
        for g in range(f + DISTINCT, F, DISTINCT):
            _assert_canon_equal(canon[f], canon[g], ("frames", f, g))
            for p in range(3):
                assert np.array_equal(coeffs[p][f], coeffs[p][g]), ("quantised plane", f, g, p)


def _device_outputs(eng):
    """What the device-resident step leaves in the engine's buffers, in block order as bench.dump_outputs
    reads it (not sampled): planes, coefficient planes, band results, pulses, skip_diff and flip."""
    from daala_b200 import engine, pvq
    d = {}
    for p in range(3):
        d["recon%d" % p] = eng.recon_plane(p)
        d["coeffs%d" % p] = eng.coeff_plane(p)
    cnt = eng.counts()
    for name, key in (("luma", "n_luma"), ("chroma", "n_chroma")):
        n = int(cnt[engine.CNT[key]])
        blocks = eng.download(getattr(eng.buf, name + "_blocks"), (n,), pvq.BLOCK_DTYPE)
        order = np.lexsort((blocks["x0"], blocks["y0"], blocks["pli"], blocks["frame"]))
        coefs = int(cnt[engine.CNT[name + "_coefs"]])
        d[name + "_band_results"] = eng.download(getattr(eng.buf, name + "_res"), (n, 9, 4), np.int16)[order]
        d[name + "_pulses"] = _segments(eng.download(getattr(eng.buf, name + "_y16"), (coefs,), np.int16), blocks, order)
        d[name + "_skip_diff"] = eng.download(getattr(eng.buf, name + "_skip_diff"), (n,), np.float64)[order]
        if name == "chroma":
            d["chroma_flip"] = eng.download(eng.buf.chroma_flip, (n,), np.int32)[order]
    return d


def test_steady_state_after_the_bench_timing_sequence(first_pass):
    """(c) The outputs left on the device after bench.py's timing calls (graph replays, every single-phase
    timing including the search-only ones, the closing replay) equal those of the first pass bit for bit."""
    from daala_b200 import engine
    eng = first_pass["eng"]
    before = _device_outputs(eng)
    # the first pass, as the host received it, is what the device holds
    for p in range(3):
        assert np.array_equal(before["recon%d" % p], first_pass["out"]["recon%d" % p])
    eng.time_device(engine.PH_ALL, True, 3)
    eng.time_device(engine.PH_ALL, True, 10)
    for ph in (engine.PH_LISTS, engine.PH_FORWARD, engine.PH_PVQ_LUMA, engine.PH_PVQ_CHROMA, engine.PH_INVERSE,
               engine.PH_PVQ_LUMA | engine.PH_SEARCH_ONLY, engine.PH_PVQ_CHROMA | engine.PH_SEARCH_ONLY):
        eng.time_device(ph, False, 1)
        eng.time_device(ph, False, 10)
    eng.time_device(engine.PH_ALL, True, 1)
    after = _device_outputs(eng)
    assert int(eng.counts()[engine.CNT["error"]]) == 0
    for k in before:
        assert before[k].dtype == after[k].dtype and before[k].tobytes() == after[k].tobytes(), k


def test_two_engines_used_alternately_match_oracle(workload, first_pass):
    """(d) bench.py's end-to-end loop: its two engines on batches rotated by 0 and 1 frames (the first is the
    engine of the first pass, as in bench.py), submit / wait alternating over 6 submits; after every wait that
    engine's outputs equal the oracle-checked outputs of its frames."""
    from daala_b200 import engine
    want = first_pass["canon"][:DISTINCT]          # checked against the oracle by test (a)
    rots = (0, 1)
    second = _engine(workload["geom"])
    _stage(second, _batch(workload, 1))
    slots = [first_pass["eng"], second]
    checked = [0, 0]

    def check(s):
        out = slots[s].wait()
        assert int(out["counts"][engine.CNT["error"]]) == 0
        for f in range(F):
            _assert_canon_equal(_canon(out, f), want[(f + rots[s]) % DISTINCT], ("engine", s, "frame", f))
        checked[s] += 1

    try:
        steps = 6
        for i in range(steps):
            s = i % 2
            if i >= 2:
                check(s)
            slots[s].submit()
        for s in range(2):
            check(s)
        assert checked == [3, 3]
    finally:
        second.close()


def test_dering_search_at_4k_matches_reference(workload):
    """(e) dering = 2 on the 4 distinct frames at 4K: every superblock's level equals the reference's own search
    loop (oracle_ref_dering_search), and the reconstruction equals the oracle's at those levels."""
    if workload["prefix"] != "ref":
        pytest.skip("needs the reference build (od_compute_dist, od_dering, od_encode_cdf_*)")
    geom = workload["geom"]
    hf = workload["frames"]
    eng = _engine(geom, nframes=DISTINCT, dering=2)
    try:
        _stage(eng, hf, dering_levels=False)
        eng.submit()
        out = eng.wait()
        seen = set()
        for f in range(DISTINCT):
            s = workload["search"][f]
            bad = np.argwhere(out["dering_levels"][f] != s["levels"])
            assert len(bad) == 0, ("levels", f, len(bad), bad[:8].tolist())
            seen |= set(s["levels"].ravel().tolist())
            for p in range(3):
                assert np.array_equal(out["recon%d" % p][f], s["recon"][p]), ("recon at the searched levels", f, p)
        assert len(seen) >= 2, seen
    finally:
        eng.close()
