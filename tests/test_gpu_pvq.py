"""GPU parity of the PVQ stage (through the C ABI) against the oracle:
indices (gain code, theta, K, pulses), synthesised coefficients and flags must
be bit-exact; the double-precision skip_diff within 1e-5 relative (north-star
tolerance for float gain/theta terms; it is normally exact too)."""
import numpy as np
import pytest

from tests import oracle_lib, pvq_oracle

pytestmark = pytest.mark.gpu


def _oracle():
    ref = oracle_lib.load_ref()
    return (ref, "ref") if ref is not None else (oracle_lib.load_port(), "port")


def _setup(size, is_keyframe, with_pred, mode="mixed", q0=38, seed=5):
    import torch
    from daala_b200 import pvq, synth
    from daala_b200.frame import FrameBuffers, Geometry
    geom = Geometry(*size)
    bsize = synth.block_size_map(geom, mode, seed=seed)
    cur = FrameBuffers(geom)
    planes, _ = synth.frame(size[0], size[1], f=3)
    cur.upload(synth.pad_planes(planes, geom), bsize)
    cur.haar_dc = 1 if is_keyframe else 0
    cur.forward()
    pred = None
    if with_pred:
        pred = FrameBuffers(geom)
        planes, _ = synth.frame(size[0], size[1], f=2, seed=777)
        pred.upload(synth.pad_planes(planes, geom), bsize)
        pred.haar_dc = 0
        pred.forward()
    torch.cuda.synchronize()
    blocks = pvq.block_list(bsize, geom)
    qm_q4 = np.full((3, 30), 16, np.uint8)
    qm_q4[0, :] = np.linspace(14, 40, 30).astype(np.uint8)
    qm_q4[1:, :] = np.linspace(20, 60, 30).astype(np.uint8)
    batch = pvq.PvqBatch(blocks, cur.coeffs, pred.coeffs if pred else None, q0=q0, is_keyframe=is_keyframe,
                         use_masking=1, pvq_qm_q4=qm_q4)
    return geom, cur, pred, batch, qm_q4


@pytest.mark.parametrize("is_keyframe,with_pred", [(1, False), (0, True), (1, True)])
def test_pvq_blocks_match_oracle(is_keyframe, with_pred):
    import torch
    from daala_b200 import pvq
    lib, prefix = _oracle()
    geom, cur, pred, batch, qm_q4 = _setup((256, 192), is_keyframe, with_pred)
    d_before = [t[0].cpu().numpy().copy() for t in cur.coeffs]
    p_planes = [t[0].cpu().numpy() for t in pred.coeffs] if pred else None
    batch.run()
    torch.cuda.synchronize()
    qm, qm_inv = pvq.default_qm(True)
    B = batch.blocks_np
    g_in, g_ref, g_out, g_y = (t.cpu().numpy() for t in (batch.in_, batch.ref, batch.out, batch.y))
    res = {k: getattr(batch, "res_" + k).cpu().numpy() for k in
           ("gain", "theta", "max_theta", "k", "skip_term", "skip_diff", "flip", "dc")}
    rng = np.random.default_rng(1)
    # every large block, a sample of the (many) small ones
    pick = [i for i in range(len(B)) if B["bs"][i] >= 2 or rng.random() < 0.12]
    assert len(pick) > 100
    nz = 0
    d_expect = [a.copy() for a in d_before]
    checked = set(pick)
    for i in pick:
        b = B[i]
        bs, pli, xdec = int(b["bs"]), int(b["pli"]), int(b["xdec"])
        n = 4 << bs
        ln = min(n * n, 512)
        off = int(b["coef_off"])
        dvec = pvq_oracle.coding_order(lib, prefix, d_before[pli], int(b["x0"]), int(b["y0"]), n)
        pvec = (pvq_oracle.coding_order(lib, prefix, p_planes[pli], int(b["x0"]), int(b["y0"]), n)
                if p_planes else np.zeros(n * n, np.int32))
        assert np.array_equal(g_in[off:off + ln], dvec[:ln])
        o = pvq_oracle.block(lib, prefix, dvec, pvec, bs, pli, xdec, 38, is_keyframe, 1, 0.147, qm, qm_inv, qm_q4)
        assert res["flip"][i] == o["flip"]
        assert np.array_equal(g_ref[off:off + ln], o["ref"][:ln])
        for band, r in enumerate(o["bands"]):
            j = i * 9 + band
            key = (i, band, bs, pli)
            assert (res["gain"][j], res["theta"][j], res["max_theta"][j], res["k"][j]) == \
                (r["gain"], r["itheta"], r["max_theta"], r["k"]), key
            assert res["skip_term"][j] == pytest.approx(r["skip_diff"], rel=1e-5, abs=1e-9), key
            nz += r["k"] > 0
        assert np.array_equal(g_y[off + 1:off + ln], o["y"][1:ln]), (i, bs, pli)
        assert np.array_equal(g_out[off + 1:off + ln], o["out"][1:ln]), (i, bs, pli)
        assert res["skip_diff"][i] == pytest.approx(o["skip_diff"], rel=1e-5, abs=1e-9)
    assert nz > 50
    # scatter: coded prefix written back, rest = skipped-coefficient init
    d_after = [t[0].cpu().numpy() for t in cur.coeffs]
    for i in pick[:200]:
        b = B[i]
        bs, pli = int(b["bs"]), int(b["pli"])
        n = 4 << bs
        x0, y0, off = int(b["x0"]), int(b["y0"]), int(b["coef_off"])
        ln = min(n * n, 512)
        exp = np.zeros((n, n), np.int32)
        if not is_keyframe:
            exp[:] = p_planes[pli][y0:y0 + n, x0:x0 + n]
        vec = np.zeros(n * n, np.int32)
        vec[:ln] = g_out[off:off + ln]
        if is_keyframe:
            vec[0] = d_before[pli][y0, x0]
        tmp = np.zeros((n, n), np.int32)
        tmp[:] = exp
        pvq_oracle.from_coding_order(lib, prefix, tmp, 0, 0, n, vec)
        assert np.array_equal(d_after[pli][y0:y0 + n, x0:x0 + n], tmp), (i, bs, pli)


@pytest.mark.parametrize("is_keyframe", [1, 0])
def test_hot_path_planes_match_frame_oracle(is_keyframe):
    """forward -> PVQ -> inverse on the GPU against the same chain of the CPU
    oracle, whole planes: quantised coefficient planes and the 8-bit
    reconstruction must be identical."""
    import torch
    from daala_b200 import pvq, synth
    from daala_b200.frame import FrameBuffers, Geometry
    from daala_b200.pipeline import HotPath
    from tests import frame_oracle
    lib, prefix = _oracle()
    geom = Geometry(320, 200)
    planes, _ = synth.frame(320, 200, f=4)
    planes = synth.pad_planes(planes, geom)
    prev, _ = synth.frame(320, 200, f=3, seed=4242)
    prev = synth.pad_planes(prev, geom)
    bsize = synth.block_size_map(geom, "mixed", seed=9)
    q4 = np.full((3, 30), 20, np.uint8)
    hp = HotPath(geom, q0=45, is_keyframe=is_keyframe, pvq_qm_q4=q4)
    hp.fb.upload(planes, bsize)
    if not is_keyframe:
        pred = FrameBuffers(geom)
        pred.upload(prev, bsize)
        pred.haar_dc = 0
        pred.forward()
        hp.use_prediction(pred)
    hp.set_block_sizes([bsize])
    hp.run()
    torch.cuda.synchronize()
    qm, qm_inv = pvq.default_qm(True)
    for pli in range(3):
        d = frame_oracle.forward_plane(lib, prefix, planes[pli], geom, pli, bsize, is_keyframe)
        md = frame_oracle.forward_plane(lib, prefix, prev[pli], geom, pli, bsize, 0) if not is_keyframe else None
        dq, stats = frame_oracle.pvq_plane(lib, prefix, d, md, geom, pli, bsize, 45, is_keyframe, 1, 0.147,
                                           qm, qm_inv, q4)
        assert stats[0] > 0
        assert np.array_equal(hp.fb.coeffs[pli][0].cpu().numpy(), dq), "quantised plane %d" % pli
        rec = frame_oracle.inverse_plane(lib, prefix, dq, geom, pli, bsize, is_keyframe)
        assert np.array_equal(hp.fb.pixels_out[pli][0].cpu().numpy(), rec), "recon plane %d" % pli
        k_gpu = int(hp.batch.res_k.sum().item())
    # K checksum over all planes
    total_k = 0
    for pli in range(3):
        d = frame_oracle.forward_plane(lib, prefix, planes[pli], geom, pli, bsize, is_keyframe)
        md = frame_oracle.forward_plane(lib, prefix, prev[pli], geom, pli, bsize, 0) if not is_keyframe else None
        total_k += int(frame_oracle.pvq_plane(lib, prefix, d, md, geom, pli, bsize, 45, is_keyframe, 1, 0.147,
                                              qm, qm_inv, q4)[1][0])
    assert k_gpu == total_k


@pytest.mark.parametrize("is_keyframe,with_pred", [(1, False), (0, True), (1, True)])
def test_pvq_kernel_variants_agree(is_keyframe, with_pred):
    """The group-cooperative kernels (default), the same with the literal
    sequential arg-max scan forced, and the scalar thread-per-band kernels must
    produce identical indices, pulses and coefficients on a large batch."""
    import torch
    geom, cur, pred, batch, qm_q4 = _setup((640, 384), is_keyframe, with_pred, q0=30, seed=12)
    outs = []
    for mode in (2, 0, 1, 3):
        batch.mode = mode
        for t in (batch.out, batch.y, batch.res_gain, batch.res_theta, batch.res_k, batch.res_skip_term):
            t.zero_()
        batch.gather()
        batch.quantise()
        torch.cuda.synchronize()
        outs.append([t.clone() for t in (batch.out, batch.y, batch.res_gain, batch.res_theta, batch.res_max_theta,
                                         batch.res_k, batch.res_skip_term, batch.res_skip_diff)])
    assert int(outs[0][5].sum().item()) > 1000
    for other in outs[1:]:
        for a, b in zip(outs[0], other):
            assert torch.equal(a, b)


def test_keyframe_with_intra_and_cfl_prediction_matches_frame_oracle():
    """The complete keyframe chain of the reference on the GPU: forward, luma PVQ
    with H/V intra prediction (dependency wavefront), chroma PVQ with CfL, inverse."""
    import torch
    from daala_b200 import pvq, synth
    from daala_b200.frame import Geometry
    from daala_b200.pipeline import HotPath
    from tests import frame_oracle
    lib, prefix = _oracle()
    geom = Geometry(384, 256)
    q4 = np.full((3, 30), 20, np.uint8)
    nf = 2
    hp = HotPath(geom, nframes=nf, q0=45, is_keyframe=1, pvq_qm_q4=q4, keyframe_prediction=True)
    frames = []
    for f in range(nf):
        planes, _ = synth.frame(384, 256, f=5 + f)
        planes = synth.pad_planes(planes, geom)
        bsize = synth.block_size_map(geom, "mixed" if f == 0 else "8", seed=31 + f)
        hp.fb.upload(planes, bsize, frame=f)
        frames.append((planes, bsize))
    hp.set_block_sizes([b for _, b in frames])
    hp.run()
    torch.cuda.synchronize()
    qm, qm_inv = pvq.default_qm(True)
    for f, (planes, bsize) in enumerate(frames):
        d0 = frame_oracle.forward_plane(lib, prefix, planes[0], geom, 0, bsize, 1)
        q0, s0 = frame_oracle.pvq_plane_pred(lib, prefix, d0, geom, 0, bsize, 45, 1, 0.147, qm, qm_inv, q4)
        assert np.array_equal(hp.fb.coeffs[0][f].cpu().numpy(), q0), "luma frame %d" % f
        assert s0[2] > -s0[3]  # predictions were used
        for pli in (1, 2):
            dc = frame_oracle.forward_plane(lib, prefix, planes[pli], geom, pli, bsize, 1)
            qc, _ = frame_oracle.pvq_plane_pred(lib, prefix, dc, geom, pli, bsize, 45, 1, 0.147, qm, qm_inv, q4,
                                                luma_d=q0)
            assert np.array_equal(hp.fb.coeffs[pli][f].cpu().numpy(), qc), "chroma %d frame %d" % (pli, f)
            rec = frame_oracle.inverse_plane(lib, prefix, qc, geom, pli, bsize, 1)
            assert np.array_equal(hp.fb.pixels_out[pli][f].cpu().numpy(), rec)
        rec0 = frame_oracle.inverse_plane(lib, prefix, q0, geom, 0, bsize, 1)
        assert np.array_equal(hp.fb.pixels_out[0][f].cpu().numpy(), rec0)


def test_work_ordering_is_a_wave_preserving_permutation_and_does_not_change_results():
    """daala_b200_pvq_order_by_work only reorders a launch: same entries, every entry stays inside its
    wave's slice, heavier bins first; symbols with and without ordering are identical."""
    import torch
    from daala_b200 import synth
    from daala_b200.frame import Geometry
    from daala_b200.pipeline import HotPath
    geom = Geometry(384, 256)
    q4 = np.full((3, 30), 20, np.uint8)
    outs = []
    for order in (True, False):
        hp = HotPath(geom, nframes=1, q0=45, is_keyframe=1, pvq_qm_q4=q4, keyframe_prediction=True)
        planes, _ = synth.frame(384, 256, f=9)
        bsize = synth.block_size_map(geom, "mixed", seed=77)
        hp.fb.upload(synth.pad_planes(planes, geom), bsize, frame=0)
        hp.set_block_sizes([bsize])
        hp.batch_luma.order_by_work = hp.batch_chroma.order_by_work = order
        hp.run()
        torch.cuda.synchronize()
        outs.append([t.clone() for b in (hp.batch_luma, hp.batch_chroma) for t in b.symbol_tensors()])
        if order:
            bl = hp.batch_luma
            for k in (16, 32, 128):
                src, dst = bl.chain_lists[k].cpu().numpy(), bl.chain_ordered[k].cpu().numpy()
                for a, c in bl.chain_slices[k]:
                    assert np.array_equal(np.sort(src[a:a + c]), np.sort(dst[a:a + c]))
                assert np.array_equal(np.sort(bl.bulk_lists[k].cpu().numpy()), np.sort(bl.bulk_ordered[k].cpu().numpy()))
                bc = hp.batch_chroma
                assert np.array_equal(np.sort(bc.lists[k].cpu().numpy()), np.sort(bc.ordered[k].cpu().numpy()))
            # heaviest first: the energy of the first tenth of a chroma launch exceeds that of the last tenth
            lst = hp.batch_chroma.ordered[16].cpu().numpy().view(np.uint32)
            blk, band = (lst >> 4).astype(np.int64), (lst & 15).astype(np.int64)
            off = hp.batch_chroma.blocks_np["coef_off"].astype(np.int64)[blk]
            x = hp.batch_chroma.in_.cpu().numpy().astype(np.float64)
            from daala_b200.pvq import BAND_EDGES
            e = np.array([np.sum(x[o + BAND_EDGES[b]:o + BAND_EDGES[b + 1]] ** 2) for o, b in zip(off, band)])
            m = max(1, len(e) // 10)
            assert e[:m].mean() > e[-m:].mean()
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_frame_groups_and_graph_replay_give_the_same_planes():
    """pvq_groups only changes scheduling (per-group batches on their own streams) and a CUDA-graph
    replay re-issues the identical launches: coefficient and pixel planes are bit-identical."""
    import torch
    from daala_b200 import synth
    from daala_b200.frame import Geometry
    from daala_b200.pipeline import HotPath
    geom = Geometry(320, 192)
    q4 = np.full((3, 30), 18, np.uint8)
    frames = []
    for f in range(3):
        planes, _ = synth.frame(320, 192, f=20 + f)
        frames.append((synth.pad_planes(planes, geom), synth.block_size_map(geom, "mixed", seed=50 + f)))
    outs = []
    for groups, graph in ((1, False), (2, False), (3, True)):
        hp = HotPath(geom, nframes=3, q0=40, is_keyframe=1, pvq_qm_q4=q4, keyframe_prediction=True,
                     pvq_groups=groups)
        for f, (planes, bsize) in enumerate(frames):
            hp.fb.upload(planes, bsize, frame=f)
        hp.set_block_sizes([b for _, b in frames])
        if graph:
            hp.capture()
            for t in hp.fb.coeffs + hp.fb.pixels_out:
                t.zero_()
            assert hp.replay() == hp.graph_launches > 0
        else:
            hp.run()
        torch.cuda.synchronize()
        outs.append([t.clone() for t in hp.fb.coeffs + hp.fb.pixels_out])
        assert int(sum(b.res_k.sum().item() for b in hp.pvq_batches())) > 0
    for other in outs[1:]:
        for a, b in zip(outs[0], other):
            assert torch.equal(a, b)


def test_hot_path_matches_recorded_reference_checksums():
    """The device chain against tests/golden/reference_vectors.npz (plane CRC-32s recorded from the real
    reference build by tests/golden/make_golden.py): forward, keyframe / inter PVQ + inverse, and the
    keyframe chain with intra + CfL prediction.  Needs neither oracle/_ref nor the port."""
    import os
    import torch
    from daala_b200.frame import FrameBuffers
    from daala_b200.pipeline import HotPath
    from tests.golden import make_golden
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_vectors.npz"))
    want = dict(zip(gold["frame_keys"].tolist(), gold["frame_crc"].tolist()))
    F = make_golden.FRAME
    geom, planes, prev, bsize = make_golden.frame_inputs()
    q4 = np.full((3, 30), F["q4"], np.uint8)
    crc = make_golden.crc
    for key in (1, 0):
        hp = HotPath(geom, q0=F["q0"], is_keyframe=key, pvq_qm_q4=q4)
        hp.fb.upload(planes, bsize)
        if not key:
            pred = FrameBuffers(geom)
            pred.upload(prev, bsize)
            pred.haar_dc = 0
            pred.forward()
            hp.use_prediction(pred)
        hp.set_block_sizes([bsize])
        hp.fb.forward()
        torch.cuda.synchronize()
        for pli in range(3):
            assert crc(hp.fb.coeffs[pli][0].cpu().numpy()) == want["fwd_p%d_k%d" % (pli, key)], (pli, key)
        hp.run()
        torch.cuda.synchronize()
        for pli in range(3):
            assert crc(hp.fb.coeffs[pli][0].cpu().numpy()) == want["pvq_p%d_k%d" % (pli, key)], (pli, key)
            assert crc(hp.fb.pixels_out[pli][0].cpu().numpy()) == want["inv_p%d_k%d" % (pli, key)], (pli, key)
    hp = HotPath(geom, q0=F["q0"], is_keyframe=1, pvq_qm_q4=q4, keyframe_prediction=True)
    hp.fb.upload(planes, bsize)
    hp.set_block_sizes([bsize])
    hp.run()
    torch.cuda.synchronize()
    for pli in range(3):
        assert crc(hp.fb.coeffs[pli][0].cpu().numpy()) == want["pred_p%d" % pli], pli


def test_dropin_pvq_helper_symbols_match_oracle():
    """Host-pointer od_pvq_* helpers and od_rdo_quant against the reference build
    (or the port when oracle/_ref is absent)."""
    import ctypes
    from daala_b200 import _native
    from tests.oracle_lib import addr
    L = _native.lib()
    lib, prefix = _oracle()
    rng = np.random.default_rng(9)
    for fn in (L.od_pvq_sin, L.od_pvq_cos):
        fn.restype = ctypes.c_int16
    L.od_rdo_quant.restype = ctypes.c_int

    def o(name):
        return getattr(lib, ("od_" if prefix == "ref" else "port_") + name)
    if prefix == "ref":
        lib.od_pvq_sin.restype = lib.od_pvq_cos.restype = ctypes.c_int16
    for x in (0, 5, 20000, 32768, 40000, 70000, -300):
        assert L.od_pvq_sin(x) == np.int16(o("pvq_sin")(x)) and L.od_pvq_cos(x) == np.int16(o("pvq_cos")(x))
    for beta in (4096, 6144):
        for cg0, q0 in ((300, 64), (1000, 400), (20000, 8)):
            assert L.od_gain_expand(cg0, q0, beta) == o("gain_expand")(cg0, q0, beta)
        for qcg in (100, 358, 900, 4000):
            assert L.od_pvq_compute_max_theta(qcg, beta) == o("pvq_compute_max_theta")(qcg, beta)
            for n in (15, 8, 32, 128):
                exp = lib.od_pvq_compute_k(qcg, -1, -1, 1, n, beta, 1) if prefix == "ref" else \
                    lib.port_pvq_compute_k(qcg, -1, 1, n, beta)
                assert L.od_pvq_compute_k(qcg, -1, -1, 1, n, beta, 1) == exp
    for ts in (1, 5, 12):
        for t in (0, 3, 11):
            assert L.od_pvq_compute_theta(t, ts) == o("pvq_compute_theta")(t, ts)
    for n in (15, 8, 32, 128):
        x = rng.integers(-3000, 3000, size=n).astype(np.int16)
        r = rng.integers(-3000, 3000, size=n).astype(np.int16)
        g1, g2 = ctypes.c_int32(0), ctypes.c_int32(0)
        assert L.od_pvq_compute_gain(addr(x), n, 100, ctypes.byref(g1), 6144, 1) == \
            o("pvq_compute_gain")(addr(x), n, 100, ctypes.byref(g2), 6144, 1)
        assert g1.value == g2.value
        x32 = x.astype(np.int32) * 41
        assert L.od_vector_log_mag(addr(x32), n) == o("vector_log_mag")(addr(x32), n)
        ra, rb = r.copy(), r.copy()
        sa, sb = ctypes.c_int(0), ctypes.c_int(0)
        gr = int(np.sqrt(float((r.astype(np.int64) ** 2).sum())))
        assert L.od_compute_householder(addr(ra), n, gr, ctypes.byref(sa), 0) == \
            o("compute_householder")(addr(rb), n, gr, ctypes.byref(sb), 0)
        assert sa.value == sb.value and np.array_equal(ra, rb)
        oa, ob = np.zeros(n, np.int16), np.zeros(n, np.int16)
        L.od_apply_householder(addr(oa), addr(x), addr(ra), n)
        o("apply_householder")(addr(ob), addr(x), addr(rb), n)
        assert np.array_equal(oa, ob)
        qmi = rng.integers(2000, 6000, size=n).astype(np.int16)
        for noref in (1, 0):
            y = np.zeros(n, np.int32)
            y[rng.integers(0, n - 1, size=5)] = rng.integers(-3, 4, size=5)
            xa, xb = np.zeros(n, np.int32), np.zeros(n, np.int32)
            L.od_pvq_synthesis_partial(addr(xa), addr(y), addr(ra), n, noref, 5000, 9000, 3, -1, addr(qmi))
            o("pvq_synthesis_partial")(addr(xb), addr(y), addr(rb), n, noref, 5000, 9000, 3, -1, addr(qmi))
            assert np.array_equal(xa, xb)
    if prefix == "ref":
        lib.od_rdo_quant.restype = ctypes.c_int
        for x in (-900, -100, -3, 0, 5, 77, 400, 12345):
            for q in (7, 64, 300):
                for d0 in (0.0, 1.3, 7.5):
                    assert L.od_rdo_quant(x, q, ctypes.c_double(d0), ctypes.c_double(0.147)) == \
                        lib.od_rdo_quant(x, q, ctypes.c_double(d0), ctypes.c_double(0.147))
