#!/usr/bin/env python
"""Generates tests/golden/reference_vectors.npz by EXECUTING the reference build (oracle/_ref, compiled
from the reference sources by oracle/Makefile) on seeded inputs.  The reference ships no golden vectors
(SURVEY.md 4 / 8(c)); these are ours, so that the plain-C port (and through it the CUDA path) stays
pinned where oracle/_ref cannot be rebuilt.  Run from the repo root:  python tests/golden/make_golden.py
(`... make_golden.py digests` writes tests/golden/reference_digests.npz instead, `... make_golden.py settings`
tests/golden/encoder_settings.npz).

Inputs are stored next to the outputs (not regenerated from seeds), except for whole planes, which are
rebuilt by daala_b200.synth (deterministic integer generator) and stored as CRC-32 of the reference output.
"""
import ctypes
import os
import sys
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import frame_oracle, oracle_lib, pvq_cases  # noqa: E402
from tests.oracle_lib import addr  # noqa: E402

FRAME = dict(w=200, h=130, f=3, prev_f=2, prev_seed=77, bsize_seed=5, q0=45, q4=20, lam=0.147)
MC_IMG = dict(h=160, w=192, seed=5)


def crc(a):
    return zlib.crc32(np.ascontiguousarray(a).tobytes()) & 0xffffffff


def mc_image():
    rng = np.random.default_rng(MC_IMG["seed"])
    h, w = MC_IMG["h"], MC_IMG["w"]
    y, x = np.mgrid[0:h, 0:w]
    img = 128 + 60 * np.sin(x / 7.0) + 40 * np.cos(y / 5.0) + rng.integers(-20, 21, size=(h, w))
    return np.clip(img, 0, 255).astype(np.uint8)


def frame_inputs():
    from daala_b200 import synth
    from daala_b200.frame import Geometry
    geom = Geometry(FRAME["w"], FRAME["h"])
    planes, _ = synth.frame(FRAME["w"], FRAME["h"], f=FRAME["f"])
    prev, _ = synth.frame(FRAME["w"], FRAME["h"], f=FRAME["prev_f"], seed=FRAME["prev_seed"])
    return geom, synth.pad_planes(planes, geom), synth.pad_planes(prev, geom), \
        synth.block_size_map(geom, "mixed", seed=FRAME["bsize_seed"])


def frame_crcs(lib, prefix, qm, qm_inv):
    """CRC-32 of every plane the frame drivers produce (forward, PVQ key / inter / predicted, inverse)."""
    geom, planes, prev, bsize = frame_inputs()
    q4 = np.full((3, 30), FRAME["q4"], np.uint8)
    out = {}
    luma_q = None
    for pli in range(3):
        for key in (1, 0):
            d = frame_oracle.forward_plane(lib, prefix, planes[pli], geom, pli, bsize, key)
            out["fwd_p%d_k%d" % (pli, key)] = crc(d)
            md = frame_oracle.forward_plane(lib, prefix, prev[pli], geom, pli, bsize, 0) if not key else None
            dq, stats = frame_oracle.pvq_plane(lib, prefix, d, md, geom, pli, bsize, FRAME["q0"], key, 1, FRAME["lam"],
                                               qm, qm_inv, q4)
            out["pvq_p%d_k%d" % (pli, key)] = crc(dq)
            out["inv_p%d_k%d" % (pli, key)] = crc(frame_oracle.inverse_plane(lib, prefix, dq, geom, pli, bsize, key))
        d = frame_oracle.forward_plane(lib, prefix, planes[pli], geom, pli, bsize, 1)
        dq, _ = frame_oracle.pvq_plane_pred(lib, prefix, d, geom, pli, bsize, FRAME["q0"], 1, FRAME["lam"], qm, qm_inv,
                                            q4, luma_d=luma_q)
        if pli == 0:
            luma_q = dq
        out["pred_p%d" % pli] = crc(dq)
    return out


def dering_image(nvsb, nhsb, sb, seed):
    rng = np.random.default_rng(seed)
    h, w = nvsb * sb, nhsb * sb
    yy, xx = np.mgrid[0:h, 0:w]
    img = 900 * np.sign(np.sin((xx * 0.9 + yy * 0.4) / 6.0)) + 300 * np.sin(yy / 3.0) + rng.integers(-40, 41, size=(h, w))
    return np.clip(np.round(img), -2048, 2047).astype(np.int16)


def dering_cases(fn):
    """fn(y, ystride, x, xstride, nhb, nvb, sbx, sby, nhsb, nvsb, xdec, dir, pli, bskip, skip_stride, threshold,
    overlap, coeff_shift) -- od_dering without the vtable.  Returns (case rows, CRC of output + directions)."""
    rows, crcs = [], []
    nhsb, nvsb = 3, 2
    Dir = (ctypes.c_int * 8) * 8
    for xdec in (0, 1):
        sb = 64 >> xdec
        img = dering_image(nvsb, nhsb, sb, 31 + xdec)
        w = img.shape[1]
        rng = np.random.default_rng(17 + xdec)
        skip_stride = nhsb * 16
        for threshold, overlap in ((19, 0), (64, 1), (200, 1)):
            bskip = (rng.random((nvsb * 16, skip_stride)) < 0.4).astype(np.uint8)
            for sby in range(nvsb):
                for sbx in range(nhsb):
                    d = Dir()
                    vals = rng.integers(0, 8, size=(8, 8))
                    for r in range(8):
                        for c in range(8):
                            d[r][c] = int(vals[r, c])
                    y = np.zeros((sb, sb), np.int16)
                    fn(addr(y), sb, addr(img, sby * sb * w + sbx * sb), w, 8, 8, sbx, sby, nhsb, nvsb, xdec, d,
                       1 if xdec else 0, addr(bskip, (sby * 16) * skip_stride + sbx * 16), skip_stride, threshold,
                       overlap, 4)
                    rows.append([xdec, threshold, overlap, sbx, sby])
                    crcs.append(crc(y) ^ crc(np.array([list(r) for r in d], np.int32)))
    return rows, crcs


def real_map_crcs(lib, prefix, qm, qm_inv, bsize):
    """Keyframe chain with prediction on the golden picture with an externally decided block-size map."""
    geom, planes, _, _ = frame_inputs()
    q4 = np.full((3, 30), FRAME["q4"], np.uint8)
    out, luma_q = {}, None
    for pli in range(3):
        d = frame_oracle.forward_plane(lib, prefix, planes[pli], geom, pli, bsize, 1)
        dq, _ = frame_oracle.pvq_plane_pred(lib, prefix, d, geom, pli, bsize, FRAME["q0"], 1, FRAME["lam"], qm, qm_inv,
                                            q4, luma_d=luma_q)
        if pli == 0:
            luma_q = dq
        out["fwd_p%d" % pli], out["pred_p%d" % pli] = crc(d), crc(dq)
        out["inv_p%d" % pli] = crc(frame_oracle.inverse_plane(lib, prefix, dq, geom, pli, bsize, 1))
    return out


def main():
    ref = oracle_lib.load_ref()
    assert ref is not None, "needs oracle/_ref (make -C oracle ref, with the reference sources present)"
    rng = np.random.default_rng(20260923)
    g = {}
    # 2-D DCTs, Haar
    for ln in (2, 3, 4, 5, 6):
        n = 1 << ln
        x = (rng.integers(-300, 301, size=(2, n, n)) * 16).astype(np.int32)
        y = np.zeros_like(x)
        for i in range(2):
            getattr(ref, "od_bin_fdct%dx%d" % (n, n))(addr(y[i]), n, addr(x[i]), n)
        g["dct_x_%d" % ln], g["dct_y_%d" % ln] = x, y
    for ln in (1, 2, 3, 4, 5, 6):
        n = 1 << ln
        x = rng.integers(-(1 << 14), 1 << 14, size=(n, n)).astype(np.int32)
        y = np.zeros_like(x)
        ref.od_haar(addr(y), n, addr(x), n, ln)
        g["haar_x_%d" % ln], g["haar_y_%d" % ln] = x, y
    # lapping filters
    for n in (4, 8, 16, 32):
        x = rng.integers(-40000, 40000, size=(40, n)).astype(np.int32)
        y = np.zeros_like(x)
        z = np.zeros_like(x)
        for i in range(len(x)):
            getattr(ref, "od_pre_filter%d" % n)(addr(y[i]), addr(x[i]))
            getattr(ref, "od_post_filter%d" % n)(addr(z[i]), addr(x[i]))
        g["filt_x_%d" % n], g["filt_pre_%d" % n], g["filt_post_%d" % n] = x, y, z
    # pvq_theta (speed = 1): scalar results + vectors, inputs regenerated from pvq_cases (stored too)
    qm, qm_inv = pvq_cases.reference_qm(ref)
    g["qm"], g["qm_inv"] = qm, qm_inv
    rows, ys, outs, xs, rs = [], [], [], [], []
    for c in pvq_cases.cases(seed=7, per_combo=2):
        if np.abs(c["x0"]).max() > 1500 * c["q0"]:
            continue   # gain / quantiser ratios the codec cannot reach; the reference overruns its candidate list there
        a = pvq_cases.run_theta(ref, "ref", c, qm, qm_inv)
        rows.append([c["n"], c["is_keyframe"], c["pli"], c["beta"], c["q0"], c["qm_off"], a["gain"], a["itheta"],
                     a["max_theta"], a["k"], len(a["y"])])
        xs.append(c["x0"]); rs.append(c["r0"]); ys.append(a["y"]); outs.append(a["out"])
        g.setdefault("theta_lam", []).append(c["lam"])
        g.setdefault("theta_skip_diff", []).append(a["skip_diff"])
    g["theta_rows"] = np.array(rows, np.int64)
    g["theta_lam"] = np.array(g["theta_lam"], np.float64)
    g["theta_skip_diff"] = np.array(g["theta_skip_diff"], np.float64)
    g["theta_x"], g["theta_r"] = np.concatenate(xs).astype(np.int32), np.concatenate(rs).astype(np.int32)
    g["theta_y"], g["theta_out"] = np.concatenate(ys).astype(np.int32), np.concatenate(outs).astype(np.int32)
    # motion compensation / matching
    img = mc_image()
    w = img.shape[1]
    I4 = ctypes.c_int32 * 4
    mrows, mcrc = [], []
    for lx, ly in ((2, 2), (3, 3), (4, 4), (5, 5), (6, 6), (3, 2)):
        for t in range(12):
            mvx, mvy = int(rng.integers(-60, 61)), int(rng.integers(-60, 61))
            if lx != ly and not (mvx & 7 or mvy & 7):
                mvx |= 1
            x0, y0 = 40 + int(rng.integers(0, 40)), 40 + int(rng.integers(0, 30))
            a = np.zeros((1 << lx) * (1 << ly), np.uint8)
            ref.oracle_ref_mc_predict1fmv8(addr(a), addr(img, y0 * w + x0), w, mvx, mvy, lx, ly)
            mrows.append([lx, ly, mvx, mvy, x0, y0]); mcrc.append(crc(a))
    g["mc1_rows"], g["mc1_crc"] = np.array(mrows, np.int64), np.array(mcrc, np.uint32)
    orows, ocrc = [], []
    for ln in (2, 3, 4, 5):
        n = 1 << ln
        for t in range(12):
            mvx = [int(v) for v in rng.integers(-40, 41, size=4)]
            mvy = [int(v) for v in rng.integers(-40, 41, size=4)]
            if t % 4 == 0:
                mvx[1], mvy[1] = mvx[0], mvy[0]
            oc, s = int(rng.integers(0, 4)), int(rng.integers(0, 4))
            a = np.zeros((n, n), np.uint8)
            ref.oracle_ref_mc_predict(addr(a), n, addr(img, 45 * w + 50), w, I4(*mvx), I4(*mvy), oc, s, ln, ln)
            orows.append([ln, oc, s] + mvx + mvy); ocrc.append(crc(a))
    g["obmc_rows"], g["obmc_crc"] = np.array(orows, np.int64), np.array(ocrc, np.uint32)
    srows = []
    for ln in (2, 3, 4, 5, 6):
        n = 1 << ln
        a = rng.integers(0, 256, size=(n, n), dtype=np.uint8)
        b = np.clip(a.astype(int) + rng.integers(-30, 31, size=a.shape), 0, 255).astype(np.uint8)
        g["sad_a_%d" % ln], g["sad_b_%d" % ln] = a, b
        srows.append([ln, getattr(ref, "od_mc_compute_sad8_%dx%d_c" % (n, n))(addr(a), n, addr(b), n),
                      getattr(ref, "od_mc_compute_satd8_%dx%d_c" % (n, n))(addr(a), n, addr(b), n)])
    g["sad_rows"] = np.array(srows, np.int64)
    # whole planes
    fc = frame_crcs(ref, "ref", qm, qm_inv)
    g["frame_keys"] = np.array(sorted(fc))
    g["frame_crc"] = np.array([fc[k] for k in sorted(fc)], np.uint32)
    # deringing of whole superblocks (oracle of the next hot-path row)
    drows, dcrc = dering_cases(lambda *a: ref.od_dering(
        ctypes.c_void_p(ctypes.addressof(ctypes.c_void_p.in_dll(ref, "OD_DERING_VTBL_C"))), *a))
    g["dering_rows"], g["dering_crc"] = np.array(drows, np.int64), np.array(dcrc, np.uint32)
    # the same picture with the block sizes the whole reference encoder decides (public API, complexity 7)
    from daala_b200 import synth
    src, _ = synth.frame(FRAME["w"], FRAME["h"], f=FRAME["f"])
    geom = frame_inputs()[0]
    real = np.zeros(geom.bsize_shape, np.uint8)
    dering = np.zeros((geom.nvsb, geom.nhsb), np.uint8)
    nbytes, csum = ctypes.c_long(0), ctypes.c_uint(0)
    rc = ref.oracle_ref_encode_keyframe(FRAME["w"], FRAME["h"], addr(np.ascontiguousarray(src[0])),
                                        addr(np.ascontiguousarray(src[1])), addr(np.ascontiguousarray(src[2])), 20, 7,
                                        addr(real), addr(dering), ctypes.byref(nbytes), ctypes.byref(csum))
    assert rc == 0
    g["real_bsize"], g["real_dering_levels"] = real, dering
    g["real_packet"] = np.array([nbytes.value, csum.value], np.int64)
    rc_crc = real_map_crcs(ref, "ref", qm, qm_inv, real)
    g["real_keys"] = np.array(sorted(rc_crc))
    g["real_crc"] = np.array([rc_crc[k] for k in sorted(rc_crc)], np.uint32)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_vectors.npz")
    np.savez_compressed(path, **g)
    print("wrote %s (%d arrays, %d bytes)" % (path, len(g), os.path.getsize(path)))


THETA_SETS = ([("seed%d" % s, dict(seed=s, per_combo=3)) for s in (1, 2, 3, 4, 5)] + [("large_k", None)] +
              [("quantizer_range", "quantizer_range")])


def theta_case_set(name):
    """The pvq_theta cases of tests/test_emu_pvq_warp.py recorded under `name`."""
    kw = dict(THETA_SETS)[name]
    if kw == "quantizer_range":
        return pvq_cases.quantizer_range_cases()
    return pvq_cases.large_k_cases() if kw is None else pvq_cases.cases(**kw)


def tf_cases():
    """Seeded calls of the TF helpers (src/tf.c:38-277) with strided source and destination, every size the
    codec's blocks can take: (name, destination shape, source, trailing arguments)."""
    rng = np.random.default_rng(5)

    def case(name, shape_dst, shape_src, *args):
        return name, shape_dst, rng.integers(-4000, 4000, size=shape_src).astype(np.int32), args

    for n in (4, 8, 16, 32, 64):
        h = n // 2
        yield case("od_tf_up_h_lp", (n, n + 2), (n, n + 5), h, n)
        yield case("od_tf_up_v_lp", (n, n + 2), (n, n + 5), h, n)
        yield case("od_tf_up_hv_lp", (n, n + 2), (n, n + 5), h, h, n)
        yield case("od_tf_down_hv", (n, n + 2), (n, n + 5), n)
        yield case("od_tf_filter_2d", (n, n + 2), (n, n + 5), n)
        yield case("od_tf_filter_inv_2d", (n, n + 2), (n, n + 5), n)
    for n in (4, 8, 16, 32):
        yield case("od_tf_up_hv", (2 * n, 2 * n + 1), (2 * n, 2 * n + 3), n)
    for cur in range(5):
        for dest in range(cur + 1):
            for filt in (0, 1):
                n = 4 << cur
                yield case("od_convert_block_down", (n, n + 1), (n, n + 3), cur, dest, filt)


def run_tf(lib, case):
    """One tf_cases() call through `lib`; the destination starts filled with 77 so that stray writes show."""
    name, shape_dst, src, args = case
    d = np.full(shape_dst, 77, np.int32)
    getattr(lib, name)(addr(d), shape_dst[1], addr(src), src.shape[1], *args)
    return d


def main_digests():
    """tests/golden/reference_digests.npz: the reference's pvq_theta (speed = 1) on every case the device
    quantiser's CPU emulation is checked on, as pvq_cases.digest rows and skip_diff, and the CRC-32 of
    every tf_cases() result of the reference's TF helpers."""
    ref = oracle_lib.load_ref()
    assert ref is not None, "needs oracle/_ref (make -C oracle ref, with the reference sources present)"
    qm, qm_inv = pvq_cases.reference_qm(ref)
    g = {}
    for name, _ in THETA_SETS:
        rows, sd = [], []
        for c in theta_case_set(name):
            a = pvq_cases.run_theta(ref, "ref", c, qm, qm_inv)
            rows.append(pvq_cases.digest(a))
            sd.append(a["skip_diff"])
        g[name], g[name + "_skip_diff"] = np.array(rows, np.int64), np.array(sd, np.float64)
    g["tf_crc"] = np.array([crc(run_tf(ref, c)) for c in tf_cases()], np.uint32)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_digests.npz")
    np.savez_compressed(path, **g)
    print("wrote %s (%d arrays, %d bytes)" % (path, len(g), os.path.getsize(path)))


# The encoder's quantizer setting (OD_SET_QUANT) at each sweep point of tests/test_gpu_engine_quantizer_range.py.  The
# keyframe gets a finer coded quantizer than the P frame that follows it (src/rate.c:765-835): 1 is the finest setting
# (keyframe 4, P frame 6), 435 the first whose keyframe reaches 60 and P frame 63, the coarsest coded quantizer; 49's
# frames (40, 44) lie in od_compute_dist's interpolated range, coded quantizers 36..47.
SETTINGS_QUANT = (1, 5, 12, 18, 28, 49, 162, 435)
# (use_activity_masking, qm): OD_HVS_QM = 1 with and without masking, OD_FLAT_QM = 0 with masking
SETTINGS_CONFIGS = ((1, 1), (0, 1), (1, 0))
SETTINGS_PIC = (64, 64)


def capture_settings(ref, quant, masking, qm):
    """oracle_ref_encoder_settings: what the encoder set for its keyframe (index 0) and the P frame after it (1)."""
    S = 2 * pvq_cases.OD_QM_STRIDE
    out = dict(quantizer=np.zeros(2, np.int32), coded_quantizer=np.zeros(2, np.int32),
               pvq_qm_q4=np.zeros((2, 3, 30), np.uint8), qm=np.zeros((2, S), np.int16), qm_inv=np.zeros((2, S), np.int16),
               pvq_norm_lambda=np.zeros(2), dering_lambda=np.zeros(2))
    rc = ref.oracle_ref_encoder_settings(SETTINGS_PIC[0], SETTINGS_PIC[1], int(quant), int(masking), int(qm),
                                         *[addr(out[k]) for k in ("quantizer", "coded_quantizer", "pvq_qm_q4", "qm",
                                                                  "qm_inv", "pvq_norm_lambda", "dering_lambda")])
    assert rc == 0, rc
    # od_init_qm (src/pvq.c:322) writes only part of the state's buffers; the rest is whatever the allocator left there
    written = pvq_cases.reference_qm(ref, hvs=bool(qm))[0] != 0
    out["qm"][:, ~written] = 0
    out["qm_inv"][:, ~written] = 0
    return out


def main_settings():
    """tests/golden/encoder_settings.npz: capture_settings at every SETTINGS_QUANT x SETTINGS_CONFIGS point, arrays
    [point][config][frame]...; the matrices, which depend on qm alone, once per kind (qm_hvs / qm_flat)."""
    ref = oracle_lib.load_ref()
    assert ref is not None, "needs oracle/_ref (make -C oracle ref, with the reference sources present)"
    keys = ("quantizer", "coded_quantizer", "pvq_qm_q4", "pvq_norm_lambda", "dering_lambda")
    g = {k: [] for k in keys}
    mats = {}
    for quant in SETTINGS_QUANT:
        rows = {k: [] for k in keys}
        for masking, qm in SETTINGS_CONFIGS:
            s = capture_settings(ref, quant, masking, qm)
            name = "hvs" if qm else "flat"
            for m in ("qm", "qm_inv"):
                assert np.array_equal(s[m][0], s[m][1])
                mats.setdefault(m + "_" + name, s[m][0])
                assert np.array_equal(mats[m + "_" + name], s[m][0])
            for k in keys:
                rows[k].append(s[k])
        for k in keys:
            g[k].append(np.stack(rows[k]))
    g = {k: np.stack(v) for k, v in g.items()}
    g.update(mats)
    g["quant"] = np.array(SETTINGS_QUANT, np.int32)
    g["configs"] = np.array(SETTINGS_CONFIGS, np.int32)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "encoder_settings.npz")
    np.savez_compressed(path, **g)
    print("wrote %s (%d arrays, %d bytes)" % (path, len(g), os.path.getsize(path)))


if __name__ == "__main__":
    mode = sys.argv[1:]
    main_digests() if mode == ["digests"] else main_settings() if mode == ["settings"] else main()
