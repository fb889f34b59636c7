"""The warp-per-band PVQ quantiser of the device (daala_b200/csrc/pvq_warp.cuh) compiled for the host
on a SIMT emulation (tests/emu/simt_emu.h: 32 fibres, warp collectives as rendezvous) and pinned
against the reference build's pvq_theta, whose results on these cases tests/golden/make_golden.py recorded
in tests/golden/reference_digests.npz -- the same source the CUDA kernels include, so the candidate
parallelisation, the event order and the redux-screened pulse search are checked on the CPU."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from tests import pvq_cases
from tests.golden import make_golden
from tests.oracle_lib import addr

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
BUILD = os.path.join(HERE, "emu", "_build")
GOLDEN = os.path.join(HERE, "golden")


def _build(name, extra):
    os.makedirs(BUILD, exist_ok=True)
    out = os.path.join(BUILD, name)
    srcs = [os.path.join(HERE, "emu", "pvq_warp_emu.cpp"), os.path.join(HERE, "emu", "simt_emu.h"),
            os.path.join(ROOT, "daala_b200", "csrc", "pvq_warp.cuh"), os.path.join(ROOT, "daala_b200", "csrc", "pvq_math.cuh")]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in srcs):
        subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas"] + extra +
                       ["-I", os.path.join(ROOT, "daala_b200", "csrc"), "-I", os.path.join(HERE, "emu"), srcs[0], "-o", out],
                       check=True)
    lib = ctypes.CDLL(out)
    lib.emu_quantise_band.restype = ctypes.c_int
    return lib


def _run(emu, c, qm, qm_inv):
    n = c["n"]
    out = np.zeros(n, np.int32)
    y = np.zeros(n, np.int32)
    it, mt, vk = ctypes.c_int(0), ctypes.c_int(0), ctypes.c_int(0)
    sd = ctypes.c_double(0.0)
    x0 = np.ascontiguousarray(c["x0"])
    r0 = np.ascontiguousarray(c["r0"])
    q = np.ascontiguousarray(qm[c["qm_off"]:c["qm_off"] + n])
    qi = np.ascontiguousarray(qm_inv[c["qm_off"]:c["qm_off"] + n])
    g = emu.emu_quantise_band(addr(out), addr(x0), addr(r0), n, c["q0"], addr(y), ctypes.byref(it), ctypes.byref(mt),
                              ctypes.byref(vk), c["beta"], ctypes.byref(sd), c["is_keyframe"], c["pli"], addr(q), addr(qi),
                              ctypes.c_double(c["lam"]))
    ny = n if it.value == -1 else n - 1
    return dict(gain=g, itheta=it.value, max_theta=mt.value, k=vk.value, y=y[:ny].copy(), out=out, skip_diff=sd.value)


def _reference_qm():
    g = np.load(os.path.join(GOLDEN, "reference_vectors.npz"))
    return g["qm"], g["qm_inv"]


def _check_case_set(emu, name, qm, qm_inv):
    """Runs the emulated quantiser on the recorded case set `name`; returns the reference's K of every case."""
    gold = np.load(os.path.join(GOLDEN, "reference_digests.npz"))
    rows, skip_diff = gold[name], gold[name + "_skip_diff"]
    cases = list(make_golden.theta_case_set(name))
    assert len(cases) == len(rows)
    for c, want, want_sd in zip(cases, rows.tolist(), skip_diff.tolist()):
        got = _run(emu, c, qm, qm_inv)
        assert pvq_cases.digest(got) == want and got["skip_diff"] == want_sd, (
            {k: c[k] for k in ("n", "kind", "is_keyframe", "pli", "beta", "q0", "lam")}, want, want_sd, got)
    return rows[:, 3]


# the second build lowers the "products are exact" bound so that the literal-scan path of the plain
# pulses (taken on the device only when a product could exceed 2^53) runs on ordinary inputs
# third run: the same bands through the three phases with the band context parked in a record in between
# (the split kernels of the engine), size-class specialised instantiations
@pytest.mark.parametrize("name,extra,seeds,split", [("libpvq_warp_emu.so", [], (1, 2, 3, 5), False),
                                                    ("libpvq_warp_emu_scan.so", ["-DDAALA_B200_PVQ_EXACT_BOUND=1e12"], (1,), False),
                                                    ("libpvq_warp_emu.so", [], (4,), True)])
def test_warp_quantiser_matches_reference(name, extra, seeds, split, monkeypatch):
    emu = _build(name, extra)
    monkeypatch.delenv("DAALA_B200_EMU_SPLIT", raising=False)
    if split:
        monkeypatch.setenv("DAALA_B200_EMU_SPLIT", "1")
    qm, qm_inv = _reference_qm()
    stats = (ctypes.c_longlong * 4).in_dll(emu, "daala_b200_pvq_warp_stats")
    n = 0
    for seed in seeds:
        n += len(_check_case_set(emu, "seed%d" % seed, qm, qm_inv))
    # coverage: unique-contender fast path, both exact fallbacks, and (second build) the literal scan
    assert n >= 400 and stats[0] > 0 and stats[1] > 0 and stats[2] > 0
    if extra:
        assert stats[3] > 0


def test_warp_quantiser_large_k():
    """Fine quantisers on large vectors: K in the hundreds to thousands (all-RDO searches, 64-bit sums)."""
    emu = _build("libpvq_warp_emu.so", [])
    qm, qm_inv = _reference_qm()
    ks = _check_case_set(emu, "large_k", qm, qm_inv)
    assert len(ks) == 48 and ks.max() > 1000


def test_warp_quantiser_quantizer_range():
    """Band quantisers 1101 to 130521 (pvq_cases.quantizer_range_cases): the coarse end of the encoder's coded
    quantizers times its quantisation matrices, where most bands code a handful of pulses or none."""
    emu = _build("libpvq_warp_emu.so", [])
    qm, qm_inv = _reference_qm()
    ks = _check_case_set(emu, "quantizer_range", qm, qm_inv)
    assert (ks == 0).any() and ks.max() > 100


def test_port_quantiser_quantizer_range():
    """The oracle's plain-C port of pvq_theta on the same recorded cases."""
    from tests import oracle_lib
    port = oracle_lib.load_port()
    qm, qm_inv = _reference_qm()
    gold = np.load(os.path.join(GOLDEN, "reference_digests.npz"))
    rows, skip_diff = gold["quantizer_range"], gold["quantizer_range_skip_diff"]
    cases = list(make_golden.theta_case_set("quantizer_range"))
    assert len(cases) == len(rows)
    for c, want, want_sd in zip(cases, rows.tolist(), skip_diff.tolist()):
        got = pvq_cases.run_theta(port, "port", c, qm, qm_inv)
        assert pvq_cases.digest(got) == want and got["skip_diff"] == want_sd, (
            {k: c[k] for k in ("n", "kind", "is_keyframe", "pli", "beta", "q0", "lam")}, want, want_sd, got)
