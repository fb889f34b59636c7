"""GPU parity of the fused lapped-transform kernels (through the C ABI of
libdaala_b200.so) against the CPU oracle: bit-exact, integer work."""
import ctypes
import os
import zlib

import numpy as np
import pytest

from tests import frame_oracle, oracle_lib

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch


def checkers():
    """(name, lib, prefix) for every available oracle: the real reference when
    oracle/_ref is present, and always the plain-C port."""
    out = [("port", oracle_lib.load_port(), "port")]
    ref = oracle_lib.load_ref()
    if ref is not None:
        out.append(("ref", ref, "ref"))
    return out


@pytest.mark.parametrize("mode", ["mixed", "4", "8", "16", "32", "64"])
@pytest.mark.parametrize("size", [(200, 130), (64, 64), (320, 192)])
@pytest.mark.parametrize("haar", [1, 0])
def test_forward_inverse_frame_matches_oracle(torch_cuda, mode, size, haar):
    torch = torch_cuda
    from daala_b200 import synth
    from daala_b200.frame import FrameBuffers, Geometry
    geom = Geometry(*size)
    planes, _ = synth.frame(size[0], size[1], f=1)
    planes = synth.pad_planes(planes, geom)
    bsize = synth.block_size_map(geom, mode, seed=zlib.crc32(repr((mode, size)).encode()) & 0xffff)
    fb = FrameBuffers(geom)
    fb.haar_dc = haar
    fb.upload(planes, bsize)
    fb.forward()
    fb.inverse()
    torch.cuda.synchronize()
    for name, lib, prefix in checkers():
        for pli in range(3):
            d_gpu = fb.coeffs[pli][0].cpu().numpy()
            d_cpu = frame_oracle.forward_plane(lib, prefix, planes[pli], geom, pli, bsize, haar)
            assert np.array_equal(d_gpu, d_cpu), "forward %s plane %d" % (name, pli)
            lap_cpu = frame_oracle.inverse_plane(lib, prefix, d_cpu, geom, pli, bsize, haar, lapped_only=True)
            assert np.array_equal(fb.lapped[pli][0].cpu().numpy(), lap_cpu), "lapped %s plane %d" % (name, pli)
            rec_cpu = frame_oracle.inverse_plane(lib, prefix, d_cpu, geom, pli, bsize, haar)
            rec_gpu = fb.pixels_out[pli][0].cpu().numpy()
            assert np.array_equal(rec_gpu, rec_cpu), "recon %s plane %d" % (name, pli)
            # lossless transform chain: reconstruction == source
            assert np.array_equal(rec_gpu, planes[pli])


@pytest.mark.parametrize("size", [(1920, 1080), (3840, 2160)])
def test_full_size_round_trip_is_lossless(torch_cuda, size):
    """BASELINE.json sizes: no quantisation => inverse(forward(x)) == x exactly
    (the reversibility property dcttest checks per block, src/dct.c:8825)."""
    torch = torch_cuda
    from daala_b200 import synth
    from daala_b200.frame import FrameBuffers, Geometry
    geom = Geometry(*size)
    planes, _ = synth.frame(size[0], size[1], f=0)
    planes = synth.pad_planes(planes, geom)
    bsize = synth.block_size_map(geom, "mixed", seed=3)
    fb = FrameBuffers(geom)
    fb.upload(planes, bsize)
    fb.forward()
    fb.inverse()
    torch.cuda.synchronize()
    for pli in range(3):
        assert np.array_equal(fb.pixels_out[pli][0].cpu().numpy(), planes[pli])
    # and the coefficient plane is not trivially the input
    assert fb.coeffs[0].abs().max().item() > 255


@pytest.mark.parametrize("ln", [2, 3, 4, 5, 6])
def test_dropin_dct_symbols_match_oracle(torch_cuda, ln):
    """Section A of include/daala_b200.h: od_bin_fdctNxN / od_bin_idctNxN /
    od_bin_fdctN with host pointers, like dcttest's function tables
    (src/dct.c:8259-8260)."""
    from daala_b200 import _native
    L = _native.lib()
    port = oracle_lib.load_port()
    n = 1 << ln
    rng = np.random.default_rng(ln)
    fwd = getattr(L, "od_bin_fdct%dx%d" % (n, n))
    inv = getattr(L, "od_bin_idct%dx%d" % (n, n))
    f1 = getattr(L, "od_bin_fdct%d" % n)
    i1 = getattr(L, "od_bin_idct%d" % n)
    a = oracle_lib.addr
    for t in range(5):
        # ieee1180-style ranges (src/dct.c:8379-8409): (-256,255), (-5,5), (-300,300), scaled by 16
        lo, hi = [(-256, 255), (-5, 5), (-300, 300), (-256, 255), (-300, 300)][t]
        x = (rng.integers(lo, hi + 1, size=(n, n + 3)) * 16).astype(np.int32)
        y_gpu = np.zeros((n, n + 1), np.int32)
        y_cpu = np.zeros((n, n + 1), np.int32)
        fwd(a(y_gpu), n + 1, a(x), n + 3)
        port.port_bin_fdct2d(ln, a(y_cpu), n + 1, a(x), n + 3)
        assert np.array_equal(y_gpu, y_cpu)
        x_gpu = np.zeros((n, n + 3), np.int32)
        inv(a(x_gpu), n + 3, a(y_gpu), n + 1)
        assert np.array_equal(x_gpu[:, :n], x[:, :n])
        v = np.ascontiguousarray(x[0, :n])
        y1g = np.zeros(n, np.int32)
        y1c = np.zeros(n, np.int32)
        f1(a(y1g), a(v), 1)
        port.port_bin_fdct(ln, a(y1c), a(v), 1)
        assert np.array_equal(y1g, y1c)
        v2 = np.zeros(n, np.int32)
        i1(a(v2), 1, a(y1g))
        assert np.array_equal(v2, v)


@pytest.mark.parametrize("ln", [1, 2, 3, 4, 5, 6])
def test_haar_wavelet_matches_oracle(torch_cuda, ln):
    """od_haar / od_haar_inv drop-in symbols (host pointers, strided) and the batched device entry point
    daala_b200_haar_blocks against the reference build / the port (src/dct.c:4822, :4861)."""
    torch = torch_cuda
    from daala_b200 import _native
    L = _native.lib()
    L.daala_b200_haar_blocks.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    L.daala_b200_haar_blocks.restype = ctypes.c_int
    a = oracle_lib.addr
    n = 1 << ln
    rng = np.random.default_rng(40 + ln)
    for name, lib, prefix in checkers():
        fwd = lib.od_haar if prefix == "ref" else lib.port_haar
        inv = lib.od_haar_inv if prefix == "ref" else lib.port_haar_inv
        for t in range(3):
            x = np.zeros((n, n + 3), np.int32)
            x[:, :n] = rng.integers(-(1 << 14), 1 << 14, size=(n, n))
            y_gpu = np.zeros((n, n + 1), np.int32)
            y_cpu = np.zeros((n, n + 1), np.int32)
            L.od_haar(a(y_gpu), n + 1, a(x), n + 3, ln)
            fwd(a(y_cpu), n + 1, a(x), n + 3, ln)
            assert np.array_equal(y_gpu, y_cpu), name
            x_gpu = np.zeros((n, n + 2), np.int32)
            x_cpu = np.zeros((n, n + 2), np.int32)
            L.od_haar_inv(a(x_gpu), n + 2, a(y_gpu), n + 1, ln)
            inv(a(x_cpu), n + 2, a(y_cpu), n + 1, ln)
            assert np.array_equal(x_gpu, x_cpu), name
            assert np.array_equal(x_gpu[:, :n], x[:, :n])
    # batch of packed blocks on the device, in place: forward equals the per-block oracle, inverse restores
    port = oracle_lib.load_port()
    blocks = rng.integers(-(1 << 14), 1 << 14, size=(37, n, n)).astype(np.int32)
    dev = torch.from_numpy(blocks.copy()).cuda()
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert L.daala_b200_haar_blocks(dev.data_ptr(), len(blocks), ln, 0, s) == 0
    got = dev.cpu().numpy()
    for i in (0, 17, 36):
        exp = np.zeros((n, n), np.int32)
        port.port_haar(a(exp), n, a(np.ascontiguousarray(blocks[i])), n, ln)
        assert np.array_equal(got[i], exp)
    assert L.daala_b200_haar_blocks(dev.data_ptr(), len(blocks), ln, 1, s) == 0
    assert np.array_equal(dev.cpu().numpy(), blocks)


def test_dropin_filter_symbols_match_oracle(torch_cuda):
    from daala_b200 import _native
    L = _native.lib()
    port = oracle_lib.load_port()
    a = oracle_lib.addr
    rng = np.random.default_rng(5)
    x = rng.integers(-4096, 4096, size=4, dtype=np.int32)
    yg, yc = np.zeros(4, np.int32), np.zeros(4, np.int32)
    L.od_pre_filter4(a(yg), a(x))
    port.port_pre_filter4(a(yc), a(x))
    assert np.array_equal(yg, yc)
    xg = np.zeros(4, np.int32)
    L.od_post_filter4(a(xg), a(yg))
    assert np.array_equal(xg, x)
    for n in (8, 16, 32):
        x = rng.integers(-30000, 30000, size=n, dtype=np.int32)
        yg, yc = np.zeros(n, np.int32), np.zeros(n, np.int32)
        getattr(L, "od_pre_filter%d" % n)(a(yg), a(x))
        port.port_pre_filter_n(n, a(yc), a(x))
        assert np.array_equal(yg, yc)
        xg = np.zeros(n, np.int32)
        getattr(L, "od_post_filter%d" % n)(a(xg), a(yg))
        assert np.array_equal(xg, x)
    for xdec in (0, 1):
        nhsb, nvsb = 3, 2
        w, h = (nhsb * 64) >> xdec, (nvsb * 64) >> xdec
        c = rng.integers(-2048, 2048, size=(h, w + 8), dtype=np.int32)
        g, p = c.copy(), c.copy()
        L.od_apply_prefilter_frame_sbs(a(g), w + 8, nhsb, nvsb, xdec, xdec)
        port.port_apply_prefilter_frame_sbs(a(p), w + 8, nhsb, nvsb, xdec, xdec)
        assert np.array_equal(g, p)
        L.od_apply_postfilter_frame_sbs(a(g), w + 8, nhsb, nvsb, xdec, xdec, 0, None, 0)
        assert np.array_equal(g, c)
    for bs in (1, 2, 3, 4):
        n = 4 << bs
        c = rng.integers(-2048, 2048, size=(n, n + 4), dtype=np.int32)
        g, p = c.copy(), c.copy()
        L.od_prefilter_split(a(g), n + 4, bs, 0, 1, 1)
        port.port_prefilter_split(a(p), n + 4, bs, 1, 1)
        assert np.array_equal(g, p)
        L.od_postfilter_split(a(g), n + 4, bs, 0, 0, None, 0, 1, 1)
        assert np.array_equal(g, c)


def test_batched_and_row_sharded_launches_equal_whole_frame(torch_cuda):
    """nframes > 1 batches and sb_row0/sb_rows shards (the multi-GPU split of
    SURVEY.md 8(e)) must reproduce the single whole-frame launch bit for bit."""
    torch = torch_cuda
    from daala_b200 import synth
    from daala_b200.frame import FrameBuffers, Geometry
    geom = Geometry(320, 250)
    nf = 3
    whole = FrameBuffers(geom, nframes=nf)
    parts = FrameBuffers(geom, nframes=nf)
    singles = []
    for f in range(nf):
        planes, _ = synth.frame(320, 250, f=f)
        planes = synth.pad_planes(planes, geom)
        bsize = synth.block_size_map(geom, "mixed", seed=f)
        whole.upload(planes, bsize, frame=f)
        parts.upload(planes, bsize, frame=f)
        one = FrameBuffers(geom)
        one.upload(planes, bsize)
        one.forward()
        one.inverse()
        singles.append(one)
    whole.forward()
    whole.inverse()
    # shards: superblock rows split 3 ways; lapped halo rows come from the
    # neighbouring shard's output, which lives in the same buffer here.
    for rank in range(3):
        parts.sb_row0, parts.sb_rows = geom.shard_rows(rank, 3)
        parts.forward()
        parts.inverse(lapped_only=True)
    for rank in range(3):
        parts.sb_row0, parts.sb_rows = geom.shard_rows(rank, 3)
        parts.sb_postfilter_store()
    torch.cuda.synchronize()
    for pli in range(3):
        assert torch.equal(whole.coeffs[pli], parts.coeffs[pli])
        assert torch.equal(whole.pixels_out[pli], parts.pixels_out[pli])
        for f in range(nf):
            assert torch.equal(whole.coeffs[pli][f], singles[f].coeffs[pli][0])
            assert torch.equal(whole.pixels_out[pli][f], singles[f].pixels_out[pli][0])
            assert torch.equal(whole.pixels_out[pli][f], whole.pixels[pli][f])


def test_tma_and_plain_load_forward_agree(torch_cuda):
    """The TMA-staged forward kernel and its plain-load twin (used for
    unaligned planes) must write identical coefficient planes."""
    torch = torch_cuda
    from daala_b200 import synth
    from daala_b200.frame import FrameBuffers, Geometry
    geom = Geometry(704, 300)
    a = FrameBuffers(geom, nframes=2)
    b = FrameBuffers(geom, nframes=2)
    for f in range(2):
        planes, _ = synth.frame(704, 300, f=f)
        planes = synth.pad_planes(planes, geom)
        bsize = synth.block_size_map(geom, "mixed", seed=20 + f)
        a.upload(planes, bsize, frame=f)
        b.upload(planes, bsize, frame=f)
    a.forward(tma=True)
    b.forward(tma=False)
    torch.cuda.synchronize()
    for pli in range(3):
        assert torch.equal(a.coeffs[pli], b.coeffs[pli])


def test_dropin_tf_symbols_match_reference(torch_cuda):
    """The TF helpers of src/tf.c:38-277 with host pointers (csrc/tf_kernels.cu) against the reference
    build's own functions (their results recorded as CRC-32 in tests/golden/reference_digests.npz by
    tests/golden/make_golden.py), strided source and destination, every size the codec's blocks can take;
    the reversibility the reference documents (od_tf_down_hv inverts od_tf_up_hv, the inverse filter
    undoes the filter) is checked on the device results as well."""
    from daala_b200 import _native
    from tests.golden import make_golden
    L = _native.lib()
    a = oracle_lib.addr
    gold = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_digests.npz")
    want = np.load(gold)["tf_crc"].tolist()
    cases = list(make_golden.tf_cases())
    assert len(cases) == len(want)
    for case, crc in zip(cases, want):
        name, _, src, args = case
        d = make_golden.run_tf(L, case)
        assert make_golden.crc(d) == crc, (name, src.shape, args)
        n = args[-1]
        if name == "od_tf_filter_inv_2d":
            back = np.zeros((n, n), np.int32)
            fc = np.ascontiguousarray(d[:, :n])   # keep alive across the call
            L.od_tf_filter_2d(a(back), n, a(fc), n, n)
            assert np.array_equal(back, src[:, :n])
        if name == "od_tf_up_hv":
            down = np.zeros((2 * n, 2 * n), np.int32)
            upc = np.ascontiguousarray(d[:, :2 * n])
            L.od_tf_down_hv(a(down), 2 * n, a(upc), 2 * n, 2 * n)
            assert np.array_equal(down, src[:, :2 * n])
