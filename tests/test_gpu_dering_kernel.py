"""GPU parity of the deringing kernel (csrc/dering_kernels.cu) against the pinned CPU oracle (oracle/port_dering.c)
on content the 3x2-superblock case of tests/test_gpu_dering.py does not reach:

  * flat blocks, where the 8 direction costs tie;
  * each of the 8 pure directional patterns (every 8x8 block constant along the lines of one direction);
  * saturated 8-bit reconstructions (samples at and beyond the ends of the u8 range);
  * frame-edge superblocks on non-square grids, with row strides that are not a multiple of 4 samples.

Both plane types and every dir_format: 0 (plain directions), 1 (luma stores direction | variance << 3, checked
against the port's direction search), 2 (luma reads that back; its thresholds follow from the stored variance), and
chroma reading plain or packed maps.  The batch entry point is checked with several frames of one geometry, per-frame
thresholds and the u8 destination, which must equal the int16 output pushed through od_coeff_to_ref_plane."""
import ctypes

import numpy as np
import pytest

from tests import oracle_lib
from tests.oracle_lib import addr
from tests.test_gpu_dering import DeringParams

pytestmark = pytest.mark.gpu

COEFF_SHIFT = 4


def _lib():
    from daala_b200 import _native
    L = _native.lib()
    L.daala_b200_dering_plane.argtypes = [ctypes.POINTER(DeringParams), ctypes.c_void_p]
    L.daala_b200_dering_plane_batch.argtypes = [ctypes.POINTER(DeringParams), ctypes.c_int, ctypes.c_longlong,
                                                ctypes.c_longlong, ctypes.c_longlong, ctypes.c_longlong,
                                                ctypes.c_void_p, ctypes.c_void_p]
    return L


def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


# ---- content ----------------------------------------------------------------------------------------------------
def _line(d, i, j):
    """Line of direction d through sample (i, j), on the whole plane (od_dir_find8's lines, extended)."""
    return [i + j, i + j // 2, i, i - j // 2, i - j, j - i // 2, j, j + i // 2][d]


def _directional(nvsb, nhsb, sb, seed, amp):
    """Every 8x8 luma block (4x4 chroma) constant along the lines of one direction, the 8 directions in turn."""
    rng = np.random.default_rng(seed)
    h, w = nvsb * sb, nhsb * sb
    n = sb // 8
    yy, xx = np.mgrid[0:h, 0:w]
    vals = rng.integers(-amp, amp + 1, size=(8, 4 * (h + w) + 8))
    img = np.zeros((h, w), np.int64)
    blk = (yy // n) * (w // n) + (xx // n)
    for d in range(8):
        sel = (blk + (yy // n)) % 8 == d
        img[sel] = vals[d][np.asarray(_line(d, yy[sel], xx[sel])) + 2 * (h + w)]
    return img.astype(np.int16)


def _flat(nvsb, nhsb, sb, seed):
    """Flat 8x8 blocks: zero, mid grey, both saturated ends, and flat blocks with a one-sample bump."""
    rng = np.random.default_rng(seed)
    h, w = nvsb * sb, nhsb * sb
    n = sb // 8
    levels = np.array([0, -2048, 2032, 400, -7])
    img = levels[rng.integers(0, len(levels), size=(h // n, w // n))].repeat(n, 0).repeat(n, 1)
    bump = rng.random((h, w)) < 0.002
    img = np.where(bump, img + rng.integers(-30, 31, size=(h, w)), img)
    return np.clip(img, -2048, 2047).astype(np.int16)


def _saturated(nvsb, nhsb, sb, seed):
    """8-bit reconstructions at the ends of the range: regions of 0 and 255 ((p - 128) << 4), ringing that
    overshoots both ends (past what od_coeff_to_ref_plane clamps), and texture in between."""
    rng = np.random.default_rng(seed)
    h, w = nvsb * sb, nhsb * sb
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.where(np.sin(xx / 5.0 + yy / 9.0) > 0, 2032, -2048)
    ring = (260 * np.sin(xx * 1.3) * np.cos(yy * 0.7)).astype(np.int64)
    noise = rng.integers(-60, 61, size=(h, w))
    img = np.where(rng.random((h, w)) < 0.3, base + ring, base + noise)
    return np.clip(img, -2600, 2600).astype(np.int16)


def _edges(nvsb, nhsb, sb, seed):
    from tests.golden.make_golden import dering_image
    return dering_image(nvsb, nhsb, sb, seed)


def _embed(img, stride):
    """img in a plane of row stride `stride` (extra columns hold junk the filter must not read)."""
    h, w = img.shape
    out = np.full((h, stride), -1234, np.int16)
    out[:, :w] = img
    return out


# ---- the oracle ---------------------------------------------------------------------------------------------------
def _oracle(x, nhsb, nvsb, xdec, dirs, bskip, thr, overlap):
    """port_dering superblock by superblock: (filtered plane [h][w], direction map).  thr[sby][sbx]."""
    port = oracle_lib.load_port()
    sb = 64 >> xdec
    units = 16 >> xdec
    stride = x.shape[1]
    skip_stride = bskip.shape[1]
    want = np.zeros((nvsb * sb, nhsb * sb), np.int16)
    want_dir = dirs.copy()
    Dir = (ctypes.c_int * 8) * 8
    for sby in range(nvsb):
        for sbx in range(nhsb):
            d = Dir()
            for r in range(8):
                for c in range(8):
                    d[r][c] = int(dirs[sby * 8 + r, sbx * 8 + c])
            y = np.zeros((sb, sb), np.int16)
            port.port_dering(addr(y), sb, addr(x, sby * sb * stride + sbx * sb), stride, 8, 8, sbx, sby, nhsb, nvsb,
                             xdec, d, 1 if xdec else 0, addr(bskip, sby * units * skip_stride + sbx * units), skip_stride,
                             int(thr[sby][sbx]), overlap, COEFF_SHIFT)
            want[sby * sb:(sby + 1) * sb, sbx * sb:(sbx + 1) * sb] = y
            want_dir[sby * 8:(sby + 1) * 8, sbx * 8:(sbx + 1) * 8] = np.array([list(r) for r in d])
    return want, want_dir


def _port_direction(x, by, bx):
    """(direction, variance) of the 8x8 luma block (by, bx) by the port's od_dir_find8."""
    port = oracle_lib.load_port()
    port.port_dering_find_direction.restype = ctypes.c_int
    var = ctypes.c_int32()
    stride = x.shape[1]
    d = port.port_dering_find_direction(addr(x, by * 8 * stride + bx * 8), stride, ctypes.byref(var), COEFF_SHIFT)
    return d, var.value


def _packed(x, nhsb, nvsb):
    """The direction | variance << 3 map a dir_format 1 luma pass must write."""
    out = np.zeros((nvsb * 8, nhsb * 8), np.int64)
    for by in range(nvsb * 8):
        for bx in range(nhsb * 8):
            d, var = _port_direction(x, by, bx)
            out[by, bx] = d | (var << 3)
    return out.astype(np.int32)


# ---- the kernel ---------------------------------------------------------------------------------------------------
def _run(x, nhsb, nvsb, xdec, dirs, bskip, threshold, overlap, dir_format, ystride=None):
    """One plane through daala_b200_dering_plane: (int16 output [h][ystride], direction map)."""
    import torch
    L = _lib()
    sb = 64 >> xdec
    h = nvsb * sb
    ystride = ystride or x.shape[1]
    x_dev = torch.from_numpy(x).cuda()
    y_dev = torch.full((h, ystride), 4321, dtype=torch.int16, device="cuda")
    dir_dev = torch.from_numpy(np.ascontiguousarray(dirs, np.int32)).cuda()
    skip_dev = torch.from_numpy(bskip).cuda()
    p = DeringParams(y=y_dev.data_ptr(), x=x_dev.data_ptr(), dir=dir_dev.data_ptr(), bskip=skip_dev.data_ptr(),
                     sb_threshold=None, ystride=ystride, xstride=x.shape[1], dir_stride=dirs.shape[1],
                     skip_stride=bskip.shape[1], nhsb=nhsb, nvsb=nvsb, xdec=xdec, pli=1 if xdec else 0,
                     threshold=threshold, overlap=overlap, coeff_shift=COEFF_SHIFT, dir_format=dir_format)
    assert L.daala_b200_dering_plane(ctypes.byref(p), _stream()) == 0
    torch.cuda.synchronize()
    return y_dev.cpu().numpy(), dir_dev.cpu().numpy()


def _skips(nvsb, nhsb, xdec, seed, p=0.4):
    units = 16 >> xdec
    rng = np.random.default_rng(seed)
    return (rng.random((nvsb * units, nhsb * units + 5)) < p).astype(np.uint8)


CONTENT = {"flat": _flat, "directional": _directional, "saturated": _saturated, "edges": _edges}
# (content, nhsb, nvsb, luma row stride over the plane width)
CASES = [("flat", 3, 2, 0), ("directional", 3, 2, 0), ("saturated", 3, 2, 0), ("edges", 5, 2, 2), ("edges", 2, 5, 6),
         ("edges", 1, 3, 0), ("directional", 4, 1, 10)]


def _content(name, nvsb, nhsb, sb, seed, amp=None):
    if name == "directional":
        return _directional(nvsb, nhsb, sb, seed, amp or 600)
    return CONTENT[name](nvsb, nhsb, sb, seed)


@pytest.mark.parametrize("content,nhsb,nvsb,pad", CASES)
@pytest.mark.parametrize("threshold,overlap", [(40, 1), (180, 0)])
def test_luma_dir_formats(content, nhsb, nvsb, pad, threshold, overlap):
    """Luma: dir_format 0 and 1 search the direction (1 also stores the port's variance), 2 reads the packed map
    back at another threshold; every output equals the port's."""
    img = _content(content, nvsb, nhsb, 64, 7 + nhsb * 3 + nvsb)
    x = _embed(img, img.shape[1] + pad)
    bskip = _skips(nvsb, nhsb, 0, 5 + pad, 0.3)
    junk = np.random.default_rng(1).integers(0, 8, size=(nvsb * 8, nhsb * 8 + 3)).astype(np.int32)
    thr = np.full((nvsb, nhsb), threshold)
    want, want_dir = _oracle(x, nhsb, nvsb, 0, junk, bskip, thr, overlap)
    ystride = nhsb * 64 + (pad and pad + 1)
    # 0: plain directions
    y, dirs = _run(x, nhsb, nvsb, 0, junk, bskip, threshold, overlap, 0, ystride)
    assert np.array_equal(dirs, want_dir)
    assert np.array_equal(y[:, :nhsb * 64], want)
    assert np.all(y[:, nhsb * 64:] == 4321), "wrote past the plane"
    # 1: direction | variance << 3, as the port's od_dir_find8
    y, packed = _run(x, nhsb, nvsb, 0, junk, bskip, threshold, overlap, 1, ystride)
    assert np.array_equal(y[:, :nhsb * 64], want)
    assert np.array_equal(packed[:, :nhsb * 8] & 7, want_dir[:, :nhsb * 8])
    assert np.array_equal(packed[:, :nhsb * 8], _packed(x, nhsb, nvsb))
    assert np.array_equal(packed[:, nhsb * 8:], junk[:, nhsb * 8:])
    # 2: the packed map read back (another threshold: the variance sets the thresholds)
    thr2 = threshold * 2 + 3
    want2, _ = _oracle(x, nhsb, nvsb, 0, junk, bskip, np.full((nvsb, nhsb), thr2), overlap)
    y2, again = _run(x, nhsb, nvsb, 0, packed, bskip, thr2, overlap, 2, ystride)
    assert np.array_equal(again, packed), "dir_format 2 must not write the map"
    assert np.array_equal(y2[:, :nhsb * 64], want2)
    if content == "directional":
        # the content is what it claims: the search finds the pattern's direction on (almost) every block
        by, bx = np.mgrid[0:nvsb * 8, 0:nhsb * 8]
        expect = (by * nhsb * 8 + bx + by) % 8
        assert np.mean(want_dir[:, :nhsb * 8] == expect) > 0.8
    if content == "flat":
        assert np.count_nonzero(packed[:, :nhsb * 8] == 0) > packed[:, :nhsb * 8].size // 2, "flat blocks tie at d=0"


def test_luma_stored_variance_sets_thresholds():
    """dir_format 2 takes the variance from the map, not from the plane.  A map whose variances are forged within
    the same threshold class (the bit length of variance >> 6) gives the port's output; a map whose variances are
    all zero gives another."""
    nhsb, nvsb = 3, 2
    img = _content("directional", nvsb, nhsb, 64, 3, amp=300)
    bskip = np.zeros((nvsb * 16, nhsb * 16), np.uint8)
    real = _packed(img, nhsb, nvsb).astype(np.int64)
    d, v = real & 7, np.minimum((real >> 3) >> 6, 32767)
    lg = np.array([int(t).bit_length() for t in v.ravel()]).reshape(v.shape)
    rng = np.random.default_rng(8)
    same = np.where(lg > 0, 1 << np.maximum(lg - 1, 0), 0) << 6 | rng.integers(0, 64, size=v.shape)
    want, _ = _oracle(img, nhsb, nvsb, 0, np.zeros_like(d, np.int32), bskip, np.full((nvsb, nhsb), 100), 1)
    y, _ = _run(img, nhsb, nvsb, 0, (d | same << 3).astype(np.int32), bskip, 100, 1, 2)
    assert np.array_equal(y, want)
    assert np.count_nonzero(lg) > lg.size // 2, "the content has variance"
    y0, _ = _run(img, nhsb, nvsb, 0, d.astype(np.int32), bskip, 100, 1, 2)
    assert not np.array_equal(y0, want), "the stored variance must set the thresholds"


@pytest.mark.parametrize("content,nhsb,nvsb,pad", CASES)
@pytest.mark.parametrize("dir_format", [0, 1, 2])
def test_chroma(content, nhsb, nvsb, pad, dir_format):
    """4:2:0 chroma reads the direction map: plain for dir_format 0, masked with & 7 otherwise."""
    img = _content(content, nvsb, nhsb, 32, 11 + nhsb + 2 * nvsb)
    x = _embed(img, img.shape[1] + pad)
    bskip = _skips(nvsb, nhsb, 1, 9 + pad, 0.4)
    rng = np.random.default_rng(21 + dir_format)
    d = rng.integers(0, 8, size=(nvsb * 8, nhsb * 8)).astype(np.int32)
    if content == "directional":
        by, bx = np.mgrid[0:nvsb * 8, 0:nhsb * 8]
        d = ((by * nhsb * 8 + bx + by) % 8).astype(np.int32)
    dmap = d if dir_format == 0 else (d | (rng.integers(0, 1 << 20, size=d.shape) << 3)).astype(np.int32)
    for threshold, overlap in ((30, 1), (120, 0)):
        want, _ = _oracle(x, nhsb, nvsb, 1, d, bskip, np.full((nvsb, nhsb), threshold), overlap)
        y, got_map = _run(x, nhsb, nvsb, 1, dmap, bskip, threshold, overlap, dir_format, nhsb * 32 + (pad and 1))
        assert np.array_equal(got_map, dmap), "chroma must not write the map"
        assert np.array_equal(y[:, :nhsb * 32], want)


def _to_u8(v):
    """od_coeff_to_ref_plane: (v + 8 >> 4) + 128, clamped to 0..255."""
    return np.clip(((v.astype(np.int32) + 8) >> 4) + 128, 0, 255).astype(np.uint8)


@pytest.mark.parametrize("nhsb,nvsb", [(3, 2), (2, 3)])
def test_batch_int16_and_u8(nhsb, nvsb):
    """daala_b200_dering_plane_batch over 3 frames of luma then chroma (per-frame thresholds and direction maps, one
    skip map):
    int16 output equal to the port frame by frame, and the u8 destination equal to that through
    od_coeff_to_ref_plane, with the int16 plane left untouched."""
    import torch
    L = _lib()
    F = 3
    makers = [lambda v, h, s, k: _saturated(v, h, s, 40 + k), lambda v, h, s, k: _content("directional", v, h, s, 50 + k),
              lambda v, h, s, k: _edges(v, h, s, 60 + k)]
    rng = np.random.default_rng(5)
    thr = rng.integers(0, 220, size=(F, nvsb, nhsb)).astype(np.int32)
    thr_c = (thr * 6 // 10).astype(np.int32)
    dir_dev = torch.full((F, nvsb * 8, nhsb * 8), -1, dtype=torch.int32, device="cuda")
    want_dirs = []
    for xdec, thr_f in ((0, thr), (1, thr_c)):
        sb = 64 >> xdec
        h, w = nvsb * sb, nhsb * sb
        planes = np.stack([makers[f](nvsb, nhsb, sb, 7 * xdec + f) for f in range(F)])
        bskip = np.ascontiguousarray(_skips(nvsb, nhsb, xdec, 70 + xdec, 0.25)[:, :nhsb * (16 >> xdec)])   # all frames
        x_dev = torch.from_numpy(planes).cuda()
        skip_dev = torch.from_numpy(bskip).cuda()
        thr_dev = torch.from_numpy(np.ascontiguousarray(thr_f)).cuda()
        y_dev = torch.full((F, h, w), 4321, dtype=torch.int16, device="cuda")
        u8_dev = torch.zeros((F, h, w), dtype=torch.uint8, device="cuda")
        outs = []
        for target in ("int16", "u8"):
            p = DeringParams(y=y_dev.data_ptr() if target == "int16" else None, x=x_dev.data_ptr(),
                             dir=dir_dev.data_ptr(), bskip=skip_dev.data_ptr(), sb_threshold=thr_dev.data_ptr(),
                             ystride=w, xstride=w, dir_stride=nhsb * 8, skip_stride=bskip.shape[1], nhsb=nhsb,
                             nvsb=nvsb, xdec=xdec, pli=xdec, threshold=0, overlap=1, coeff_shift=COEFF_SHIFT,
                             dir_format=0)
            u8 = ctypes.c_void_p(u8_dev.data_ptr()) if target == "u8" else None
            assert L.daala_b200_dering_plane_batch(ctypes.byref(p), F, h * w, h * w, nvsb * nhsb * 64, nvsb * nhsb,
                                                   u8, _stream()) == 0
            torch.cuda.synchronize()
            outs.append(y_dev.cpu().numpy().copy())
        y16, y16_after = outs
        assert np.array_equal(y16_after, y16), "the u8 pass must not write the int16 plane"
        got_u8 = u8_dev.cpu().numpy()
        dirs = dir_dev.cpu().numpy()
        for f in range(F):
            if xdec == 0:
                want_dirs.append(dirs[f].copy())
                d_in = np.zeros_like(dirs[f])
            else:
                d_in = want_dirs[f]
                assert np.array_equal(dirs[f], want_dirs[f])
            want, want_dir = _oracle(planes[f], nhsb, nvsb, xdec, d_in, bskip, thr_f[f], 1)
            if xdec == 0:
                assert np.array_equal(dirs[f], want_dir), "frame %d directions" % f
            assert np.array_equal(y16[f], want), "frame %d plane %d" % (f, xdec)
            assert np.array_equal(got_u8[f], _to_u8(want)), "frame %d plane %d u8" % (f, xdec)
        assert got_u8.min() == 0 and got_u8.max() == 255, "the saturated frame reaches both clamps"
