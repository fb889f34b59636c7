"""Order of the luma chain heads: the keyframe engine hands the row / column chains of the H/V intra predictor to
warps heaviest first (chain length in blocks times the cost of the band's size class), so that the longest serial
work starts early instead of after every chain that precedes it in block order.

A numpy model of the dependency structure k_luma_deps builds (same-size top / left neighbours, chain heads, chain
lengths) is checked against the counts of the bench workload on the CPU, and against the engine's device-built
lists on the GPU.
"""
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NBANDS = np.array([1, 4, 7, 9, 9])
CHAIN_BANDS = (1, 2, 4, 5, 7, 8)
COST = (7, 9, 18)       # kf_engine.cu kChainCost0..2: item cost of the n <= 16 / 32 / 128 bands, in 10 us
BINS = 12288            # kf_engine.cu kLevelBins


def weight_bin(length, band):
    c = 0 if band < 3 else 1 if band < 6 else 2
    return BINS - 1 - np.minimum(np.asarray(length) * COST[c], BINS - 1)


def frame_model(m):
    """Luma blocks of one block-size map [UH, UW] (unit raster, the 4x4 blocks of a unit in raster order), their
    same-size top / left neighbour flags and the length of the column / row chain from each block on."""
    uh, uw = m.shape
    uy, ux = np.mgrid[0:uh, 0:uw]
    span = np.where(m > 0, 1 << np.maximum(m.astype(np.int64) - 1, 0), 1)
    origin = ((ux % span) == 0) & ((uy % span) == 0)
    ys, xs, bss = [], [], []
    for q in range(4):   # a unit coded as 4x4 blocks holds four of them
        sel = origin & ((m == 0) | (q == 0))
        ys.append(np.where(sel, uy * 8 + (q >> 1) * 4 * (m == 0), -1))
        xs.append(np.where(sel, ux * 8 + (q & 1) * 4 * (m == 0), -1))
        bss.append(m)
    y = np.stack(ys, -1).reshape(-1)
    x = np.stack(xs, -1).reshape(-1)
    bs = np.stack(bss, -1).reshape(-1).astype(np.int64)
    keep = y >= 0
    y, x, bs = y[keep], x[keep], bs[keep]
    n = 4 << bs
    top = (y - n >= 0) & (m[np.maximum(y - 1, 0) >> 3, x >> 3] == bs)
    left = (x > 0) & (m[y >> 3, np.maximum(x - 1, 0) >> 3] == bs)
    # successors: the block whose top (left) neighbour this one is; chain lengths by walking them
    grid = np.full((uh * 2 + 1, uw * 2 + 1), -1, np.int64)
    grid[y >> 2, x >> 2] = np.arange(len(y))
    lengths = {}
    for name, dy, dx, dep in (("down", 1, 0, top), ("across", 0, 1, left)):
        j = grid[np.minimum((y + dy * n) >> 2, uh * 2), np.minimum((x + dx * n) >> 2, uw * 2)]
        succ = np.where((j >= 0) & (bs[np.maximum(j, 0)] == bs) & dep[np.maximum(j, 0)], j, -1)
        length = np.ones(len(y), np.int64)
        cur = np.arange(len(y))
        alive = succ[cur] >= 0
        while alive.any():
            cur = np.where(alive, succ[np.maximum(cur, 0)], cur)
            length += alive
            alive = alive & (succ[cur] >= 0)
        lengths[name] = length
    return dict(y=y, x=x, bs=bs, top=top, left=left, down=lengths["down"], across=lengths["across"])


def heads_of(fm):
    """{(y0, x0, band): weight bin} of every row / column chain head of one frame."""
    nb = NBANDS[fm["bs"]]
    out = {}
    for band in CHAIN_BANDS:
        down = band % 3 == 1
        sel = (nb > band) & ~(fm["top"] if down else fm["left"])
        bins = weight_bin((fm["down"] if down else fm["across"])[sel], band)
        out.update(zip(zip(fm["y"][sel].tolist(), fm["x"][sel].tolist(), [band] * int(sel.sum())), bins.tolist()))
    return out


def bench_maps():
    real = np.load(os.path.join(ROOT, "daala_b200", "data", "bench_bsize_4k.npz"))
    return [np.ascontiguousarray(real["bsize_%d" % (f % 4)]) for f in range(16)]   # bench.py's 16-frame batch


def test_model_matches_the_bench_dependency_counts():
    per_band = {b: [0, 0, 0] for b in CHAIN_BANDS}   # heads, items, longest chain
    band0 = free = 0
    for m in bench_maps():
        fm = frame_model(m)
        nb = NBANDS[fm["bs"]]
        band0 += len(nb)
        free += int((nb > 3).sum() + (nb > 6).sum())
        for band in CHAIN_BANDS:
            down = band % 3 == 1
            sel = (nb > band) & ~(fm["top"] if down else fm["left"])
            length = (fm["down"] if down else fm["across"])[sel]
            per_band[band][0] += int(sel.sum())
            per_band[band][1] += int(length.sum())
            per_band[band][2] = max(per_band[band][2], int(length.max()))
            assert length.sum() == (nb > band).sum()   # the chains of a band cover its items exactly once
    want = {1: (35408, 5.0, 68), 2: (44400, 4.0, 120), 4: (16612, 8.4, 68), 5: (20932, 6.7, 120),
            7: (6288, 19.2, 68), 8: (8128, 14.8, 120)}
    for band, (heads, mean, longest) in want.items():
        h, items, mx = per_band[band]
        assert (h, round(items / h, 1), mx) == (heads, mean, longest), band
    assert sum(v[0] for v in per_band.values()) == 131768
    assert sum(v[1] for v in per_band.values()) == 876824
    assert band0 == 348996 and free == 317728
    # 1,225,820 chain items = row / column chains + band 0
    assert sum(v[1] for v in per_band.values()) + band0 == 1225820


def test_weight_bins_order_heaviest_first():
    assert weight_bin(120, 8) < weight_bin(68, 7) < weight_bin(1, 7) < weight_bin(1, 4) < weight_bin(1, 1)
    assert weight_bin(10 ** 6, 1) == 0 and weight_bin(1, 1) == BINS - 1 - COST[0]


def _check_sorted_heads(geom, maps):
    from daala_b200 import engine, pvq, synth
    F = len(maps)
    eng = engine.KeyframeEngine(geom, nframes=F, q0=72, pvq_qm_q4=np.full((3, 30), 16, np.uint8),
                                max_blocks_div=2 if geom.pic_w == 3840 else 0)
    planes = []
    seed = 12345
    for f in range(min(F, 2)):
        p, seed = synth.frame(geom.pic_w, geom.pic_h, f=f, seed=seed)
        planes.append(synth.pad_planes(p, geom))
    eng.upload([np.stack([planes[f % len(planes)][p] for f in range(F)]) for p in range(3)], np.stack(maps))
    eng.run_device(engine.PH_ALL, graph=False)
    cnt = eng.counts()
    assert int(cnt[engine.CNT["error"]]) == 0
    nl, nh = int(cnt[engine.CNT["n_luma"]]), int(cnt[engine.CNT["n_heads"]])
    blocks = eng.download(eng.buf.luma_blocks, (nl,), pvq.BLOCK_DTYPE)
    heads = eng.download(eng.buf.luma_heads, (nh,), np.uint32)
    raw = eng.download(eng.buf.luma_heads_raw, (nh,), np.uint32)
    bins = eng.download(eng.buf.luma_head_bin, (nh,), np.int32)
    eng.close()
    # the sorted list is a permutation of the list k_luma_deps emitted
    assert np.array_equal(np.sort(heads), np.sort(raw)) and len(np.unique(heads)) == nh
    # every head and its weight bin as the model has them
    want = {}
    for f, m in enumerate(maps):
        want.update({(f,) + k: v for k, v in heads_of(frame_model(m)).items()})
    b = blocks[raw >> 4]
    got = dict(zip(zip(b["frame"].tolist(), b["y0"].tolist(), b["x0"].tolist(), (raw & 15).tolist()), bins.tolist()))
    assert len(got) == nh and got == want
    # heaviest first: the model's bins along the sorted list never decrease
    bh = blocks[heads >> 4]
    order = np.array([want[k] for k in zip(bh["frame"].tolist(), bh["y0"].tolist(), bh["x0"].tolist(),
                                           (heads & 15).tolist())])
    assert (np.diff(order) >= 0).all()
    return order


@pytest.mark.gpu
def test_heads_heaviest_first_1080p():
    from daala_b200 import synth
    from daala_b200.frame import Geometry
    geom = Geometry(1920, 1080)
    maps = [synth.block_size_map(geom, "mixed", seed=101 + f) for f in range(2)]
    order = _check_sorted_heads(geom, maps)
    assert len(np.unique(order)) > 10


@pytest.mark.gpu
def test_heads_heaviest_first_bench_maps():
    from daala_b200.frame import Geometry
    order = _check_sorted_heads(Geometry(3840, 2160), bench_maps())
    assert len(order) == 131768
    # the first head is one of the longest 128-coefficient row chains (120 blocks)
    assert order[0] == weight_bin(120, 8)
