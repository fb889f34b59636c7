"""Seeded synthetic 4:2:0 content (SURVEY.md 8(d)): translating ramps plus
LCG noise, so transforms, PVQ and motion search all have work to do.  The same
bytes feed the CPU oracle and the GPU path."""
import numpy as np


def _lcg_stream(seed, count):
    """s = s*1103515245 + 12345 (uint32); out = (s >> 16) & 0x7fff -- vectorised
    with the closed form of the affine recurrence in uint32 arithmetic."""
    a = np.uint64(1103515245)
    c = np.uint64(12345)
    mask = np.uint64(0xFFFFFFFF)
    # doubling: compute (A_k, C_k) with s_{i+k} = A_k s_i + C_k
    out = np.empty(count, dtype=np.uint32)
    s = np.uint64(seed)
    # block recurrence: generate first block serially, then jump
    block = min(count, 1 << 12)
    for i in range(block):
        s = (s * a + c) & mask
        out[i] = s
    if count > block:
        # A^block, sum_{j<block} A^j * c
        A = np.uint64(1)
        C = np.uint64(0)
        for _ in range(block):
            C = (C * a + c) & mask
            A = (A * a) & mask
        done = block
        while done < count:
            n = min(block, count - done)
            prev = out[done - block:done - block + n].astype(np.uint64)
            out[done:done + n] = ((prev * A + C) & mask).astype(np.uint32)
            done += n
    return (out >> np.uint32(16)) & np.uint32(0x7FFF), int(out[-1]) if count else seed


def frame(pic_w, pic_h, f=0, seed=12345, xdec=1):
    """Returns ([Y, U, V] uint8 arrays at picture resolution, next seed)."""
    planes = []
    s = seed
    for pli in range(3):
        w = pic_w >> (xdec if pli else 0)
        h = pic_h >> (xdec if pli else 0)
        x = np.arange(w)[None, :]
        y = np.arange(h)[:, None]
        noise, s = _lcg_stream(s, w * h)
        v = (128 + (60 * ((x + 3 * f) % 97)) // 97 + (40 * ((y + 2 * f) % 61)) // 61 - 50
             + (noise.reshape(h, w).astype(np.int64) % 9) - 4)
        planes.append(np.clip(v, 0, 255).astype(np.uint8))
    return planes, s


def pad_planes(planes, geom):
    """Replicate the last row/column out to the padded frame size, like
    daala_image_copy_pad (src/encode.c:1896) does for the encoder input."""
    out = []
    for pli, a in enumerate(planes):
        ph, pw = geom.plane_shape(pli)
        out.append(np.pad(a, ((0, ph - a.shape[0]), (0, pw - a.shape[1])), mode="edge"))
    return out


def block_size_map(geom, mode="mixed", seed=7):
    """A valid quadtree block-size map (one byte per 8x8 luma unit, values 0..4
    = 4x4..64x64), standing in for the encoder's RDO decision."""
    rng = np.random.default_rng(seed)
    bh, bw = geom.bsize_shape
    m = np.zeros((bh, bw), np.uint8)
    if mode in ("4", "8", "16", "32", "64"):
        m[:] = {"4": 0, "8": 1, "16": 2, "32": 3, "64": 4}[mode]
        return m

    def fill(y, x, lvl):
        n = 1 << (lvl - 1) if lvl > 0 else 1  # units per side: lvl 4 -> 8, 1 -> 1
        if lvl <= 1:
            m[y, x] = rng.integers(0, 2)  # 4x4 or 8x8
            return
        if rng.random() < 0.45:
            m[y:y + n, x:x + n] = lvl
            return
        h = n // 2
        for dy in (0, h):
            for dx in (0, h):
                fill(y + dy, x + dx, lvl - 1)

    for sy in range(0, bh, 8):
        for sx in range(0, bw, 8):
            fill(sy, sx, 4)
    return m


def mv_grid(geom, seed=0, p_split=(0.6, 0.5, 0.4), p_gold=0.5, umv=32):
    """A seeded MV grid for one P frame of `geom`: (valid, mv, ref) with (nvsb*8 + 1) x (nhsb*8 + 1) vertices.
    The corners of every 64x64 MV block are valid; a vertex that is the centre of a 64, 32 or 16 block is valid
    with probability p_split[0], [1], [2] (every split level occurs), the other vertices with 1/2.  Vectors are
    uniform in +-umv luma pixels (od_mv_est keeps them within OD_UMV_CLAMP = 32, src/mcenc.c:2467-2478) in 1/8
    pel; ref is GOLD (0) with probability p_gold, else PREV (1)."""
    rng = np.random.default_rng(seed)
    nv, nh = geom.nvsb * 8 + 1, geom.nhsb * 8 + 1
    vy, vx = np.mgrid[0:nv, 0:nh]
    p = np.full((nv, nh), 0.5)
    for lvl, step in enumerate((8, 4, 2)):
        centre = (vx % step == step // 2) & (vy % step == step // 2)
        p[centre] = p_split[lvl]
    valid = rng.random((nv, nh)) < p
    valid[(vx % 8 == 0) & (vy % 8 == 0)] = True
    mv = rng.integers(-umv * 8, umv * 8 + 1, size=(nv, nh, 2)).astype(np.int32)
    ref = (rng.random((nv, nh)) >= p_gold).astype(np.uint8)
    return valid.astype(np.uint8), mv, ref


def mv_grid_b(geom, seed=0, p_split=(0.6, 0.5, 0.4), p_next=0.5, p_gold=0.3, umv=32):
    """A seeded MV grid for one B frame of `geom`: (valid, mv, mv1, ref), valid / mv / split levels as mv_grid.  ref
    is NEXT (2) with probability p_next, else GOLD (0) with probability p_gold, else PREV (1), mixed per vertex (the
    reference's B frames use PREV and NEXT, src/encode.c:1855 rules out 3; GOLD covers the engine's third slot).  mv1 is random on every
    vertex, as od_mv_est leaves it (stale on the vertices whose ref is not NEXT).  A stream of its own: mv_grid's
    output for a seed does not change."""
    rng = np.random.default_rng([seed, 2])
    nv, nh = geom.nvsb * 8 + 1, geom.nhsb * 8 + 1
    vy, vx = np.mgrid[0:nv, 0:nh]
    p = np.full((nv, nh), 0.5)
    for lvl, step in enumerate((8, 4, 2)):
        centre = (vx % step == step // 2) & (vy % step == step // 2)
        p[centre] = p_split[lvl]
    valid = rng.random((nv, nh)) < p
    valid[(vx % 8 == 0) & (vy % 8 == 0)] = True
    mv = rng.integers(-umv * 8, umv * 8 + 1, size=(nv, nh, 2)).astype(np.int32)
    mv1 = rng.integers(-umv * 8, umv * 8 + 1, size=(nv, nh, 2)).astype(np.int32)
    u = rng.random((nv, nh))
    ref = np.where(u < p_next, 2, np.where(u < p_next + (1 - p_next) * p_gold, 0, 1)).astype(np.uint8)
    return valid.astype(np.uint8), mv, mv1, ref
