"""numpy restatement of the P-frame finishing pass's first two kernels (csrc/kf_engine.cu, k_fin_patch and
k_fin_skip_map): the host coder's per-block skip / DC decisions applied to the coefficient planes of a step, and the
skip maps they imply.  It builds the inputs of the oracle's frame driver (oracle/inter_finish_driver.inc,
inverse_frame_inter_finish), which then runs the reference's inverse, postfilters and od_dering."""
import numpy as np


def dc_quant(q0, qm_q4, pli, bs):
    """The band-0 quantiser of a block of plane pli, bs = log2(n) - 2 (src/encode.c:1333-1334)."""
    return max(1, (int(q0) * int(qm_q4[pli][bs * (bs + 1)])) >> 4)


def _select(blocks, frame, pli):
    return np.nonzero((blocks["frame"] == frame) & (blocks["pli"] == pli))[0]


def patch(d, md, blocks, skip, dc, frame, pli, q0, qm_q4):
    """One plane of one frame: d / md the step's coefficient and prediction planes, blocks / skip / dc the block
    records of the plane's list (luma or chroma) with the decisions in the same order.  skip = 0 keeps the coded
    coefficients, skip = 1 takes md over the whole block; either way DC = md[0] + dc * dc_quant."""
    out = np.array(d, np.int32, copy=True)
    for i in _select(blocks, frame, pli):
        b = blocks[i]
        n, y0, x0 = 4 << int(b["bs"]), int(b["y0"]), int(b["x0"])
        if skip[i]:
            out[y0:y0 + n, x0:x0 + n] = md[y0:y0 + n, x0:x0 + n]
        out[y0, x0] = int(md[y0, x0]) + int(dc[i]) * dc_quant(q0, qm_q4, pli, int(b["bs"]))
    return out


def skip_map(blocks, skip, dc, frame, pli, geom):
    """state->bskip[pli] of one frame: [plane_h / 4, nhsb * 16] u8, skip && dc == 0 over each block's 4x4 units
    (src/encode.c:1690-1691); row stride state->skip_stride for every plane, a chroma row's tail stays 0."""
    h = geom.plane_shape(pli)[0]
    m = np.zeros((h // 4, geom.nhsb * 16), np.uint8)
    for i in _select(blocks, frame, pli):
        b = blocks[i]
        u, y, x = 1 << int(b["bs"]), int(b["y0"]) >> 2, int(b["x0"]) >> 2
        m[y:y + u, x:x + u] = 1 if skip[i] and dc[i] == 0 else 0
    return m


def coded_superblocks(bskip_luma, geom):
    """[nvsb, nhsb] bool: the superblock has a coded 4x4 luma unit (src/encode.c:2724-2738); the others are not
    deringed."""
    m = bskip_luma[:geom.nvsb * 16, :geom.nhsb * 16].reshape(geom.nvsb, 16, geom.nhsb, 16)
    return (m == 0).any(axis=(1, 3))
