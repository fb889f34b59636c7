"""The late-skip decision of a P-frame block (od_block_encode, reference src/encode.c:1412-1450) taken by the host coder
from a step's late-skip record (config.late_skip; include/daala_b200.h, daala_b200_kf_late_skip; symbols.LATE_SKIP_DTYPE).

After coding a block with bs > 0 the reference compares dist_noskip + lambda * rate_noskip with
dist_skip + lambda * rate_skip, and codes the block as md when skipping is strictly better.  The rates are the host
entropy coder's; the distortions are the record's.  Which dist_noskip applies depends on the two decisions the coder
took just before for the same block: od_rdo_quant's DC index (src/pvq_encoder.c:730-741), which is 0 or q1 whatever the
DC rate, and the PVQ skip of the AC (src/pvq_encoder.c:975).  `field` restates that choice; `q1` the DC candidate."""
import numpy as np


def dc_quant(q0, pvq_qm_q4, pli, bs):
    """The step's band-0 quantiser: max(1, q0 * pvq_qm_q4[pli][bs * (bs + 1)] >> 4), elementwise."""
    q4 = np.asarray(pvq_qm_q4, np.int64)
    return np.maximum(1, (int(q0) * q4[np.asarray(pli), np.asarray(bs) * (np.asarray(bs) + 1)]) >> 4)


def q1(dc_resid, dq):
    """OD_DIV_R0(dc_resid, dc_quant) (src/odintrin.h:123): the non-zero DC index od_rdo_quant may return."""
    x = np.asarray(dc_resid, np.int64)
    dq = np.asarray(dq, np.int64)
    h = ((dq + 1) >> 1) - 1
    num = x + np.where(x < 0, -h, h)
    return np.sign(num) * (np.abs(num) // dq)   # C division truncates toward zero


def field(pvq_skip, dc):
    """The record field holding dist_noskip of a block whose AC was PVQ-skipped (pvq_skip) or coded, with DC index dc
    (0 or q1).  None for (pvq_skip, 0): od_pvq_encode has skipped the block already and there is no late-skip test."""
    if pvq_skip:
        return "noskip_pred_dcq" if dc else None
    return "noskip_coded_dcq" if dc else "noskip_coded_dc0"


def decide(rec, pvq_skip, dc, rate_noskip, rate_skip, lam):
    """True when the reference late-skips the block (src/encode.c:1431): rec is its late-skip record, pvq_skip and dc
    the coder's decisions so far, rate_noskip / rate_skip its rates in 1/8 bit (OD_BITRES) and lam enc->bs_rdo_lambda.
    A PVQ-skipped block with dc = 0 has no test and returns False.  Blocks with bs = 0 have no test either (their
    record is all zero): the caller leaves them out."""
    f = field(pvq_skip, dc)
    if f is None:
        return False
    return bool(rec["dist_skip"] + lam * rate_skip < rec[f] + lam * rate_noskip)
