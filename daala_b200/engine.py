"""Host side of the keyframe engine (include/daala_b200.h, "Keyframe engine"; csrc/kf_engine.cu):
ctypes binding + numpy marshalling.  The engine is the batched equivalent of od_encode_coefficients
(reference src/encode.c:2539) for keyframes without the entropy coder: u8 planes + block-size maps in,
reconstruction + PVQ symbols out, everything in between on the GPU (work lists included).  Created with
inter=1 the same engine codes P-frame residuals: the motion-compensated prediction planes are a second input
(`pred=`), and each block's scalar-quantised DC index is a further output.  With inter_mc=1 the engine makes
that prediction itself from each frame's MV grid and its GOLD / PREV pictures in a pool of reference pictures
(`refs=`, `ref_slot=`, `mv_grid=`), as od_state_mc_predict does, and returns it as `pred0..2`.  With inter_finish=1
`encode` also returns each block's unquantised DC residual, and `finish` takes the host coder's skip and DC decisions
and deringing levels and returns the reconstruction the decoder makes, with its skip maps.  With inter_finish=2 the pass
searches the deringing levels itself (the reference's P-frame search: real skip maps, uncoded superblocks left out,
one CDF context) and returns them with the reconstruction made at those levels.  An engine with inter_mc and
inter_finish codes a sequence without moving pictures through the host: `finish(..., ref_slot_out=)` stores each
frame's reconstruction into a pool slot on the device, `encode(..., resident=True)` predicts from the pool as it stands,
and `pool_load` seeds a slot from host memory or from another engine's device buffer (a GOP's keyframe).
With inter=1 and symbol_stream=2 each step also returns the P-frame symbol stream (the stream of symbol_stream=1 with a
DC record per block: qdc and the unquantised residual), and `finish_stream` takes the decisions back in that order.
With inter=1 and late_skip=1 each step also returns the four late-skip distortions of every block
(symbols.LATE_SKIP_DTYPE; `luma_late_skip` / `chroma_late_skip`, and `sym_late_skip` in stream order), from which the
host coder takes the reference's late-skip decision (daala_b200/lateskip.py).
With inter_mc=1 and mc_next=1 the engine predicts B frames: `ref_slot=` is [F, 3] (GOLD, PREV, NEXT) and `mv1_grid=`
holds each vertex's second vector, which a vertex with ref 2 (NEXT) is predicted with (gop.py gives the reference's
B-frame order and buffer rotation).
With inter=1 and frame_quant=1 every frame of a batch has its own quantizer: `encode(..., frame_quant=)` takes one
FRAME_QUANT_DTYPE record per frame (frame_quant_records builds them) in place of the engine-wide q0, coded_quantizer,
dering_lambda and pvq_qm_q4, so P and B frames of different types or streams share one batch.
With keyframe_quant=1 (keyframes) the same records code every keyframe of a batch at its own quantizer: the keyframes
of several streams, or several sweep points of one, share one step.  use_masking, qm and pvq_norm_lambda stay
engine-wide (stream settings).
With lossless=1 every frame is coded at quantizer 0, the reference's Haar-wavelet path (keyframes, or P / B frames with
inter=1 and host or inter_mc prediction): `encode` takes no block-size map and returns each block's residual
(`ll_coeffs0..2`, int16 planes), the three root tree sums of every block (`ll_blocks`, [F, nvsb, nhsb, 3, 4] int32) and
the reconstruction; `encode(..., ll_ref_slot_out=)` stores each frame's reconstruction into a pool slot (inter_mc).
daala_b200/lossless.py restates the path in numpy.
With haar_dc_quant=1 (keyframes) the step quantises the keyframe DCs as the reference encoder does (its superblock DC
predictor and Haar-level quantiser, with the adaptive DC rate): the reconstruction, the coefficient planes and the CfL
reference carry the quantised DCs, and `encode` returns the coded indices as dc_index0..2 ([F, h / 4, w / 4] int32 per
plane).  daala_b200/haardc.py restates the chain in numpy.  With symbol_stream=1 too the stream carries the same
indices in coding order, one symbols.HDC_DTYPE record per block record (`sym_hdc`), and `encode(..., dc_grids=False)`
leaves the grids out.
With frame_types=1 (on an inter=1, frame_quant=1, haar_dc_quant=1 engine with inter_finish) one batch holds keyframes
and P / B frames: `encode(..., frame_type=)` takes one type per frame (1 = keyframe, 0 = P or B frame), each keyframe is
coded as a keyframe_quant=1, haar_dc_quant=1 engine codes it and each P / B frame as the frame_quant=1 inter engine
does, and the results are those of both kinds.  The finishing pass deringes the keyframes too, and ref_slot_out stores
them in the pool, so one engine codes a whole GOP.  With symbol_stream=3 too each step returns the mixed stream: every
frame's block records in the kind of its frame (a keyframe's with its CfL flips and sym_hdc records, a P / B frame's
with its sym_dc records; the other kind's records are zero), and `finish_stream` takes the decisions in its order.

No torch here: device memory, streams and the CUDA graph belong to the engine."""
import ctypes

import numpy as np

from . import _native, mvgrid, pvq
from .frame import Geometry

c_int, c_ll, c_void_p = ctypes.c_int, ctypes.c_longlong, ctypes.c_void_p

PH_LISTS, PH_FORWARD, PH_PVQ_LUMA, PH_INVERSE, PH_PVQ_CHROMA = 1, 2, 4, 8, 16
PH_PVQ, PH_ALL, PH_SEARCH_ONLY = 20, 31, 64
CNT = dict(n_luma=0, n_chroma=1, luma_coefs=2, chroma_coefs=3, items_l=4, items_c=7,
           total_hi=14, n_heads=15, n_heads0=16, error=17, mc_bad_ref=19, mc_beyond=20)


class Config(ctypes.Structure):
    _fields_ = [("pic_w", c_int), ("pic_h", c_int), ("nframes", c_int), ("q0", c_int), ("use_masking", c_int),
                ("qm_stride", c_int), ("pvq_norm_lambda", ctypes.c_double), ("pvq_qm_q4", (ctypes.c_ubyte * 32) * 3),
                ("qm", c_void_p), ("qm_inv", c_void_p), ("sb_row0", c_int), ("sb_rows", c_int),
                ("max_blocks_div", c_int), ("persist_ctas_per_sm", c_int), ("dering", c_int), ("stream", c_void_p),
                ("coded_quantizer", c_int), ("qm_is_flat", c_int), ("dering_lambda", ctypes.c_double),
                ("symbol_stream", c_int), ("inter", c_int), ("inter_mc", c_int), ("mc_refs", c_int),
                ("inter_finish", c_int), ("late_skip", c_int), ("mc_next", c_int), ("frame_quant", c_int),
                ("lossless", c_int), ("haar_dc_quant", c_int), ("keyframe_quant", c_int), ("frame_types", c_int)]


# daala_b200_kf_frame_quant: one frame's quantizer on a frame_quant or keyframe_quant engine.  A keyframe's record:
# q0 = max(1, state->quantizer), state->coded_quantizer, enc->dering_lambda and the pvq_qm_q4 od_interp_qm set for it
FRAME_QUANT_DTYPE = np.dtype([("q0", "<i4"), ("coded_quantizer", "<i4"), ("dering_lambda", "<f8"),
                              ("pvq_qm_q4", "u1", (3, 32))])
MAX_Q0 = 8191   # od_codedquantizer_to_quantizer(63), the largest quantizer a record may carry


def frame_quant_records(q0, coded_quantizer, dering_lambda=None, pvq_qm_q4=None):
    """[F] FRAME_QUANT_DTYPE records from per-frame values: q0 and coded_quantizer [F]; dering_lambda [F] (None: each
    frame's 0.67 * OD_PVQ_LAMBDA * q0^2, the engine's default, src/rate.c:1086); pvq_qm_q4 [F, 3, 30] or one [3, 30]
    table for every frame (None: all 16)."""
    q0 = np.atleast_1d(np.asarray(q0, np.int64))
    rec = np.zeros(q0.shape[0], FRAME_QUANT_DTYPE)
    rec["q0"] = q0
    rec["coded_quantizer"] = np.broadcast_to(np.asarray(coded_quantizer, np.int64), q0.shape)
    lam = 0.67 * pvq.PVQ_LAMBDA * q0.astype(np.float64) ** 2 if dering_lambda is None else dering_lambda
    rec["dering_lambda"] = np.broadcast_to(np.asarray(lam, np.float64), q0.shape)
    q4 = np.full((3, 30), 16, np.uint8) if pvq_qm_q4 is None else np.asarray(pvq_qm_q4, np.uint8)
    rec["pvq_qm_q4"][:, :, :30] = np.broadcast_to(q4[..., :30], (q0.shape[0], 3, 30))
    return rec


class Totals(ctypes.Structure):
    _fields_ = [("n_luma", c_ll), ("luma_coefs", c_ll), ("n_chroma", c_ll), ("chroma_coefs", c_ll)]


class IO(ctypes.Structure):
    _fields_ = [("pixels", c_void_p * 3), ("bsize", c_void_p), ("dering_level", c_void_p), ("totals", ctypes.POINTER(Totals)),
                ("pixels_out", c_void_p * 3), ("luma_blocks", c_void_p), ("chroma_blocks", c_void_p),
                ("luma_res", c_void_p), ("chroma_res", c_void_p), ("luma_y16", c_void_p), ("chroma_y16", c_void_p),
                ("luma_skip_diff", c_void_p), ("chroma_skip_diff", c_void_p), ("chroma_flip", c_void_p),
                ("counts", c_void_p), ("dering_level_out", c_void_p),
                ("sym_index", c_void_p), ("sym_index_cap", c_ll), ("sym_blocks", c_void_p), ("sym_blocks_cap", c_ll),
                ("sym_bands", c_void_p), ("sym_bands_cap", c_ll), ("sym_pulses", c_void_p), ("sym_pulses_cap", c_ll),
                ("pred_pixels", c_void_p * 3), ("luma_dc", c_void_p), ("chroma_dc", c_void_p),
                ("ref_pixels", c_void_p * 3), ("nrefs", c_int), ("ref_slot", c_void_p), ("mv_grid", c_void_p),
                ("pred_pixels_out", c_void_p * 3), ("luma_dc_resid", c_void_p), ("chroma_dc_resid", c_void_p),
                ("ref_resident", c_int), ("sym_dc", c_void_p), ("sym_dc_cap", c_ll),
                ("luma_late_skip", c_void_p), ("chroma_late_skip", c_void_p), ("sym_late_skip", c_void_p),
                ("sym_late_skip_cap", c_ll), ("ref_slot_next", c_void_p), ("mv1_grid", c_void_p),
                ("frame_quant", c_void_p), ("ll_coeffs", c_void_p * 3), ("ll_blocks", c_void_p),
                ("ll_ref_slot_out", c_void_p), ("dc_index", c_void_p * 3), ("sym_hdc", c_void_p),
                ("sym_hdc_cap", c_ll), ("frame_type", c_void_p)]


class FinishIO(ctypes.Structure):
    _fields_ = [("luma_skip", c_void_p), ("chroma_skip", c_void_p), ("luma_dc", c_void_p), ("chroma_dc", c_void_p),
                ("dering_level", c_void_p), ("pixels_out", c_void_p * 3), ("bskip_out", c_void_p * 3),
                ("dering_level_out", c_void_p), ("ref_slot_out", c_void_p), ("stream_skip", c_void_p),
                ("stream_dc", c_void_p)]


class SymBounds(ctypes.Structure):
    _fields_ = [("index", c_ll), ("blocks", c_ll), ("bands", c_ll), ("pulse_bytes", c_ll)]


class Buffers(ctypes.Structure):
    _fields_ = [("pixels", c_void_p * 3), ("coeffs", c_void_p * 3), ("lapped", c_void_p * 3),
                ("pixels_out", c_void_p * 3), ("plane_w", c_int * 3), ("plane_h", c_int * 3), ("bsize", c_void_p),
                ("counts", c_void_p), ("luma_blocks", c_void_p), ("chroma_blocks", c_void_p), ("dep_top", c_void_p),
                ("dep_left", c_void_p), ("succ_bottom", c_void_p), ("succ_right", c_void_p), ("luma_items", c_void_p * 3),
                ("luma_heads", c_void_p), ("luma_heads0", c_void_p), ("chroma_items", c_void_p * 3),
                ("luma_res", c_void_p), ("chroma_res", c_void_p), ("luma_y16", c_void_p), ("chroma_y16", c_void_p),
                ("luma_skip_diff", c_void_p), ("chroma_skip_diff", c_void_p), ("chroma_flip", c_void_p),
                ("max_luma_blocks", c_int), ("max_chroma_blocks", c_int), ("stream", c_void_p),
                ("bytes_allocated", c_ll), ("pred_pixels", c_void_p * 3), ("pred_coeffs", c_void_p * 3),
                ("luma_heads_raw", c_void_p), ("luma_head_bin", c_void_p), ("ref_pixels", c_void_p * 3),
                ("ref_slot", c_void_p), ("mv_grid", c_void_p), ("mc_refs", c_int), ("ref_slot_next", c_void_p),
                ("mv1_grid", c_void_p), ("frame_quant", c_void_p), ("haar_dc", c_void_p * 3),
                ("dc_index", c_void_p * 3), ("sym_hdc", c_void_p)]


def _bind():
    L = _native.lib()
    if getattr(L, "_kf_bound", False):
        return L
    L.daala_b200_kf_create.argtypes = [ctypes.POINTER(Config)]
    L.daala_b200_kf_create.restype = c_void_p
    L.daala_b200_kf_destroy.argtypes = [c_void_p]
    L.daala_b200_kf_destroy.restype = None
    L.daala_b200_kf_error.argtypes = [c_void_p]
    L.daala_b200_kf_error.restype = ctypes.c_char_p
    L.daala_b200_kf_device_buffers.argtypes = [c_void_p, ctypes.POINTER(Buffers)]
    L.daala_b200_kf_launches_per_step.argtypes = [c_void_p]
    L.daala_b200_kf_run_device.argtypes = [c_void_p, c_int, c_int]
    L.daala_b200_kf_time_device.argtypes = [c_void_p, c_int, c_int, c_int, ctypes.POINTER(ctypes.c_float)]
    L.daala_b200_kf_count_blocks.argtypes = [c_void_p, c_int, c_ll, c_int, c_int, c_int, c_int, c_int,
                                             ctypes.POINTER(Totals)]
    for name in ("daala_b200_kf_submit", "daala_b200_kf_encode"):
        getattr(L, name).argtypes = [c_void_p, ctypes.POINTER(IO)]
    L.daala_b200_kf_finish.argtypes = [c_void_p, ctypes.POINTER(FinishIO)]
    L.daala_b200_kf_pool_load.argtypes = [c_void_p, c_int, ctypes.POINTER(c_void_p)]
    L.daala_b200_kf_symbol_bounds.argtypes = [ctypes.POINTER(Totals), c_int, ctypes.POINTER(SymBounds)]
    L.daala_b200_kf_frame_quant_derive.argtypes = [c_void_p, c_int, c_void_p]
    L.daala_b200_kf_load_frame_quant.argtypes = [c_void_p, c_void_p]
    L.daala_b200_kf_wait.argtypes = [c_void_p]
    L.daala_b200_device_copy.argtypes = [c_void_p, c_void_p, ctypes.c_size_t, c_int]
    L.daala_b200_host_alloc.argtypes = [ctypes.c_size_t]
    L.daala_b200_host_alloc.restype = c_void_p
    L.daala_b200_host_free.argtypes = [c_void_p]
    L.daala_b200_host_free.restype = None
    L._kf_bound = True
    return L


def frame_quant_derive(records):
    """What submit derives from a frame_quant step's records (daala_b200_kf_frame_quant_derive): each frame's
    deringing thresholds [F, 2, 6] int32 (luma, chroma per level) and the finishing pass's DC limit."""
    r = np.ascontiguousarray(records, FRAME_QUANT_DTYPE)
    tbl = np.zeros((r.shape[0], 2, 6), np.int32)
    limit = _bind().daala_b200_kf_frame_quant_derive(r.ctypes.data, r.shape[0], tbl.ctypes.data)
    return tbl, int(limit)


class Pinned:
    """A numpy array over page-locked host memory (daala_b200_host_alloc)."""

    def __init__(self, shape, dtype):
        self.L = _bind()
        self.nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
        self.ptr = self.L.daala_b200_host_alloc(max(self.nbytes, 1))
        if not self.ptr:
            raise MemoryError("daala_b200_host_alloc(%d) failed" % self.nbytes)
        buf = (ctypes.c_char * max(self.nbytes, 1)).from_address(self.ptr)
        self.array = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)

    def free(self):
        if self.ptr:
            self.array = None
            self.L.daala_b200_host_free(self.ptr)
            self.ptr = None


class KeyframeEngine:
    """One engine = one set of device buffers + one CUDA graph for batches of `nframes` keyframes."""

    def __init__(self, geom, nframes=1, q0=38, use_masking=1, lam=pvq.PVQ_LAMBDA, pvq_qm_q4=None, qm=None,
                 qm_inv=None, sb_row0=0, sb_rows=0, max_blocks_div=0, persist_ctas_per_sm=0, split_free=1, level_chains=0, noref_prepass=0, dering=0, coded_quantizer=0,
                 qm_is_flat=0, dering_lambda=None, pinned=True, symbol_stream=0, inter=0, inter_mc=0, mc_refs=0,
                 inter_finish=0, late_skip=0, mc_next=0, frame_quant=0, lossless=0, haar_dc_quant=0, keyframe_quant=0,
                 frame_types=0):
        # split_free, level_chains and noref_prepass exist only for bench.py, which passes them: one schedule is left
        retired = ("split_free=%r (chroma through the persistent kernel)" % split_free if split_free == 0 else
                   "split_free=%r (luma bands 3 / 6 through the phase kernels)" % split_free if split_free != 1 else
                   "level_chains=%r (level-synchronous luma chains)" % level_chains if level_chains != 0 else
                   "noref_prepass=%r (the no-reference prepass)" % noref_prepass if noref_prepass != 0 else None)
        if retired:
            raise ValueError("KeyframeEngine: %s is a retired PVQ schedule; split_free=1, level_chains=0, noref_prepass=0 "
                             "is the one the engine has" % retired)
        self.L = _bind()
        self.geom, self.F = geom, nframes
        if qm is None:
            qm, qm_inv = pvq.default_qm(True)
        self._qm = np.ascontiguousarray(qm, np.int16)
        self._qm_inv = np.ascontiguousarray(qm_inv, np.int16)
        cfg = Config()
        cfg.pic_w, cfg.pic_h, cfg.nframes, cfg.q0, cfg.use_masking = geom.pic_w, geom.pic_h, nframes, int(q0), int(use_masking)
        cfg.qm_stride = pvq.OD_QM_STRIDE
        cfg.pvq_norm_lambda = float(lam)
        q4 = pvq_qm_q4 if pvq_qm_q4 is not None else np.full((3, 30), 16, np.uint8)
        for p in range(3):
            for i in range(30):
                cfg.pvq_qm_q4[p][i] = int(q4[p][i])
        cfg.qm, cfg.qm_inv = self._qm.ctypes.data, self._qm_inv.ctypes.data
        cfg.sb_row0, cfg.sb_rows = int(sb_row0), int(sb_rows)
        cfg.max_blocks_div, cfg.persist_ctas_per_sm = int(max_blocks_div), int(persist_ctas_per_sm)
        cfg.dering = int(dering)
        # dering == 2 or inter_finish == 2 (level search): scale of od_compute_dist and enc->dering_lambda =
        # 0.67 * OD_PVQ_LAMBDA * q^2 (src/rate.c:1086; the target quantizer is this engine's q0)
        cfg.coded_quantizer = int(coded_quantizer)
        cfg.qm_is_flat = int(qm_is_flat)
        cfg.dering_lambda = float(0.67 * pvq.PVQ_LAMBDA * q0 * q0 if dering_lambda is None else dering_lambda)
        self.dering_lambda = cfg.dering_lambda
        self.dering = int(dering)
        cfg.symbol_stream = int(symbol_stream)
        self.symbol_stream = int(symbol_stream)
        cfg.inter = int(inter)
        self.inter = int(inter)
        cfg.inter_mc, cfg.mc_refs = int(inter_mc), int(mc_refs)
        self.inter_mc = int(inter_mc)
        cfg.inter_finish = int(inter_finish)
        self.inter_finish = int(inter_finish)
        # late_skip: od_compute_dist with coded_quantizer, qm_is_flat and use_masking above
        cfg.late_skip = int(late_skip)
        self.late_skip = int(late_skip)
        # mc_next: B frames, a third picture (NEXT) per frame and the mv1 grid
        cfg.mc_next = int(mc_next)
        self.mc_next = int(mc_next)
        # frame_quant: each step takes one FRAME_QUANT_DTYPE record per frame (encode(..., frame_quant=)); the config's
        # q0, coded_quantizer, dering_lambda and pvq_qm_q4 are then not read
        cfg.frame_quant = int(frame_quant)
        self.frame_quant = int(frame_quant)
        self._fq = None
        # lossless: quantizer 0 (the Haar-wavelet path); q0, pvq_qm_q4 and the block-size maps are not read
        cfg.lossless = int(lossless)
        self.lossless = int(lossless)
        # haar_dc_quant: keyframe DCs quantised on the device, indices returned as dc_index0..2
        cfg.haar_dc_quant = int(haar_dc_quant)
        self.haar_dc_quant = int(haar_dc_quant)
        # keyframe_quant: keyframes take one FRAME_QUANT_DTYPE record per frame, as frame_quant engines do
        cfg.keyframe_quant = int(keyframe_quant)
        self.keyframe_quant = int(keyframe_quant)
        # frame_types: keyframes and P / B frames in one batch, one type per frame (encode(..., frame_type=))
        cfg.frame_types = int(frame_types)
        self.frame_types = int(frame_types)
        self._ftype = None
        self._ll_slot = None
        self.nrefs = 0
        self.resident = False
        self._pool_src = []
        self.kf = self.L.daala_b200_kf_create(ctypes.byref(cfg))
        if not self.kf:
            raise RuntimeError("daala_b200_kf_create failed (refused configuration, no CUDA device, or out of memory): %s"
                               % self.L.daala_b200_kf_error(None).decode())
        self.buf = Buffers()
        self._check(self.L.daala_b200_kf_device_buffers(self.kf, ctypes.byref(self.buf)), "device_buffers")
        self.sb_row0 = sb_row0
        self.sb_rows = sb_rows if sb_rows > 0 else geom.nvsb
        self.pinned = pinned
        self._host = {}
        self._io = None
        self._out = None
        self.totals = None

    def launches_per_step(self):
        return int(self.L.daala_b200_kf_launches_per_step(self.kf))

    def close(self):
        if getattr(self, "kf", None):
            self.L.daala_b200_kf_destroy(self.kf)
            self.kf = None
        for v in self._host.values():
            if isinstance(v, Pinned):
                v.free()
        self._host = {}

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, what):
        if rc != 0:
            raise _native.CudaError("%s failed with cudaError %d (%s)" % (
                what, rc, self.L.daala_b200_kf_error(self.kf).decode() if self.kf else ""))

    # --- host buffers --------------------------------------------------------------------------
    def _arr(self, name, shape, dtype, pinned=None):
        """(Re)usable host array `name`; pinned when the engine was created with pinned=True (or `pinned`)."""
        cur = self._host.get(name)
        n = int(np.prod(shape))
        if cur is not None:
            a = cur.array if isinstance(cur, Pinned) else cur
            if a.dtype == np.dtype(dtype) and a.size >= n:
                return a.reshape(-1)[:n].reshape(shape)
            if isinstance(cur, Pinned):
                cur.free()
        if self.pinned if pinned is None else pinned:
            cur = Pinned((max(n, 1),), dtype)
            self._host[name] = cur
            return cur.array[:n].reshape(shape)
        a = np.zeros(max(n, 1), dtype)
        self._host[name] = a
        return a[:n].reshape(shape)

    def count_blocks(self, bsize):
        t = Totals()
        g = self.geom
        b = np.ascontiguousarray(bsize, np.uint8)
        assert b.shape == (self.F,) + tuple(g.bsize_shape)
        self._check(self.L.daala_b200_kf_count_blocks(b.ctypes.data, self.F, b.strides[0], b.strides[1], g.nhsb, g.nvsb,
                                                      self.sb_row0, self.sb_rows if self.sb_rows != g.nvsb else 0,
                                                      ctypes.byref(t)), "count_blocks")
        return t

    def stage_dering_levels(self, levels):
        """levels: [F, nvsb, nhsb] uint8 (0..5), staged next to the other inputs (engines created with dering=1)."""
        g = self.geom
        a = self._arr("dlev", (self.F, g.nvsb, g.nhsb), np.uint8)
        a[...] = levels

    def _check_pred(self, pred):
        if bool(self.inter and not self.inter_mc) != (pred is not None):
            raise ValueError("pred= planes are required by an inter engine and refused by a keyframe engine "
                             "and by an inter_mc engine")

    def stage_mc(self, refs, ref_slot, mv_grid, resident=False, mv1_grid=None):
        """Copies one batch's prediction inputs (inter_mc engines) into the host buffers.  refs: per plane an
        array [nrefs, h, w] u8 (frame-sized reference pictures), uploaded into pool slots [0, nrefs); ref_slot: [F, 2]
        pool slots of each frame's GOLD and PREV picture ([F, 3] GOLD, PREV, NEXT on an mc_next engine); mv_grid:
        [F, nvsb*8 + 1, nhsb*8 + 1] mvgrid.MV_PT_DTYPE (mvgrid.pack); mv1_grid (mc_next engines only, required there):
        [F, nvsb*8 + 1, nhsb*8 + 1, 2] int32, each vertex's second vector.  resident=True: the step reads the pool as it
        stands (ref_resident), refs must be None and every slot named must hold a picture (pool_load, an earlier upload,
        or a finish with ref_slot_out)."""
        g = self.geom
        nslot = 3 if self.mc_next else 2
        if (mv1_grid is not None) != bool(self.mc_next):
            raise ValueError("mv1_grid= goes with an mc_next engine, and it needs one")
        if ref_slot is not None and np.shape(ref_slot) != (self.F, nslot):
            raise ValueError("ref_slot= is [F, %d] on this engine (GOLD, PREV%s)" % (nslot, ", NEXT" if self.mc_next else ""))
        if resident:
            if not self.inter_mc or refs is not None or ref_slot is None or mv_grid is None:
                raise ValueError("resident=True goes with an inter_mc engine, needs ref_slot= and mv_grid=, and "
                                 "refuses refs= (the step reads the pool as it stands)")
        elif not self.inter_mc or refs is None or ref_slot is None or mv_grid is None:
            raise ValueError("refs=, ref_slot= and mv_grid= go with an inter_mc engine, and it needs all three")
        self.resident = bool(resident)
        self.nrefs = 0 if resident else int(np.shape(refs[0])[0])
        if not resident:
            for p in range(3):
                a = self._arr("ref%d" % p, (self.nrefs,) + g.plane_shape(p), np.uint8)
                a[...] = refs[p]
        a = self._arr("slot", (self.F, 2), np.int32)
        a[...] = np.asarray(ref_slot)[:, :2]
        a = self._arr("grid", (self.F, g.nvsb * 8 + 1, g.nhsb * 8 + 1), mvgrid.MV_PT_DTYPE)
        a[...] = mv_grid
        if self.mc_next:
            a = self._arr("slot_next", (self.F,), np.int32)
            a[...] = np.asarray(ref_slot)[:, 2]
            a = self._arr("grid1", (self.F, g.nvsb * 8 + 1, g.nhsb * 8 + 1, 2), np.int32)
            a[...] = mv1_grid

    def stage_frame_quant(self, records):
        """Copies the [F] FRAME_QUANT_DTYPE records of one batch into the host buffers (frame_quant and keyframe_quant
        engines; the C call refuses them elsewhere).  None: the next step is submitted without records."""
        if records is None:
            self._fq = None
            return
        r = np.asarray(records)
        if r.dtype != FRAME_QUANT_DTYPE or r.shape != (self.F,):
            raise ValueError("frame_quant= is [%d] FRAME_QUANT_DTYPE records (frame_quant_records builds them)" % self.F)
        self._fq = self._arr("fq", (self.F,), FRAME_QUANT_DTYPE)
        self._fq[...] = r

    def stage_frame_type(self, frame_type):
        """Copies the [F] frame types of one batch (1 = keyframe, 0 = P or B frame) into the host buffers: required by a
        frame_types engine and refused by any other with a ValueError.  The C call refuses values other than 0 and 1."""
        if bool(self.frame_types) != (frame_type is not None):
            raise ValueError("frame_type= is required by an engine created with frame_types=1 and refused by any other")
        if frame_type is None:
            self._ftype = None
            return
        t = np.asarray(frame_type)
        if t.shape != (self.F,):
            raise ValueError("frame_type= is [%d] values, 1 = keyframe, 0 = P or B frame" % self.F)
        self._ftype = self._arr("ftype", (self.F,), np.uint8)
        self._ftype[...] = t

    def stage_inputs(self, planes, bsize, pred=None):
        """Copies one batch into the engine's (pinned) host input buffers.  planes: per plane an array
        [F, h, w] u8 (padded geometry); bsize: [F, nvsb*8, nhsb*8]; pred (inter engines): the
        motion-compensated prediction planes, shaped like `planes`."""
        g = self.geom
        self._check_pred(pred)
        for p in range(3):
            a = self._arr("in%d" % p, (self.F,) + g.plane_shape(p), np.uint8)
            a[...] = planes[p]
            if self.inter and not self.inter_mc:
                a = self._arr("pred%d" % p, (self.F,) + g.plane_shape(p), np.uint8)
                a[...] = pred[p]
        if self.lossless:   # every block is 64x64: no map, no block lists
            self.totals = None
            return
        b = self._arr("bsize", (self.F,) + tuple(g.bsize_shape), np.uint8)
        b[...] = bsize
        self.totals = self.count_blocks(b)

    def symbol_bounds(self, totals=None):
        """Worst-case lengths (index, blocks, bands, pulse_bytes) of the symbol stream arrays for `totals`
        (default: those of the staged batch), from daala_b200_kf_symbol_bounds."""
        b = SymBounds()
        self._check(self.L.daala_b200_kf_symbol_bounds(ctypes.byref(totals or self.totals), self.F, ctypes.byref(b)),
                    "symbol_bounds")
        return b

    def prepare_io(self, symbols=True, recon=True, stream=None, pred=True, dc_grids=True):
        """Builds the daala_b200_kf_io record over the staged inputs and result buffers sized for them.
        stream (default: whether the engine was created with symbol_stream) adds the symbol stream buffers
        sym_index, sym_blocks, sym_bands and sym_pulses (daala_b200/symbols.py), and sym_dc on a symbol_stream=2
        engine (and sym_late_skip on one with late_skip too), sym_hdc on a symbol_stream=1 engine with
        haar_dc_quant, or both sym_dc and sym_hdc on a symbol_stream=3 engine, pinned and sized by
        daala_b200_kf_symbol_bounds; only their used part is copied back.
        late_skip engines return luma_late_skip / chroma_late_skip (symbols.LATE_SKIP_DTYPE per block, block order)
        with the symbols.  On a symbol_stream=2 or 3 engine symbols=False also leaves out the classic DC arrays (the
        stream carries them).  pred=False (inter_mc engines): the prediction planes are not copied back.  dc_grids=False
        (haar_dc_quant engines): the index grids dc_index0..2 are not copied back (sym_hdc carries the same indices)."""
        if self.lossless:
            return self._prepare_io_lossless(recon, pred)
        g, t = self.geom, self.totals
        io = IO()
        for p in range(3):
            io.pixels[p] = self._arr("in%d" % p, (self.F,) + g.plane_shape(p), np.uint8).ctypes.data
        io.bsize = self._arr("bsize", (self.F,) + tuple(g.bsize_shape), np.uint8).ctypes.data
        if self.dering == 1:
            io.dering_level = self._arr("dlev", (self.F, g.nvsb, g.nhsb), np.uint8).ctypes.data
        io.totals = ctypes.pointer(t)
        out = {}
        if recon:
            for p in range(3):
                out["recon%d" % p] = self._arr("out%d" % p, (self.F,) + g.plane_shape(p), np.uint8)
                io.pixels_out[p] = out["recon%d" % p].ctypes.data
        if symbols:
            nl, nc = int(t.n_luma), int(t.n_chroma)
            out["luma_blocks"] = self._arr("lb", (nl,), pvq.BLOCK_DTYPE)
            out["chroma_blocks"] = self._arr("cb", (nc,), pvq.BLOCK_DTYPE)
            out["luma_res"] = self._arr("lr", (nl, 9, 4), np.int16)
            out["chroma_res"] = self._arr("cr", (nc, 9, 4), np.int16)
            out["luma_y16"] = self._arr("ly", (int(t.luma_coefs),), np.int16)
            out["chroma_y16"] = self._arr("cy", (int(t.chroma_coefs),), np.int16)
            out["luma_skip_diff"] = self._arr("ls", (nl,), np.float64)
            out["chroma_skip_diff"] = self._arr("cs", (nc,), np.float64)
            out["chroma_flip"] = self._arr("cf", (nc,), np.int32)
            for k in ("luma_blocks", "chroma_blocks", "luma_res", "chroma_res", "luma_y16", "chroma_y16",
                      "luma_skip_diff", "chroma_skip_diff", "chroma_flip"):
                setattr(io, k, out[k].ctypes.data)
            if self.late_skip:
                from . import symbols as sym
                out["luma_late_skip"] = self._arr("lls", (nl,), sym.LATE_SKIP_DTYPE)
                out["chroma_late_skip"] = self._arr("cls", (nc,), sym.LATE_SKIP_DTYPE)
                io.luma_late_skip, io.chroma_late_skip = out["luma_late_skip"].ctypes.data, out["chroma_late_skip"].ctypes.data
        mc_h2d = self._prepare_io_mc(io, out, pred)
        if self.inter:
            if not self.inter_mc:
                for p in range(3):
                    io.pred_pixels[p] = self._arr("pred%d" % p, (self.F,) + g.plane_shape(p), np.uint8).ctypes.data
        classic_dc = symbols or self.symbol_stream < 2
        if self.inter and classic_dc:
            out["luma_dc"] = self._arr("ld", (int(t.n_luma),), np.int32)
            out["chroma_dc"] = self._arr("cd", (int(t.n_chroma),), np.int32)
            io.luma_dc, io.chroma_dc = out["luma_dc"].ctypes.data, out["chroma_dc"].ctypes.data
        if (self.inter_finish or self.symbol_stream >= 2) and classic_dc:
            out["luma_dc_resid"] = self._arr("ldr", (int(t.n_luma),), np.int32)
            out["chroma_dc_resid"] = self._arr("cdr", (int(t.n_chroma),), np.int32)
            io.luma_dc_resid, io.chroma_dc_resid = out["luma_dc_resid"].ctypes.data, out["chroma_dc_resid"].ctypes.data
        if self._fq is not None:
            io.frame_quant = self._fq.ctypes.data
        if self._ftype is not None:
            io.frame_type = self._ftype.ctypes.data
        if self._ll_slot is not None:   # refused by the C call: a lossy engine has no lossless step
            io.ll_ref_slot_out = self._ll_slot.ctypes.data
        if self.haar_dc_quant and dc_grids:
            for p in range(3):
                h, w = g.plane_shape(p)
                out["dc_index%d" % p] = self._arr("dci%d" % p, (self.F, h >> 2, w >> 2), np.int32)
                io.dc_index[p] = out["dc_index%d" % p].ctypes.data
        out["counts"] = self._arr("cnt", (32,), np.int32)
        io.counts = out["counts"].ctypes.data
        if self.dering:
            out["dering_levels"] = self._arr("dlev_out", (self.F, g.nvsb, g.nhsb), np.uint8)
            io.dering_level_out = out["dering_levels"].ctypes.data
        self.d2h_bytes = sum(v.nbytes for v in out.values())
        if self.symbol_stream if stream is None else stream:
            from . import symbols as sym
            b = self.symbol_bounds(t)
            out["sym_index"] = self._arr("si", (self.F, 6), np.int64, pinned=True)
            out["sym_blocks"] = self._arr("sb", (int(b.blocks),), sym.BLOCK_DTYPE, pinned=True)
            out["sym_bands"] = self._arr("sn", (int(b.bands), 4), np.int16, pinned=True)
            out["sym_pulses"] = self._arr("sp", (int(b.pulse_bytes),), np.uint8, pinned=True)
            for k, cap in (("sym_index", b.index), ("sym_blocks", b.blocks), ("sym_bands", b.bands),
                           ("sym_pulses", b.pulse_bytes)):
                setattr(io, k, out[k].ctypes.data)
                setattr(io, k + "_cap", int(cap))
            if self.symbol_stream >= 2:
                out["sym_dc"] = self._arr("sd", (int(b.blocks),), sym.DC_DTYPE, pinned=True)
                io.sym_dc, io.sym_dc_cap = out["sym_dc"].ctypes.data, int(b.blocks)
                if self.late_skip:
                    out["sym_late_skip"] = self._arr("sls", (int(b.blocks),), sym.LATE_SKIP_DTYPE, pinned=True)
                    io.sym_late_skip, io.sym_late_skip_cap = out["sym_late_skip"].ctypes.data, int(b.blocks)
            if self.haar_dc_quant:
                out["sym_hdc"] = self._arr("shdc", (int(b.blocks),), sym.HDC_DTYPE, pinned=True)
                io.sym_hdc, io.sym_hdc_cap = out["sym_hdc"].ctypes.data, int(b.blocks)
        self._io, self._out = io, out
        px = sum(int(np.prod(g.plane_shape(p))) for p in range(3))
        self.h2d_bytes = (px * self.F * (2 if self.inter and not self.inter_mc else 1) + int(np.prod(g.bsize_shape)) * self.F
                          + mc_h2d)
        if self._fq is not None:   # the records, each frame's deringing thresholds (int32 [2][6]) and band quantisers ([3][32])
            self.h2d_bytes += self.F * (FRAME_QUANT_DTYPE.itemsize + 48 + 384)
        if self._ftype is not None:
            self.h2d_bytes += self.F
        return out

    def stage_ll_ref_slot_out(self, slots):
        """[F] int32 pool slots that receive each frame's lossless reconstruction (-1 = not stored), or None: nothing
        stored (lossless engines with inter_mc; the C call refuses the table elsewhere)."""
        if slots is None:
            self._ll_slot = None
            return
        self._ll_slot = self._arr("llslot", (self.F,), np.int32)
        self._ll_slot[...] = slots

    def _prepare_io_mc(self, io, out, pred):
        """The inter_mc inputs of `io` staged by stage_mc (the reference pictures unless resident, the slot map, the MV
        grids) and, with pred, the prediction planes as outputs pred0..2; returns the bytes of those inputs (0 on an
        engine without inter_mc)."""
        if not self.inter_mc:
            return 0
        g = self.geom
        io.ref_resident = int(self.resident)
        for p in range(3):
            if not self.resident:
                io.ref_pixels[p] = self._arr("ref%d" % p, (self.nrefs,) + g.plane_shape(p), np.uint8).ctypes.data
            if pred:
                out["pred%d" % p] = self._arr("pred%d" % p, (self.F,) + g.plane_shape(p), np.uint8)
                io.pred_pixels_out[p] = out["pred%d" % p].ctypes.data
        io.nrefs = self.nrefs
        nvert = self.F * (g.nvsb * 8 + 1) * (g.nhsb * 8 + 1)
        io.ref_slot = self._arr("slot", (self.F, 2), np.int32).ctypes.data
        io.mv_grid = self._arr("grid", (self.F, g.nvsb * 8 + 1, g.nhsb * 8 + 1), mvgrid.MV_PT_DTYPE).ctypes.data
        px = sum(int(np.prod(g.plane_shape(p))) for p in range(3))
        h2d = px * self.nrefs + 8 * self.F + nvert * mvgrid.MV_PT_DTYPE.itemsize
        if self.mc_next:   # the NEXT slot of each frame and the mv1 of each vertex
            io.ref_slot_next = self._arr("slot_next", (self.F,), np.int32).ctypes.data
            io.mv1_grid = self._arr("grid1", (self.F, g.nvsb * 8 + 1, g.nhsb * 8 + 1, 2), np.int32).ctypes.data
            h2d += 4 * self.F + nvert * 8
        return h2d

    def _prepare_io_lossless(self, recon, pred):
        """prepare_io of a lossless engine: the inputs, [the prediction inputs], and as outputs the reconstruction
        (recon0..2), the residual planes ll_coeffs0..2 ([F, h, w] int16), the root sums ll_blocks ([F, nvsb, nhsb, 3, 4]
        int32: tree_sum[0][1], [1][0], [1][1], 0 per plane), [pred0..2] and the counters."""
        g = self.geom
        io = IO()
        out = {}
        for p in range(3):
            io.pixels[p] = self._arr("in%d" % p, (self.F,) + g.plane_shape(p), np.uint8).ctypes.data
            if recon:
                out["recon%d" % p] = self._arr("out%d" % p, (self.F,) + g.plane_shape(p), np.uint8)
                io.pixels_out[p] = out["recon%d" % p].ctypes.data
            out["ll_coeffs%d" % p] = self._arr("llc%d" % p, (self.F,) + g.plane_shape(p), np.int16)
            io.ll_coeffs[p] = out["ll_coeffs%d" % p].ctypes.data
            if self.inter and not self.inter_mc:
                io.pred_pixels[p] = self._arr("pred%d" % p, (self.F,) + g.plane_shape(p), np.uint8).ctypes.data
        out["ll_blocks"] = self._arr("llb", (self.F, g.nvsb, g.nhsb, 3, 4), np.int32)
        io.ll_blocks = out["ll_blocks"].ctypes.data
        mc_h2d = self._prepare_io_mc(io, out, pred)
        if self._ll_slot is not None:
            io.ll_ref_slot_out = self._ll_slot.ctypes.data
        out["counts"] = self._arr("cnt", (32,), np.int32)
        io.counts = out["counts"].ctypes.data
        self.d2h_bytes = sum(v.nbytes for v in out.values())
        self._io, self._out = io, out
        px = sum(int(np.prod(g.plane_shape(p))) for p in range(3))
        self.h2d_bytes = px * self.F * (2 if self.inter and not self.inter_mc else 1) + mc_h2d
        if self._ll_slot is not None:
            self.h2d_bytes += 4 * self.F
        return out

    def submit(self):
        self._check(self.L.daala_b200_kf_submit(self.kf, ctypes.byref(self._io)), "kf_submit")

    def wait(self):
        self._check(self.L.daala_b200_kf_wait(self.kf), "kf_wait")
        self._pool_src = []
        return self._out

    def stream_d2h_bytes(self):
        """Bytes the last submit copied of the symbol stream (after wait): the index and the used part of the
        other arrays (block records, band records, pulses and, on symbol_stream=2 engines, DC records and, with
        late_skip, late-skip records; with haar_dc_quant, the keyframe DC records; on symbol_stream=3 engines both the
        DC records and the keyframe DC records)."""
        from . import symbols as sym
        idx = self._out["sym_index"]
        blocks = int(idx[:, 1].sum())
        dc = blocks * sym.DC_DTYPE.itemsize if "sym_dc" in self._out else 0
        dc += blocks * sym.LATE_SKIP_DTYPE.itemsize if "sym_late_skip" in self._out else 0
        dc += blocks * sym.HDC_DTYPE.itemsize if "sym_hdc" in self._out else 0
        return idx.nbytes + blocks * sym.BLOCK_DTYPE.itemsize + int(idx[:, 3].sum()) * 8 + int(idx[:, 5].sum()) + dc

    def encode(self, planes, bsize, symbols=True, recon=True, dering_levels=None, stream=None, pred=None, refs=None,
               ref_slot=None, mv_grid=None, resident=False, mv1_grid=None, frame_quant=None, ll_ref_slot_out=None,
               dc_grids=True, frame_type=None):
        """One batch end to end through the C ABI with host buffers; returns the result arrays (views of
        the engine's host buffers: copy what must survive the next call).  pred: see stage_inputs; refs, ref_slot,
        mv_grid, resident, mv1_grid (inter_mc engines, which also return the prediction as pred0..2): see stage_mc;
        frame_quant (frame_quant and keyframe_quant engines, required there): [F] FRAME_QUANT_DTYPE records, see
        stage_frame_quant;
        frame_type (frame_types engines, required there and refused elsewhere): see stage_frame_type; such an engine
        returns the outputs of both kinds, each 0 on the blocks and frames of the other kind (include/daala_b200.h);
        ll_ref_slot_out (lossless engines with inter_mc): see stage_ll_ref_slot_out; dc_grids: see prepare_io.  On a lossless engine bsize is not
        read (None is fine) and the results are those of _prepare_io_lossless.  Raises
        when the batch exceeded the block capacity, or (inter_mc) when a used vertex names a picture other than GOLD /
        PREV (/ NEXT on mc_next engines) or a vector reaches past the reference's edge extension: the reference
        encoder's result is undefined there."""
        self.stage_frame_type(frame_type)
        self.stage_inputs(planes, bsize, pred)
        if (self.inter_mc or refs is not None or ref_slot is not None or mv_grid is not None or resident
                or mv1_grid is not None):
            self.stage_mc(refs, ref_slot, mv_grid, resident, mv1_grid)
        if self.dering == 1:
            self.stage_dering_levels(dering_levels)
        self.stage_frame_quant(frame_quant)
        self.stage_ll_ref_slot_out(ll_ref_slot_out)
        self.prepare_io(symbols, recon, stream, dc_grids=dc_grids)
        self.submit()
        out = self.wait()
        if int(out["counts"][CNT["error"]]):
            raise RuntimeError("keyframe engine: block capacity exceeded (max_blocks_div too large)")
        if self.inter_mc:
            bad, beyond = int(out["counts"][CNT["mc_bad_ref"]]), int(out["counts"][CNT["mc_beyond"]])
            if bad or beyond:
                raise RuntimeError("keyframe engine: MV grid outside the reference's definition: %d leaf corners with a "
                                   "ref other than GOLD / PREV%s, %d corner windows past the edge extension"
                                   % (bad, " / NEXT" if self.mc_next else "", beyond))
        return out

    def prepare_finish(self, luma_skip, luma_dc, chroma_skip, chroma_dc, dering_levels=None, ref_slot_out=None):
        """Stages the host coder's decisions for the last submitted batch (inter_finish engines) and builds the
        daala_b200_kf_finish_io record; returns the result arrays finish_submit fills: recon0..2, bskip0..2
        ([F, plane_h / 4, nhsb * 16] u8, state->bskip[pli] of each frame with row stride state->skip_stride; a chroma
        row's columns past plane_w / 4 stay 0) and dering_levels ([F, nvsb, nhsb], the levels applied; on an
        inter_finish=2 engine the levels the pass searched, and dering_levels must be None: the C call refuses
        levels there).  ref_slot_out (engines with inter_mc too): [F] int32, the pool slot that receives each frame's
        reconstruction, -1 = not stored; None stores nothing."""
        t = self.totals
        fio = FinishIO()
        n = {"luma": int(t.n_luma), "chroma": int(t.n_chroma)}
        for kind, sk, dc in (("luma", luma_skip, luma_dc), ("chroma", chroma_skip, chroma_dc)):
            a = self._arr("fs_" + kind, (n[kind],), np.uint8)
            a[...] = sk
            setattr(fio, kind + "_skip", a.ctypes.data)
            a = self._arr("fd_" + kind, (n[kind],), np.int32)
            a[...] = dc
            setattr(fio, kind + "_dc", a.ctypes.data)
        return self._prepare_finish_rest(fio, sum(n.values()), dering_levels, ref_slot_out)

    def prepare_finish_stream(self, skip, dc, dering_levels=None, ref_slot_out=None):
        """prepare_finish with the decisions in stream order (symbol_stream=2 or 3 engines with inter_finish): skip
        and dc have one entry per block record of the last step's stream, frames one after the other (the order of its
        sym_blocks).  symbols.stream_to_classic gives each record's index in the classic block order.  On a
        symbol_stream=3 engine the keyframes' entries are checked as any other and otherwise not read."""
        t = self.totals
        fio = FinishIO()
        n = int(t.n_luma) + int(t.n_chroma)
        a = self._arr("fs_stream", (n,), np.uint8)
        a[...] = skip
        fio.stream_skip = a.ctypes.data
        a = self._arr("fd_stream", (n,), np.int32)
        a[...] = dc
        fio.stream_dc = a.ctypes.data
        return self._prepare_finish_rest(fio, n, dering_levels, ref_slot_out)

    def _prepare_finish_rest(self, fio, nblocks, dering_levels, ref_slot_out):
        """The levels, the slot table and the result buffers of a finish record whose decisions are staged."""
        g = self.geom
        if dering_levels is not None:
            a = self._arr("flev", (self.F, g.nvsb, g.nhsb), np.uint8)
            a[...] = dering_levels
            fio.dering_level = a.ctypes.data
        if ref_slot_out is not None:
            a = self._arr("fslot", (self.F,), np.int32)
            a[...] = ref_slot_out
            fio.ref_slot_out = a.ctypes.data
        out = {}
        for p in range(3):
            out["recon%d" % p] = self._arr("fout%d" % p, (self.F,) + g.plane_shape(p), np.uint8)
            fio.pixels_out[p] = out["recon%d" % p].ctypes.data
            out["bskip%d" % p] = self._arr("fskip%d" % p, (self.F, g.plane_shape(p)[0] // 4, g.nhsb * 16), np.uint8)
            fio.bskip_out[p] = out["bskip%d" % p].ctypes.data
        out["dering_levels"] = self._arr("flev_out", (self.F, g.nvsb, g.nhsb), np.uint8)
        fio.dering_level_out = out["dering_levels"].ctypes.data
        # one skip byte and one int32 DC per block, the levels, the slot table
        self.finish_h2d_bytes = (5 * nblocks + (self.F * g.nvsb * g.nhsb if dering_levels is not None else 0)
                                 + (4 * self.F if ref_slot_out is not None else 0))
        self.finish_d2h_bytes = sum(v.nbytes for v in out.values())
        self._fio, self._fout = fio, out
        return out

    def finish_submit(self):
        self._check(self.L.daala_b200_kf_finish(self.kf, ctypes.byref(self._fio)), "kf_finish")

    def finish(self, luma_skip, luma_dc, chroma_skip, chroma_dc, dering_levels=None, ref_slot_out=None):
        """The finishing pass of the last encoded P-frame batch (inter_finish engines): per block (block order of
        the luma / chroma results of encode) the host coder's skip decision (0 or 1) and final DC index, per
        superblock the deringing level (None: all 0; inter_finish=2 engines search the levels, so None there), and
        per frame the pool slot that receives its reconstruction (ref_slot_out, engines with inter_mc; None: none).
        Returns the reconstruction the decoder makes, the skip maps and the levels applied (see prepare_finish);
        views of the engine's host buffers."""
        self.prepare_finish(luma_skip, luma_dc, chroma_skip, chroma_dc, dering_levels, ref_slot_out)
        self.finish_submit()
        self.wait()
        return self._fout

    def finish_stream(self, skip, dc, dering_levels=None, ref_slot_out=None):
        """finish with the decisions in the order of the last step's symbol stream (see prepare_finish_stream)."""
        self.prepare_finish_stream(skip, dc, dering_levels, ref_slot_out)
        self.finish_submit()
        self.wait()
        return self._fout

    def pool_load(self, slot, planes):
        """Enqueues the copy of one frame-sized picture into pool slot `slot` (inter_mc engines), ordered with submit
        and finish on the engine's stream.  planes: three [h, w] u8 host arrays (padded geometry), or three device
        addresses, e.g. a keyframe engine's buf.pixels_out[p] + f * plane bytes (that engine waited for first)."""
        g = self.geom
        ptrs = (c_void_p * 3)()
        for p in range(3):
            if isinstance(planes[p], (int, np.integer)):
                ptrs[p] = int(planes[p])
            elif planes[p] is not None:
                a = np.ascontiguousarray(planes[p], np.uint8)
                if a.shape != g.plane_shape(p):
                    raise ValueError("pool_load: plane %d is %s, the engine's plane is %s" % (p, a.shape, g.plane_shape(p)))
                self._pool_src.append(a)   # the copy may still read it until wait()
                ptrs[p] = a.ctypes.data
        self._check(self.L.daala_b200_kf_pool_load(self.kf, int(slot), ptrs), "kf_pool_load")

    # --- device-resident use -------------------------------------------------------------------
    def run_device(self, phases=PH_ALL, graph=True):
        self._check(self.L.daala_b200_kf_run_device(self.kf, phases, 1 if graph else 0), "kf_run_device")

    def time_device(self, phases=PH_ALL, graph=True, reps=1):
        """Milliseconds (CUDA events on the engine's stream) for `reps` repetitions of the phases."""
        ms = ctypes.c_float()
        self._check(self.L.daala_b200_kf_time_device(self.kf, phases, 1 if graph else 0, reps, ctypes.byref(ms)),
                    "kf_time_device")
        return float(ms.value)

    def upload(self, planes, bsize, pred=None, frame_quant=None):
        """Copies one batch straight into the engine's device buffers for run_device; frame_quant (frame_quant and
        keyframe_quant engines): the [F] FRAME_QUANT_DTYPE records the step's kernels read, checked and loaded with the
        tables submit derives from them (daala_b200_kf_load_frame_quant)."""
        g = self.geom
        self._check_pred(pred)
        if frame_quant is not None:
            if not (self.frame_quant or self.keyframe_quant):
                raise ValueError("frame_quant= needs an engine created with frame_quant=1 or keyframe_quant=1")
            r = np.ascontiguousarray(frame_quant, FRAME_QUANT_DTYPE)
            assert r.shape == (self.F,)
            self._check(self.L.daala_b200_kf_load_frame_quant(self.kf, r.ctypes.data), "upload")
        for p in range(3):
            for dst, src in ((self.buf.pixels[p], planes[p]),) + (((self.buf.pred_pixels[p], pred[p]),) if pred is not None else ()):
                a = np.ascontiguousarray(src, np.uint8)
                assert a.shape == (self.F,) + g.plane_shape(p)
                self._check(self.L.daala_b200_device_copy(dst, a.ctypes.data, a.nbytes, 0), "upload")
        b = np.ascontiguousarray(bsize, np.uint8)
        assert b.shape == (self.F,) + tuple(g.bsize_shape)
        self._check(self.L.daala_b200_device_copy(self.buf.bsize, b.ctypes.data, b.nbytes, 0), "upload")

    def download(self, ptr, shape, dtype):
        self.wait()
        a = np.zeros(shape, dtype)
        if a.nbytes:
            self._check(self.L.daala_b200_device_copy(a.ctypes.data, ptr, a.nbytes, 1), "download")
        return a

    def counts(self):
        return self.download(self.buf.counts, (32,), np.int32)

    def coeff_plane(self, p):
        return self.download(self.buf.coeffs[p], (self.F,) + self.geom.plane_shape(p), np.int32)

    def pred_coeff_plane(self, p):
        """The transformed prediction md of plane p (inter engines)."""
        return self.download(self.buf.pred_coeffs[p], (self.F,) + self.geom.plane_shape(p), np.int32)

    def pool_plane(self, p):
        """The reference-picture pool of plane p, [mc_refs, h, w] u8 (inter_mc engines)."""
        return self.download(self.buf.ref_pixels[p], (self.buf.mc_refs,) + self.geom.plane_shape(p), np.uint8)

    def recon_plane(self, p):
        return self.download(self.buf.pixels_out[p], (self.F,) + self.geom.plane_shape(p), np.uint8)


def band_records(blocks, res, geom, pli, frame):
    """[h/4, w/4, 9, 4] int16 array of one plane of one frame with each block's band records stored at
    its origin (the layout the oracle's recording hook uses); unwritten entries are -32768."""
    h, w = geom.plane_shape(pli)
    out = np.full((h // 4, w // 4, 9, 4), -32768, np.int16)
    sel = (blocks["pli"] == pli) & (blocks["frame"] == frame)
    b = blocks[sel]
    r = res[sel]
    nb = np.array([1, 4, 7, 9, 9])[b["bs"]]
    for band in range(9):
        m = nb > band
        out[b["y0"][m] >> 2, b["x0"][m] >> 2, band] = r[m, band]
    return out
