"""CPU tests of the host logic: geometry, sharding, block/band lists, the
exported C ABI, and the N>1 border exchange over gloo (world_size 2)."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_geometry_and_row_shards():
    from daala_b200.frame import Geometry
    g = Geometry(3840, 2160)
    assert (g.nhsb, g.nvsb, g.frame_w, g.frame_h) == (60, 34, 3840, 2176)
    assert g.plane_shape(1) == (1088, 1920)
    rows = [g.shard_rows(r, 8) for r in range(8)]
    assert [n for _, n in rows] == [5, 5, 4, 4, 4, 4, 4, 4]          # SURVEY.md 8(d) config 4
    assert rows[0][0] == 0 and all(rows[i][0] + rows[i][1] == rows[i + 1][0] for i in range(7))
    g8 = Geometry(7680, 4320)
    assert [g8.shard_rows(r, 8)[1] for r in range(8)] == [9, 9, 9, 9, 8, 8, 8, 8]


@pytest.mark.parametrize("mode", ["mixed", "4", "8", "16", "32", "64"])
def test_block_and_band_lists_cover_every_plane_once(mode):
    from daala_b200 import pvq, synth
    from daala_b200.frame import Geometry
    g = Geometry(320, 200)
    bsize = synth.block_size_map(g, mode, seed=4)
    blocks = pvq.block_list(bsize, g)
    for pli in range(3):
        ph, pw = g.plane_shape(pli)
        cover = np.zeros((ph, pw), np.int32)
        for b in blocks[blocks["pli"] == pli]:
            n = 4 << int(b["bs"])
            assert b["x0"] % n == 0 and b["y0"] % n == 0
            cover[b["y0"]:b["y0"] + n, b["x0"]:b["x0"] + n] += 1
        assert (cover == 1).all()
    total = pvq.assign_offsets(blocks)
    assert total == int(np.minimum(16 << (2 * blocks["bs"].astype(np.int64)), 512).sum())
    lists = pvq.band_lists(blocks)
    nb = sum(pvq.NBANDS[int(b)] for b in blocks["bs"])
    assert sum(len(v) for v in lists.values()) == nb
    # every (block, band) pair exactly once
    allb = np.concatenate(list(lists.values()))
    assert len(np.unique(allb)) == len(allb)
    # shards partition the block list
    parts = [pvq.block_list(bsize, g, sb_row0=r0, sb_rows=n) for r0, n in (g.shard_rows(r, 2) for r in range(2))]
    assert sum(len(p) for p in parts) == len(blocks)


def test_band_wave_lists_respect_the_intra_dependencies():
    """Every (block, band) entry appears once; an entry of wave w > 1 has the same band of a
    same-size neighbour in wave w - 1 and none later (od_hv_intra_pred, src/intra.c:37)."""
    from daala_b200 import pvq, synth
    from daala_b200.frame import Geometry
    geom = Geometry(512, 320)
    maps = [synth.block_size_map(geom, "mixed", seed=s) for s in (3, 4)]
    blocks = np.concatenate([pvq.block_list(b, geom, frame=f) for f, b in enumerate(maps)])
    luma, top, left, depth = pvq.sort_by_depth(pvq.raster_order(blocks[blocks["pli"] == 0]), maps, geom)
    bulk, chain, slices = pvq.band_wave_lists(luma, top, left, depth)
    wave = {}
    for k in (16, 32, 128):
        assert set((bulk[k] & 15).tolist()) <= {3, 6}
        for e in bulk[k].tolist():
            wave[e] = 0
        assert sum(c for _, c in slices[k]) == len(chain[k])
        for w, (a, c) in enumerate(slices[k]):
            assert c > 0
            for e in chain[k][a:a + c].tolist():
                assert e not in wave
                wave[e] = w + 1
    total = sum(pvq.NBANDS[int(b)] for b in luma["bs"])
    assert len(wave) == total
    for e, w in wave.items():
        blk, band = e >> 4, e & 15
        need = []
        if band in (0, 1, 4, 7) and top[blk] >= 0:
            need.append((int(top[blk]) << 4) | band)
        if band in (0, 2, 5, 8) and left[blk] >= 0:
            need.append((int(left[blk]) << 4) | band)
        if band in (3, 6):
            assert w == 0
            continue
        assert luma["bs"][blk] == luma["bs"][top[blk]] if top[blk] >= 0 else True
        assert w == 1 + max([wave[x] for x in need], default=0)


@pytest.mark.parametrize("mode", ["mixed", "4", "8", "64"])
def test_native_list_builder_equals_the_numpy_construction(mode):
    """daala_b200_host_keyframe_lists (C++, csrc/host_lists.cu) against the numpy builders HotPath uses:
    identical arrays in identical order (host code only -- no GPU)."""
    import time
    from daala_b200 import pvq, synth
    from daala_b200.frame import Geometry
    geom = Geometry(704, 448)
    maps = [synth.block_size_map(geom, mode, seed=s) for s in (3, 4, 5)]
    t0 = time.perf_counter()
    nat = pvq.native_keyframe_lists(maps, geom)
    t_native = time.perf_counter() - t0
    t0 = time.perf_counter()
    blocks = np.concatenate([pvq.block_list(b, geom, frame=f) for f, b in enumerate(maps)])
    luma, top, left, depth = pvq.sort_by_depth(pvq.raster_order(blocks[blocks["pli"] == 0]), maps, geom)
    luma = luma.copy()
    luma_total = pvq.assign_offsets(luma)
    bulk, chain, slices = pvq.band_wave_lists(luma, top, left, depth)
    chroma = pvq.mark_luma4x4(blocks[blocks["pli"] != 0].copy(), maps)
    chroma = chroma[np.argsort(chroma["bs"], kind="stable")].copy()
    chroma_total = pvq.assign_offsets(chroma)
    chroma_lists = pvq.band_lists(chroma)
    t_numpy = time.perf_counter() - t0
    assert np.array_equal(nat["luma"], luma)
    assert np.array_equal(nat["dep_top"], top) and np.array_equal(nat["dep_left"], left)
    assert np.array_equal(nat["depth"], depth)
    assert nat["luma_total"] == luma_total and nat["chroma_total"] == chroma_total
    assert np.array_equal(nat["chroma"], chroma)
    for k in (16, 32, 128):
        assert np.array_equal(nat["chain"][k], chain[k]), k
        assert nat["chain_slices"][k] == slices[k], k
        assert np.array_equal(nat["bulk"][k], bulk[k]), k
        assert np.array_equal(nat["chroma_lists"][k], chroma_lists[k]), k
        waves = np.repeat(np.arange(len(slices[k]), dtype=np.uint16), [c for _, c in slices[k]])
        assert np.array_equal(nat["chain_wave"][k], waves), k
    del t_native, t_numpy    # timings belong in DESIGN.md, not in an assertion


@pytest.mark.parametrize("mode", ["mixed", "4", "16", "64"])
def test_tensor_op_list_builder_equals_the_native_builder(mode):
    """daala_b200/lists_torch.py (device-agnostic tensor ops, meant to run where the block-size maps
    already live) against the C++ host builder: identical arrays (run here on CPU tensors)."""
    import torch
    from daala_b200 import lists_torch, pvq, synth
    from daala_b200.frame import Geometry
    geom = Geometry(576, 320)
    maps = [synth.block_size_map(geom, mode, seed=s) for s in (7, 8, 9)]
    nat = pvq.native_keyframe_lists(maps, geom)
    got = lists_torch.keyframe_lists(torch.from_numpy(np.stack(maps)), geom.nhsb, geom.nvsb)
    assert np.array_equal(got["luma"].numpy().reshape(-1).view(pvq.BLOCK_DTYPE), nat["luma"])
    assert np.array_equal(got["chroma"].numpy().reshape(-1).view(pvq.BLOCK_DTYPE), nat["chroma"])
    for k in ("dep_top", "dep_left", "depth"):
        assert np.array_equal(got[k].numpy(), nat[k]), k
    assert got["luma_total"] == nat["luma_total"] and got["chroma_total"] == nat["chroma_total"]
    for k in (16, 32, 128):
        assert np.array_equal(got["chain"][k].numpy().view(np.uint32), nat["chain"][k]), k
        assert np.array_equal(got["chain_wave"][k].numpy().view(np.uint16), nat["chain_wave"][k]), k
        assert got["chain_slices"][k] == nat["chain_slices"][k], k
        assert np.array_equal(got["bulk"][k].numpy().view(np.uint32), nat["bulk"][k]), k
        assert np.array_equal(got["chroma_lists"][k].numpy().view(np.uint32), nat["chroma_lists"][k]), k


@pytest.mark.parametrize("name", ["hvs", "flat"])
def test_host_init_qm_reproduces_the_reference_tables(name):
    """daala_b200.pvq.init_qm (restatement of od_init_qm, src/pvq.c:322) against the tables exported from the
    reference build (daala_b200/data/qm_*.npy) and, when oracle/_ref is present, against od_init_qm itself."""
    from daala_b200 import pvq
    from tests import oracle_lib, pvq_cases
    inputs = pvq.qm_inputs()
    qm, qm_inv = pvq.init_qm(inputs["qm8_" + name], inputs)
    want, want_inv = pvq.default_qm(name == "hvs")
    assert np.array_equal(qm, want) and np.array_equal(qm_inv, want_inv)
    ref = oracle_lib.load_ref()
    if ref is not None:
        a, b = pvq_cases.reference_qm(ref, name == "hvs")
        assert np.array_equal(qm, a) and np.array_equal(qm_inv, b)
    # a custom matrix goes through the same path: doubling every entry halves the (non-DC) scale
    q2, _ = pvq.init_qm(inputs["qm8_" + name] * 2, inputs)
    assert q2[0] == 2048 and abs(int(q2[5]) * 2 - int(qm[5])) <= 1


def test_hot_path_plumbing_is_identical_with_device_built_lists():
    """HotPath.set_block_sizes(device_lists=True) (tensor-op construction where the maps live) must hand the
    kernels byte-identical descriptors, lists, neighbour indices and wave slices as the numpy path.  Dry run on
    CPU tensors: buffers are allocated, no kernel is launched."""
    import torch
    from daala_b200 import synth
    from daala_b200.frame import Geometry
    from daala_b200.pipeline import HotPath
    geom = Geometry(448, 320)
    maps = [synth.block_size_map(geom, "mixed", seed=s) for s in (11, 12)]
    hps = []
    for device_lists in (False, True):
        hp = HotPath(geom, nframes=2, device="cpu", q0=40, is_keyframe=1, keyframe_prediction=True)
        hp.set_block_sizes(maps, device_lists=device_lists)
        hps.append(hp)
    a, b = hps
    for x, y in ((a.batch_luma, b.batch_luma), (a.batch_chroma, b.batch_chroma)):
        assert torch.equal(x.blocks, y.blocks) and (x.total, x.nblocks) == (y.total, y.nblocks)
        assert x.in_.shape == y.in_.shape and x.res_k.shape == y.res_k.shape and x.y16.shape == y.y16.shape
        assert (x.params.q0, x.params.is_keyframe, x.params.use_masking) == (y.params.q0, y.params.is_keyframe,
                                                                               y.params.use_masking)
    for k in (16, 32, 128):
        assert torch.equal(a.batch_chroma.lists[k], b.batch_chroma.lists[k])
        assert torch.equal(a.batch_luma.chain_lists[k], b.batch_luma.chain_lists[k])
        assert torch.equal(a.batch_luma.bulk_lists[k], b.batch_luma.bulk_lists[k])
        assert torch.equal(a.batch_luma.chain_waves[k], b.batch_luma.chain_waves[k])
        assert a.batch_luma.chain_slices[k] == b.batch_luma.chain_slices[k]
        assert b.batch_luma._order_keys.numel() >= max(b.batch_luma.chain_lists[k].numel(),
                                                       b.batch_luma.bulk_lists[k].numel())
    assert torch.equal(a.batch_luma.dep_top, b.batch_luma.dep_top)
    assert torch.equal(a.batch_luma.dep_left, b.batch_luma.dep_left)
    assert a.batch_luma.max_depth == b.batch_luma.max_depth


def test_header_is_plain_c_and_reference_arm_prints_the_contract_line(tmp_path):
    """include/daala_b200.h must compile as C99 (the reference is C and binds to it directly), and
    `bench.py --impl reference` must print one JSON line with the contract's keys (CPU only)."""
    import json
    src = tmp_path / "hdr.c"
    src.write_text('#include "daala_b200.h"\nint main(void) { daala_b200_pvq_params p; (void)p; return 0; }\n')
    inc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include")
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only", "-I", inc, str(src)],
                   check=True)
    root = os.path.dirname(inc)
    r = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--steps", "1",
                        "--warmup", "1"], capture_output=True, text=True, timeout=600, cwd=root)
    assert r.returncode == 0, r.stderr[-2000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    for key in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better",
                "config", "cpu_baseline", "e2e"):
        assert key in line, key
    assert line["impl"] == "reference" and line["value"] > 0
    assert line["cpu_baseline"]["kind"] in ("reference", "port") and line["cpu_baseline"]["cores"] >= 1
    assert line["e2e"]["h2d_bytes_per_step"] == 0 and line["e2e"]["d2h_bytes_per_step"] == 0


def test_library_exports_every_declared_symbol():
    """The built library must export everything include/daala_b200.h declares
    (no compute calls here: the build container has no GPU)."""
    import ctypes
    from daala_b200 import _native
    L = _native.lib()
    hdr = open(os.path.join(ROOT, "include", "daala_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    names = set(re.findall(r"\b((?:od|daala_b200)_[a-z0-9_]+)\s*\(", hdr))
    names |= {"OD_FDCT_2D_CUDA", "OD_IDCT_2D_CUDA", "OD_PRE_FILTER_CUDA", "OD_POST_FILTER_CUDA"}
    # the reference's own table names: what its objects resolve when this library replaces dct.o / filter.o
    names |= {"OD_FDCT_2D_C", "OD_IDCT_2D_C", "OD_FDCT_1D", "OD_IDCT_1D", "OD_PRE_FILTER", "OD_POST_FILTER",
              "OD_FILTER_PARAMS4"}
    assert len(names) >= 60
    missing = [n for n in sorted(names) if not hasattr(L, n)]
    assert not missing, missing
    assert L.daala_b200_version().startswith(b"daala_b200")
    assert L.daala_b200_device_count() >= 0


def test_unknown_pvq_kernel_modes_are_refused_before_any_launch():
    """daala_b200_pvq_encode_bands_mode knows modes 0-3; any other mode returns cudaErrorInvalidValue (1) even for
    an empty band list, so nothing is launched and no device is needed to check it."""
    import ctypes
    from daala_b200 import pvq
    L = pvq._bind()
    prm = pvq.PvqParams()
    for mode in (4, 11, 20, 30, -1):
        assert L.daala_b200_pvq_encode_bands_mode(ctypes.byref(prm), None, 0, 128, mode, None) == 1, mode
    for mode in range(4):
        assert L.daala_b200_pvq_encode_bands_mode(ctypes.byref(prm), None, 0, 128, mode, None) == 0, mode


def test_native_struct_layouts_match_the_header():
    import ctypes
    from daala_b200 import _native, mc, pvq
    assert ctypes.sizeof(_native.Plane) == 4 * 8 + 6 * 4 + 4 * 8
    assert ctypes.sizeof(_native.Frame) == 3 * ctypes.sizeof(_native.Plane) + 8 + 10 * 4 + 8 + 3 * 8   # + post16[3]
    assert pvq.BLOCK_DTYPE.itemsize == 12
    assert mc.MC_BLOCK_DTYPE.itemsize == 40 and mc.MATCH_JOB_DTYPE.itemsize == 16
    assert ctypes.sizeof(pvq.PvqParams) % 8 == 0


def test_ctypes_mirrors_have_the_sizes_the_c_compiler_gives(tmp_path):
    """sizeof() of every ABI struct as gcc lays it out vs the ctypes / numpy mirrors on the Python side."""
    import ctypes
    from daala_b200 import _native, mc, pvq
    from tests.test_gpu_dering import DeringParams
    from daala_b200 import engine
    names = ["daala_b200_plane", "daala_b200_frame", "daala_b200_pvq_block", "daala_b200_pvq_params",
             "daala_b200_mc_block", "daala_b200_match_job", "daala_b200_dering_params", "daala_b200_keyframe_lists",
             "daala_b200_kf_config", "daala_b200_kf_totals", "daala_b200_kf_io", "daala_b200_kf_buffers"]
    src = tmp_path / "sizes.c"
    src.write_text('#include <stdio.h>\n#include "daala_b200.h"\nint main(void) {\n'
                   + "".join('  printf("%%zu\\n", sizeof(%s));\n' % n for n in names) + "  return 0;\n}\n")
    exe = tmp_path / "sizes"
    inc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include")
    subprocess.run(["gcc", "-std=c99", "-I", inc, str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    want = [ctypes.sizeof(_native.Plane), ctypes.sizeof(_native.Frame), pvq.BLOCK_DTYPE.itemsize,
            ctypes.sizeof(pvq.PvqParams), mc.MC_BLOCK_DTYPE.itemsize, mc.MATCH_JOB_DTYPE.itemsize,
            ctypes.sizeof(DeringParams), ctypes.sizeof(pvq._KeyframeLists), ctypes.sizeof(engine.Config),
            ctypes.sizeof(engine.Totals), ctypes.sizeof(engine.IO), ctypes.sizeof(engine.Buffers)]
    assert got == want, list(zip(names, got, want))


WORKER = r'''
import os, sys
sys.path.insert(0, %r)
import numpy as np, torch, torch.distributed as dist
from daala_b200.frame import Geometry
from daala_b200.sharding import BorderExchange, plane_rows
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo", rank=rank, world_size=world)
geom = Geometry(256, 320)            # 4 x 5 superblocks
F = 2
g = torch.Generator().manual_seed(7)
full = [torch.randint(-5000, 5000, (F,) + geom.plane_shape(p), generator=g, dtype=torch.int32) for p in range(3)]
mine = [torch.zeros_like(t) for t in full]
r0, n = geom.shard_rows(rank, world)
for p in range(3):
    a, b = plane_rows(geom, p, r0, n)
    mine[p][:, a:b] = full[p][:, a:b]      # what this rank computed
ex = BorderExchange(geom, mine, rank, world)
ex()
for p in range(3):
    a, b = plane_rows(geom, p, r0, n, halo=2)
    assert torch.equal(mine[p][:, a:b], full[p][:, a:b]), (rank, p)
    # nothing else was touched
    rest = mine[p].clone(); rest[:, a:b] = 0
    assert int(rest.abs().sum()) == 0
dist.barrier()
dist.destroy_process_group()
print("rank %%d ok" %% rank)
'''


def test_border_exchange_two_ranks_gloo(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(WORKER % ROOT)
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT="29577", WORLD_SIZE="2")
    procs = [subprocess.Popen([sys.executable, str(script)], env=dict(env, RANK=str(r)), stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT, text=True) for r in range(2)]
    outs = [p.communicate(timeout=240)[0] for p in procs]
    for r, (p, o) in enumerate(zip(procs, outs)):
        assert p.returncode == 0, o
        assert "rank %d ok" % r in o


def test_dropin_link_test_binary_resolves_filter_and_dct_symbols_from_the_library():
    """oracle/_ref/daala_dropin_test = the reference encoder's objects minus filter.o / dct.o, shim/cudastate.o and
    libdaala_b200.so: every filter / DCT symbol of the reference must be UNDEFINED in the program (so the
    dynamic linker takes it from the library) and the vtable initialisers must come from the shim."""
    exe = os.path.join(ROOT, "oracle", "_ref", "daala_dropin_test")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/daala_dropin_test not built (needs the reference sources)")
    syms = subprocess.run(["nm", exe], capture_output=True, text=True, check=True).stdout.splitlines()
    kind = {ln.split()[-1]: ln.split()[-2] for ln in syms if len(ln.split()) >= 2}
    for name in ("od_apply_prefilter_frame_sbs", "od_apply_postfilter_frame_sbs", "od_prefilter_split",
                 "od_postfilter_split", "od_haar", "od_haar_inv", "OD_FDCT_2D_C", "OD_IDCT_2D_C", "OD_FDCT_2D_CUDA",
                 "od_mc_predict1fmv8_cuda", "od_mc_compute_sad8_8x8_cuda"):
        assert kind.get(name) in ("U", "B", "D", "R") and kind.get(name) != "T", (name, kind.get(name))
    for name in ("od_state_opt_vtbl_init_cuda", "od_enc_opt_vtbl_init_cuda", "od_state_opt_vtbl_init_x86",
                 "od_enc_opt_vtbl_init_x86", "daala_encode_create", "od_pvq_encode"):
        assert kind.get(name) == "T", (name, kind.get(name))
    assert "od_bin_fdct8" not in kind or kind["od_bin_fdct8"] == "U"


def test_no_gpu_means_a_loud_failure_not_a_cpu_fallback():
    """Without a CUDA device the product path refuses to run: the engine's constructor raises, a drop-in symbol
    (void signature, nothing to return an error through) terminates the process with a message.  Only meaningful
    where there is no GPU (the build container); skipped on a GPU box."""
    import subprocess
    import sys
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from daala_b200 import engine
    from daala_b200.frame import Geometry
    with pytest.raises(RuntimeError, match="daala_b200_kf_create failed"):
        engine.KeyframeEngine(Geometry(128, 128), nframes=1)
    code = ("import ctypes, numpy as np\n"
            "from daala_b200 import _native\n"
            "L = _native.lib()\n"
            "x = np.zeros(16, np.int32); y = np.zeros(16, np.int32)\n"
            "L.od_bin_fdct4x4.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]\n"
            "L.od_bin_fdct4x4(y.ctypes.data, 4, x.ctypes.data, 4)\n"
            "print('computed without a GPU')\n")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120,
                       cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert r.returncode != 0 and "computed without a GPU" not in r.stdout
    assert "no CPU fallback exists" in r.stderr
