"""Drop-in link test on the GPU (SURVEY.md 8(b), 8(c)(5)): the reference encoder's own objects linked
against libdaala_b200.so instead of its filter.o / dct.o, vtables filled by shim/cudastate.c.  The
program (oracle/dropin_main.c) checks the function tables dcttest-style and encodes frames through
daala_encode_*; packets must be byte-identical to the pure-C reference build's, and the same packets decoded by
the reference DECODER of each build (daala_decode_*: its inverse transforms, postfilters and motion compensation
run on the CUDA back end in the drop-in build) must give identical pictures (SURVEY.md 8(f) rank 4)."""
import os
import subprocess

import pytest

pytestmark = [pytest.mark.gpu]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "oracle", "_ref", "daala_dropin_test")
REF = os.path.join(ROOT, "oracle", "_ref", "libdaala_ref.so")


def _run(w, h, nframes, timeout):
    if not (os.path.exists(EXE) and os.path.exists(REF)):
        pytest.skip("oracle/_ref/daala_dropin_test not built (needs the reference sources)")
    r = subprocess.run([EXE, REF, str(w), str(h), str(nframes)], capture_output=True, text=True, timeout=timeout)
    print(r.stdout)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-2000:])
    assert "drop-in link test ok" in r.stdout and "table checks: ok" in r.stdout
    assert r.stdout.count("decoded picture sum") == nframes and "DIFFERENT" not in r.stdout
    return r.stdout


def test_reference_encoder_on_the_cuda_back_end_emits_identical_keyframe_packet():
    out = _run(128, 128, 1, 600)
    assert "frame 0" in out


def test_reference_encoder_on_the_cuda_back_end_emits_identical_inter_packets():
    """Keyframe + P frame: the MC / SAD vtable slots (od_mc_predict1fmv8_cuda, blends, SADs) carry the
    motion search of the reference's od_mv_est."""
    out = _run(64, 64, 2, 900)
    assert "frame 1" in out
