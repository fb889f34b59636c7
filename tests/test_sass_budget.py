"""Instruction-footprint budget of the luma chain kernel k_pvq_persist<true> (CPU: nvcc cross-compiles).

The kernel walks the luma intra chains one band per warp and runs a band's setup, search and finish back to
back, so its straight-line code competes for the instruction cache (DESIGN.md 3.3).  This pins what
tools/sass_footprint.py reports for it, so that a change cannot quietly make the code larger again:
SASS bytes, the stack frame, and 64 registers (32 one-warp CTAs per SM).
"""
import importlib.util
import os

import pytest

from daala_b200 import build as _build

HAVE_NVCC = os.path.exists(_build.NVCC)

# Ratchet values, not the design budget: what the kernel compiles to with CUDA 12.9 (97,920 bytes, a 224-byte frame),
# so that it cannot grow back.  The goal the instruction cache asks for is far smaller (DESIGN.md 3.3), and no
# stack frame at all.  Another nvcc may lay the code out differently; lower these when the kernel shrinks.
MAX_SASS_BYTES = 96 * 1024
MAX_STACK_BYTES = 224
REGISTERS = 64


@pytest.mark.skipif(not HAVE_NVCC, reason="nvcc not available")
def test_luma_chain_kernel_within_footprint_budget():
    path = os.path.join(_build.ROOT, "tools", "sass_footprint.py")
    spec = importlib.util.spec_from_file_location("sass_footprint", path)
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    rows, _ = tool.footprint()
    row = next(r for r in rows if r["kernel"] == "k_pvq_persist<true>")
    assert row["sass_bytes"] <= MAX_SASS_BYTES, row
    assert row["stack"] <= MAX_STACK_BYTES, row
    assert row["regs"] == REGISTERS, row
