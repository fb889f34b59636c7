"""GPU parity of the distortion kernel (csrc/dist_kernels.cu) against the pinned CPU oracle
(oracle/port_dist.c, bit-identical to od_compute_dist by tests/test_oracle_dering.py)."""
import ctypes
import os

import numpy as np
import pytest

from tests import oracle_lib
from tests.oracle_lib import addr

pytestmark = [pytest.mark.gpu]


@pytest.mark.parametrize("n", [8, 16, 32, 64])
def test_compute_dist_matches_oracle(n):
    import torch
    from daala_b200 import _native
    L = _native.lib()
    L.daala_b200_compute_dist.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                          ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    port = oracle_lib.load_port()
    port.port_compute_dist.restype = ctypes.c_double
    rng = np.random.default_rng(n)
    count = 23
    x = (rng.integers(-128, 128, size=(count, n, n)) * 16 + rng.integers(-8, 9, size=(count, n, n))).astype(np.int32)
    x[::3] = (x[::3] // 64) * 64
    y = (x + rng.integers(-60, 61, size=x.shape) * rng.integers(1, 5, size=(count, 1, 1))).astype(np.int32)
    y[5] = x[5]                                          # identical pair: distortion exactly 0
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    out = torch.zeros(count, dtype=torch.float64, device="cuda")
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    for flat, masking, cq in ((0, 1, 20), (0, 0, 40), (0, 1, 60), (1, 1, 20)):
        assert L.daala_b200_compute_dist(xd.data_ptr(), yd.data_ptr(), count, n, flat, masking, cq, out.data_ptr(), s) == 0
        got = out.cpu().numpy()
        want = np.array([port.port_compute_dist(addr(x[i]), addr(y[i]), n, flat, masking, cq) for i in range(count)])
        # integer stages are exact; pow() of the CUDA math library may differ from libm in the last ulps
        assert np.allclose(got, want, rtol=1e-12, atol=0), (flat, masking, cq, np.abs(got - want).max())
        assert abs(got[5]) <= 1e-9 and (got[np.arange(count) != 5] > 0).all()
        if flat:
            assert np.array_equal(got, want)
