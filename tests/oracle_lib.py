"""ctypes loaders for the CHECKER libraries (test infrastructure only).

  load_port(): oracle/libdaala_port.so  -- our plain-C restatement (always buildable)
  load_ref():  oracle/_ref/libdaala_ref.so -- the unmodified xiph/daala sources
               compiled by oracle/Makefile from REF_SRC (may be absent)
"""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE = os.path.join(ROOT, "oracle")
# a checkout of the xiph/daala sources: the one named by DAALA_REF, else one next to this repository, else the
# read-only system-wide checkout at /root/reference; without any of them the checker libraries under oracle/_ref
# are used as they are (or are absent)
_REF_CANDIDATES = ([os.environ["DAALA_REF"]] if os.environ.get("DAALA_REF") else
                   [os.path.join(os.path.dirname(ROOT), "reference"), "/root/reference"])
REF_SRC = next((p for p in _REF_CANDIDATES if os.path.isdir(os.path.join(p, "src"))), _REF_CANDIDATES[0])

c_int = ctypes.c_int
c_double = ctypes.c_double
i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
i16p = np.ctypeslib.ndpointer(np.int16, flags="C_CONTIGUOUS")
u8p = np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")

_cache = {}


def _make(target):
    subprocess.run(["make", "-C", ORACLE, target, "-j8", "REF=" + os.path.abspath(REF_SRC)], check=True,
                   stdout=subprocess.DEVNULL, stderr=subprocess.PIPE)


def have_ref_sources():
    return os.path.isdir(REF_SRC)


def load_port():
    if "port" not in _cache:
        _make("port")
        _cache["port"] = ctypes.CDLL(os.path.join(ORACLE, "libdaala_port.so"))
    return _cache["port"]


def load_ref(simd=False):
    key = "ref_simd" if simd else "ref"
    if key not in _cache:
        name = "libdaala_ref_simd.so" if simd else "libdaala_ref.so"
        path = os.path.join(ORACLE, "_ref", name)
        if have_ref_sources():
            _make("ref")
        _cache[key] = ctypes.CDLL(path) if os.path.exists(path) else None
    return _cache[key]


def addr(a, off=0):
    """Raw pointer into a numpy array (element offset `off`)."""
    return ctypes.c_void_p(a.ctypes.data + off * a.itemsize)
