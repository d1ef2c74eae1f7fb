"""TEST INFRASTRUCTURE — ctypes binding of the C Jubjub oracle (jubjub_oracle.c on oracle/field_tmpl.inc).

The shared object is compiled on first use into the system temporary directory, under a name derived from the sources'
hash, so neither the tests nor tools/verify_tx_bench.py write into the repository tree."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_SRC = os.path.join(_HERE, "jubjub_oracle.c")
_INC = os.path.join(_ROOT, "oracle")
_lib = None


def build() -> str:
    h = hashlib.sha256()
    for p in (_SRC, os.path.join(_INC, "field_tmpl.inc")):
        h.update(open(p, "rb").read())
    so = os.path.join(tempfile.gettempdir(), "zkb200_jjoracle_%s_%d.so" % (h.hexdigest()[:16], os.getuid()))
    if not os.path.exists(so):
        tmp = so + ".%d.tmp" % os.getpid()
        subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-shared", "-std=gnu99", "-Wall",
                               "-Wno-unused-function", "-I", _INC, "-o", tmp, _SRC])
        os.replace(tmp, so)
    return so


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.jjo_threads.restype = C.c_int
        _lib.jjo_sqrt.restype = C.c_int
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def into_xy(encodings: bytes):
    """(xy uint64 (n, 2, 4) canonical, status uint8 (n,)) — the layout of zero_chain_b200.groth16.jubjub_into_xy."""
    n = len(encodings) // 32
    assert len(encodings) == 32 * n
    xy = np.zeros((max(n, 1), 2, 4), np.uint64)
    st = np.zeros(max(n, 1), np.uint8)
    if n:
        enc = np.frombuffer(encodings, np.uint8)
        lib().jjo_into_xy(_p(enc), C.c_size_t(n), _p(xy), _p(st))
    return xy[:n], st[:n]


def sqrt(a: int):
    """A square root of a (< r) or None."""
    out = np.zeros(4, np.uint64)
    inp = np.array([(a >> (64 * i)) & (2 ** 64 - 1) for i in range(4)], np.uint64)
    r = lib().jjo_sqrt(_p(inp), _p(out))
    return None if r else sum(int(v) << (64 * i) for i, v in enumerate(out))


def threads() -> int:
    return int(lib().jjo_threads())
