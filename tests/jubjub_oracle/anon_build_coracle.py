"""TEST INFRASTRUCTURE — ctypes binding of the C anonymous-transfer oracle (anon_build_oracle.c, which includes
tx_build_oracle.c, elgamal_oracle.c, redjubjub_oracle.c and jubjub_oracle.c on oracle/field_tmpl.inc), in the byte layout
of tests/jubjub_oracle/anon_build.py.

The shared object is compiled on first use into the system temporary directory, under a name derived from the sources'
hash, so neither the tests nor tools/anon_build_bench.py write into the repository tree."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_SRC = os.path.join(_HERE, "anon_build_oracle.c")
_INC = os.path.join(_ROOT, "oracle")
_lib = None


def build() -> str:
    h = hashlib.sha256()
    for p in (_SRC, os.path.join(_HERE, "tx_build_oracle.c"), os.path.join(_HERE, "elgamal_oracle.c"), os.path.join(_HERE, "redjubjub_oracle.c"),
              os.path.join(_HERE, "jubjub_oracle.c"), os.path.join(_INC, "field_tmpl.inc")):
        h.update(open(p, "rb").read())
    so = os.path.join(tempfile.gettempdir(), "zkb200_aboracle_%s_%d.so" % (h.hexdigest()[:16], os.getuid()))
    if not os.path.exists(so):
        tmp = so + ".%d.tmp" % os.getpid()
        subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-shared", "-std=gnu99", "-Wall",
                               "-Wno-unused-function", "-I", _INC, "-I", _HERE, "-o", tmp, _SRC])
        os.replace(tmp, so)
    return so


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.jjo_threads.restype = C.c_int
        _lib.abo_fields.restype = C.c_int
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _buf(b: bytes):
    return np.frombuffer(b, np.uint8) if b else np.zeros(1, np.uint8)


def _rows(out: np.ndarray, size: int, n: int) -> list:
    b = out.tobytes()
    return [b[size * i:size * (i + 1)] for i in range(n)]


def anonymous_fields(keys: bytes, sks: bytes, rings, positions, amounts, rs: bytes, alphas: bytes, g_epoch_enc: bytes):
    """[(fields, rsk, dk, status)] per row, as anon_build.anonymous_fields returns them; keys is the concatenated key
    table, sks / rs / alphas concatenations of 32-byte values, rings n rows of 11 indices, positions n pairs (s, t).
    Raises ValueError for a g_epoch that fails Point::read + as_prime_order."""
    n = len(amounts)
    rg = np.ascontiguousarray(np.asarray(rings, np.int64).reshape(-1).astype(np.uint32)) if n else np.zeros(1, np.uint32)
    pos = np.ascontiguousarray(np.asarray(positions, np.int64).reshape(-1).astype(np.uint8)) if n else np.zeros(1, np.uint8)
    f = np.zeros(max(864 * n, 1), np.uint8)
    rsk, dk, st = np.zeros(max(32 * n, 1), np.uint8), np.zeros(max(32 * n, 1), np.uint8), np.zeros(max(n, 1), np.uint8)
    if lib().abo_fields(C.c_size_t(len(keys) // 32), _p(_buf(keys)), C.c_size_t(n), _p(_buf(sks)), _p(rg), _p(pos),
                        _p(np.ascontiguousarray(amounts, np.uint32) if n else np.zeros(1, np.uint32)), _p(_buf(rs)), _p(_buf(alphas)),
                        _p(_buf(g_epoch_enc)), _p(f), _p(rsk), _p(dk), _p(st)):
        raise ValueError("g_epoch fails Point::read or is not of prime order")
    return list(zip(_rows(f, 864, n), _rows(rsk, 32, n), _rows(dk, 32, n), [int(s) for s in st[:n]]))


def threads() -> int:
    return int(lib().jjo_threads())
