"""TEST INFRASTRUCTURE — ctypes binding of the C transaction-building oracle (tx_build_oracle.c, which includes
elgamal_oracle.c, redjubjub_oracle.c and jubjub_oracle.c on oracle/field_tmpl.inc), in the byte layouts of
tests/jubjub_oracle/tx_build.py.  Signing is redjubjub_oracle.c's, through rj_coracle.py.

The shared object is compiled on first use into the system temporary directory, under a name derived from the sources'
hash, so neither the tests nor tools/tx_build_bench.py write into the repository tree."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_SRC = os.path.join(_HERE, "tx_build_oracle.c")
_INC = os.path.join(_ROOT, "oracle")
_lib = None


def build() -> str:
    h = hashlib.sha256()
    for p in (_SRC, os.path.join(_HERE, "elgamal_oracle.c"), os.path.join(_HERE, "redjubjub_oracle.c"), os.path.join(_HERE, "jubjub_oracle.c"),
              os.path.join(_INC, "field_tmpl.inc")):
        h.update(open(p, "rb").read())
    so = os.path.join(tempfile.gettempdir(), "zkb200_txoracle_%s_%d.so" % (h.hexdigest()[:16], os.getuid()))
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
        _lib.txo_fields.restype = C.c_int
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _buf(b: bytes):
    return np.frombuffer(b, np.uint8) if b else np.zeros(1, np.uint8)


def _rows(out: np.ndarray, size: int, n: int) -> list:
    b = out.tobytes()
    return [b[size * i:size * (i + 1)] for i in range(n)]


def blake2s(data: bytes, person: bytes) -> bytes:
    out = np.zeros(32, np.uint8)
    lib().txo_blake2s(_p(_buf(person)), _p(_buf(data)), C.c_size_t(len(data)), _p(out))
    return out.tobytes()


def keys(seeds):
    """(sks, dks, eks): lists of 32-byte values, one per seed"""
    n = len(seeds)
    off = np.zeros(n + 1, np.uint64)
    np.cumsum([len(s) for s in seeds], out=off[1:])
    sk, dk, ek = (np.zeros(max(32 * n, 1), np.uint8) for _ in range(3))
    lib().txo_keys(C.c_size_t(n), _p(_buf(b"".join(seeds))), _p(off), _p(sk), _p(dk), _p(ek))
    return _rows(sk, 32, n), _rows(dk, 32, n), _rows(ek, 32, n)


def g_epoch(epochs):
    """[(encoding, tag byte)] per epoch; (None, -1) when no tag below 255 gives a point"""
    n = len(epochs)
    out = np.zeros(max(32 * n, 1), np.uint8)
    tags = np.zeros(max(n, 1), np.int32)
    lib().txo_g_epoch(C.c_size_t(n), _p(np.ascontiguousarray(epochs, np.uint32)), _p(out), _p(tags))
    return [(out[32 * i:32 * i + 32].tobytes() if tags[i] >= 0 else None, int(tags[i])) for i in range(n)]


def confidential_fields(sks: bytes, eks: bytes, amounts, fees, rs: bytes, alphas: bytes, g_epoch_enc: bytes):
    """[(fields, rsk, dk, status)] per row, as tx_build.confidential_fields returns them; sks / eks / rs / alphas are
    concatenations of 32-byte values.  Raises ValueError for a g_epoch that fails Point::read + as_prime_order."""
    n = len(amounts)
    f = np.zeros(max(288 * n, 1), np.uint8)
    rsk, dk, st = np.zeros(max(32 * n, 1), np.uint8), np.zeros(max(32 * n, 1), np.uint8), np.zeros(max(n, 1), np.uint8)
    if lib().txo_fields(C.c_size_t(n), _p(_buf(sks)), _p(_buf(eks)), _p(np.ascontiguousarray(amounts, np.uint32)),
                        _p(np.ascontiguousarray(fees, np.uint32)), _p(_buf(rs)), _p(_buf(alphas)), _p(_buf(g_epoch_enc)), _p(f), _p(rsk),
                        _p(dk), _p(st)):
        raise ValueError("g_epoch fails Point::read or is not of prime order")
    return list(zip(_rows(f, 288, n), _rows(rsk, 32, n), _rows(dk, 32, n), [int(s) for s in st[:n]]))


def threads() -> int:
    return int(lib().jjo_threads())
