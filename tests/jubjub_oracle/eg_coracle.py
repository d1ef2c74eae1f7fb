"""TEST INFRASTRUCTURE — ctypes binding of the C ElGamal oracle (elgamal_oracle.c, which includes redjubjub_oracle.c and
through it jubjub_oracle.c on oracle/field_tmpl.inc).

The shared object is compiled on first use into the system temporary directory, under a name derived from the sources'
hash, so neither the tests nor tools/elgamal_bench.py write into the repository tree."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_SRC = os.path.join(_HERE, "elgamal_oracle.c")
_INC = os.path.join(_ROOT, "oracle")
_lib = None


def build() -> str:
    h = hashlib.sha256()
    for p in (_SRC, os.path.join(_HERE, "redjubjub_oracle.c"), os.path.join(_HERE, "jubjub_oracle.c"), os.path.join(_INC, "field_tmpl.inc")):
        h.update(open(p, "rb").read())
    so = os.path.join(tempfile.gettempdir(), "zkb200_egoracle_%s_%d.so" % (h.hexdigest()[:16], os.getuid()))
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
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _buf(b: bytes):
    return np.frombuffer(b, np.uint8) if b else np.zeros(1, np.uint8)


def decrypt(dks: bytes, cts: bytes, pending: bytes | None = None):
    """(status uint8, values uint32) of zk_elgamal_decrypt_batch for concatenated 32-byte keys and 64-byte ciphertexts, by
    the reference's loop; the ciphertexts are split over the OpenMP threads."""
    n = len(dks) // 32
    assert len(dks) == 32 * n and len(cts) == 64 * n and (pending is None or len(pending) == 64 * n)
    st = np.zeros(max(n, 1), np.uint8)
    val = np.zeros(max(n, 1), np.uint32)
    lib().ego_decrypt(C.c_size_t(n), _p(_buf(dks)), _p(_buf(cts)), None if pending is None else _p(_buf(pending)), _p(val), _p(st))
    return st[:n], val[:n]


def encrypt(amounts, rs, eks: bytes, neg: bool = False) -> bytes:
    """Ciphertext::encrypt (or neg_encrypt) of each amount (< 2^32) with randomness rs[i] (< r_J) to the 32-byte encryption
    key eks[32 i ..]: concatenated 64-byte ciphertexts."""
    n = len(amounts)
    assert len(rs) == n and len(eks) == 32 * n
    a = np.ascontiguousarray(amounts, np.uint32) if n else np.zeros(1, np.uint32)
    r = _buf(b"".join(int(x).to_bytes(32, "little") for x in rs))
    out = np.zeros(max(64 * n, 1), np.uint8)
    lib().ego_encrypt(C.c_size_t(n), _p(a), _p(r), _p(_buf(eks)), C.c_int(int(neg)), _p(out))
    return out[:64 * n].tobytes()


def multiples(n: int) -> np.ndarray:
    """(n, 32) uint8: the encoding of i P_G in row i, by successive addition."""
    out = np.zeros((max(n, 1), 32), np.uint8)
    lib().ego_multiples(C.c_size_t(n), _p(out))
    return out[:n]


def threads() -> int:
    return int(lib().jjo_threads())
