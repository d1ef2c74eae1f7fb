"""TEST INFRASTRUCTURE — ctypes binding of the C RedJubjub oracle (redjubjub_oracle.c, which includes jubjub_oracle.c on
oracle/field_tmpl.inc).

The shared object is compiled on first use into the system temporary directory, under a name derived from the sources'
hash, so neither the tests nor tools/redjubjub_bench.py write into the repository tree."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_SRC = os.path.join(_HERE, "redjubjub_oracle.c")
_INC = os.path.join(_ROOT, "oracle")
_lib = None


def build() -> str:
    h = hashlib.sha256()
    for p in (_SRC, os.path.join(_HERE, "jubjub_oracle.c"), os.path.join(_INC, "field_tmpl.inc")):
        h.update(open(p, "rb").read())
    so = os.path.join(tempfile.gettempdir(), "zkb200_rjoracle_%s_%d.so" % (h.hexdigest()[:16], os.getuid()))
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


def _msgs(msgs):
    off = np.zeros(len(msgs) + 1, np.uint64)
    np.cumsum([len(m) for m in msgs], out=off[1:])
    return _buf(b"".join(msgs)), off


def _sk_bytes(sks) -> bytes:
    return b"".join(int(k).to_bytes(32, "little") for k in sks)


def redjubjub_verify(vks: bytes, sigs: bytes, msgs) -> np.ndarray:
    """Verdicts (uint8, the codes of zk_redjubjub_verify_batch) for concatenated 32-byte keys, 64-byte signatures and a list
    of messages; the signatures are split over the OpenMP threads."""
    n = len(msgs)
    assert len(vks) == 32 * n and len(sigs) == 64 * n
    out = np.zeros(max(n, 1), np.uint8)
    mb, off = _msgs(msgs)
    lib().rjo_verify(C.c_size_t(n), _p(_buf(vks)), _p(_buf(sigs)), _p(mb), _p(off), _p(out))
    return out[:n]


def redjubjub_sign(sks, ts: bytes, msgs) -> bytes:
    """PrivateKey::sign for each (sk < r_J, 80 bytes of T, msg): concatenated 64-byte signatures."""
    n = len(msgs)
    assert len(sks) == n and len(ts) == 80 * n
    out = np.zeros(max(64 * n, 1), np.uint8)
    mb, off = _msgs(msgs)
    lib().rjo_sign(C.c_size_t(n), _p(_buf(_sk_bytes(sks))), _p(_buf(ts)), _p(mb), _p(off), _p(out))
    return out[:64 * n].tobytes()


def redjubjub_public_key(sks) -> bytes:
    """sk P_G for each key, concatenated 32-byte encodings."""
    n = len(sks)
    out = np.zeros(max(32 * n, 1), np.uint8)
    lib().rjo_public_key(C.c_size_t(n), _p(_buf(_sk_bytes(sks))), _p(out))
    return out[:32 * n].tobytes()


def h_star(a: bytes, b: bytes) -> int:
    out = np.zeros(4, np.uint64)
    lib().rjo_h_star(_p(_buf(a)), C.c_size_t(len(a)), _p(_buf(b)), C.c_size_t(len(b)), _p(out))
    return sum(int(v) << (64 * i) for i, v in enumerate(out))


def blake2b(data: bytes, person: bytes = bytes(16)) -> bytes:
    out = np.zeros(64, np.uint8)
    lib().rjo_blake2b(_p(_buf(person)), _p(_buf(data)), C.c_size_t(len(data)), _p(out))
    return out.tobytes()


def threads() -> int:
    return int(lib().jjo_threads())
