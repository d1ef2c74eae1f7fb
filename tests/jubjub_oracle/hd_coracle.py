"""TEST INFRASTRUCTURE — ctypes binding of the C key-derivation oracle (hd_keys_oracle.c, which includes tx_build_oracle.c,
elgamal_oracle.c, redjubjub_oracle.c and jubjub_oracle.c on oracle/field_tmpl.inc), in the row layout of
tests/jubjub_oracle/hd_keys.py.

The shared object is compiled on first use into the system temporary directory, under a name derived from the sources'
hash, so neither the tests nor tools/hd_bench.py write into the repository tree."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from .hd_keys import XK, NotInField

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_SRC = os.path.join(_HERE, "hd_keys_oracle.c")
_INC = os.path.join(_ROOT, "oracle")
_lib = None


def build() -> str:
    h = hashlib.sha256()
    for p in (_SRC, os.path.join(_HERE, "tx_build_oracle.c"), os.path.join(_HERE, "elgamal_oracle.c"), os.path.join(_HERE, "redjubjub_oracle.c"),
              os.path.join(_HERE, "jubjub_oracle.c"), os.path.join(_INC, "field_tmpl.inc")):
        h.update(open(p, "rb").read())
    so = os.path.join(tempfile.gettempdir(), "zkb200_hdoracle_%s_%d.so" % (h.hexdigest()[:16], os.getuid()))
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
        _lib.hdo_xsk_derive.restype = C.c_longlong
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _buf(b: bytes):
    return np.frombuffer(b, np.uint8) if b else np.zeros(1, np.uint8)


def _out(size: int, n: int, want: bool = True):
    return np.zeros(max(size * n, 1), np.uint8) if want else None


def _rows(out, size: int, n: int) -> list:
    if out is None:
        return [None] * n
    b = out.tobytes()
    return [b[size * i:size * (i + 1)] for i in range(n)]


def _idx(v, n: int):
    return np.ascontiguousarray(np.asarray(v, np.int64).astype(np.uint32)) if n else np.zeros(1, np.uint32)


def master(seeds, outputs: bool = True) -> list:
    """[(xsk, xpgk, dk, ek)] per seed, as hd_keys.master_row; outputs=False leaves the last three None"""
    n = len(seeds)
    off = np.zeros(n + 1, np.uint64)
    off[1:] = np.cumsum([len(s) for s in seeds]) if n else []
    xsk, xpgk, dk, ek = _out(XK, n), _out(XK, n, outputs), _out(32, n, outputs), _out(32, n, outputs)
    lib().hdo_master(C.c_size_t(n), _p(_buf(b"".join(seeds))), _p(off), _p(xsk), _p(xpgk), _p(dk), _p(ek))
    return list(zip(_rows(xsk, XK, n), _rows(xpgk, XK, n), _rows(dk, 32, n), _rows(ek, 32, n)))


def xsk_derive(parents, parent_idx, child_idx, outputs: bool = True) -> list:
    """[(xsk, xpgk, dk, ek, status)] as hd_keys.xsk_derive_rows; parents a list of 73-byte xsks or their concatenation"""
    pb = parents if isinstance(parents, (bytes, bytearray)) else b"".join(parents)
    n = len(parent_idx)
    xsk, xpgk, dk, ek, st = _out(XK, n), _out(XK, n, outputs), _out(32, n, outputs), _out(32, n, outputs), _out(1, n)
    bad = lib().hdo_xsk_derive(C.c_size_t(len(pb) // XK), _p(_buf(pb)), C.c_size_t(n), _p(_idx(parent_idx, n)), _p(_idx(child_idx, n)),
                               _p(xsk), _p(xpgk), _p(dk), _p(ek), _p(st))
    if bad >= 0:
        raise NotInField("parents[%d]" % bad)
    return list(zip(_rows(xsk, XK, n), _rows(xpgk, XK, n), _rows(dk, 32, n), _rows(ek, 32, n), [int(s) for s in st[:n]]))


def xpgk_derive(parents, parent_idx, child_idx, outputs: bool = True) -> list:
    """[(xpgk, dk, ek, status)] as hd_keys.xpgk_derive_rows"""
    pb = parents if isinstance(parents, (bytes, bytearray)) else b"".join(parents)
    n = len(parent_idx)
    xpgk, dk, ek, st = _out(XK, n), _out(32, n, outputs), _out(32, n, outputs), _out(1, n)
    lib().hdo_xpgk_derive(C.c_size_t(len(pb) // XK), _p(_buf(pb)), C.c_size_t(n), _p(_idx(parent_idx, n)), _p(_idx(child_idx, n)),
                          _p(xpgk), _p(dk), _p(ek), _p(st))
    return list(zip(_rows(xpgk, XK, n), _rows(dk, 32, n), _rows(ek, 32, n), [int(s) for s in st[:n]]))


def tag(pgk: bytes) -> bytes:
    out = np.zeros(4, np.uint8)
    lib().hdo_tag(_p(_buf(pgk)), _p(out))
    return out.tobytes()


def threads() -> int:
    return int(lib().jjo_threads())
