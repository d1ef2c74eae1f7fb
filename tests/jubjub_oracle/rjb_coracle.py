"""TEST INFRASTRUCTURE — ctypes binding of the C batch-verification oracle (rj_batch_oracle.c, which includes
redjubjub_oracle.c and through it jubjub_oracle.c on oracle/field_tmpl.inc).

The shared object is compiled on first use into the system temporary directory, under a name derived from the sources'
hash, so neither the tests nor tools/redjubjub_batch_bench.py write into the repository tree."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from .rj_coracle import _buf, _msgs, _p

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_SRC = os.path.join(_HERE, "rj_batch_oracle.c")
_INC = os.path.join(_ROOT, "oracle")
_lib = None


def build() -> str:
    h = hashlib.sha256()
    for p in (_SRC, os.path.join(_HERE, "redjubjub_oracle.c"), os.path.join(_HERE, "jubjub_oracle.c"),
              os.path.join(_INC, "field_tmpl.inc")):
        h.update(open(p, "rb").read())
    so = os.path.join(tempfile.gettempdir(), "zkb200_rjboracle_%s_%d.so" % (h.hexdigest()[:16], os.getuid()))
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
    return _lib


def redjubjub_batch_verify(vks: bytes, sigs: bytes, msgs, zs: bytes):
    """redjubjub::batch_verify with the randomizers zs (n * 32 bytes, canonical): (verdict, first_bad), first_bad None
    unless the verdict is a rejected entry's code (2 / 3 / 4).  The entries are split over the OpenMP threads."""
    n = len(msgs)
    assert len(vks) == 32 * n and len(sigs) == 64 * n and len(zs) == 32 * n
    verdict = np.zeros(1, np.uint8)
    first = np.zeros(1, np.uint64)
    mb, off = _msgs(msgs)
    lib().rjo_batch_verify(C.c_size_t(n), _p(_buf(vks)), _p(_buf(sigs)), _p(mb), _p(off), _p(_buf(zs)), _p(verdict), _p(first))
    v = int(verdict[0])
    return v, (int(first[0]) if v > 1 else None)
