"""TEST INFRASTRUCTURE — ctypes binding of the C oracle of both anonymous-balances calls (anon_issue_oracle.c, which
includes anon_balances_oracle.c and through it the confidential-transfer, ElGamal, RedJubjub and point-decoding oracles).

The shared object is compiled on first use into the system temporary directory, under a name derived from the sources'
hash, so neither the tests nor tools/anon_balances_bench.py write into the repository tree."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from .anon_coracle import _arr, _p

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_SRC = os.path.join(_HERE, "anon_issue_oracle.c")
_INC = os.path.join(_ROOT, "oracle")
_lib = None


def build() -> str:
    h = hashlib.sha256()
    for p in (_SRC, os.path.join(_HERE, "anon_balances_oracle.c"), os.path.join(_HERE, "balances_oracle.c"),
              os.path.join(_HERE, "elgamal_oracle.c"), os.path.join(_HERE, "redjubjub_oracle.c"), os.path.join(_HERE, "jubjub_oracle.c"),
              os.path.join(_INC, "field_tmpl.inc")):
        h.update(open(p, "rb").read())
    so = os.path.join(tempfile.gettempdir(), "zkb200_anonissue_%s_%d.so" % (h.hexdigest()[:16], os.getuid()))
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
        _lib.aio_block.restype = C.c_longlong
    return _lib


def block(keys: bytes, balances: bytes, pendings: bytes, flags: bytes, kind: bytes, members, tx_points: bytes, tx_extra: bytes,
          g_epoch: bytes, applied: bytes, issued_in: bytes | None = None):
    """zk_anonymous_calls_block by the sequential loop.  Returns (bad, outputs): bad is the failing account or None;
    outputs = (enc_balances, verify_points, issued, status, new_balances, new_pendings, new_flags) as bytes; issued starts
    as issued_in (zero bytes)."""
    n_acct = len(flags)
    mem = np.ascontiguousarray(np.asarray(members, np.int64).reshape(-1).astype(np.uint32))
    n_tx = len(mem) // 12
    assert len(kind) == n_tx
    nb, npd, nf = _arr(balances), _arr(pendings), _arr(flags)
    seen = np.zeros(max(n_acct, 1), np.uint8)
    eb = np.zeros(max(768 * n_tx, 1), np.uint8)
    vp = np.zeros(max(1664 * n_tx, 1), np.uint8)
    iss = _arr(issued_in if issued_in is not None else bytes(64 * n_tx)) if n_tx else np.zeros(1, np.uint8)
    st = np.zeros(max(n_tx, 1), np.uint8)
    bad = lib().aio_block(C.c_size_t(n_acct), _p(_arr(keys)), _p(nb), _p(npd), _p(nf), _p(seen), C.c_size_t(n_tx), _p(_arr(kind)),
                          _p(mem if n_tx else np.zeros(1, np.uint32)), _p(_arr(tx_points)), _p(_arr(tx_extra)), _p(_arr(g_epoch)),
                          _p(_arr(applied)), _p(eb), _p(vp), _p(iss), _p(st))
    out = (eb[:768 * n_tx].tobytes(), vp[:1664 * n_tx].tobytes(), iss[:64 * n_tx].tobytes(), st[:n_tx].tobytes(),
           nb[:64 * n_acct].tobytes(), npd[:64 * n_acct].tobytes(), nf[:n_acct].tobytes())
    return (None if bad < 0 else int(bad)), out
