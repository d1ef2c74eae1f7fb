"""TEST INFRASTRUCTURE — ctypes binding of the C encrypted-asset oracle (assets_oracle.c, which includes balances_oracle.c
and through it the ElGamal, RedJubjub and point-decoding oracles on oracle/field_tmpl.inc).

The shared object is compiled on first use into the system temporary directory, under a name derived from the sources'
hash, so neither the tests nor tools/assets_bench.py write into the repository tree."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_SRC = os.path.join(_HERE, "assets_oracle.c")
_INC = os.path.join(_ROOT, "oracle")
_lib = None


def build() -> str:
    h = hashlib.sha256()
    for p in (_SRC, os.path.join(_HERE, "balances_oracle.c"), os.path.join(_HERE, "elgamal_oracle.c"),
              os.path.join(_HERE, "redjubjub_oracle.c"), os.path.join(_HERE, "jubjub_oracle.c"), os.path.join(_INC, "field_tmpl.inc")):
        h.update(open(p, "rb").read())
    so = os.path.join(tempfile.gettempdir(), "zkb200_assetoracle_%s_%d.so" % (h.hexdigest()[:16], os.getuid()))
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
        _lib.ao_block.restype = C.c_longlong
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _arr(b, dtype=np.uint8):
    return np.array(np.frombuffer(bytes(b), dtype) if len(b) else np.zeros(1, dtype), dtype)   # a writable copy


def _idx(v, n):
    return np.ascontiguousarray(np.asarray(v, np.int64).astype(np.uint32)) if n else np.zeros(1, np.uint32)


def block(balances: bytes, pendings: bytes, flags: bytes, kind, slot_a, slot_b, tx_points: bytes, applied: bytes):
    """zk_assets_block by the sequential loop.  Returns (bad, outputs): bad is the failing slot or None; outputs =
    (balance_sender, balance_after, event_ct, event_flags, status, new_balances, new_pendings, new_flags) as bytes, with
    zero bytes where the call writes nothing."""
    n_slots, n_tx = len(flags), len(kind)
    nb, npd, nf = _arr(balances), _arr(pendings), _arr(flags)
    seen = np.zeros(max(n_slots, 1), np.uint8)
    bs, ba = np.zeros(max(64 * n_tx, 1), np.uint8), np.zeros(max(64 * n_tx, 1), np.uint8)
    ev, ef, st = np.zeros(max(128 * n_tx, 1), np.uint8), np.zeros(max(n_tx, 1), np.uint8), np.zeros(max(n_tx, 1), np.uint8)
    bad = lib().ao_block(C.c_size_t(n_slots), _p(nb), _p(npd), _p(nf), _p(seen), C.c_size_t(n_tx), _p(_arr(bytes(kind))),
                         _p(_idx(slot_a, n_tx)), _p(_idx(slot_b, n_tx)), _p(_arr(tx_points)), _p(_arr(applied)), _p(bs), _p(ba), _p(ev),
                         _p(ef), _p(st))
    out = (bs[:64 * n_tx].tobytes(), ba[:64 * n_tx].tobytes(), ev[:128 * n_tx].tobytes(), ef[:n_tx].tobytes(), st[:n_tx].tobytes(),
           nb[:64 * n_slots].tobytes(), npd[:64 * n_slots].tobytes(), nf[:n_slots].tobytes())
    return (None if bad < 0 else int(bad)), out
