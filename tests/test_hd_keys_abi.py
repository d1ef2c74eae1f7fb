"""CPU check that the key-derivation calls (hd_keys.cu) are declared in include/zkb200.h, exported by the built library and
bound by the ctypes layer with size_t in their size places, and that their argument checks — NULL pointers, sizes, and the
host form's SpendingKey::read of every named parent — run before any device is touched.  The calls refused here return
before they read the context, so a zeroed stand-in serves for one."""
import os
import re
import subprocess

import numpy as np

from tests.jubjub_oracle import hd_keys as hd
from tests.jubjub_oracle import redjubjub as rj
from zero_chain_b200 import _lib

CALLS = {"zk_xsk_master_batch": 8, "zk_xsk_derive_batch": 11, "zk_xpgk_derive_batch": 10}


def test_symbols_are_declared_exported_and_bound():
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "zkb200.h")).read()
    out = subprocess.check_output(["nm", "-D", "--defined-only", _lib.SO_PATH]).decode()
    exported = set(re.findall(r" T (zk_[a-z0-9_]+)", out))
    L = _lib.lib()
    for base, nargs in CALLS.items():
        for name in (base, base + "_device"):
            assert re.search(r"\b%s\s*\(" % name, hdr), name
            assert name in exported, name
            assert name in _lib.SIGNATURES and getattr(L, name).restype is _lib.i32
            args = _lib.SIGNATURES[name][1]
            assert len(args) == nargs
            sizes = (1,) if base == "zk_xsk_master_batch" else (1, 3)
            assert all(args[i] is _lib.sz for i in sizes)
            assert [a for i, a in enumerate(args) if i not in sizes] == [_lib.vp] * (nargs - len(sizes))


def test_null_size_and_parent_refusals_without_a_device():
    L = _lib.lib()
    ctx = np.zeros(4096, np.uint8).ctypes.data       # never read: every call below is refused first
    p = np.zeros(4096, np.uint8).ctypes.data
    for name in ("zk_xsk_master_batch", "zk_xsk_master_batch_device"):
        assert getattr(L, name)(None, 0, *([None] * 6)) == -2                       # no context
        assert getattr(L, name)(ctx, 1, p, p, None, p, p, p) == -2                  # xsks NULL
        assert getattr(L, name)(ctx, 0, *([None] * 6)) == 0                         # an empty call
    assert L.zk_xsk_master_batch(ctx, 2, p, np.array([0, 5, 3], np.uint64).ctypes.data, p, None, None, None) == -2   # offsets decrease
    for name, nout in (("zk_xsk_derive_batch", 5), ("zk_xpgk_derive_batch", 4)):
        for f in (getattr(L, name), getattr(L, name + "_device")):
            assert f(None, 0, None, 0, *([None] * (nout + 2))) == -2
            assert f(ctx, 1, None, 1, *([p] * (nout + 2))) == -2                    # parents NULL with n_parents > 0
            assert f(ctx, 1, p, 1, p, None, *([p] * nout)) == -2                   # child_idx NULL
            assert f(ctx, 1, p, 1, p, p, None, *([p] * (nout - 1))) == -2          # the first output NULL
            assert f(ctx, 1, p, 1, p, p, *([p] * (nout - 1)), None) == -2          # status NULL
            assert f(ctx, 1, p, (1 << 26) + 1, *([p] * (nout + 2))) == -2          # too many rows
            assert f(ctx, (1 << 24) + 1, p, 1, *([p] * (nout + 2))) == -2          # too many parents
            assert f(ctx, 0, None, 0, *([None] * (nout + 2))) == 0
    # the host form reads every named parent's sk first, and names the lowest that is >= r_J
    parents = hd.random_xsk_parents(5, seed=1)
    parents[4] = parents[4][:41] + rj.scalar_bytes(rj.R_J)
    parents[2] = parents[2][:41] + b"\xff" * 32
    pb = np.frombuffer(b"".join(parents), np.uint8)
    pidx = np.array([0, 4, 2, 9], np.uint32)
    assert L.zk_xsk_derive_batch(ctx, 5, pb.ctypes.data, 4, pidx.ctypes.data, p, p, None, None, None, p) == -8
    assert "parents[2]" in L.zk_last_error().decode()


def test_python_layer_refuses_indices_outside_u32():
    """the C calls take raw u32 indices; the wrappers refuse a value they would otherwise wrap (-1 would become the
    hardened index 2^32 - 1) before any call is made, so a stand-in context serves"""
    import types

    import pytest

    from zero_chain_b200 import groth16 as zk
    ctx = types.SimpleNamespace(_h=None)
    parents = hd.random_xsk_parents(2, seed=2)
    for pidx, cidx, what in (([0], [-1], r"child_idx\[0\] = -1"), ([0, 1], [3, 1 << 32], r"child_idx\[1\]"),
                             ([-1], [0], r"parent_idx\[0\]"), ([1 << 40], [0], r"parent_idx\[0\]"), ([0, 1], [0], "child_idx: 1 values")):
        with pytest.raises(ValueError, match=what):
            zk.xsk_derive(ctx, parents, pidx, cidx)
        with pytest.raises(ValueError, match=what):
            zk.xpgk_derive(ctx, [hd.xpgk_from_xsk(p) for p in parents], pidx, cidx)
