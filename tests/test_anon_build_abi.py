"""CPU check that zk_anonymous_fields_batch and its _device form (tx_build.cu) are declared in include/zkb200.h, exported
by the built library and bound by the ctypes layer, with n_keys and n as size_t in their places."""
import os
import re
import subprocess

from zero_chain_b200 import _lib

NAMES = ["zk_anonymous_fields_batch", "zk_anonymous_fields_batch_device"]


def test_anonymous_fields_symbols_are_declared_exported_and_bound():
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "zkb200.h")).read()
    out = subprocess.check_output(["nm", "-D", "--defined-only", _lib.SO_PATH]).decode()
    exported = set(re.findall(r" T (zk_[a-z0-9_]+)", out))
    L = _lib.lib()
    for name in NAMES:
        assert re.search(r"\b%s\s*\(" % name, hdr), name
        assert name in exported, name
        assert name in _lib.SIGNATURES and getattr(L, name).restype is _lib.i32
        # ctx, the key table (n_keys, keys), n, seven row inputs, four outputs
        args = _lib.SIGNATURES[name][1]
        assert len(args) == 15
        assert args[1] is _lib.sz and args[3] is _lib.sz
        assert [a for i, a in enumerate(args) if i not in (1, 3)] == [_lib.vp] * 13


def test_null_and_size_arguments_are_refused_without_a_device():
    """the argument checks run before any device is touched"""
    L = _lib.lib()
    assert L.zk_anonymous_fields_batch(None, 0, None, 0, *([None] * 11)) == -2
    assert L.zk_anonymous_fields_batch_device(None, 0, None, 0, *([None] * 11)) == -2
