"""CPU check that zk_import_anonymous_block and its _device form (import.cu) are declared in include/zkb200.h, exported by
the built library and bound by the ctypes layer."""
import os
import re
import subprocess

from zero_chain_b200 import _lib

NAMES = ["zk_import_anonymous_block", "zk_import_anonymous_block_device"]


def test_anonymous_import_symbols_are_declared_exported_and_bound():
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "zkb200.h")).read()
    out = subprocess.check_output(["nm", "-D", "--defined-only", _lib.SO_PATH]).decode()
    exported = set(re.findall(r" T (zk_[a-z0-9_]+)", out))
    L = _lib.lib()
    for name in NAMES:
        assert re.search(r"\b%s\s*\(" % name, hdr), name
        assert name in exported, name
        assert name in _lib.SIGNATURES and getattr(L, name).restype is _lib.i32
        # ctx, both keys, the account table (n_accounts and four arrays), n_tx, eight transaction arrays, seven outputs
        assert len(_lib.SIGNATURES[name][1]) == 23
        assert _lib.SIGNATURES[name][1][3] is _lib.sz and _lib.SIGNATURES[name][1][8] is _lib.sz
