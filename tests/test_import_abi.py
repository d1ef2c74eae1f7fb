"""CPU check that the block-import entry points (zk_import_confidential_block, zk_import_assets_block and their _device
forms, import.cu) are declared in include/zkb200.h, exported by the built library and bound by the ctypes layer."""
import re
import subprocess

from zero_chain_b200 import _lib

NAMES = ["zk_import_confidential_block", "zk_import_confidential_block_device", "zk_import_assets_block", "zk_import_assets_block_device"]


def test_import_symbols_are_declared_exported_and_bound():
    import os
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "zkb200.h")).read()
    out = subprocess.check_output(["nm", "-D", "--defined-only", _lib.SO_PATH]).decode()
    exported = set(re.findall(r" T (zk_[a-z0-9_]+)", out))
    L = _lib.lib()
    for name in NAMES:
        assert re.search(r"\b%s\s*\(" % name, hdr), name
        assert name in exported, name
        assert name in _lib.SIGNATURES and getattr(L, name).restype is _lib.i32
    # ctx, pvk, the table size and its three arrays, n_tx, then the transaction arrays and outputs, then the rounds
    assert [len(_lib.SIGNATURES[n][1]) for n in NAMES] == [18, 18, 23, 23]
