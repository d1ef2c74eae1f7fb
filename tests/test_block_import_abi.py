"""CPU check that zk_import_block and its _device form (import.cu) are declared in include/zkb200.h, exported by the built
library and bound by the ctypes layer with their argument counts and the types at the section boundaries."""
import ctypes as C
import os
import re
import subprocess

from zero_chain_b200 import _lib

NAMES = ["zk_import_block", "zk_import_block_device"]
HDR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "zkb200.h")


def test_block_import_symbols_are_declared_exported_and_bound():
    hdr = open(HDR).read()
    out = subprocess.check_output(["nm", "-D", "--defined-only", _lib.SO_PATH]).decode()
    exported = set(re.findall(r" T (zk_[a-z0-9_]+)", out))
    L = _lib.lib()
    for name in NAMES:
        m = re.search(r"\bint %s\s*\(([^;]*)\);" % name, hdr)
        assert m, name
        assert name in exported, name
        assert name in _lib.SIGNATURES and getattr(L, name).restype is _lib.i32
        # ctx and the two keys, six signature arguments, then the confidential (16), asset (26) and anonymous (20)
        # sections, first_bad_sig and launches
        args = _lib.SIGNATURES[name][1]
        assert len(args) == 73 == len(m.group(1).split(","))
        assert args[3] is _lib.sz                                                  # n_sig
        assert args[9] is _lib.sz and args[13] is _lib.sz and args[24] == C.POINTER(_lib.u32)      # confidential
        assert args[25] is _lib.sz and args[31] is _lib.u32 and args[32] is C.c_uint8 and args[33] is _lib.sz
        assert args[49] == C.POINTER(_lib.sz) and args[50] == C.POINTER(_lib.u32)                  # assets
        assert args[51] is _lib.sz and args[56] is _lib.sz                                         # anonymous
        assert args[71] == C.POINTER(_lib.sz) and args[72] == C.POINTER(_lib.u32)


def test_bad_signature_code():
    assert re.search(r"#define ZK_ERR_BAD_SIGNATURE \(-10\)", open(HDR).read())
    assert _lib.ZK_ERR_BAD_SIGNATURE == -10
