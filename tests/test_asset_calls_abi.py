"""CPU check that zk_import_asset_calls and its _device form (import.cu) are declared in include/zkb200.h, exported by the
built library and bound by the ctypes layer with their argument counts."""
import ctypes as C
import os
import re
import subprocess

from zero_chain_b200 import _lib

NAMES = ["zk_import_asset_calls", "zk_import_asset_calls_device"]


def test_asset_calls_symbols_are_declared_exported_and_bound():
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "zkb200.h")).read()
    out = subprocess.check_output(["nm", "-D", "--defined-only", _lib.SO_PATH]).decode()
    exported = set(re.findall(r" T (zk_[a-z0-9_]+)", out))
    L = _lib.lib()
    for name in NAMES:
        m = re.search(r"\bint %s\s*\(([^;]*)\);" % name, hdr)
        assert m, name
        assert name in exported, name
        assert name in _lib.SIGNATURES and getattr(L, name).restype is _lib.i32
        # ctx, pvk, the slot table (n_slots and five arrays), next_asset_id, new_slot_flags, n_tx, four transaction arrays,
        # eleven outputs, n_slots_out, rounds
        args = _lib.SIGNATURES[name][1]
        assert len(args) == 28 == len(m.group(1).split(","))
        assert args[2] is _lib.sz and args[10] is _lib.sz
        assert args[8] is _lib.u32 and args[9] is C.c_uint8
        assert args[26] == C.POINTER(_lib.sz) and args[27] == C.POINTER(_lib.u32)
