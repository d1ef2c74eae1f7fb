"""CPU check of the compiled passes of zk_import_asset_calls (import.cu, import.cuh section 6): the hash-table probes, key
compares and row copies keep everything in registers (no LDL / STL, no stack frame)."""
import re
import subprocess

import pytest

KERNELS = [("k_imp_as_start", 10), ("k_imp_as_row_insert", 40), ("k_imp_as_row_dup", 40), ("k_imp_as_compact", 20),
           ("k_imp_as_issue_flag", 10), ("k_imp_as_refs", 20), ("k_imp_as_ref_insert", 40), ("k_imp_as_new", 40), ("k_imp_as_slot", 40),
           ("k_imp_as_tx_points", 10)]


@pytest.mark.parametrize("kernel, min_lines", KERNELS)
def test_asset_calls_kernels_have_no_local_memory(kernel, min_lines):
    from zero_chain_b200 import _lib
    names = subprocess.check_output("cuobjdump -sass %s | grep 'Function :'" % _lib.SO_PATH, shell=True).decode()
    fn = [l.split(":")[1].strip() for l in names.splitlines() if re.search(r"\d%s[mP]" % kernel, l)]
    assert len(fn) == 1, names
    sass = subprocess.check_output(["cuobjdump", "-sass", "-fun", fn[0], _lib.SO_PATH], stderr=subprocess.STDOUT).decode()
    body = [l for l in sass.splitlines() if re.search(r"/\*[0-9a-f]{4,}\*/", l)]
    assert len(body) > min_lines                                   # the kernel itself, not an empty stub
    assert not [l for l in body if "LDL" in l or "STL" in l]
    res = subprocess.check_output(["cuobjdump", "-res-usage", _lib.SO_PATH], stderr=subprocess.STDOUT).decode()
    m = re.search(r"Function %s:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)" % re.escape(fn[0]), res)
    assert m, res
    assert int(m.group(2)) == 0 and int(m.group(3)) == 0
