"""CPU check of the kernels zk_import_block adds or gives a section offset (import.cu, import.cuh sections 2, 4, 5 and
7): no local memory (no LDL / STL, no stack frame)."""
import re
import subprocess

import pytest

KERNELS = [("k_imp_gather", 20), ("k_imp_fail", 10), ("k_imp_decide", 10), ("k_imp_an_issue_row", 20), ("k_imp_an_scatter", 10),
           ("k_imp_as_compact", 20), ("k_imp_sig_first", 5), ("k_imp_sig_code", 3), ("k_imp_sig_z", 10)]


@pytest.mark.parametrize("kernel, min_lines", KERNELS)
def test_block_import_kernels_have_no_local_memory(kernel, min_lines):
    from zero_chain_b200 import _lib
    names = subprocess.check_output("cuobjdump -sass %s | grep 'Function :'" % _lib.SO_PATH, shell=True).decode()
    fn = [l.split(":")[1].strip() for l in names.splitlines() if re.search(r"\d%s[mP]" % kernel, l)]
    assert len(fn) == 1, names
    sass = subprocess.check_output(["cuobjdump", "-sass", "-fun", fn[0], _lib.SO_PATH], stderr=subprocess.STDOUT).decode()
    body = [l for l in sass.splitlines() if re.search(r"/\*[0-9a-f]{4,}\*/", l)]
    assert len(body) > min_lines
    assert not [l for l in body if "LDL" in l or "STL" in l]
    res = subprocess.check_output(["cuobjdump", "-res-usage", _lib.SO_PATH], stderr=subprocess.STDOUT).decode()
    m = re.search(r"Function %s:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)" % re.escape(fn[0]), res)
    assert m, res
    assert int(m.group(2)) == 0 and int(m.group(3)) == 0
