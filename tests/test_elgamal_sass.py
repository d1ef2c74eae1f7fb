"""CPU check of the compiled ElGamal kernels: the per-ciphertext kernel carries its points and the double-and-add chain in
registers, and the table build and the index go through global memory only, so none of the three may touch local memory
(no LDL / STL) or have a stack frame."""
import re
import subprocess

import pytest


@pytest.mark.parametrize("kernel, min_lines", [("k_elgamal_decrypt", 1000), ("k_elgamal_table", 300), ("k_elgamal_index", 10)])
def test_elgamal_kernels_have_no_local_memory(kernel, min_lines):
    from zero_chain_b200 import _lib
    names = subprocess.check_output("cuobjdump -sass %s | grep 'Function :'" % _lib.SO_PATH, shell=True).decode()
    fn = [l.split(":")[1].strip() for l in names.splitlines() if kernel in l]
    assert len(fn) == 1, names
    sass = subprocess.check_output(["cuobjdump", "-sass", "-fun", fn[0], _lib.SO_PATH], stderr=subprocess.STDOUT).decode()
    body = [l for l in sass.splitlines() if re.search(r"/\*[0-9a-f]{4,}\*/", l)]
    assert len(body) > min_lines                                   # the kernel itself, not an empty stub
    assert not [l for l in body if "LDL" in l or "STL" in l]
    res = subprocess.check_output(["cuobjdump", "-res-usage", _lib.SO_PATH], stderr=subprocess.STDOUT).decode()
    m = re.search(r"Function %s:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)" % re.escape(fn[0]), res)
    assert m, res
    assert int(m.group(2)) == 0 and int(m.group(3)) == 0
