"""CPU check of the compiled key-derivation kernels (hd_keys.cu): each thread carries its hash state, scalars and points in
registers and reads the window table and the parents' Niels points from global memory, so no kernel's SASS may touch
local memory (no LDL / STL) or have a stack frame."""
import re
import subprocess

import pytest

KERNELS = ["k_hd_master", "k_hd_named", "k_hd_xsk_parents", "k_hd_xsk_rows", "k_hd_xpgk_parents", "k_hd_xpgk_rows"]


@pytest.fixture(scope="module")
def names():
    from zero_chain_b200 import _lib
    return subprocess.check_output("cuobjdump -sass %s | grep 'Function :'" % _lib.SO_PATH, shell=True).decode()


@pytest.mark.parametrize("kernel", KERNELS)
def test_hd_kernel_has_no_local_memory(kernel, names):
    from zero_chain_b200 import _lib
    fn = [l.split(":")[1].strip() for l in names.splitlines() if re.search(r"\b_Z\d+%s" % kernel, l)]
    assert len(fn) == 1, names
    sass = subprocess.check_output(["cuobjdump", "-sass", "-fun", fn[0], _lib.SO_PATH], stderr=subprocess.STDOUT).decode()
    body = [l for l in sass.splitlines() if re.search(r"/\*[0-9a-f]{4,}\*/", l)]
    assert len(body) > (10 if kernel == "k_hd_named" else 500)
    assert not [l for l in body if "LDL" in l or "STL" in l]
    res = subprocess.check_output(["cuobjdump", "-res-usage", _lib.SO_PATH], stderr=subprocess.STDOUT).decode()
    m = re.search(r"Function %s:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)" % re.escape(fn[0]), res)
    assert m, res
    assert int(m.group(2)) == 0 and int(m.group(3)) == 0
