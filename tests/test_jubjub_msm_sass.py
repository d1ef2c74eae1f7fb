"""CPU check of the compiled Jubjub MSM and batch-verification kernels: the per-entry stage (BLAKE2b and two Point::reads),
the bucket accumulation and the bucket reduction carry their points in registers, so their SASS must have no local-memory
access (no LDL / STL) and no stack frame."""
import re
import subprocess

import pytest

KERNELS = ["k_rj_batch_prep", "k_jm_read_points", "k_jm_accumulate", "k_jm_combine", "k_jm_combine_warp", "k_jm_slices",
           "k_jm_windows", "k_jm_horner", "k_rj_batch_verdict", "k_jm_encode"]


@pytest.mark.parametrize("kernel", KERNELS)
def test_kernel_has_no_local_memory(kernel):
    from zero_chain_b200 import _lib
    names = subprocess.check_output("cuobjdump -sass %s | grep 'Function :'" % _lib.SO_PATH, shell=True).decode()
    fn = [l.split(":")[1].strip() for l in names.splitlines() if "_Z%d%s" % (len(kernel), kernel) in l]
    assert len(fn) == 1, names
    sass = subprocess.check_output(["cuobjdump", "-sass", "-fun", fn[0], _lib.SO_PATH], stderr=subprocess.STDOUT).decode()
    body = [l for l in sass.splitlines() if re.search(r"/\*[0-9a-f]{4,}\*/", l)]
    assert len(body) > 100
    assert not [l for l in body if "LDL" in l or "STL" in l]
    res = subprocess.check_output(["cuobjdump", "-res-usage", _lib.SO_PATH], stderr=subprocess.STDOUT).decode()
    m = re.search(r"Function %s:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)" % re.escape(fn[0]), res)
    assert m, res
    assert int(m.group(2)) == 0 and int(m.group(3)) == 0
