"""CPU check of the compiled issue passes of zk_anonymous_calls_block: every new kernel of anon_balances.cu keeps its
state in registers (no LDL / STL, no stack frame)."""
import re
import subprocess

import pytest

KERNELS = [("k_an_call_touch", 20), ("k_an_call_tx", 50), ("k_an_issue_account", 300), ("k_an_issue_read", 30), ("k_an_issued", 20),
           ("k_an_issue_finish_acct", 50)]


@pytest.mark.parametrize("kernel, min_lines", KERNELS)
def test_issue_kernels_have_no_local_memory(kernel, min_lines):
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
