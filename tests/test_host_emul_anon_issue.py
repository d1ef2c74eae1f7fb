"""CPU check of the PRODUCT's issue passes of zk_anonymous_calls_block (zero_chain_b200/csrc/anon_balances.cuh, with the
balances.cuh passes it reuses) compiled with ZK_HOST_EMUL: every pass of run_block with a kind array, run as loops over
its items, against the Python oracle of the module's loop on small mixed blocks and against the C oracle on a block where
one account takes issues among hundreds of rings.  The real PTX path is covered by tests/test_gpu_anon_issue.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.jubjub_oracle import anon_issue as ai
from tests.jubjub_oracle import anon_issue_coracle as aic
from tests.jubjub_oracle import anon_issue_corpus
from tests.jubjub_oracle import bal_corpus
from tests.jubjub_oracle import balances as bal

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_anon_issue") / "libemul_anon_issue.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "zero_chain_b200", "csrc"),
                           "-o", so, os.path.join(HERE, "host_emul", "emul_anon_issue.cpp")])
    lib = C.CDLL(so)
    lib.emu_anon_calls_block.restype = C.c_longlong
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _a(b, dtype=np.uint8):
    return np.array(np.frombuffer(bytes(b), dtype) if len(b) else np.zeros(1, dtype), dtype)


def run(emu, keys, balances, pendings, flags, kind, members, tx_points, tx_extra, g_epoch, applied):
    n_acct = len(flags)
    mem = np.ascontiguousarray(np.asarray(members, np.int64).reshape(-1).astype(np.uint32))
    n_tx = len(mem) // 12
    eb, vp, iss = np.zeros(768 * n_tx, np.uint8), np.zeros(1664 * n_tx, np.uint8), np.zeros(64 * n_tx, np.uint8)
    st = np.zeros(n_tx, np.uint8)
    nb, npd, nf = np.zeros(max(64 * n_acct, 1), np.uint8), np.zeros(max(64 * n_acct, 1), np.uint8), np.zeros(max(n_acct, 1), np.uint8)
    bad = emu.emu_anon_calls_block(C.c_size_t(n_acct), _p(_a(keys)), _p(_a(balances)), _p(_a(pendings)), _p(_a(flags)), C.c_size_t(n_tx),
                                   _p(_a(kind)), _p(mem), _p(_a(tx_points)), _p(_a(tx_extra)), _p(_a(g_epoch)), _p(_a(applied)), _p(eb),
                                   _p(vp), _p(iss), _p(st), _p(nb), _p(npd), _p(nf))
    out = (eb.tobytes(), vp.tobytes(), iss.tobytes(), st.tobytes(), nb[:64 * n_acct].tobytes(), npd[:64 * n_acct].tobytes(),
           nf[:n_acct].tobytes())
    return (None if bad < 0 else int(bad)), out


@pytest.mark.parametrize("seed, n_acct, n_tx", [(61, 6, 10), (62, 16, 8)])
def test_header_equals_python_oracle(emu, seed, n_acct, n_tx):
    b = anon_issue_corpus.make(n_acct, n_tx, seed, issue_frac=0.4, bad_issue_points=1, bad_kind=True, bad_points=1, bad_index=True,
                               dup_frac=0.5, mask_p=(0.0, 0.75, 0.0, 0.0, 0.25))
    bad, got = run(emu, *b.args())
    assert bad is None
    assert got == ai.run_abi(*b.args())
    assert set(got[3]) >= {0, 3}


def test_issues_among_hundreds_of_rings_equal_c_oracle(emu):
    """300 transactions over 8 accounts, a third of them issues: account 0 sits in most rings and takes issues before,
    between and after them; the entry sort spans several scan levels"""
    b = anon_issue_corpus.make(8, 300, 63, issue_frac=0.3, skew=3.0, bad_issue_points=4, bad_kind=True, bad_points=4, bad_index=True)
    k = np.frombuffer(b.kind, np.uint8)
    issuers = b.members.reshape(-1, 12)[k == 1, 0]
    assert (issuers == 0).sum() > 20 and ((issuers >= 6) & (issuers < 8)).sum() > 0
    bad, got = run(emu, *b.args())
    assert bad is None
    assert (None, got) == aic.block(*b.args())
    assert set(got[3]) == {0, 1, 2, 3}


def test_bad_account_behind_an_issue(emu):
    """an issue before an account's first touch does not excuse its unreadable stored balance; an account only issues
    name is never decoded"""
    b = anon_issue_corpus.make(16, 4, 64, issue_frac=0.0, free=0, dup_frac=0.0)
    bal_b = bytearray(b.balances)
    for a in (14, 15):
        bal_b[64 * a:64 * a + 32] = bal_corpus.bad_curve()
    flags = bytearray(b.flags)
    flags[14] |= bal.BALANCE
    flags[15] |= bal.BALANCE
    mem = (np.arange(48, dtype=np.uint32) % 14).reshape(4, 12)
    mem[0, 0] = 15                                                 # issue 0 to account 15, which no ring names
    kind = bytes([1, 0, 0, 0])
    args = (b.keys, bytes(bal_b), b.pendings, bytes(flags), kind, mem.reshape(-1), b.tx_points, b.tx_extra, b.g_epoch, b"\x01" * 4)
    bad, got = run(emu, *args)
    assert bad is None and (None, got) == aic.block(*args)
    assert got[6][15] == flags[15] and got[4][64 * 15:] == got[2][:64] and got[5][64 * 15:] == b.pendings[64 * 15:]
    mem[0, 0] = 14
    mem[2, 3] = 14                                                 # issued to, then touched
    args = args[:5] + (mem.reshape(-1),) + args[6:]
    assert run(emu, *args)[0] == 14 == aic.block(*args)[0]
    with pytest.raises(bal.BadAccount):
        ai.run_abi(*args)
