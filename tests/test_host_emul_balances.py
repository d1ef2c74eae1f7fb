"""CPU check of the PRODUCT's balance-update header (zero_chain_b200/csrc/balances.cuh) compiled with ZK_HOST_EMUL: every
pass of the device pipeline, run as loops over its items, against the Python oracle of the module's loop on small blocks
(the scan across several levels, rollover rules, absent balances, self-transfers, every status), and on a block long
enough for one chain to span several scan levels against the C oracle.  The real PTX path is covered by
tests/test_gpu_balances.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.jubjub_oracle import bal_coracle as bc
from tests.jubjub_oracle import bal_corpus
from tests.jubjub_oracle import balances as bal

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_bal") / "libemul_bal.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "zero_chain_b200", "csrc"),
                           "-o", so, os.path.join(HERE, "host_emul", "emul_balances.cpp")])
    lib = C.CDLL(so)
    lib.emu_bal_block.restype = C.c_longlong
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _a(b, dtype=np.uint8):
    return np.array(np.frombuffer(bytes(b), dtype) if len(b) else np.zeros(1, dtype), dtype)


def run(emu, balances, pendings, flags, sender, recipient, tx_points, applied):
    n_acct, n_tx = len(flags), len(sender)
    s = np.ascontiguousarray(sender, np.uint32) if n_tx else np.zeros(1, np.uint32)
    r = np.ascontiguousarray(recipient, np.uint32) if n_tx else np.zeros(1, np.uint32)
    bs, ba = np.zeros(max(64 * n_tx, 1), np.uint8), np.zeros(max(64 * n_tx, 1), np.uint8)
    st = np.zeros(max(n_tx, 1), np.uint8)
    nb, npd, nf = np.zeros(max(64 * n_acct, 1), np.uint8), np.zeros(max(64 * n_acct, 1), np.uint8), np.zeros(max(n_acct, 1), np.uint8)
    bad = emu.emu_bal_block(C.c_size_t(n_acct), _p(_a(balances)), _p(_a(pendings)), _p(_a(flags)), C.c_size_t(n_tx), _p(s), _p(r),
                            _p(_a(tx_points)), _p(_a(applied)), _p(bs), _p(ba), _p(st), _p(nb), _p(npd), _p(nf))
    out = (bs[:64 * n_tx].tobytes(), ba[:64 * n_tx].tobytes(), st[:n_tx].tobytes(), nb[:64 * n_acct].tobytes(),
           npd[:64 * n_acct].tobytes(), nf[:n_acct].tobytes())
    return (None if bad < 0 else int(bad)), out


@pytest.mark.parametrize("seed, n_acct, n_tx", [(11, 4, 10), (12, 2, 24), (13, 7, 5), (14, 300, 40)])
def test_header_equals_python_oracle(emu, seed, n_acct, n_tx):
    b = bal_corpus.make(n_acct, n_tx, seed, bad_points=2, bad_index=True, self_frac=0.2)
    bad, got = run(emu, *b.args())
    assert bad is None
    assert got == bal.run_abi(*b.args())


def test_long_chain_equals_c_oracle(emu):
    """one sender holds most of 700 transactions: its chain crosses every level of the scan (8, 64, 512 elements)"""
    b = bal_corpus.make(6, 700, 15, skew=4.0, bad_points=5)
    assert np.bincount(b.sender).max() > 520
    bad, got = run(emu, *b.args())
    assert bad is None
    assert (None, got) == bc.block(*b.args())


def test_no_transactions(emu):
    b = bal_corpus.make(5, 0, 16)
    assert run(emu, *b.args()) == (None, (b"", b"", b"", b.balances, b.pendings, b.flags))


def test_bad_account(emu):
    b = bal_corpus.make(4, 3, 17)
    pend = bytearray(b.pendings)
    pend[64 * 3 + 32:64 * 3 + 64] = bal_corpus.bad_curve()
    flags = bytearray(b.flags)
    flags[3] |= bal.PENDING
    args = (b.balances, bytes(pend), bytes(flags), [0, 1, 3], [1, 0, 0], b.tx_points, b"\x01" * 3)
    assert run(emu, *args)[0] == 3
    args = (b.balances, bytes(pend), bytes(flags), [0, 1, 2], [1, 0, 0], b.tx_points, b"\x01" * 3)
    bad, got = run(emu, *args)
    assert bad is None and got == bal.run_abi(*args) and got[4][192:256] == bytes(pend[192:256])
