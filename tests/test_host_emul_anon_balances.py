"""CPU check of the PRODUCT's anonymous-transfer header (zero_chain_b200/csrc/anon_balances.cuh, with the balances.cuh
passes it reuses) compiled with ZK_HOST_EMUL: every pass of the device pipeline, run as loops over its items, against the
Python oracle of the module's loop on small blocks (rollover rules, absent balances, members listed twice, every status),
and against the C oracle on a block where one account's entries span several levels of the scan.  The real PTX path is
covered by tests/test_gpu_anon_balances.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.jubjub_oracle import anon_balances as ab
from tests.jubjub_oracle import anon_coracle as aco
from tests.jubjub_oracle import anon_corpus
from tests.jubjub_oracle import bal_corpus
from tests.jubjub_oracle import balances as bal

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_anon") / "libemul_anon.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "zero_chain_b200", "csrc"),
                           "-o", so, os.path.join(HERE, "host_emul", "emul_anon_balances.cpp")])
    lib = C.CDLL(so)
    lib.emu_anon_block.restype = C.c_longlong
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _a(b, dtype=np.uint8):
    return np.array(np.frombuffer(bytes(b), dtype) if len(b) else np.zeros(1, dtype), dtype)


def run(emu, keys, balances, pendings, flags, members, tx_points, tx_extra, g_epoch, applied):
    n_acct = len(flags)
    mem = np.ascontiguousarray(np.asarray(members, np.int64).reshape(-1).astype(np.uint32))
    n_tx = len(mem) // 12
    eb, vp = np.zeros(max(768 * n_tx, 1), np.uint8), np.zeros(max(1664 * n_tx, 1), np.uint8)
    st = np.zeros(max(n_tx, 1), np.uint8)
    nb, npd, nf = np.zeros(max(64 * n_acct, 1), np.uint8), np.zeros(max(64 * n_acct, 1), np.uint8), np.zeros(max(n_acct, 1), np.uint8)
    bad = emu.emu_anon_block(C.c_size_t(n_acct), _p(_a(keys)), _p(_a(balances)), _p(_a(pendings)), _p(_a(flags)), C.c_size_t(n_tx),
                             _p(mem if n_tx else np.zeros(1, np.uint32)), _p(_a(tx_points)), _p(_a(tx_extra)), _p(_a(g_epoch)),
                             _p(_a(applied)), _p(eb), _p(vp), _p(st), _p(nb), _p(npd), _p(nf))
    out = (eb[:768 * n_tx].tobytes(), vp[:1664 * n_tx].tobytes(), st[:n_tx].tobytes(), nb[:64 * n_acct].tobytes(),
           npd[:64 * n_acct].tobytes(), nf[:n_acct].tobytes())
    return (None if bad < 0 else int(bad)), out


@pytest.mark.parametrize("seed, n_acct, n_tx", [(31, 4, 5), (32, 14, 4)])
def test_header_equals_python_oracle(emu, seed, n_acct, n_tx):
    b = anon_corpus.make(n_acct, n_tx, seed, bad_points=1, bad_index=True, dup_frac=0.5, mask_p=(0.0, 0.75, 0.0, 0.0, 0.25))
    bad, got = run(emu, *b.args())
    assert bad is None
    assert got == ab.run_abi(*b.args())
    assert set(got[2]) >= {0, 3}


def test_segments_across_scan_levels_equal_c_oracle(emu):
    """400 rings over 5 accounts: account 0 holds 4000 of the 4800 entries, so its applied entries (over two thousand)
    span the first three levels of the scan (8, 64 and 512 elements per item)"""
    b = anon_corpus.make(5, 400, 33, skew=3.0, bad_points=6, bad_index=True)
    assert np.bincount(b.members[b.members < 5]).max() > 4000
    bad, got = run(emu, *b.args())
    assert bad is None
    assert (None, got) == aco.block(*b.args())
    assert set(got[2]) == {0, 1, 2, 3}


def test_no_transactions(emu):
    b = anon_corpus.make(5, 0, 34)
    assert run(emu, *b.args()) == (None, (b"", b"", b"", b.balances, b.pendings, b.flags))


def test_bad_account(emu):
    b = anon_corpus.make(16, 2, 35, dup_frac=0.0)
    pend = bytearray(b.pendings)
    pend[64 * 15 + 32:64 * 15 + 64] = bal_corpus.bad_curve()
    flags = bytearray(b.flags)
    flags[15] |= bal.PENDING
    mem = np.arange(24, dtype=np.uint32) % 15                      # account 15 untouched
    args = (b.keys, b.balances, bytes(pend), bytes(flags), mem, b.tx_points, b.tx_extra, b.g_epoch, b"\x01\x01")
    bad, got = run(emu, *args)
    assert bad is None and (None, got) == aco.block(*args) and got[4][64 * 15:] == bytes(pend[64 * 15:])
    mem[20] = 15                                                   # touched
    args = args[:4] + (mem,) + args[5:]
    assert run(emu, *args)[0] == 15 == aco.block(*args)[0]
