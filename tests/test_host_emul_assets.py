"""CPU check of the PRODUCT's encrypted-asset header (zero_chain_b200/csrc/assets.cuh) compiled with ZK_HOST_EMUL: every
pass of the device pipeline, run as loops over its items, against the C oracle of the module's loop on random blocks of
mixed kinds (restarts by issue and destroy, rollovers, every status), on a block where one slot's chain crosses every
level of the scan with restarts inside it, and against the Python oracle on the hand-made rules.  The real PTX path is
covered by tests/test_gpu_assets.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.jubjub_oracle import assets as asr
from tests.jubjub_oracle import assets_coracle as ac
from tests.jubjub_oracle import assets_corpus
from tests.jubjub_oracle import bal_corpus
from tests.jubjub_oracle import balances as bal

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_assets") / "libemul_assets.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "zero_chain_b200", "csrc"),
                           "-o", so, os.path.join(HERE, "host_emul", "emul_assets.cpp")])
    lib = C.CDLL(so)
    lib.emu_as_block.restype = C.c_longlong
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _a(b, dtype=np.uint8):
    return np.array(np.frombuffer(bytes(b), dtype) if len(b) else np.zeros(1, dtype), dtype)


def run(emu, balances, pendings, flags, kind, slot_a, slot_b, tx_points, applied):
    n, n_tx = len(flags), len(kind)
    idx = lambda v: np.ascontiguousarray(np.asarray(v, np.int64).astype(np.uint32)) if n_tx else np.zeros(1, np.uint32)
    bs, ba = np.zeros(max(64 * n_tx, 1), np.uint8), np.zeros(max(64 * n_tx, 1), np.uint8)
    ev, ef, st = np.zeros(max(128 * n_tx, 1), np.uint8), np.zeros(max(n_tx, 1), np.uint8), np.zeros(max(n_tx, 1), np.uint8)
    nb, npd, nf = np.zeros(max(64 * n, 1), np.uint8), np.zeros(max(64 * n, 1), np.uint8), np.zeros(max(n, 1), np.uint8)
    bad = emu.emu_as_block(C.c_size_t(n), _p(_a(balances)), _p(_a(pendings)), _p(_a(flags)), C.c_size_t(n_tx), _p(_a(bytes(kind))),
                           _p(idx(slot_a)), _p(idx(slot_b)), _p(_a(tx_points)), _p(_a(applied)), _p(bs), _p(ba), _p(ev), _p(ef), _p(st),
                           _p(nb), _p(npd), _p(nf))
    out = (bs[:64 * n_tx].tobytes(), ba[:64 * n_tx].tobytes(), ev[:128 * n_tx].tobytes(), ef[:n_tx].tobytes(), st[:n_tx].tobytes(),
           nb[:64 * n].tobytes(), npd[:64 * n].tobytes(), nf[:n].tobytes())
    return (None if bad < 0 else int(bad)), out


@pytest.mark.parametrize("seed, n_slots, n_tx", [(31, 4, 30), (32, 2, 40), (33, 9, 25), (34, 300, 120)])
def test_header_equals_c_oracle(emu, seed, n_slots, n_tx):
    b = assets_corpus.make(n_slots, n_tx, seed, issue_frac=0.2, destroy_frac=0.15, bad_points=3, bad_index=True, zero_frac=0.3,
                           self_frac=0.2)
    bad, got = run(emu, *b.args())
    assert bad is None
    assert (None, got) == ac.block(*b.args())


def test_small_block_equals_python_oracle(emu):
    b = assets_corpus.make(3, 10, 35, issue_frac=0.3, destroy_frac=0.2, bad_points=1, bad_index=True, zero_frac=0.3)
    assert run(emu, *b.args()) == (None, asr.run_abi(*b.args()))


def test_long_chain_with_restarts(emu):
    """one slot holds most of 700 transactions, issues and destroys among them: its chains cross every scan level"""
    b = assets_corpus.make(6, 700, 36, skew=4.0, issue_frac=0.03, destroy_frac=0.02, bad_points=5)
    assert np.bincount(b.slot_a).max() > 500
    kinds = np.frombuffer(b.kind, np.uint8)
    assert ((kinds != 0) & (b.slot_a == 0)).sum() >= 10
    bad, got = run(emu, *b.args())
    assert bad is None
    assert (None, got) == ac.block(*b.args())


def test_transfers_only_equal_the_confidential_header(emu):
    b = assets_corpus.make(7, 60, 37, issue_frac=0.0, destroy_frac=0.0, bad_points=2)
    b.applied = bytes(int(v == 1) for v in b.applied)
    got = run(emu, *b.args())[1]
    assert (got[0], got[1], got[4]) + got[5:] == bal.run_abi(*b.transfers())


def test_no_transactions(emu):
    b = assets_corpus.make(5, 0, 38)
    assert run(emu, *b.args()) == (None, (b"", b"", b"", b"", b"", b.balances, b.pendings, b.flags))


def test_bad_slot(emu):
    b = assets_corpus.make(4, 3, 39, issue_frac=0.0, destroy_frac=0.0)
    pend = bytearray(b.pendings)
    pend[64 * 3 + 32:64 * 3 + 64] = bal_corpus.bad_curve()
    flags = bytearray(b.flags)
    flags[3] |= bal.PENDING
    args = (b.balances, bytes(pend), bytes(flags), bytes([0, 2, 1]), [0, 3, 2], [1, 0, 0], b.tx_points, b"\x01" * 3)
    assert run(emu, *args)[0] == 3                                   # named by a destroy
    args = (b.balances, bytes(pend), bytes(flags), bytes([0, 2, 1]), [0, 2, 2], [1, 3, 3], b.tx_points, b"\x01" * 3)
    bad, got = run(emu, *args)
    assert bad is None and got == ac.block(*args)[1] and got[6][192:256] == bytes(pend[192:256])
