"""CPU check of the PRODUCT's anonymous-transfer functions (zero_chain_b200/csrc/tx_build.cuh: anon_key_entry,
anon_status, anonymous_row, anon_position, anonymous_left) compiled with ZK_HOST_EMUL and run in the order of
zk_anonymous_fields_batch's passes, against the Python oracle (tests/jubjub_oracle/tx_build.py) on edge and random rows.
The real PTX path is covered by tests/test_gpu_anon_build.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.jubjub_oracle import anon_build as ab
from tests.jubjub_oracle import tx_build as tb

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_anon") / "libemul_anon.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "zero_chain_b200", "csrc"),
                           "-o", so, os.path.join(HERE, "host_emul", "emul_anon_build.cpp")])
    return C.CDLL(so)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _b(data: bytes):
    return np.frombuffer(data, np.uint8) if data else np.zeros(1, np.uint8)


def _fields(emu, table, rows, g):
    n = len(rows)
    sks, rings, s, t, amounts, rs, alphas = zip(*rows)
    sc = lambda v: b"".join(x.to_bytes(32, "little") for x in v)
    f = np.full(864 * n, 0xEE, np.uint8)
    rsk, dk, st = np.zeros(32 * n, np.uint8), np.zeros(32 * n, np.uint8), np.zeros(n, np.uint8)
    assert emu.emu_anon_fields(C.c_size_t(len(table)), _p(_b(b"".join(table))), C.c_size_t(n), _p(_b(sc(sks))),
                               _p(np.array(rings, np.uint32).reshape(-1)), _p(np.array(list(zip(s, t)), np.uint8).reshape(-1)),
                               _p(np.array(amounts, np.uint32)), _p(_b(sc(rs))), _p(_b(sc(alphas))), _p(_b(g)), _p(f), _p(rsk), _p(dk),
                               _p(st)) == 0
    return [(f[864 * i:864 * i + 864].tobytes(), rsk[32 * i:32 * i + 32].tobytes(), dk[32 * i:32 * i + 32].tobytes(), int(st[i]))
            for i in range(n)]


def test_positions(emu):
    for s in range(12):
        for t in range(12):
            if s == t:
                continue
            got = [emu.emu_anon_position(s, t, j) for j in range(11)]
            assert got[0] == t
            assert got[1:] == [p for p in range(12) if p not in (s, t)]


def test_edge_rows(emu):
    table = ab.key_table()
    rows = ab.edge_rows()
    g = tb.g_epoch(5)[0]
    got = _fields(emu, table, rows, g)
    for row, out in zip(rows, got):
        assert out == ab.anonymous_fields(table, *row, g), row
    assert {o[3] for o in got} == {0, 1, 2, 3, ab.ANON_BAD_INDEX, ab.ANON_BAD_POSITIONS}


def test_random_rows_over_a_larger_table(emu):
    """a table with failing keys no ring names: they are never read and change nothing"""
    table = [tb.keys(b"table key %d" % i)[2] for i in range(20)] + [k for k, _ in tb.bad_recipient_keys()]
    rows = ab.random_rows(5, 20, seed=6)
    g = tb.g_epoch(8)[0]
    assert _fields(emu, table, rows, g) == [ab.anonymous_fields(table, *r, g) for r in rows]
