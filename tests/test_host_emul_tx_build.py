"""CPU check of the PRODUCT's transaction-building header (zero_chain_b200/csrc/tx_build.cuh): the device source compiled
with ZK_HOST_EMUL against hashlib and the Python oracle (tests/jubjub_oracle/redjubjub.py, elgamal.py) — BLAKE2s at every
block edge, the committed P_G window table and the table built for a g_epoch, key derivation, GEpoch::group_hash,
the confidential fields with edge rows, and signatures.  The real PTX path is covered by tests/test_gpu_tx_build.py."""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np
import pytest

from tests.jubjub_oracle import pyref as jj
from tests.jubjub_oracle import redjubjub as rj
from tests.jubjub_oracle import tx_build as tb

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
TABLE_ENTRIES = 64 * 9


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_tb") / "libemul_tb.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "zero_chain_b200", "csrc"),
                           "-o", so, os.path.join(HERE, "host_emul", "emul_tx_build.cpp")])
    return C.CDLL(so)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _b(data: bytes):
    return np.frombuffer(data, np.uint8) if data else np.zeros(1, np.uint8)


def test_blake2s(emu):
    rng = np.random.default_rng(3)
    for pers in (b"zech_bdk", b"zcgepoch", b"Zcash_PH"):
        for n in (0, 1, 31, 32, 33, 55, 63, 64, 65, 69, 127, 128, 129, 200):
            msg = rng.bytes(n)
            out = np.zeros(32, np.uint8)
            emu.emu_tb_blake2s(_p(_b(pers)), _p(_b(msg)), C.c_uint32(n), _p(out))
            assert out.tobytes() == hashlib.blake2s(msg, digest_size=32, person=pers).digest(), (pers, n)


def _table_words(points) -> bytes:
    return b"".join(b"".join(((v << 256) % jj.R).to_bytes(32, "little") for v in tb.niels(p)) for p in points)


def test_pg_table_matches_oracle(emu):
    out = np.zeros(TABLE_ENTRIES * 24, np.uint32)
    emu.emu_tb_pg_table(_p(out))
    assert out.tobytes() == _table_words(tb.window_table(rj.P_G))


def test_epoch_table_matches_oracle(emu):
    g = tb.g_epoch(5)[0]
    out = np.zeros(TABLE_ENTRIES * 24, np.uint32)
    assert emu.emu_tb_epoch_table(_p(_b(g)), _p(out)) == 0
    assert out.tobytes() == _table_words(tb.window_table(jj.read(g)[1]))
    # the builder run on P_G gives the committed table
    pg = np.zeros(TABLE_ENTRIES * 24, np.uint32)
    emu.emu_tb_pg_table(_p(pg))
    assert emu.emu_tb_epoch_table(_p(_b(jj.encode(rj.P_G))), _p(out)) == 0
    assert np.array_equal(out, pg)


def test_keys_from_seed(emu):
    seeds = [b"", b"a", b"Alice" + b" " * 27, bytes(range(127)), bytes(128), bytes(range(129)) + b"x" * 200]
    off = np.zeros(len(seeds) + 1, np.uint64)
    np.cumsum([len(s) for s in seeds], out=off[1:])
    n = len(seeds)
    sks, dks, eks = (np.zeros(32 * n, np.uint8) for _ in range(3))
    emu.emu_tb_keys(C.c_size_t(n), _p(_b(b"".join(seeds))), _p(off), _p(sks), _p(dks), _p(eks))
    for i, s in enumerate(seeds):
        assert (sks[32 * i:32 * i + 32].tobytes(), dks[32 * i:32 * i + 32].tobytes(), eks[32 * i:32 * i + 32].tobytes()) == tb.keys(s)


def test_g_epoch(emu):
    for e in list(range(65)) + [2 ** 32 - 1]:
        out, tag = np.zeros(32, np.uint8), C.c_uint32(0)
        assert emu.emu_tb_g_epoch(C.c_uint32(e), _p(out), C.byref(tag)) == 1
        assert (out.tobytes(), tag.value) == tb.g_epoch(e), e


def _fields(emu, rows, g_epoch):
    n = len(rows)
    cols = list(zip(*rows))
    sks, eks, amounts, fees, rs, alphas = cols
    f = np.zeros(32 * 9 * n, np.uint8)
    rsk, dk, st = np.zeros(32 * n, np.uint8), np.zeros(32 * n, np.uint8), np.zeros(n, np.uint8)
    sc = lambda v: b"".join(x.to_bytes(32, "little") for x in v)
    emu.emu_tb_fields(C.c_size_t(n), _p(_b(sc(sks))), _p(_b(b"".join(eks))), _p(np.array(amounts, np.uint32)), _p(np.array(fees, np.uint32)),
                      _p(_b(sc(rs))), _p(_b(sc(alphas))), _p(_b(g_epoch)), _p(f), _p(rsk), _p(dk), _p(st))
    return [(f[288 * i:288 * i + 288].tobytes(), rsk[32 * i:32 * i + 32].tobytes(), dk[32 * i:32 * i + 32].tobytes(), int(st[i]))
            for i in range(n)]


def test_confidential_fields(emu):
    rows = tb.edge_rows() + tb.random_rows(6, seed=11)
    g = tb.g_epoch(3)[0]
    got = _fields(emu, rows, g)
    for row, out in zip(rows, got):
        assert out == tb.confidential_fields(*row, g), row


def test_sign(emu):
    rng = np.random.default_rng(9)
    lengths = [0, 1, 47, 48, 49, 127, 128, 129, 300]
    sks = [0, 1, rj.R_J - 1] + [int.from_bytes(rng.bytes(32), "little") % rj.R_J for _ in lengths[3:]]
    ts = [rng.bytes(80) for _ in lengths]
    msgs = [rng.bytes(n) for n in lengths]
    n = len(msgs)
    off = np.zeros(n + 1, np.uint64)
    np.cumsum(lengths, out=off[1:])
    sigs = np.zeros(64 * n, np.uint8)
    emu.emu_tb_sign(C.c_size_t(n), _p(_b(b"".join(rj.scalar_bytes(s) for s in sks))), _p(_b(b"".join(ts))), _p(_b(b"".join(msgs))), _p(off),
                    _p(sigs))
    for i in range(n):
        sig = sigs[64 * i:64 * i + 64].tobytes()
        assert sig == rj.sign(sks[i], msgs[i], ts[i]), i
        assert rj.verify(rj.public_key(sks[i]), msgs[i], sig) == rj.OK
