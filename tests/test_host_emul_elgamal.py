"""CPU check of the PRODUCT's ElGamal header (zero_chain_b200/csrc/elgamal.cuh) compiled with ZK_HOST_EMUL: the
per-ciphertext stage (status and the encoding of V = left - dk right) against the Python oracle on a corpus with every
status, the chunked table build against the C oracle's successive additions, and the index, also on a reduced-size index
with forced fingerprint collisions.  The real PTX path is covered by tests/test_gpu_elgamal.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.jubjub_oracle import eg_coracle as ec
from tests.jubjub_oracle import eg_corpus
from tests.jubjub_oracle import elgamal as eg

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
EG_CHUNK = 16                       # table entries per thread of the build (elgamal.cuh)
EMPTY = 0xFFFFFFFF


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_eg") / "libemul_eg.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "zero_chain_b200", "csrc"),
                           "-o", so, os.path.join(HERE, "host_emul", "emul_elgamal.cpp")])
    return C.CDLL(so)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _b(data: bytes):
    return np.frombuffer(data, np.uint8) if data else np.zeros(1, np.uint8)


def _stage(emu, dks, cts, pds):
    n = len(dks) // 32
    venc = np.zeros((n, 32), np.uint8)
    st = np.zeros(n, np.uint8)
    emu.emu_eg_stage(C.c_size_t(n), _p(_b(dks)), _p(_b(cts)), None if pds is None else _p(_b(pds)), _p(venc), _p(st))
    return [int(s) for s in st], [bytes(v) for v in venc]


def test_stage_matches_python_oracle(emu):
    entries = eg_corpus.special_entries(5) + eg_corpus.random_entries(16, seed=6)
    dks, cts, pds, want_null, want_pend = eg_corpus.columns(entries)
    for pending in (None, pds):
        st, venc = _stage(emu, dks, cts, pending)
        for i, e in enumerate(entries):
            ws, wv = eg.stage(e[0], e[1], None if pending is None else e[2])
            assert st[i] == ws, i
            if ws == eg.OK:
                assert venc[i] == wv, i
        want = want_null if pending is None else want_pend
        # the statuses the construction intends: OK and NOT_FOUND differ only in the lookup, which comes after the stage
        assert st == [s if s >= 2 else 0 for s in want[0]]
    assert set(want_pend[0]) == {0, 1, 2, 3, 4}


def test_stage_encodings_are_table_entries(emu):
    """For small amounts the encoding of V is the reference's i P_G, the sign of x included (neg_encrypt is not)."""
    entries = eg_corpus.special_entries(8)
    dks, cts, pds, _, want = eg_corpus.columns(entries[:2])
    st, venc = _stage(emu, dks, cts, pds)
    table = ec.multiples(11)
    assert st == [0, 0] and venc == [bytes(table[10]), bytes(table[0])]
    neg = entries[5]
    st, venc = _stage(emu, neg[0], neg[1], None)
    assert st == [0] and venc[0] == bytes(ec.multiples(6)[5])[:31] + bytes([ec.multiples(6)[5][31] ^ 0x80])


@pytest.mark.parametrize("n", [1, EG_CHUNK - 1, EG_CHUNK, EG_CHUNK + 1, 5 * EG_CHUNK + 3, 4099])
def test_table_chunks_match_successive_additions(emu, n):
    out = np.zeros((n, 32), np.uint8)
    emu.emu_eg_table(C.c_uint32(n), _p(out))
    assert np.array_equal(out, ec.multiples(n))


def _index(emu, log_slots, keys, order, probes):
    keys = np.ascontiguousarray(keys, np.uint8)
    probes = np.ascontiguousarray(probes, np.uint8)
    order = np.ascontiguousarray(order, np.uint32)
    found = np.zeros(len(probes), np.uint32)
    emu.emu_eg_index(C.c_int(log_slots), C.c_uint32(len(keys)), _p(keys), _p(order), C.c_uint32(len(probes)), _p(probes), _p(found))
    return [int(v) for v in found]


def test_index_finds_every_key(emu):
    keys = ec.multiples(20000)
    rng = np.random.default_rng(1)
    order = rng.permutation(len(keys))
    misses = rng.integers(0, 256, (500, 32), dtype=np.uint8)
    neg = keys[1:500].copy()
    neg[:, 31] ^= 0x80                                            # -i P_G: same y, the other sign
    got = _index(emu, 15, keys, order, np.concatenate([keys, misses, neg]))
    assert got[:len(keys)] == list(range(len(keys)))
    assert got[len(keys):] == [EMPTY] * (len(misses) + len(neg))


def test_index_with_forced_fingerprint_collisions(emu):
    """Keys that share the slot bits and the fingerprint and differ only elsewhere: every one is still found, and a probe
    with the same slot and fingerprint but no entry is not."""
    rng = np.random.default_rng(2)
    keys = rng.integers(0, 256, (40, 32), dtype=np.uint8)
    keys[:30, 0:4] = [0x35, 0x02, 0, 0]                           # slot 0x235 in a 2^10 index for 30 of them
    keys[:30, 4:8] = [0x11, 0x22, 0x3c, 0xab]                     # and one fingerprint (the top 12 bits of word 1)
    keys[:30, 8] = np.arange(30)                                  # distinct keys
    absent = keys[:5].copy()
    absent[:, 8] = 200 + np.arange(5)
    for order in (np.arange(40), np.arange(40)[::-1], rng.permutation(40)):
        got = _index(emu, 10, keys, order, np.concatenate([keys, absent]))
        assert got == list(range(40)) + [EMPTY] * 5
