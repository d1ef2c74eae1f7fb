"""CPU check of the PRODUCT's key-derivation functions (zero_chain_b200/csrc/hd_keys.cuh) compiled with ZK_HOST_EMUL: the
hashes against hashlib (the master hash, both 69-byte PRF messages, the 0x13 expansion and the 32-byte fingerprint), and
whole rows of the three calls, run in the order of their passes, against the Python oracle (tests/jubjub_oracle/hd_keys.py)
on edge and random rows.  The real PTX path is covered by tests/test_gpu_hd_keys.py."""
import ctypes as C
import hashlib
import os
import struct
import subprocess

import numpy as np
import pytest

from tests.jubjub_oracle import hd_keys as hd
from tests.jubjub_oracle import redjubjub as rj

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
XK = hd.XK


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_hd") / "libemul_hd.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "zero_chain_b200", "csrc"),
                           "-o", so, os.path.join(HERE, "host_emul", "emul_hd_keys.cpp")])
    lib = C.CDLL(so)
    lib.emu_tag.restype = C.c_uint32
    lib.emu_xsk_derive.restype = C.c_longlong
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _b(data: bytes):
    return np.frombuffer(data, np.uint8) if data else np.zeros(1, np.uint8)


def _rows(a, size, n):
    return [a[size * i:size * (i + 1)].tobytes() for i in range(n)] if a is not None else [None] * n


def _out(size, n):
    return np.full(max(size * n, 1), 0xEE, np.uint8)


def _seeds():
    rng = np.random.default_rng(3)
    return [b"", b"\x00", b"Alice" + b" " * 27] + [rng.bytes(int(k)) for k in (31, 32, 64, 127, 128, 129, 300)]


def test_hashes_match_hashlib(emu):
    for seed in _seeds():
        sk, chain = _out(32, 1), _out(32, 1)
        emu.emu_master_hash(_p(_b(seed)), C.c_uint64(len(seed)), _p(sk), _p(chain))
        i = hashlib.blake2b(seed, digest_size=64, person=hd.MASTER_PERSONALIZATION).digest()
        assert chain.tobytes() == i[32:]
        assert int.from_bytes(sk.tobytes(), "little") == rj.spending_key(i[:32])
    rng = np.random.default_rng(4)
    for c, key, index in [(bytes(32), bytes(32), 0), (b"\xff" * 32, b"\xff" * 32, 2 ** 32 - 1), (rng.bytes(32), rng.bytes(32), 2 ** 31),
                          (rng.bytes(32), rng.bytes(32), 2 ** 31 - 1), (rng.bytes(32), rng.bytes(32), 0x01020304)]:
        for t in (0x11, 0x12):
            out = _out(64, 1)
            emu.emu_prf_child(_p(_b(c)), C.c_uint32(t), _p(_b(key)), C.c_uint32(index), _p(out))
            assert out.tobytes() == hd.prf_expand_vec(c, [bytes([t]), key, struct.pack("<I", index)])
    for i in [bytes(64), b"\xff" * 64, rng.bytes(64)]:
        out = _out(32, 1)
        emu.emu_tweak(_p(_b(i)), _p(out))
        want = hashlib.blake2b(i[:32] + b"\x13", digest_size=64, person=rj.EXPAND_SEED_PERSONALIZATION).digest()
        assert int.from_bytes(out.tobytes(), "little") == rj.to_uniform(want)
    for pgk in [bytes(32), b"\xff" * 32, rng.bytes(32), hd.IDENTITY_SIGNED]:
        want = hashlib.blake2b(pgk, digest_size=32, person=hd.EKFP_PERSONALIZATION).digest()[:4]
        assert struct.pack("<I", emu.emu_tag(_p(_b(pgk)))) == want


def _master(emu, seeds):
    n = len(seeds)
    off = np.zeros(n + 1, np.uint64)
    np.cumsum([len(s) for s in seeds], out=off[1:])
    outs = [_out(XK, n), _out(XK, n), _out(32, n), _out(32, n)]
    emu.emu_master(C.c_size_t(n), _p(_b(b"".join(seeds))), _p(off), *(_p(o) for o in outs))
    return list(zip(_rows(outs[0], XK, n), _rows(outs[1], XK, n), _rows(outs[2], 32, n), _rows(outs[3], 32, n)))


def _xsk(emu, parents, pidx, cidx, outputs=True):
    n = len(pidx)
    outs = [_out(XK, n)] + ([_out(XK, n), _out(32, n), _out(32, n)] if outputs else [None] * 3)
    st = _out(1, n)
    bad = emu.emu_xsk_derive(C.c_size_t(len(parents)), _p(_b(b"".join(parents))), C.c_size_t(n), _p(np.array(pidx, np.uint32)),
                             _p(np.array(cidx, np.uint32)), *(_p(o) for o in outs), _p(st))
    return bad, list(zip(_rows(outs[0], XK, n), _rows(outs[1], XK, n), _rows(outs[2], 32, n), _rows(outs[3], 32, n), [int(s) for s in st[:n]]))


def _xpgk(emu, parents, pidx, cidx):
    n = len(pidx)
    outs = [_out(XK, n), _out(32, n), _out(32, n)]
    st = _out(1, n)
    emu.emu_xpgk_derive(C.c_size_t(len(parents)), _p(_b(b"".join(parents))), C.c_size_t(n), _p(np.array(pidx, np.uint32)),
                        _p(np.array(cidx, np.uint32)), *(_p(o) for o in outs), _p(st))
    return list(zip(_rows(outs[0], XK, n), _rows(outs[1], 32, n), _rows(outs[2], 32, n), [int(s) for s in st[:n]]))


def test_master_rows(emu):
    seeds = _seeds()
    assert _master(emu, seeds) == [hd.master_row(s) for s in seeds]


def test_xsk_edge_and_random_rows(emu):
    parents = hd.edge_xsk_parents()
    pidx, cidx = hd.edge_rows(len(parents))
    bad, got = _xsk(emu, parents, pidx, cidx)
    assert bad == -1
    assert got == hd.xsk_derive_rows(parents, pidx, cidx)
    assert {g[4] for g in got} == {0, hd.BAD_INDEX, hd.DEPTH}
    parents = hd.random_xsk_parents(6, seed=1)
    pidx, cidx = hd.random_rows(60, 6, seed=2)
    assert _xsk(emu, parents, pidx, cidx)[1] == hd.xsk_derive_rows(parents, pidx, cidx)
    # no optional outputs: the same xsks
    assert [g[0] for g in _xsk(emu, parents, pidx, cidx, outputs=False)[1]] == [w[0] for w in hd.xsk_derive_rows(parents, pidx, cidx)]


def test_xsk_bad_named_parent_leaves_its_rows_unwritten(emu):
    parents = hd.random_xsk_parents(4, seed=5)
    parents[2] = parents[2][:41] + rj.scalar_bytes(rj.R_J)
    bad, got = _xsk(emu, parents, [0, 2, 3, 9], [1, 2, 3, 4])
    assert bad == 2
    assert got[1] == (b"\xee" * XK, b"\xee" * XK, b"\xee" * 32, b"\xee" * 32, 0xEE)
    want = hd.xsk_derive_rows(parents, [0, 3, 9], [1, 3, 4])
    assert [got[0], got[2], got[3]] == want
    assert _xsk(emu, parents, [0, 1, 3], [1, 2, 3])[0] == -1          # an unnamed bad parent is never read


def test_xpgk_edge_and_random_rows(emu):
    parents = hd.edge_xpgk_parents()
    pidx, cidx = hd.edge_rows(len(parents))
    got = _xpgk(emu, parents, pidx, cidx)
    assert got == hd.xpgk_derive_rows(parents, pidx, cidx)
    assert {g[3] for g in got} == {0, 1, 2, 3, hd.BAD_INDEX, hd.HARDENED_INDEX, hd.DEPTH}
    parents = [hd.xpgk_from_xsk(x) for x in hd.random_xsk_parents(6, seed=7)]
    pidx, cidx = hd.random_rows(60, 6, seed=8)
    assert _xpgk(emu, parents, pidx, cidx) == hd.xpgk_derive_rows(parents, pidx, cidx)
