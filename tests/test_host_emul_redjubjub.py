"""CPU check of the PRODUCT's RedJubjub header (zero_chain_b200/csrc/redjubjub.cuh): the device source compiled with
ZK_HOST_EMUL against the Python oracle (tests/jubjub_oracle/redjubjub.py) — BLAKE2b over every block edge, Fs::to_uniform
on edge digests, and whole verifications over a corpus with every verdict.  The real PTX path is covered by
tests/test_gpu_redjubjub.py."""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np
import pytest

from tests.jubjub_oracle import redjubjub as rj
from tests.jubjub_oracle import rj_corpus

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_rj") / "libemul_rj.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "zero_chain_b200", "csrc"),
                           "-o", so, os.path.join(HERE, "host_emul", "emul_redjubjub.cpp")])
    return C.CDLL(so)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _b(data: bytes):
    return np.frombuffer(data, np.uint8) if data else np.zeros(1, np.uint8)


def test_blake2b(emu):
    rng = np.random.default_rng(2)
    for n in list(range(0, 301, 7)) + rj_corpus.EDGE_LENGTHS + [352, 353, 1000]:
        rbar, msg = rng.bytes(32), rng.bytes(n)
        out = np.zeros(64, np.uint8)
        emu.emu_rj_h_star_digest(_p(_b(rbar)), _p(_b(msg)), C.c_uint64(n), _p(out))
        assert out.tobytes() == hashlib.blake2b(rbar + msg, digest_size=64, person=rj.H_STAR_PERSONALIZATION).digest(), n


def test_to_uniform(emu):
    r = rj.R_J
    vals = [0, 1, r - 1, r, r + 1, 2 * r, 17 * r + 5, (1 << 256) - 1, 1 << 256, (1 << 256) * r, (1 << 256) * r + r - 1,
            (1 << 512) - 1, (1 << 512) - r, ((1 << 512) // r) * r, ((1 << 512) // r) * r - 1]
    rng = np.random.default_rng(4)
    digests = [v.to_bytes(64, "little") for v in vals] + [b"\xff" * 32 + bytes(32), bytes(32) + b"\xff" * 32]
    digests += [rng.bytes(64) for _ in range(200)]
    for d in digests:
        out = np.zeros(32, np.uint8)
        emu.emu_rj_to_uniform(_p(_b(d)), _p(out))
        assert int.from_bytes(out.tobytes(), "little") == rj.to_uniform(d), d.hex()


def test_verify_mixed_corpus(emu):
    entries, _ = rj_corpus.mixed(len(rj_corpus.EDGE_LENGTHS), seed=7)
    vks, sigs, msgs = rj_corpus.columns(entries)
    n = len(entries)
    off = np.zeros(n + 1, np.uint64)
    np.cumsum([len(m) for m in msgs], out=off[1:])
    out = np.zeros(n, np.uint8)
    emu.emu_rj_verify(C.c_size_t(n), _p(_b(vks)), _p(_b(sigs)), _p(_b(b"".join(msgs))), _p(off), _p(out))
    want = [rj_corpus.python_verdict(e) for e in entries]
    assert [int(v) for v in out] == want
    assert set(want) == {0, 1, 2, 3, 4}
