"""CPU check of the PRODUCT's Jubjub MSM header (zero_chain_b200/csrc/jubjub_msm.cuh): the device source compiled with
ZK_HOST_EMUL against the Python oracle — Niels negation, one bucket's accumulation over runs with the identity, small-order
points and both signs, the bucket reduction and Horner arithmetic of small windows, and the per-entry stage of batch
verification (z c per entry, the sum of z S).  The real PTX path is covered by tests/test_gpu_jubjub_msm.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.jubjub_oracle import pyref as jj
from tests.jubjub_oracle import redjubjub as rj
from tests.jubjub_oracle import rj_batch as rjb
from tests.jubjub_oracle import rj_corpus

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_jm") / "libemul_jm.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "zero_chain_b200", "csrc"),
                           "-o", so, os.path.join(HERE, "host_emul", "emul_jubjub_msm.cpp")])
    return C.CDLL(so)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _b(data: bytes):
    return np.frombuffer(data, np.uint8) if data else np.zeros(1, np.uint8)


def _points(seed, n):
    rng = np.random.default_rng(seed)
    t8, t4, t2 = jj.torsion_point(8), jj.torsion_point(4), jj.torsion_point(2)
    pts = [jj.IDENTITY, t8, t4, t2, rj.P_G, jj.neg(rj.P_G), jj.add(rj.P_G, t8)]
    while len(pts) < n:
        pts.append(jj.add(jj.mul(rj.P_G, int.from_bytes(rng.bytes(32), "little") % rj.R_J), (jj.IDENTITY, t8, t2)[len(pts) % 3]))
    return pts[:n]


def _niels(emu, pts):
    out = np.zeros((len(pts), 24), np.uint32)
    for i, p in enumerate(pts):
        assert emu.emu_jm_read_niels(_p(_b(jj.encode(p))), _p(out[i])) == 0
    return out


def _ext(emu, pts):
    out = np.zeros((len(pts), 32), np.uint32)
    for i, p in enumerate(pts):
        assert emu.emu_jm_ext_read(_p(_b(jj.encode(p))), _p(out[i])) == 0
    return out


def _enc(emu, ext):
    out = np.zeros(32, np.uint8)
    emu.emu_jm_encode(_p(np.ascontiguousarray(ext)), _p(out))
    return out.tobytes()


def test_niels_negation(emu):
    pts = _points(1, 24)
    n = _niels(emu, pts)
    neg = _niels(emu, [jj.neg(p) for p in pts])
    for i in range(len(pts)):
        out = np.zeros(24, np.uint32)
        emu.emu_jm_niels_cneg(_p(n[i]), 1, _p(out))
        assert (out == neg[i]).all(), i
        emu.emu_jm_niels_cneg(_p(n[i]), 0, _p(out))
        assert (out == n[i]).all(), i


def test_bucket_accumulation(emu):
    pts = _points(2, 40)
    niels = _niels(emu, pts)
    rng = np.random.default_rng(3)
    runs = [[0], [0, 0, 0], [1] * 8, [4, 4 | 1 << 31], [1, 2, 3, 1 | 1 << 31, 2 | 1 << 31], list(range(40))]
    runs += [[int(i) | (int(s) << 31) for i, s in zip(rng.integers(0, 40, 33), rng.integers(0, 2, 33))] for _ in range(6)]
    for run in runs:
        entries = np.array([7, 7] + run, np.uint32)          # two leading entries outside the run [2, 2 + len)
        out = np.zeros(32, np.uint32)
        emu.emu_jm_accumulate(_p(niels), _p(entries), 2, 2 + len(run), _p(out))
        want = jj.IDENTITY
        for e in run:
            p = pts[e & 0x7fffffff]
            want = jj.add(want, jj.neg(p) if e >> 31 else p)
        assert _enc(emu, out) == jj.encode(want), run
    out = np.zeros(32, np.uint32)
    emu.emu_jm_accumulate(_p(niels), _p(np.zeros(1, np.uint32)), 0, 0, _p(out))
    assert _enc(emu, out) == jj.encode(jj.IDENTITY)


@pytest.mark.parametrize("c", [3, 5, 8])
def test_window_reduction_and_horner(emu, c):
    nb, log_l = 1 << (c - 1), c // 2
    L, n_slices = 1 << log_l, nb >> log_l
    pts = _points(10 + c, nb)
    buckets = _ext(emu, pts)
    S = np.zeros((n_slices, 32), np.uint32)
    T = np.zeros((n_slices, 32), np.uint32)
    for j in range(n_slices):
        emu.emu_jm_slice_sums(_p(np.ascontiguousarray(buckets[j * L:(j + 1) * L])), L, _p(S[j]), _p(T[j]))
        assert _enc(emu, T[j]) == jj.encode(rjb.multiexp(pts[j * L:(j + 1) * L], [1] * L))
    R = np.zeros(32, np.uint32)
    emu.emu_jm_window_sum(_p(S), _p(T), n_slices, log_l, _p(R))
    want = rjb.multiexp(pts, range(1, nb + 1))
    assert _enc(emu, R) == jj.encode(want)
    # Horner over three windows
    wins = _ext(emu, pts[:3])
    out = np.zeros(32, np.uint32)
    emu.emu_jm_horner(_p(wins), 3, c, _p(out))
    assert _enc(emu, out) == jj.encode(rjb.multiexp(pts[:3], [1, 1 << c, 1 << (2 * c)]))


def test_batch_entry_stage(emu):
    entries, _ = rj_corpus.mixed(len(rj_corpus.EDGE_LENGTHS), seed=11)
    vks, sigs, msgs = rj_corpus.columns(entries)
    n = len(entries)
    rng = np.random.default_rng(12)
    zs = [int.from_bytes(rng.bytes(64), "little") % rj.R_J for _ in range(n)]
    zs[0], zs[1] = 0, rj.R_J - 1
    off = np.zeros(n + 1, np.uint64)
    np.cumsum([len(m) for m in msgs], out=off[1:])
    codes = np.zeros(n, np.uint8)
    zc = np.zeros(32 * n, np.uint8)
    total = np.zeros(32, np.uint8)
    emu.emu_rj_batch_prep(C.c_size_t(n), _p(_b(vks)), _p(_b(sigs)), _p(_b(b"".join(msgs))), _p(off),
                          _p(_b(b"".join(z.to_bytes(32, "little") for z in zs))), _p(codes), _p(zc), _p(total))
    want_sum = 0
    for i, (vk, sig, msg) in enumerate(zip([e[0] for e in entries], [e[1] for e in entries], msgs)):
        st_vk, _ = jj.read(vk)
        st_r, _ = jj.read(sig[:32])
        s = int.from_bytes(sig[32:], "little")
        code = rj.BAD_VK if st_vk else rj.BAD_R if st_r else rj.BAD_S if s >= rj.R_J else rj.OK
        assert codes[i] == code, i
        got = int.from_bytes(zc[32 * i:32 * i + 32].tobytes(), "little")
        if code == rj.OK:
            assert got == zs[i] * rj.h_star(sig[:32], msg) % rj.R_J
            want_sum += zs[i] * s
        else:
            assert got == 0
    assert int.from_bytes(total.tobytes(), "little") == want_sum % rj.R_J
    assert set(codes) == {1, 2, 3, 4}
