"""CPU check of the PRODUCT's Jubjub header (zero_chain_b200/csrc/jubjub.cuh): the device source compiled with ZK_HOST_EMUL
against the Python oracle (tests/jubjub_oracle/pyref.py) — the Tonelli-Shanks square root down to its deepest loop, the
extended-coordinate group law, and every decode class.  The real PTX path is covered by tests/test_gpu_jubjub.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.jubjub_oracle import pyref as jj

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
R = jj.R


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_jj") / "libemul_jj.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "zero_chain_b200", "csrc"),
                           "-o", so, os.path.join(HERE, "host_emul", "emul_jubjub.cpp")])
    return C.CDLL(so)


def _w(*vals):
    return np.array([(v >> (32 * i)) & 0xFFFFFFFF for v in vals for i in range(8)], np.uint32)


def _int(a, k=0):
    return sum(int(x) << (32 * i) for i, x in enumerate(a[8 * k:8 * k + 8]))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _sqrt(emu, a):
    o = np.zeros(8, np.uint32)
    return _int(o) if emu.emu_jj_sqrt(_p(_w(a)), _p(o)) else None


def test_square_root(emu):
    rng = np.random.default_rng(5)
    rnd = [int.from_bytes(rng.bytes(32), "little") % R for _ in range(200)]
    omega = pow(7, (R - 1) >> 32, R)                             # order 2^32
    two_adic = [pow(omega, 1 << (32 - k), R) for k in range(33)]  # order 2^k, k = 0..32 (2^32: a non-residue)
    vals = [0, 1, R - 1, 2, 7, R - 7] + rnd + [x * x % R for x in rnd[:50]] + two_adic + [s * s * w % R for s, w in zip(rnd, two_adic)]
    for a in vals:
        got = _sqrt(emu, a)
        if jj.is_square(a):
            assert got is not None and got * got % R == a, a
        else:
            assert got is None, a
    assert _sqrt(emu, 0) == 0 and _sqrt(emu, 1) in (1, R - 1)
    assert _sqrt(emu, two_adic[32]) is None and _sqrt(emu, two_adic[31]) is not None   # the full-depth residue has a root
    assert _sqrt(emu, R - 1) is not None                          # -1 is a square (r = 1 mod 4)


def test_group_law(emu):
    pts = [jj.IDENTITY, jj.torsion_point(2), jj.torsion_point(4), jj.torsion_point(8)] + [jj.prime_order_point(s) for s in (3, 11, 99)]
    pts.append(jj.add(pts[4], pts[3]))                            # a point outside the prime-order subgroup
    zs = [1, 5, R - 2]
    o = np.zeros(16, np.uint32)
    for i, p in enumerate(pts):
        for j, q in enumerate(pts):
            zp, zq = zs[i % 3], zs[(i + j) % 3]
            assert emu.emu_jj_add(_p(_w(*p)), _p(_w(zp)), _p(_w(*q)), _p(_w(zq)), _p(o)) == 1
            assert (_int(o, 0), _int(o, 1)) == jj.add(p, q), (i, j)
        assert emu.emu_jj_dbl(_p(_w(*p)), _p(_w(zs[i % 3])), _p(o)) == 1
        assert (_int(o, 0), _int(o, 1)) == jj.add(p, p), i
    kills = [emu.emu_jj_order_kills(_p(_w(*p))) for p in pts]
    assert kills == [1, 0, 0, 0, 1, 1, 1, 0]


def _decode(emu, encs):
    n = len(encs)
    xy = np.zeros(16 * n, np.uint32)
    st = np.zeros(n, np.uint8)
    emu.emu_jj_into_xy(_p(np.frombuffer(b"".join(encs), np.uint8)), C.c_size_t(n), _p(xy), _p(st))
    return [(int(st[i]), _int(xy, 2 * i), _int(xy, 2 * i + 1)) for i in range(n)]


def test_decode_every_class(emu):
    rng = np.random.default_rng(9)
    good = [jj.prime_order_point(s) for s in range(1, 9)]
    encs = [jj.encode(p) for p in good]
    encs += [jj.encode(jj.neg(p)) for p in good[:3]]                             # the other sign
    encs += [bytes([1]) + bytes(31), bytes([1]) + bytes(30) + b"\x80"]           # identity, with and without the sign bit
    encs += [jj.encode(jj.torsion_point(k)) for k in (2, 4, 8)]                  # (0, -1) and friends
    encs += [jj.encode(jj.add(good[0], jj.torsion_point(k))) for k in (2, 4, 8)]   # P + T
    encs += [(R + k).to_bytes(32, "little") for k in (0, 1, 5)]                  # y >= r
    encs += [((1 << 255) - 1).to_bytes(32, "little"), b"\xff" * 32]
    encs += [rng.bytes(32) for _ in range(120)]
    got = _decode(emu, encs)
    want = [jj.into_xy(e) for e in encs]
    assert got == want
    classes = {s for s, _, _ in want}
    assert classes == {jj.OK, jj.NOT_IN_FIELD, jj.NOT_ON_CURVE, jj.NOT_PRIME_ORDER}
    assert got[len(good) + 3] == got[len(good) + 4] == (0, 0, 1)                # `01 00..00 80` is the identity too
