"""GPU tests of zk_jubjub_msm: the sum equals the closed form (bases k_i P_G, result (sum s_i k_i mod r_J) P_G) for
n in {1, 2, 3, 100, 4097, 2^17 + 5}, and the Python oracle's naive multiexp with zero scalars, r_J - 1, repeated points,
the identity, small-order and non-prime-order points; every bucket of a window hit, one very heavy bucket; argument,
decode and canonical errors."""
import ctypes as C

import numpy as np
import pytest

from tests.jubjub_oracle import pyref as jj
from tests.jubjub_oracle import redjubjub as rj
from tests.jubjub_oracle import rj_batch as rjb
from tests.jubjub_oracle import rj_coracle as cj
from zero_chain_b200 import _lib
from zero_chain_b200 import groth16 as zk

pytestmark = pytest.mark.gpu
R_J = rj.R_J


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


def _sb(scalars) -> bytes:
    return b"".join(int(s).to_bytes(32, "little") for s in scalars)


def _closed_form(ks, ss) -> bytes:
    return cj.redjubjub_public_key([sum(int(k) * int(s) for k, s in zip(ks, ss)) % R_J])


@pytest.mark.parametrize("n", [1, 2, 3, 100, 4097, (1 << 17) + 5])
def test_closed_form(ctx, n):
    rng = np.random.default_rng(n)
    ks = [int.from_bytes(rng.bytes(32), "little") % R_J for _ in range(n)]
    ss = [int.from_bytes(rng.bytes(32), "little") % R_J for _ in range(n)]
    ss[0] = R_J - 1
    if n > 2:
        ss[1] = 0
        ks[2] = ks[0]                                     # a repeated point
    pts = cj.redjubjub_public_key(ks)
    assert zk.jubjub_msm(ctx, pts, _sb(ss)) == _closed_form(ks, ss)


def test_oracle_with_torsion_and_identity(ctx):
    rng = np.random.default_rng(5)
    t8, t4, t2 = jj.torsion_point(8), jj.torsion_point(4), jj.torsion_point(2)
    pts = [rj.P_G, jj.IDENTITY, t8, t4, t2, jj.add(rj.P_G, t8), jj.add(jj.mul(rj.P_G, 12345), t4)]
    pts += [jj.mul(rj.P_G, int.from_bytes(rng.bytes(32), "little") % R_J) for _ in range(20)]
    pts += [jj.add(pts[-1], t8), pts[-2], pts[-2]]
    ss = [int.from_bytes(rng.bytes(32), "little") % R_J for _ in pts]
    ss[1], ss[3], ss[-1] = 0, R_J - 1, R_J - 1
    for s_list in (ss, [R_J - 1] * len(pts), [0] * len(pts), [1] * len(pts), [8] * len(pts)):
        want = jj.encode(rjb.multiexp(pts, s_list))
        assert zk.jubjub_msm(ctx, [jj.encode(p) for p in pts], _sb(s_list)) == want


def test_every_bucket_and_one_heavy_bucket(ctx):
    # 4097 points: 8-bit windows, 128 buckets each.  Scalars whose every window digit runs over all of 1..128 and their
    # negatives (the carry makes digits above 128 negative), so every bucket of every window is hit from both signs.
    n = 4097
    ks = list(range(1, n + 1))
    pts = cj.redjubjub_public_key(ks)
    ss = []
    for i in range(n):
        d = i % 256
        s = sum(d << (8 * w) for w in range(31))
        ss.append(s % R_J)
    assert zk.jubjub_msm(ctx, pts, _sb(ss)) == _closed_form(ks, ss)
    # one bucket with every entry: the same small scalar for 2^15 points (runs folded by a warp)
    n = 1 << 15
    ks = [int(k) for k in np.random.default_rng(8).integers(1, 1 << 62, n)]
    pts = cj.redjubjub_public_key(ks)
    for s in (1, 77, R_J - 1):
        assert zk.jubjub_msm(ctx, pts, _sb([s] * n)) == _closed_form(ks, [s] * n)


def test_errors(ctx):
    L = _lib.lib()
    pts = cj.redjubjub_public_key([3, 5, 7])
    out = np.zeros(32, np.uint8)
    sc = np.frombuffer(_sb([1, 2, 3]), np.uint8)
    pb = np.frombuffer(pts, np.uint8)
    assert zk.jubjub_msm(ctx, [], []) == jj.encode(jj.IDENTITY)
    assert L.zk_jubjub_msm(ctx._h, 0, None, None, out.ctypes.data) == 0
    assert L.zk_jubjub_msm(None, 3, pb.ctypes.data, sc.ctypes.data, out.ctypes.data) == -2
    assert L.zk_jubjub_msm(ctx._h, 3, None, sc.ctypes.data, out.ctypes.data) == -2
    assert L.zk_jubjub_msm(ctx._h, 3, pb.ctypes.data, None, out.ctypes.data) == -2
    assert L.zk_jubjub_msm(ctx._h, 3, pb.ctypes.data, sc.ctypes.data, None) == -2
    bad_sc = np.frombuffer(_sb([1, R_J, 3]), np.uint8)
    assert L.zk_jubjub_msm(ctx._h, 3, pb.ctypes.data, bad_sc.ctypes.data, out.ctypes.data) == -8
    assert "scalar 1" in L.zk_last_error().decode()
    off_curve = 2
    while jj.point_for_y(off_curve) is not None:
        off_curve += 1
    bad_pts = np.frombuffer(pts[:64] + off_curve.to_bytes(32, "little"), np.uint8)
    assert L.zk_jubjub_msm(ctx._h, 3, bad_pts.ctypes.data, sc.ctypes.data, out.ctypes.data) == -7
    assert "point 2" in L.zk_last_error().decode()
    not_in_field = np.frombuffer(pts[:32] + jj.R.to_bytes(32, "little") + pts[64:], np.uint8)
    assert L.zk_jubjub_msm(ctx._h, 3, not_in_field.ctypes.data, sc.ctypes.data, out.ctypes.data) == -7
    assert "point 1" in L.zk_last_error().decode()
    # the context still computes
    assert zk.jubjub_msm(ctx, pts, _sb([1, 2, 3])) == _closed_form([3, 5, 7], [1, 2, 3])
