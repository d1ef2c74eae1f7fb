"""CPU checks of the two Jubjub oracles (tests/jubjub_oracle: the Python integer restatement and the C one on the oracle's Fr
code) against the reference's own literals (tests/golden/jubjub_points.json) and against each other."""
import json
import os

import numpy as np
import pytest

from tests.jubjub_oracle import coracle as cj
from tests.jubjub_oracle import pyref as jj

GOLD = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jubjub_points.json")))
R = jj.R


def _c(encs):
    xy, st = cj.into_xy(b"".join(encs))
    return [(int(st[i]), sum(int(v) << (64 * k) for k, v in enumerate(xy[i, 0])), sum(int(v) << (64 * k) for k, v in enumerate(xy[i, 1])))
            for i in range(len(encs))]


def test_curve_constants():
    assert not jj.is_square(jj.D)                                   # the addition law is complete
    assert jj.is_square(R - 1)                                      # a = -1 is a square
    g = jj.prime_order_point(1)
    assert jj.on_curve(g) and jj.mul(g, jj.R_J) == jj.IDENTITY and jj.mul(g, jj.R_J - 1) == jj.neg(g)
    assert jj.mul(jj.torsion_point(8), 8) == jj.IDENTITY and jj.mul(jj.torsion_point(8), 4) != jj.IDENTITY


def test_reference_literals():
    """modules/encrypted-balances/src/lib.rs:407, 443-450: every transaction point decodes and is of prime order.
    core/jubjub/src/curve/mod.rs:424-444: both read vectors decode to the y at :428 with opposite x parity, on the curve,
    but outside the prime-order subgroup."""
    encs = [bytes.fromhex(e["hex"]) for e in GOLD["transaction_points"]]
    assert len(encs) == 9
    want = [jj.into_xy(e) for e in encs]
    assert [w[0] for w in want] == [jj.OK] * 9
    for e, (_, x, y) in zip(encs, want):
        assert jj.on_curve((x, y)) and jj.encode((x, y)) == e       # write(read(e)) == e
    assert _c(encs) == want
    y = int(GOLD["read_vectors_y"]["decimal"])
    reads = [bytes.fromhex(e["hex"]) for e in GOLD["read_vectors"]]
    pts = [jj.read(e) for e in reads]
    assert [s for s, _ in pts] == [jj.OK, jj.OK]
    assert pts[0][1][1] == pts[1][1][1] == y
    assert pts[0][1][0] & 1 == 0 and pts[1][1][0] & 1 == 1 and pts[0][1] == jj.neg(pts[1][1])
    assert [jj.into_xy(e) for e in reads] == _c(reads) == [(jj.NOT_PRIME_ORDER, 0, 0)] * 2


def test_special_points():
    ident = bytes([1]) + bytes(31)
    ident_signed = bytes([1]) + bytes(30) + b"\x80"
    two = jj.encode(jj.torsion_point(2))                            # (0, -1)
    assert jj.torsion_point(2) == (0, R - 1)
    p = jj.prime_order_point(7)
    encs = [ident, ident_signed, two] + [jj.encode(jj.add(p, jj.torsion_point(k))) for k in (2, 4, 8)] + [jj.encode(p)]
    want = [(0, 0, 1), (0, 0, 1)] + [(jj.NOT_PRIME_ORDER, 0, 0)] * 4 + [(0, p[0], p[1])]
    assert [jj.into_xy(e) for e in encs] == want
    assert _c(encs) == want


def test_square_roots_agree():
    rng = np.random.default_rng(3)
    vals = [0, 1, R - 1, 7] + [int.from_bytes(rng.bytes(32), "little") % R for _ in range(100)]
    for a in vals:
        p, c = jj.sqrt(a), cj.sqrt(a)
        assert (p is None) == (c is None) == (not jj.is_square(a))
        if c is not None:
            assert c * c % R == a and p * p % R == a


def test_oracles_agree_on_random_encodings():
    rng = np.random.default_rng(11)
    encs = [rng.bytes(32) for _ in range(1700)]
    encs += [jj.encode(jj.prime_order_point(int.from_bytes(rng.bytes(32), "little"))) for _ in range(250)]
    encs += [(R + int(rng.integers(0, 1 << 40))).to_bytes(32, "little") for _ in range(50)]
    want = [jj.into_xy(e) for e in encs]
    assert _c(encs) == want
    counts = np.bincount([w[0] for w in want], minlength=4)
    assert all(counts > 40), counts
