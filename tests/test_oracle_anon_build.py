"""CPU check of the anonymous transfer's oracles — the Python one (tests/jubjub_oracle/tx_build.py, anonymous_fields) and
the C one (tx_build_oracle.c through tx_coracle.py): they agree on edge and random rows; the ring order is gen_proof's
for all 132 (s, t) pairs; every status comes out where it should; and the rows decrypt as neg_encrypt / encrypt /
encrypt(0) must.  The reference has no literal anonymous transfer (its tests draw r from an RNG), so these are the
semantics restated from anonymous.rs and crypto_components.rs; the GPU tests tie them to the module's import."""
import numpy as np

from tests.jubjub_oracle import anon_build as ab
from tests.jubjub_oracle import anon_build_coracle as abc
from tests.jubjub_oracle import elgamal as eg
from tests.jubjub_oracle import pyref as jj
from tests.jubjub_oracle import redjubjub as rj
from tests.jubjub_oracle import tx_build as tb

sc = lambda v: b"".join(x.to_bytes(32, "little") for x in v)


def _c_rows(table, rows, g):
    sks, rings, s, t, amounts, rs, alphas = zip(*rows)
    return abc.anonymous_fields(b"".join(table), sc(sks), rings, list(zip(s, t)), amounts, sc(rs), sc(alphas), g)


def test_edge_and_random_rows_agree():
    table = ab.key_table()
    rows = ab.edge_rows() + ab.random_rows(6, len(table) - 5, seed=3)   # random rings over the valid keys
    g = tb.g_epoch(4)[0]
    want = [ab.anonymous_fields(table, *r, g) for r in rows]
    assert _c_rows(table, rows, g) == want
    st = [w[3] for w in want]
    assert {0, 1, 2, 3, ab.ANON_BAD_INDEX, ab.ANON_BAD_POSITIONS} <= set(st)
    for w in want:
        if w[3]:
            assert w[:3] == (bytes(864), bytes(32), bytes(32))


def test_statuses_and_their_precedence():
    table = ab.key_table()
    g = tb.g_epoch(0)[0]
    base = list(range(11))
    row = lambda ring, s, t: ab.anonymous_fields(table, 5, ring, s, t, 1, 2, 3, g)[3]
    for k, (_, code) in enumerate(tb.bad_recipient_keys()):
        assert row([15 + k] + base[1:], 0, 1) == code                         # the recipient's key
        assert row(base[:9] + [15 + k] + base[10:], 0, 1) == code             # a decoy's key
    assert row([0, 1, 16, 3, 4, 5, 6, 15, 8, 9, 10], 0, 1) == jj.NOT_ON_CURVE   # the first failing key in ring order
    assert row(base[:10] + [len(table)], 0, 1) == ab.ANON_BAD_INDEX
    assert row([15] + base[1:10] + [len(table)], 0, 1) == ab.ANON_BAD_INDEX     # an index before a key code
    for s, t in ((3, 3), (12, 0), (0, 12), (255, 11)):
        assert row(base, s, t) == ab.ANON_BAD_POSITIONS
    assert row([len(table)] + base[1:], 5, 5) == ab.ANON_BAD_POSITIONS           # positions before an index
    assert abc.anonymous_fields(b"", sc([5]), [base], [(0, 1)], [1], sc([2]), sc([3]), g)[0] == (bytes(864), bytes(32), bytes(32),
                                                                                                 ab.ANON_BAD_INDEX)   # n_keys = 0


def test_ring_order_for_every_position_pair():
    """one row placed at each of the 132 (s, t) pairs: the sender's key and ciphertext at s, the recipient's at t, the
    decoys' on the other positions in their order; gen_proof's inserts (the Python oracle) give the same"""
    table = ab.key_table()[:14]
    ring = [13] + list(range(10))
    g = tb.g_epoch(2)[0]
    pairs = [(s, t) for s in range(12) for t in range(12) if s != t]
    assert len(pairs) == 132
    sk, amount, r, alpha = 4321, 17, 999, 5
    out = abc.anonymous_fields(b"".join(table), sc([sk] * 132), [ring] * 132, pairs, [amount] * 132, sc([r] * 132), sc([alpha] * 132), g)
    ref = out[pairs.index((0, 1))][0]
    ek_s, left_s, left_t = ref[:32], ref[384:416], ref[416:448]
    decoy_keys = [ref[32 * p:32 * p + 32] for p in range(2, 12)]
    decoy_lefts = [ref[384 + 32 * p:416 + 32 * p] for p in range(2, 12)]
    assert decoy_keys == [table[k] for k in ring[1:]] and ref[32:64] == table[13]
    assert ek_s == jj.encode(jj.mul(rj.P_G, int.from_bytes(out[0][2], "little")))
    for (s, t), (f, rsk, dk, st) in zip(pairs, out):
        assert st == 0
        others = [p for p in range(12) if p not in (s, t)]
        assert f[32 * s:32 * s + 32] == ek_s and f[384 + 32 * s:416 + 32 * s] == left_s
        assert f[32 * t:32 * t + 32] == table[13] and f[384 + 32 * t:416 + 32 * t] == left_t
        assert [f[32 * p:32 * p + 32] for p in others] == decoy_keys
        assert [f[384 + 32 * p:416 + 32 * p] for p in others] == decoy_lefts
        assert f[768:] == ref[768:] and rsk == out[0][1] and dk == out[0][2]
    for s, t in ((0, 1), (1, 0), (5, 2), (11, 10), (3, 9)):
        assert ab.anonymous_fields(table, sk, ring, s, t, amount, r, alpha, g) == out[pairs.index((s, t))]


def test_rows_decrypt():
    """left_s with right decrypts to -amount under the sender's dk, left_t to amount under the recipient's, each decoy's to
    0 under its own; rvk is rsk P_G"""
    seeds = [b"ring member %d" % i for i in range(12)]
    keys = [tb.keys(s) for s in seeds]
    table = [k[2] for k in keys]
    g = tb.g_epoch(1)[0]
    sk = rj.spending_key(b"sender")
    ring, s, t = [3, 0, 1, 2, 4, 5, 6, 7, 8, 9, 10], 6, 2
    f, rsk, dk, st = ab.anonymous_fields(table, sk, ring, s, t, 42, 12345, 678, g)
    assert st == 0
    right = f[768:800]
    assert eg.decrypt_bytes(keys[3][1], f[384 + 32 * t:416 + 32 * t] + right, bound=50) == (eg.OK, 42)
    v = eg.v_point(eg.read(f[384 + 32 * s:416 + 32 * s] + right)[1], int.from_bytes(dk, "little"))
    assert v == jj.neg(jj.mul(rj.P_G, 42))
    others = [p for p in range(12) if p not in (s, t)]
    for p, k in zip(others, ring[1:]):
        assert eg.decrypt_bytes(keys[k][1], f[384 + 32 * p:416 + 32 * p] + right, bound=2) == (eg.OK, 0)
    assert f[800:832] == rj.public_key(int.from_bytes(rsk, "little"))


def test_random_rows_agree():
    rng = np.random.default_rng(12)
    table = [tb.keys(b"k %d" % i)[2] for i in range(24)]
    rows = ab.random_rows(10, 24, seed=int(rng.integers(1 << 30)))
    g = tb.g_epoch(7)[0]
    assert _c_rows(table, rows, g) == [ab.anonymous_fields(table, *r, g) for r in rows]
