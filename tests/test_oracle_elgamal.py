"""CPU checks of the ElGamal oracles (tests/jubjub_oracle/elgamal.py on pyref.py and redjubjub.py, and the C restatement in
elgamal_oracle.c) against each other and against the golden facts in tests/golden/elgamal.json: the reference's transaction
literals and genesis balances, the reference's own ElGamal test properties, the bound, and every status class."""
import json
import os

import numpy as np

from tests.jubjub_oracle import eg_coracle as ec
from tests.jubjub_oracle import eg_corpus
from tests.jubjub_oracle import elgamal as eg
from tests.jubjub_oracle import pyref as jj

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "elgamal.json")))
POINTS = {e["name"]: bytes.fromhex(e["hex"]) for e in json.load(open(os.path.join(HERE, "golden", "jubjub_points.json")))["transaction_points"]}
ALICE_SEED = json.load(open(os.path.join(HERE, "golden", "redjubjub.json")))["alice_seed"]["text"].encode()
AMOUNTS = GOLD["test_amounts"]


def _c(dks, cts, pds=None):
    st, val = ec.decrypt(b"".join(dks), b"".join(cts), None if pds is None else b"".join(pds))
    return [int(x) for x in st], [int(x) for x in val]


def _key(rng):
    return int.from_bytes(rng.bytes(32), "little") % jj.R_J


def test_bound_and_bob_seed():
    assert GOLD["bound"]["value"] == eg.BOUND == 1_000_000
    dk, ek = eg.account_keys(GOLD["bob_seed"]["text"].encode())
    assert jj.encode(ek) == POINTS["pkd_addr_bob"]
    assert jj.encode(eg.account_keys(ALICE_SEED)[1]) == POINTS["pkd_addr_alice"]


def test_reference_literals():
    """modules/encrypted-balances/src/lib.rs:443-448: the amounts of the reference's own transaction, and None for Bob's
    ciphertext under Alice's key (the full walk, so only the C oracle)."""
    keys = {"alice": eg.account_keys(ALICE_SEED)[0], "bob": eg.account_keys(GOLD["bob_seed"]["text"].encode())[0]}
    lit = GOLD["literal_decryptions"]
    dks = [eg.key_bytes(keys[d["key"]]) for d in lit]
    cts = [POINTS[d["left"]] + POINTS[d["right"]] for d in lit]
    want = [d["value"] for d in lit]
    assert want == [10, 1, 10, None]
    for dk, ct, w in zip(dks, cts, want):
        if w is not None:
            assert eg.decrypt_bytes(dk, ct, bound=w + 5) == (eg.OK, w)
    assert _c(dks, cts) == ([0, 0, 0, 1], [10, 1, 10, 0])


def test_genesis_balances():
    """Both genesis balances use randomness Fs::one(): (amount P_G + ek, P_G)."""
    dk, ek = eg.account_keys(ALICE_SEED)
    for g in GOLD["genesis"]:
        assert g["randomness"] == "Fs::one()"
        ct = eg.encrypt(g["value"], 1, ek)
        assert ct[1] == eg.P_G
        assert eg.decrypt(ct, dk) == g["value"]
        assert _c([eg.key_bytes(dk)], [eg.write(ct)]) == ([0], [g["value"]])
    assert [g["value"] for g in GOLD["genesis"]] == [10_000, 100]


def test_reference_elgamal_properties():
    """elgamal.rs:198-340: the round trip, Alice's seed, 20 - 13 = 7, 15 + 4 = 19 with add == add_no_params, a wrong key
    (the reference's should_panic: None), and the read / write round trip."""
    rng = np.random.default_rng(23)
    sk, r1, r2 = _key(rng), _key(rng), _key(rng)
    ek = jj.mul(eg.P_G, sk)
    a = AMOUNTS
    assert eg.decrypt(eg.encrypt(a["enc_dec"]["value"], r1, ek), sk) == 5
    dk_alice, ek_alice = eg.account_keys(ALICE_SEED)
    assert eg.decrypt(eg.encrypt(a["enc_dec_ivk"]["value"], r1, ek_alice), dk_alice) == 100
    x20, x13, x7 = [v["value"] for v in a["homomorphic_sub"]]
    d = eg.sub(eg.encrypt(x20, r1, ek), eg.encrypt(x13, r2, ek))
    assert eg.decrypt(d, sk) == x7 == 7
    x15, x4, x19 = [v["value"] for v in a["add_no_params"]]
    s = eg.add(eg.encrypt(x15, r1, ek), eg.encrypt(x4, r2, ek))
    assert eg.decrypt(s, sk) == x19 == 19
    # add_no_params is the same group law: the C oracle's encryptions, added as points, give the same ciphertext
    c15, c4 = ec.encrypt([x15, x4], [r1, r2], jj.encode(ek) * 2)[:64], ec.encrypt([x4], [r2], jj.encode(ek))
    assert eg.write(eg.add(eg.read(c15)[1], eg.read(c4)[1])) == eg.write(s)
    sk2 = _key(rng)
    wrong = eg.sub(eg.encrypt(x20, r1, ek), eg.encrypt(x13, r2, jj.mul(eg.P_G, sk2)))
    assert _c([eg.key_bytes(sk)], [eg.write(wrong)]) == ([1], [0])
    ct = eg.encrypt(a["read_write"]["value"], r1, ek)
    ok, back = eg.read(eg.write(ct))
    assert ok and back == ct and eg.decrypt(back, sk) == 6


def test_bounds():
    rng = np.random.default_rng(29)
    sk = _key(rng)
    ek = jj.encode(jj.mul(eg.P_G, sk))
    amounts = [999_999, 1_000_000, 2 ** 32 - 1, 0, 1]
    cts = ec.encrypt(amounts, [_key(rng) for _ in amounts], ek * len(amounts))
    neg = ec.encrypt([5], [_key(rng)], ek, neg=True)
    k = eg.key_bytes(sk)
    st, val = _c([k] * 7, [cts, neg, eg.write(eg.ZERO)])
    assert (st, val) == ([0, 1, 1, 0, 0, 1, 0], [999_999, 0, 0, 0, 1, 0, 0])
    # the C encryptions are the Python oracle's
    r = _key(rng)
    assert ec.encrypt([77], [r], ek) == eg.write(eg.encrypt(77, r, jj.mul(eg.P_G, sk)))
    assert ec.encrypt([77], [r], ek, neg=True) == eg.write(eg.neg_encrypt(77, r, jj.mul(eg.P_G, sk)))


def test_every_status_class():
    """dk >= r_J; y >= r, a non-square and a torsion component in the left and in the right point of the balance and of the
    pending transfer; and the precedence among them.  Both oracles against the intended statuses."""
    entries = eg_corpus.special_entries(31) + eg_corpus.random_entries(24, seed=32)
    dks, cts, pds, want_null, want_pend = eg_corpus.columns(entries)
    assert set(want_pend[0]) == {0, 1, 2, 3, 4}
    st, val = ec.decrypt(dks, cts, pds)
    assert ([int(x) for x in st], [int(x) for x in val]) == want_pend
    st, val = ec.decrypt(dks, cts)
    assert ([int(x) for x in st], [int(x) for x in val]) == want_null
    for e in entries:
        for pend, want in ((None, e[3]), (e[2], e[4])):
            s, _ = eg.stage(e[0], e[1], pend)
            assert s == (want[0] if want[0] >= 2 else eg.OK)
            if want[0] == eg.OK and want[1] < 50:
                assert eg.decrypt_bytes(e[0], e[1], pend, bound=60) == want
