"""CPU check of the transaction-building oracles — the Python one (tests/jubjub_oracle/tx_build.py) and the C one
(tx_build_oracle.c through tx_coracle.py) — against the reference's literals in tests/golden/tx_build.json (Alice's
encryption key, GEpoch::group_hash(0) at tag byte 1, the nonce Alice's dk makes with GEpoch(0), the literal ciphertext
decrypting to 10 under Alice's dk) and against each other: BLAKE2s, keys, group hashes with their tags, the confidential
fields of edge and random rows, and signatures."""
import hashlib
import json
import os

import numpy as np

from tests.jubjub_oracle import elgamal as eg
from tests.jubjub_oracle import pyref as jj
from tests.jubjub_oracle import redjubjub as rj
from tests.jubjub_oracle import rj_coracle as cj
from tests.jubjub_oracle import tx_build as tb
from tests.jubjub_oracle import tx_coracle as tc

GOLD = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tx_build.json")))


def test_known_answers():
    sk, dk, ek = tb.keys(GOLD["alice_seed"].encode())
    assert ek.hex() == GOLD["alice_encryption_key"]["value"]
    assert tb.g_epoch(0) == (bytes.fromhex(GOLD["g_epoch_0"]["value"]), 1)
    assert tb.g_epoch(1) == (bytes.fromhex(GOLD["g_epoch_1"]["value"]), 1)
    assert tb.g_epoch(2)[1] == 7
    g = jj.read(bytes.fromhex(GOLD["g_epoch_0"]["value"]))[1]
    assert jj.encode(jj.mul(g, int.from_bytes(dk, "little"))).hex() == GOLD["alice_nonce"]["value"]
    ct = bytes.fromhex(GOLD["enc10_by_alice"]["value"]) + bytes.fromhex(GOLD["randomness"]["value"])
    assert eg.decrypt_bytes(dk, ct, bound=20) == (eg.OK, 10)


def test_fields_rows_are_consistent():
    """rvk is rsk P_G, the ciphertexts decrypt under the two keys, and a bad recipient key zeroes its row"""
    ek_r = tb.keys(b"Bob" + b" " * 29)
    g = tb.g_epoch(0)[0]
    f, rsk, dk, st = tb.confidential_fields(1234, ek_r[2], 42, 3, 99, 77, g)
    assert st == jj.OK and f[6 * 32:7 * 32] == rj.public_key(int.from_bytes(rsk, "little"))
    assert eg.decrypt_bytes(dk, f[64:96] + f[160:192], bound=50) == (eg.OK, 42)
    assert eg.decrypt_bytes(ek_r[1], f[96:128] + f[160:192], bound=50) == (eg.OK, 42)
    assert eg.decrypt_bytes(dk, f[128:160] + f[160:192], bound=50) == (eg.OK, 3)
    for key, status in tb.bad_recipient_keys():
        assert tb.confidential_fields(1, key, 1, 1, 1, 1, g) == (bytes(288), bytes(32), bytes(32), status)


def test_c_oracle_known_answers():
    sks, dks, eks = tc.keys([GOLD["alice_seed"].encode()])
    assert eks[0].hex() == GOLD["alice_encryption_key"]["value"]
    (g0, t0), (g1, t1), (_, t2) = tc.g_epoch([0, 1, 2])
    assert (g0.hex(), t0, t1, t2) == (GOLD["g_epoch_0"]["value"], 1, 1, 7)
    assert g1.hex() == GOLD["g_epoch_1"]["value"]              # the Python oracle's value, restated independently
    ek_bob = tc.keys([b"Bob" + b" " * 29])[2][0]
    f = tc.confidential_fields(sks[0], ek_bob, [10], [1], (5).to_bytes(32, "little"), (7).to_bytes(32, "little"), g0)[0][0]
    assert f[256:288].hex() == GOLD["alice_nonce"]["value"]


def test_blake2s_agrees():
    rng = np.random.default_rng(5)
    for n in (0, 1, 31, 32, 33, 63, 64, 65, 69, 127, 128, 129, 300):
        m = rng.bytes(n)
        for person in (b"zech_bdk", b"zcgepoch"):
            assert tc.blake2s(m, person) == hashlib.blake2s(m, digest_size=32, person=person).digest(), n


def test_keys_agree():
    seeds = [b"", b"a", bytes(range(127)), bytes(128), bytes(range(129)) + b"x" * 200] + [b"seed %d" % i for i in range(10)]
    sks, dks, eks = tc.keys(seeds)
    assert list(zip(sks, dks, eks)) == [tb.keys(s) for s in seeds]


def test_g_epochs_agree():
    epochs = list(range(65)) + [2 ** 31, 2 ** 32 - 1]
    assert tc.g_epoch(epochs) == [tb.g_epoch(e) for e in epochs]


def test_fields_agree():
    rows = tb.edge_rows() + tb.random_rows(12, seed=17)
    g = tb.g_epoch(6)[0]
    sc = lambda v: b"".join(x.to_bytes(32, "little") for x in v)
    sks, eks, amounts, fees, rs, alphas = zip(*rows)
    assert tc.confidential_fields(sc(sks), b"".join(eks), amounts, fees, sc(rs), sc(alphas), g) == [tb.confidential_fields(*r, g) for r in rows]


def test_signatures_agree():
    rng = np.random.default_rng(8)
    lengths = [0, 1, 47, 48, 49, 127, 128, 129]
    sks = [int.from_bytes(rng.bytes(64), "little") % rj.R_J for _ in lengths]
    ts, msgs = [rng.bytes(80) for _ in lengths], [rng.bytes(n) for n in lengths]
    sigs = cj.redjubjub_sign(sks, b"".join(ts), msgs)
    assert [sigs[64 * i:64 * i + 64] for i in range(len(lengths))] == [rj.sign(k, m, t) for k, m, t in zip(sks, msgs, ts)]
