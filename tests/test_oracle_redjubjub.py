"""CPU checks of the RedJubjub oracles (tests/jubjub_oracle/redjubjub.py on pyref.py, and the C restatement in
redjubjub_oracle.c): the Alice key derivation pinned by the reference's address literal, the generator P_G against the committed
device constants, BLAKE2b against RFC 7693, the reference's own signature test properties, and the two oracles against each
other on a corpus that hits every verdict."""
import hashlib
import json
import os
import subprocess
import sys

import numpy as np

from tests.jubjub_oracle import rj_coracle as cj
from tests.jubjub_oracle import pyref as jj
from tests.jubjub_oracle import redjubjub as rj
from tests.jubjub_oracle import rj_corpus

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = json.load(open(os.path.join(HERE, "golden", "redjubjub.json")))
POINTS = json.load(open(os.path.join(HERE, "golden", "jubjub_points.json")))


def test_literals_match_the_oracle():
    p = GOLD["personalizations"]
    assert rj.GH_FIRST_BLOCK == GOLD["gh_first_block"]["text"].encode()
    assert rj.PH_PERSONALIZATION == p["pedersen_hash_generators"]["text"].encode()
    assert rj.H_STAR_PERSONALIZATION == p["h_star"]["text"].encode()
    assert rj.EXPAND_SEED_PERSONALIZATION == p["prf_expand"]["text"].encode()
    assert rj.BDK_PERSONALIZATION == p["crh_bdk"]["text"].encode()


def test_alice_address_pin():
    """EncryptionKey::from_seed(Alice seed) == pkd_addr_alice (modules/encrypted-balances/src/lib.rs:443): BLAKE2b-512 with a
    16-byte personalization, the 512-bit little-endian reduction, P_G, the point encoding, BLAKE2s "zech_bdk" and the
    five-bit drop, all fixed by one reference value."""
    seed = GOLD["alice_seed"]["text"].encode()
    want = next(e["hex"] for e in POINTS["transaction_points"] if e["name"] == "pkd_addr_alice")
    assert rj.encryption_key(seed).hex() == want


def test_generator_matches_device_constants():
    assert jj.encode(rj.P_G).hex().startswith("ac776c79") and rj.P_G_INDEX == 4
    assert jj.on_curve(rj.P_G) and jj.mul(rj.P_G, jj.R_J) == jj.IDENTITY and rj.P_G != jj.IDENTITY
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "gen_redjubjub_consts.py"), "--check"], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    src = open(os.path.join(ROOT, "zero_chain_b200", "csrc", "redjubjub_consts.inc")).read()
    words = lambda name: sum(int(w, 16) << (32 * i) for i, w in enumerate(src.split(name)[1].split("{")[1].split("}")[0].replace("u", "").split(",")))
    assert (words("RJ_PG_X[8]"), words("RJ_PG_Y[8]")) == rj.P_G


def test_blake2b_rfc7693():
    want = ("ba80a53f981c4d0d6a2797b69f12f6e94c212f14685ac4b74b12bb6fdbffa2d1"
            "7d87c5392aab792dc252d5de4533cc9518d38aa8dbf1925ab92386edd4009923")     # RFC 7693 Appendix A, BLAKE2b-512("abc")
    assert hashlib.blake2b(b"abc", digest_size=64).hexdigest() == want
    assert cj.blake2b(b"abc").hex() == want
    for n in rj_corpus.EDGE_LENGTHS + [383, 384, 385]:
        data = bytes((5 * i + 1) & 0xFF for i in range(n))
        assert cj.blake2b(data, rj.H_STAR_PERSONALIZATION) == hashlib.blake2b(data, digest_size=64, person=rj.H_STAR_PERSONALIZATION).digest()
        assert cj.h_star(data[:32].ljust(32, b"\x01"), data) == rj.h_star(data[:32].ljust(32, b"\x01"), data)


def test_reference_signature_properties():
    """redjubjub.rs tests, with the Diversifier generator: round trip, swapped messages fail, re-randomized keys verify, and
    vk + (a point of order 8) still verifies (cofactor_check)."""
    rng = np.random.default_rng(17)
    m1, m2 = [m["text"].encode() for m in GOLD["messages"]]
    t8 = jj.torsion_point(8)
    for _ in range(2):
        sk = int.from_bytes(rng.bytes(32), "little") % rj.R_J
        vk = rj.public_key(sk)
        s1, s2 = rj.sign(sk, m1, rng.bytes(80)), rj.sign(sk, m2, rng.bytes(80))
        assert rj.verify(vk, m1, s1) == rj.verify(vk, m2, s2) == rj.OK
        assert rj.verify(vk, m1, s2) == rj.verify(vk, m2, s1) == rj.BAD_EQUATION
        alpha = int.from_bytes(rng.bytes(32), "little") % rj.R_J
        rsk, rvk = (sk + alpha) % rj.R_J, rj.randomize_public_key(vk, alpha)
        assert rvk == rj.public_key(rsk)
        r1, r2 = rj.sign(rsk, m1, rng.bytes(80)), rj.sign(rsk, m2, rng.bytes(80))
        assert rj.verify(rvk, m1, r1) == rj.verify(rvk, m2, r2) == rj.OK
        assert rj.verify(rvk, m1, r2) == rj.verify(rvk, m2, r1) == rj.BAD_EQUATION
        _, a = jj.read(vk)
        assert rj.verify(jj.encode(jj.add(a, t8)), m1, s1) == rj.OK
        # the C oracle agrees on all of it
        vks = [vk] * 4 + [rvk] * 4 + [jj.encode(jj.add(a, t8))]
        sigs = [s1, s2, s2, s1, r1, r2, r2, r1, s1]
        msgs = [m1, m2, m1, m2, m1, m2, m1, m2, m1]
        assert list(cj.redjubjub_verify(b"".join(vks), b"".join(sigs), msgs)) == [1, 1, 0, 0, 1, 1, 0, 0, 1]
        assert cj.redjubjub_sign([sk], bytes(80), [m1]) == rj.sign(sk, m1, bytes(80))


def test_oracles_agree_on_mixed_corpus():
    entries, n_special = rj_corpus.mixed(len(rj_corpus.EDGE_LENGTHS) * 2, seed=3)
    vks, sigs, msgs = rj_corpus.columns(entries)
    got = [int(v) for v in cj.redjubjub_verify(vks, sigs, msgs)]
    want = [rj_corpus.python_verdict(e) for e in entries]
    assert got == want
    assert all(w == e[3] for w, e in zip(want, entries) if e[3] is not None)
    assert set(want) == {0, 1, 2, 3, 4}
    assert {len(m) for m, v in zip(msgs, want) if v == rj.OK} >= {0, 96, 97, 224, 225, 300}
