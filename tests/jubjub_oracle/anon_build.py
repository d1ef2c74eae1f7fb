"""TEST INFRASTRUCTURE (oracle): the sender side of an anonymous transfer, restated with Python integers on pyref.py,
redjubjub.py, elgamal.py and tx_build.py (key derivation, g_epoch), in the byte layout of zk_anonymous_fields_batch
(include/zkb200.h).

  anonymous_fields   MultiCiphertexts::<Anonymous>::encrypt (neg_encrypt for the sender, encrypt for the recipient,
                     encrypt(0) for each decoy; core/proofs/src/crypto_components.rs:168-216) and gen_proof's two list
                     inserts of the sender and the recipient into the decoys (core/proofs/src/anonymous.rs:97-145), with
                     rvk = pgk + alpha P_G and nonce = dk g_epoch, every point computed the reference's way
  key_table, edge_rows, random_rows   the rows the tests run it on"""
from __future__ import annotations

import numpy as np

from . import elgamal as eg
from . import pyref as jj
from . import redjubjub as rj
from .tx_build import bad_recipient_keys, keys

RING = 12
N_ANON_FIELDS = 2 * RING + 3
ANON_BAD_INDEX, ANON_BAD_POSITIONS = 4, 5


def _ring_insert(decoys: list, s: int, t: int, sender, recipient) -> list:
    """gen_proof's two Vec::insert calls (anonymous.rs:118-125 and 138-145), in its order"""
    v = list(decoys)
    if s < t:
        v.insert(s, sender)
        v.insert(t, recipient)
    else:
        v.insert(t, recipient)
        v.insert(s, sender)
    return v


def anonymous_fields(keys: list, sk: int, ring, s: int, t: int, amount: int, r: int, alpha: int, g_epoch_enc: bytes):
    """(fields, rsk, dk, status) of one row of zk_anonymous_fields_batch: keys the table of 32-byte encryption keys, ring
    the 11 indices into it (recipient, then the ten decoys), s / t the sender's and recipient's positions.  fields: the
    27 encodings enc_keys[12] | left_ciphertexts[12] | right_ciphertext | rvk | nonce.  The recipient's and the decoys'
    enc_keys are the table's bytes.  Status ANON_BAD_POSITIONS, then ANON_BAD_INDEX, then the zk_jubjub_into_xy code of
    the first key in ring order that fails EncryptionKey::read; a non-zero status gives zeros."""
    zero = (bytes(32 * N_ANON_FIELDS), bytes(32), bytes(32))
    if s >= RING or t >= RING or s == t:
        return zero + (ANON_BAD_POSITIONS,)
    if any(k >= len(keys) for k in ring):
        return zero + (ANON_BAD_INDEX,)
    pts = []
    for k in ring:
        st, x, y = jj.into_xy(keys[k])
        if st != jj.OK:
            return zero + (st,)
        pts.append((x, y))
    pgk = rj.proof_generation_key(sk)
    dk = rj.decryption_key(pgk)
    ek_s = jj.mul(rj.P_G, dk)
    sender, right = eg.neg_encrypt(amount, r, ek_s)
    recipient = eg.encrypt(amount, r, pts[0])[0]
    decoys = [eg.encrypt(0, r, p)[0] for p in pts[1:]]
    enc_keys = _ring_insert([keys[k] for k in ring[1:]], s, t, jj.encode(ek_s), keys[ring[0]])
    lefts = _ring_insert([jj.encode(c) for c in decoys], s, t, jj.encode(sender), jj.encode(recipient))
    rvk = jj.add(pgk, jj.mul(rj.P_G, alpha))
    nonce = jj.mul(jj.read(g_epoch_enc)[1], dk)
    fields = b"".join(enc_keys + lefts + [jj.encode(right), jj.encode(rvk), jj.encode(nonce)])
    return fields, rj.scalar_bytes((sk + alpha) % rj.R_J), rj.scalar_bytes(dk), jj.OK


def key_table() -> list:
    """a key table for the anonymous edge rows: 14 derived keys, the identity, then each failing key of
    bad_recipient_keys"""
    return [keys(b"ring member %d" % i)[2] for i in range(14)] + [jj.encode(jj.IDENTITY)] + [k for k, _ in bad_recipient_keys()]


def edge_rows() -> list:
    """(sk, ring, s, t, amount, r, alpha) rows at the edges, over key_table() with the sender's own key as key 13:
    the (s, t) pairs (0, 1), (1, 0), (0, 11), (11, 0) and (10, 11); r = 0; amounts 0 and 2^32 - 1; alpha = r_J - sk; the
    recipient equal to the sender; the identity as a decoy; a decoy listed twice; each failing key at the recipient's
    entry and at a decoy's, and two at once (the first in ring order wins); an index >= n_keys; s = t; s = 12; t = 12; and
    the precedence of positions over indices over keys"""
    sk_self = rj.spending_key(b"ring member 13")
    top = 2 ** 32 - 1
    base = list(range(11))
    rows = [(77, base, 0, 1, 5, 9, 11), (78, base, 1, 0, 6, 10, 12), (79, base, 0, 11, 7, 11, 13), (80, base, 11, 0, 8, 12, 14),
            (81, base, 10, 11, 9, 13, 15), (82, base, 3, 7, 10, 0, 16), (83, base, 5, 2, 0, 14, 17), (84, base, 6, 9, top, rj.R_J - 1, 18),
            (85, base, 4, 8, 11, 15, rj.R_J - 85), (0, base, 2, 3, 1, 1, 0), (rj.R_J - 1, base, 9, 1, top, rj.R_J - 1, rj.R_J - 1),
            (sk_self, [13] + base[1:], 7, 2, 12, 16, 19),
            (86, [0, 1, 2, 14, 4, 5, 6, 7, 8, 9, 10], 2, 9, 13, 17, 20),
            (87, [0, 1, 2, 3, 4, 5, 3, 7, 8, 3, 10], 8, 4, 14, 18, 21)]
    for k in range(4):
        rows.append((88 + k, [15 + k] + base[1:], 1, 2, 1, 2, 3))
        rows.append((92 + k, base[:5] + [15 + k] + base[6:], 11, 10, 1, 2, 3))
    rows += [(96, [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 19], 0, 1, 1, 2, 3), (97, base, 4, 4, 1, 2, 3), (98, base, 12, 0, 1, 2, 3),
             (99, base, 0, 12, 1, 2, 3), (100, [2 ** 32 - 1] + base[1:], 12, 12, 1, 2, 3), (101, [15] + base[1:5] + [19] + base[6:], 3, 4, 1, 2, 3),
             (102, [0, 1, 16, 3, 4, 5, 6, 15, 8, 9, 10], 0, 5, 1, 2, 3)]
    return rows


def random_rows(n: int, n_keys: int, seed: int) -> list:
    """(sk, ring, s, t, amount, r, alpha) rows with rings drawn from n_keys keys and random distinct positions"""
    rng = np.random.default_rng(seed)
    fs = lambda: int.from_bytes(rng.bytes(64), "little") % rj.R_J
    rows = []
    for _ in range(n):
        s, t = (int(v) for v in rng.choice(RING, 2, replace=False))
        rows.append((fs(), [int(v) for v in rng.integers(0, n_keys, RING - 1)], s, t, int(rng.integers(0, 2 ** 32)), fs(), fs()))
    return rows
