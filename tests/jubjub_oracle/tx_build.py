"""TEST INFRASTRUCTURE (oracle): the sender side of a confidential transfer, restated with Python integers on pyref.py,
redjubjub.py and elgamal.py, in the byte layouts of zk_keys_from_seed_batch, zk_g_epoch_batch and
zk_confidential_fields_batch (include/zkb200.h).

  keys               SpendingKey::from_seed -> ProofGenerationKey -> DecryptionKey -> EncryptionKey (core/keys/src/lib.rs)
  g_epoch            GEpoch::group_hash: find_group_hash(epoch as u32 LE, "zcgepoch"), tag bytes from 0
                     (core/primitives/src/g_epoch.rs:102-145)
  confidential_fields  MultiCiphertexts::<Confidential>::encrypt and ProofContext's rvk / nonce (zface's gen_proof): every
                     point computed the reference's way, amount P_G + r ek for both ciphertexts, pgk + alpha P_G for rvk
  window_table       d 16^j G for j < 64, d <= 8: the layout of the device's fixed-base tables"""
from __future__ import annotations

import struct

import numpy as np

from . import elgamal as eg
from . import pyref as jj
from . import redjubjub as rj

GEPOCH_PERSONALIZATION = b"zcgepoch"
N_FIELDS = 9


def niels(p) -> list:
    """(y - x, y + x, 2d x y) of an affine point, canonical"""
    x, y = p
    return [(y - x) % jj.R, (y + x) % jj.R, 2 * jj.D * x * y % jj.R]


def window_table(g) -> list:
    """d 16^j g in entry order 9 j + d"""
    pts, base = [], g
    for _ in range(64):
        acc = jj.IDENTITY
        for _ in range(9):
            pts.append(acc)
            acc = jj.add(acc, base)
        base = jj.mul(base, 16)
    return pts


def keys(seed: bytes):
    """(sk, dk, ek) encodings of an account seed"""
    sk = rj.spending_key(seed)
    dk = rj.decryption_key(rj.proof_generation_key(sk))
    return rj.scalar_bytes(sk), rj.scalar_bytes(dk), jj.encode(jj.mul(rj.P_G, dk))


def g_epoch(epoch: int):
    """(encoding, tag byte) of GEpoch::group_hash(epoch)"""
    p, i = rj.find_group_hash(struct.pack("<I", epoch), GEPOCH_PERSONALIZATION)
    return jj.encode(p), i


def confidential_fields(sk: int, ek_recipient: bytes, amount: int, fee: int, r: int, alpha: int, g_epoch_enc: bytes):
    """(fields, rsk, dk, status) of one row: fields are the 9 encodings in ConfidentialTx order (address_sender,
    address_recipient, amount_sender, amount_recipient, fee_sender, randomness, rvk, g_epoch, nonce).  A recipient key
    that fails EncryptionKey::read gives zeros and its zk_jubjub_into_xy status."""
    st, x, y = jj.into_xy(ek_recipient)
    if st != jj.OK:
        return bytes(32 * N_FIELDS), bytes(32), bytes(32), st
    ek_r = (x, y)
    pgk = rj.proof_generation_key(sk)
    dk = rj.decryption_key(pgk)
    ek_s = jj.mul(rj.P_G, dk)
    amount_sender, randomness = eg.encrypt(amount, r, ek_s)
    amount_recipient, _ = eg.encrypt(amount, r, ek_r)
    fee_sender, _ = eg.encrypt(fee, r, ek_s)
    rvk = jj.add(pgk, jj.mul(rj.P_G, alpha))
    g = jj.read(g_epoch_enc)[1]
    nonce = jj.mul(g, dk)
    fields = b"".join([jj.encode(ek_s), ek_recipient, jj.encode(amount_sender), jj.encode(amount_recipient), jj.encode(fee_sender),
                       jj.encode(randomness), jj.encode(rvk), g_epoch_enc, jj.encode(nonce)])
    return fields, rj.scalar_bytes((sk + alpha) % rj.R_J), rj.scalar_bytes(dk), jj.OK


def bad_recipient_keys() -> list:
    """(encoding, status) for each way EncryptionKey::read fails"""
    not_in_field = (jj.R).to_bytes(32, "little")
    y = 2
    while jj.point_for_y(y) is not None:
        y += 1
    not_on_curve = y.to_bytes(32, "little")
    small = jj.encode(jj.torsion_point(4))
    mixed = jj.encode(jj.add(jj.mul(rj.P_G, 5), jj.torsion_point(2)))
    return [(not_in_field, jj.NOT_IN_FIELD), (not_on_curve, jj.NOT_ON_CURVE), (small, jj.NOT_PRIME_ORDER), (mixed, jj.NOT_PRIME_ORDER)]


def edge_rows() -> list:
    """(sk, ek_recipient, amount, fee, r, alpha) rows at the edges: sk = 0, r = 0 (identity randomness), alpha = r_J - sk
    (rsk = 0, identity rvk), amounts and fees 0 and 2^32 - 1, and recipient keys that fail each way"""
    ek = keys(b"Bob" + b" " * 29)[2]
    top = 2 ** 32 - 1
    rows = [(0, ek, 5, 1, 7, 9), (123, ek, 10, 1, 0, 77), (456, ek, 0, 0, 3, rj.R_J - 456), (rj.R_J - 1, ek, top, top, rj.R_J - 1, rj.R_J - 1),
            (789, ek, top, 0, 11, 0), (1, jj.encode(jj.IDENTITY), 3, 2, 5, 8)]
    rows += [(31, k, 1, 1, 2, 3) for k, _ in bad_recipient_keys()]
    return rows


def random_rows(n: int, seed: int) -> list:
    rng = np.random.default_rng(seed)
    fs = lambda: int.from_bytes(rng.bytes(64), "little") % rj.R_J
    eks = [keys(b"recipient %d" % i)[2] for i in range(4)]
    return [(fs(), eks[i % 4], int(rng.integers(0, 10 ** 6)), int(rng.integers(0, 1000)), fs(), fs()) for i in range(n)]
