"""TEST INFRASTRUCTURE — random blocks of confidential transfers in the layout of zk_balances_confidential_block.

Ciphertexts are real lifted-ElGamal encryptions (the C ElGamal oracle's encrypt) to a few encryption keys.  A block has a
skewed choice of sender (weight 1 / (i + 1)^skew for account i), so that a few senders have long chains, self-transfers,
due and non-due accounts, absent balances and pendings, zeros in the mask, every point-rejection class and, on request,
out-of-range indices."""
from __future__ import annotations

import numpy as np

from . import eg_coracle as ec
from . import elgamal as eg
from . import pyref as jj

BAD_FIELD = (jj.R + 3).to_bytes(32, "little")           # y >= r: NotInField


def bad_curve() -> bytes:
    """a y with no x: NotOnCurve"""
    y = 2
    while jj.point_for_y(y) is not None:
        y += 1
    return y.to_bytes(32, "little")


def bad_order(enc: bytes) -> bytes:
    """a curve point outside the prime-order subgroup: a valid point plus one of order 8"""
    return jj.encode(jj.add(jj.read(enc)[1], jj.torsion_point(8)))


_KEYS = None


def keys():
    global _KEYS
    if _KEYS is None:
        _KEYS = b"".join(jj.encode(jj.mul(eg.P_G, 1000 + 7919 * i)) for i in range(4))
    return _KEYS


def encrypt(rng, n: int, rs=None) -> bytes:
    """n ciphertexts of random amounts < 2^20 to random keys; rs: the randomness of each (default random)"""
    k = keys()
    if rs is None:
        rs = [int(x) for x in rng.integers(1, 2**62, n)]
    eks = b"".join(k[32 * i:32 * i + 32] for i in rng.integers(0, 4, n))
    return ec.encrypt([int(a) for a in rng.integers(0, 2**20, n)], rs, eks)


class Block:
    def __init__(self, balances, pendings, flags, sender, recipient, tx_points, applied):
        self.balances, self.pendings, self.flags = balances, pendings, flags
        self.sender, self.recipient, self.tx_points, self.applied = sender, recipient, tx_points, applied

    @property
    def n_tx(self):
        return len(self.sender)

    def args(self):
        return (self.balances, self.pendings, self.flags, self.sender, self.recipient, self.tx_points, self.applied)


def make(n_acct: int, n_tx: int, seed: int, skew: float = 1.0, bad_points: int = 0, bad_index: bool = False,
         self_frac: float = 0.05, zero_frac: float = 0.1) -> Block:
    rng = np.random.default_rng(seed)
    cts = encrypt(rng, 2 * n_acct)
    balances, pendings = cts[:64 * n_acct], cts[64 * n_acct:]
    flags = bytearray(int(f) for f in rng.integers(0, 8, n_acct))
    w = 1.0 / np.arange(1, n_acct + 1) ** skew
    sender = rng.choice(n_acct, n_tx, p=w / w.sum()).astype(np.uint32)
    recipient = rng.integers(0, n_acct, n_tx).astype(np.uint32)
    self_tx = rng.random(n_tx) < self_frac
    recipient[self_tx] = sender[self_tx]
    # amount_sender, amount_recipient, fee_sender share the transaction's randomness r; randomness = r P_G
    rs = [int(x) for x in rng.integers(1, 2**62, n_tx)]
    enc = encrypt(rng, 3 * n_tx, [r for r in rs for _ in range(3)])
    pts = bytearray()
    for k in range(n_tx):
        c = enc[192 * k:192 * k + 192]
        pts += c[0:32] + c[64:96] + c[128:160] + c[32:64]
    applied = bytearray((rng.random(n_tx) >= zero_frac).astype(np.uint8).tobytes())
    if bad_points:
        curve = bad_curve()
        for i, k in enumerate(rng.choice(n_tx, bad_points, replace=False)):
            slot = int(rng.integers(0, 4))
            off = 128 * int(k) + 32 * slot
            kind = i % 3
            pts[off:off + 32] = BAD_FIELD if kind == 0 else curve if kind == 1 else bad_order(bytes(pts[off:off + 32]))
    if bad_index and n_tx >= 2:
        sender[n_tx // 3] = n_acct + 5
        recipient[2 * n_tx // 3] = 0xFFFFFFFF
    return Block(bytes(balances), bytes(pendings), bytes(flags), sender, recipient, bytes(pts), bytes(applied))
