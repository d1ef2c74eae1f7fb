"""TEST INFRASTRUCTURE — random blocks of anonymous transfers in the layout of zk_balances_anonymous_block.

Account ciphertexts are real lifted-ElGamal encryptions (bal_corpus.encrypt); each account's EncKey is the left point of
one more encryption (a valid point, distinct from the others).  A ring draws its 12 members with weight 1 / (i + 1)^skew for account i, so a few accounts sit in many rings and members
repeat inside a ring; dup_frac of the rings also get member 1 = member 0 on purpose.  The transaction points (lefts,
right, rvk, nonce) and g_epoch come from a pool of encryptions' points.  The mask takes every value 0..4 (1 applies;
0, 2, 3, 4 are the verifier's other verdicts); on request some transaction points are replaced by every rejection class
of bal_corpus, and two rings get an out-of-range index."""
from __future__ import annotations

import numpy as np

from . import bal_corpus

RING = 12
MASK_P = (0.1, 0.6, 0.1, 0.1, 0.1)        # probabilities of the mask values 0 .. 4


class Block:
    def __init__(self, keys, balances, pendings, flags, members, tx_points, tx_extra, g_epoch, applied):
        self.keys, self.balances, self.pendings, self.flags = keys, balances, pendings, flags
        self.members, self.tx_points, self.tx_extra, self.g_epoch, self.applied = members, tx_points, tx_extra, g_epoch, applied

    @property
    def n_tx(self):
        return len(self.members) // RING

    def args(self):
        return (self.keys, self.balances, self.pendings, self.flags, self.members, self.tx_points, self.tx_extra, self.g_epoch,
                self.applied)


def make(n_acct: int, n_tx: int, seed: int, skew: float = 1.0, bad_points: int = 0, bad_index: bool = False, dup_frac: float = 0.1,
         pool: int | None = None, keys: bytes | None = None, mask_p=MASK_P) -> Block:
    rng = np.random.default_rng(seed)
    cts = bal_corpus.encrypt(rng, 2 * n_acct)
    balances, pendings = cts[:64 * n_acct], cts[64 * n_acct:]
    flags = bytearray(int(f) for f in rng.integers(0, 8, n_acct))
    if keys is None:
        keys = np.frombuffer(bal_corpus.encrypt(rng, n_acct), np.uint8).reshape(-1, 64)[:, :32].tobytes()
    w = 1.0 / np.arange(1, n_acct + 1) ** skew
    members = rng.choice(n_acct, (n_tx, RING), p=w / w.sum()).astype(np.uint32) if n_acct else np.zeros((n_tx, RING), np.uint32)
    dup = rng.random(n_tx) < dup_frac
    members[dup, 1] = members[dup, 0]
    # the pool of valid points: both halves of pool encryptions
    n_pool = pool if pool is not None else max(8, min(2048, 8 * n_tx))
    pts_pool = np.frombuffer(bal_corpus.encrypt(rng, n_pool), np.uint8).reshape(2 * n_pool, 32)
    tx_points = bytearray(pts_pool[rng.integers(0, 2 * n_pool, n_tx * (RING + 1))].tobytes())
    tx_extra = pts_pool[rng.integers(0, 2 * n_pool, 2 * n_tx)].tobytes()
    g_epoch = pts_pool[int(rng.integers(0, 2 * n_pool))].tobytes()
    applied = rng.choice(5, n_tx, p=mask_p).astype(np.uint8).tobytes()
    if bad_points:
        curve = bal_corpus.bad_curve()
        for i, k in enumerate(rng.choice(n_tx, bad_points, replace=False)):
            off = 32 * ((RING + 1) * int(k) + int(rng.integers(0, RING + 1)))
            kind = i % 3
            tx_points[off:off + 32] = (bal_corpus.BAD_FIELD if kind == 0 else curve if kind == 1
                                       else bal_corpus.bad_order(bytes(tx_points[off:off + 32])))
    if bad_index and n_tx >= 2:
        members[n_tx // 3, 5] = n_acct + 5
        members[2 * n_tx // 3, 11] = 0xFFFFFFFF
    return Block(keys, bytes(balances), bytes(pendings), bytes(flags), members.reshape(-1), bytes(tx_points), tx_extra, g_epoch, applied)
