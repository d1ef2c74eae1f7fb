"""TEST INFRASTRUCTURE — random blocks of encrypted-asset calls in the layout of zk_assets_block.

Ciphertexts are real lifted-ElGamal encryptions (bal_corpus.encrypt).  A block mixes transfers, issues and destroys; slot
choices are skewed (weight 1 / (i + 1)^skew for slot i), so a few slots carry long chains with issues and destroys inside
them.  It has self-transfers, due and non-due slots, absent balances and pendings, mask values 0-4, every point-rejection
class (in the points each kind reads, and garbage in the ones it ignores) and, on request, invalid slots and kinds."""
from __future__ import annotations

import numpy as np

from . import bal_corpus

TRANSFER, ISSUE, DESTROY = 0, 1, 2


class Block:
    def __init__(self, balances, pendings, flags, kind, slot_a, slot_b, tx_points, applied):
        self.balances, self.pendings, self.flags = balances, pendings, flags
        self.kind, self.slot_a, self.slot_b, self.tx_points, self.applied = kind, slot_a, slot_b, tx_points, applied

    @property
    def n_tx(self):
        return len(self.kind)

    def args(self):
        return (self.balances, self.pendings, self.flags, self.kind, self.slot_a, self.slot_b, self.tx_points, self.applied)

    def transfers(self):
        """the confidential_transfer arguments (balances, pendings, flags, sender, recipient, tx_points, applied) of a block
        of transfers only"""
        assert set(self.kind) <= {TRANSFER}
        return (self.balances, self.pendings, self.flags, self.slot_a, self.slot_b, self.tx_points, self.applied)


def make(n_slots: int, n_tx: int, seed: int, skew: float = 1.0, issue_frac: float = 0.1, destroy_frac: float = 0.05,
         bad_points: int = 0, bad_index: bool = False, self_frac: float = 0.05, zero_frac: float = 0.1) -> Block:
    rng = np.random.default_rng(seed)
    base = bal_corpus.make(n_slots, n_tx, seed + 100000, skew=skew, self_frac=self_frac, zero_frac=0.0)
    r = rng.random(n_tx)
    kind = np.where(r < issue_frac, ISSUE, np.where(r < issue_frac + destroy_frac, DESTROY, TRANSFER)).astype(np.uint8)
    slot_a, slot_b = base.sender.copy(), base.recipient.copy()
    pts = bytearray(base.tx_points)
    garbage = [bal_corpus.BAD_FIELD, bal_corpus.bad_curve()]
    for k in np.flatnonzero(kind != TRANSFER):
        k = int(k)
        slot_b[k] = int(rng.integers(0, 2**32))                       # read for transfers only
        ignored = (1, 2) if kind[k] == ISSUE else (0, 1, 2, 3)
        for i in ignored:
            if rng.random() < 0.5:
                pts[128 * k + 32 * i:128 * k + 32 * i + 32] = garbage[int(rng.integers(0, 2))]
    applied = bytearray(int(v) for v in np.where(rng.random(n_tx) < zero_frac, rng.integers(0, 5, n_tx), 1))
    if bad_points:
        curve = bal_corpus.bad_curve()
        cand = np.flatnonzero(kind != DESTROY)
        for i, k in enumerate(rng.choice(cand, min(bad_points, len(cand)), replace=False)):
            k = int(k)
            slot = int(rng.integers(0, 4)) if kind[k] == TRANSFER else (0, 3)[int(rng.integers(0, 2))]
            off = 128 * k + 32 * slot
            c = i % 3
            pts[off:off + 32] = (bal_corpus.BAD_FIELD if c == 0 else curve if c == 1 else
                                 bal_corpus.bad_order(bytes(base.tx_points[off:off + 32])))
    if bad_index and n_tx >= 4:
        slot_a[n_tx // 4] = n_slots + 5
        kind[n_tx // 2] = TRANSFER
        slot_b[n_tx // 2] = 0xFFFFFFFF
        kind[3 * n_tx // 4] = 7
    return Block(base.balances, base.pendings, base.flags, bytes(kind.tobytes()), slot_a, slot_b, bytes(pts), bytes(applied))
