"""TEST INFRASTRUCTURE — random blocks of both anonymous-balances calls in the layout of zk_anonymous_calls_block, built
on anon_corpus.

A block of anon_corpus rings, of which issue_frac become issues.  An issuer is a member of a random ring (so issues land
before an account's first touch, after it and between two touches, more often on the accounts many rings name), or, one
time in five, one of the last `free` accounts, which no ring names.  An issue's ignored fields (members 1..11, slots
1..11 of its points, its tx_extra row) are left as the ring had them, some of them out of range or unreadable.  The mask
takes every value 0..4 for issues too, so some issues fail; on request issues get a rejected total or randomness, and
two transactions an unknown kind and one issue an issuer out of range."""
from __future__ import annotations

import numpy as np

from . import anon_corpus
from . import bal_corpus

RING = 12


class Block(anon_corpus.Block):
    def __init__(self, b: anon_corpus.Block, kind: bytes):
        super().__init__(*b.args())
        self.kind = kind

    def args(self):
        return (self.keys, self.balances, self.pendings, self.flags, self.kind, self.members, self.tx_points, self.tx_extra, self.g_epoch,
                self.applied)


def make(n_acct: int, n_tx: int, seed: int, issue_frac: float = 0.1, free: int = 2, bad_issue_points: int = 0, bad_kind: bool = False,
         **kw) -> Block:
    b = anon_corpus.make(n_acct, n_tx, seed, **kw)
    rng = np.random.default_rng(seed + 1000)
    mem = b.members.reshape(-1, RING).copy()
    named = n_acct - free
    ring_free = (mem >= named) & (mem < n_acct)
    mem[ring_free] = mem[ring_free] % max(named, 1)
    kind = (rng.random(n_tx) < issue_frac).astype(np.uint8)
    issues = np.flatnonzero(kind)
    for k in issues.tolist():
        if free and rng.random() < 0.2:
            mem[k, 0] = named + int(rng.integers(0, free))
        else:
            mem[k, 0] = mem[int(rng.integers(0, n_tx)), int(rng.integers(0, RING))]
    if len(issues):
        mem[issues[0], 5] = 0xFFFFFFFF                         # an ignored member out of range
    tx_points = bytearray(b.tx_points)
    if len(issues) > 1:
        off = 32 * ((RING + 1) * int(issues[1]) + 3)           # an ignored slot that does not read
        tx_points[off:off + 32] = bal_corpus.BAD_FIELD
    curve = bal_corpus.bad_curve()
    for i, k in enumerate(rng.permutation(issues)[:bad_issue_points].tolist()):
        off = 32 * ((RING + 1) * k + (0 if i % 2 == 0 else RING))
        tx_points[off:off + 32] = curve if i % 3 == 0 else bal_corpus.BAD_FIELD if i % 3 == 1 else bal_corpus.bad_order(bytes(tx_points[off:off + 32]))
    if bad_kind and n_tx >= 4:
        kind[n_tx // 4] = 2
        kind[3 * n_tx // 4] = 255
        if len(issues) > 2:
            mem[issues[2], 0] = n_acct + 1                     # an issuer out of range
    b.members, b.tx_points = mem.reshape(-1), bytes(tx_points)
    return Block(b, kind.tobytes())
