"""TEST INFRASTRUCTURE — blocks of anonymous-balances calls (transfers and issues) with proofs forged from toy keys'
trapdoors (tests/verify_forge.py), for zk_import_anonymous_block.

Two toy keys: one of 11-point public inputs (23 inputs, the confidential shape issues are checked with) and one of 52
points (105 inputs, the anonymous transfer's).  Each transaction has an intended verdict.  A passing one gets a proof valid
for exactly the points the reference reads under the intended verdicts: an issue's own fields, and for a transfer the 52
points the C oracle (anon_issue_coracle.block) gives with the intended issue verdicts applied and no transfer (a transfer
changes pending balances only, so no transfer verdict moves them).  A failing one gets a proof valid for nothing (C + G1).
A transaction with a rejected point gets verdict 4 either way.  The rings, points and tables come from anon_issue_corpus;
no GPU."""
from __future__ import annotations

import numpy as np

from tests import verify_forge as vf
from tests.jubjub_oracle import anon_issue_coracle as aic
from tests.jubjub_oracle import anon_issue_corpus
from tests.jubjub_oracle import coracle as jco
from zero_chain_b200 import groth16 as zk

RING = zk.ANONIMITY_SIZE


class ForgeKey:
    """a toy CRS whose public inputs are the coordinates of n_points Jubjub points, with its trapdoor"""

    def __init__(self, n_points: int, seed: int):
        self.n_points = n_points
        self.toy = vf.ToyKey(n_inputs=2 * n_points + 1, seed=seed)
        self.params_bytes = self.toy.crs.params_bytes

    def proofs(self, rows: bytes, passing) -> list:
        """one proof per row of n_points encodings: valid for its points where passing, valid for nothing elsewhere"""
        P = self.n_points
        n = len(rows) // (32 * P)
        if not n:
            return []
        xy, st = jco.into_xy(rows)
        xy = xy.reshape(n, P, 2, 4)
        cs = []
        for k in range(n):
            if passing[k]:
                ins = [sum(int(v) << (64 * i) for i, v in enumerate(xy[k, p, c])) for p in range(P) for c in range(2)]
                cs.append(vf.forge(self.toy.crs, ins, vf.A_S, vf.B_S, k=self.toy.k)[2])
            else:
                cs.append(vf.forge(self.toy.crs, [k % 7] * (2 * P), vf.A_S, vf.B_S, k=self.toy.k)[2] + 1)
        return vf.proofs_from_c(vf.A_S, vf.B_S, cs)

    def rejected(self, rows: bytes):
        n = len(rows) // (32 * self.n_points)
        return jco.into_xy(rows)[1].reshape(n, self.n_points).any(axis=1) if n else np.zeros(0, bool)


class Block:
    def __init__(self, accounts, txs, g_epoch, proofs, intended):
        self.accounts, self.txs, self.g_epoch, self.proofs, self.intended = accounts, txs, g_epoch, proofs, intended

    def args(self):
        return self.accounts, self.txs, self.g_epoch, self.proofs

    def arrays(self):
        """kind, members, tx_points, tx_extra and issue_fields as the C call takes them"""
        t = self.txs
        return (bytes(x.kind for x in t), np.array([x.members for x in t], np.uint32).reshape(-1), b"".join(x.points() for x in t),
                b"".join(x.rvk + x.nonce for x in t),
                b"".join(x.fee + x.balance if x.kind == zk.ANON_ISSUE else bytes(96) for x in t))

    def oracle(self, verdicts):
        """the C oracle's zk_anonymous_calls_block outputs with the transactions whose verdict is 1 applied"""
        kind, members, tx_points, tx_extra, _ = self.arrays()
        bad, out = aic.block(*self.accounts, kind, members, tx_points, tx_extra, self.g_epoch, bytes(int(v == 1) for v in verdicts))
        assert bad is None
        return out


def block(anon: ForgeKey, conf: ForgeKey, n_acct: int, n_tx: int, seed: int, issue_frac=0.1, fail_frac=0.0, fail_at=(), issues=None,
          issuer=None, **kw) -> Block:
    """n_tx calls over n_acct accounts (anon_issue_corpus's block, its kinds and issuers unless issues / issuer give them:
    the transactions that are issues, and {transaction: issuer}); fail_frac of them, and those at fail_at, fail.  **kw goes
    to anon_issue_corpus.make (skew, bad_points, bad_issue_points, free)."""
    b = anon_issue_corpus.make(n_acct, n_tx, seed, issue_frac=issue_frac, **kw)
    rng = np.random.default_rng(seed + 2)
    kind = np.frombuffer(b.kind, np.uint8).copy()
    if issues is not None:
        kind[:] = zk.ANON_TRANSFER
        kind[list(issues)] = zk.ANON_ISSUE
    mem = b.members.reshape(-1, RING).copy()
    for k, a in (issuer or {}).items():
        mem[k, 0] = a
    pts = [b.tx_points[32 * i:32 * i + 32] for i in range((RING + 1) * n_tx)]
    extra = [b.tx_extra[32 * i:32 * i + 32] for i in range(2 * n_tx)]
    txs = []
    for k in range(n_tx):
        row = pts[(RING + 1) * k:(RING + 1) * (k + 1)]
        if kind[k] == zk.ANON_ISSUE:
            # fee and balance: a valid point of the row's ignored slots, and a stored ciphertext of the table
            a = int(rng.integers(0, n_acct))
            txs.append(zk.AnonIssueTx(int(mem[k, 0]), row[0], row[1 + k % 11], b.balances[64 * a:64 * a + 64], row[RING], extra[2 * k],
                                      extra[2 * k + 1]))
        else:
            txs.append(zk.AnonymousTx(mem[k], row[:RING], row[RING], extra[2 * k], extra[2 * k + 1]))
    passing = rng.random(n_tx) >= fail_frac
    passing[list(fail_at)] = False
    blk = Block((b.keys, b.balances, b.pendings, b.flags), txs, b.g_epoch, [None] * n_tx, None)
    is_issue = kind == zk.ANON_ISSUE
    iss, tr = np.flatnonzero(is_issue).tolist(), np.flatnonzero(~is_issue).tolist()
    intended = [0] * n_tx
    rows = b"".join(txs[k].verify_points(b.keys, b.g_epoch) for k in iss)
    for k, p, r in zip(iss, conf.proofs(rows, passing[iss]), conf.rejected(rows)):
        blk.proofs[k], intended[k] = p, (zk.VERDICT_INPUT_REJECTED if r else int(passing[k]))
    vp = blk.oracle(intended)[1]
    rows = b"".join(vp[1664 * k:1664 * k + 1664] for k in tr)
    for k, p, r in zip(tr, anon.proofs(rows, passing[tr]), anon.rejected(rows)):
        blk.proofs[k], intended[k] = p, (zk.VERDICT_INPUT_REJECTED if r else int(passing[k]))
    blk.intended = intended
    return blk
