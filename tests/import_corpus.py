"""TEST INFRASTRUCTURE — blocks of confidential transfers and of encrypted-asset calls with proofs forged from a toy key's
trapdoor (tests/verify_forge.py), for the block imports (zk_import_confidential_block / zk_import_assets_block).

Each transaction has an intended verdict.  A passing one gets a proof valid for exactly the points it reads when the
block is applied with the intended verdicts: its sender's balance excludes every earlier failed transfer of its chain.
So a transfer after a failure fails while that failure still counts as applied, and passes a round later, which is what
makes the rounds matter.  A failing one gets a proof that verifies for nothing (C + G1).  The balances come from the C
oracles (balances_oracle.c, assets_oracle.c) run with the intended mask; public inputs from the C Jubjub oracle; no GPU."""
from __future__ import annotations

import numpy as np

from tests import verify_forge as vf
from tests.jubjub_oracle import assets_coracle as ac
from tests.jubjub_oracle import bal_coracle as bc
from tests.jubjub_oracle import bal_corpus
from tests.jubjub_oracle import coracle as jco
from zero_chain_b200 import groth16 as zk

POINTS = zk.CONFIDENTIAL_POINTS
ROW = 32 * POINTS


class ForgeKey:
    """A toy CRS of 11-point public inputs (the confidential proof's shape) with its trapdoor."""

    def __init__(self, seed=5):
        self.toy = vf.ToyKey(n_inputs=2 * POINTS + 1, seed=seed)
        self.params_bytes = self.toy.crs.params_bytes

    def proofs(self, rows: bytes, passing) -> list:
        """one proof per 352-byte row: valid for its points where passing, valid for nothing elsewhere"""
        n = len(rows) // ROW
        xy, st = jco.into_xy(rows)
        xy = xy.reshape(n, POINTS, 2, 4)
        st = st.reshape(n, POINTS)
        cs = []
        for k in range(n):
            if passing[k] and not st[k].any():
                ins = [sum(int(v) << (64 * i) for i, v in enumerate(xy[k, p, c])) for p in range(POINTS) for c in range(2)]
                cs.append(vf.forge(self.toy.crs, ins, vf.A_S, vf.B_S, k=self.toy.k)[2])
            else:
                cs.append(vf.forge(self.toy.crs, [k % 7] * (2 * POINTS), vf.A_S, vf.B_S, k=self.toy.k)[2] + 1)
        return vf.proofs_from_c(vf.A_S, vf.B_S, cs) if n else []


class ConfBlock:
    """rows: each transfer's 11 verifier points with the balance its proof was made for"""

    def __init__(self, accounts, txs, proofs, intended, rows):
        self.accounts, self.txs, self.proofs, self.intended, self.rows = accounts, txs, proofs, intended, rows

    def oracle(self, verdicts):
        """the C oracle's (balance_after, status, new_balances, new_pendings, new_flags) for the final verdicts"""
        bad, out = bc.block(*self.accounts, [t.sender for t in self.txs], [t.recipient for t in self.txs],
                            b"".join(t.points() for t in self.txs), bytes(int(v == 1) for v in verdicts))
        assert bad is None
        return out[1:]


def _oracle_conf(*args):
    bad, out = bc.block(*args)
    assert bad is None
    return out


def _oracle_assets(*args):
    bad, out = ac.block(*args)
    assert bad is None
    return out


def confidential(key: ForgeKey, n_acct: int, n_tx: int, seed: int, fail_frac=0.0, fail_at=(), skew=1.0, bad_points=0,
                 sender=None, state_call=_oracle_conf) -> ConfBlock:
    """n_tx transfers over n_acct accounts (bal_corpus's tables and points); fail_frac of them, and those at fail_at, fail.
    sender: fixed senders instead of the corpus's draw.  A transfer with a rejected point gets verdict 4 either way.
    state_call: what computes the balances the proofs are made for, with zk.confidential_block's arguments and result (the
    C oracle by default; a GPU run may pass the device call, which its tests check against the oracle byte for byte)."""
    b = bal_corpus.make(n_acct, n_tx, seed, skew=skew, bad_points=bad_points, zero_frac=0.0)
    rng = np.random.default_rng(seed + 1)
    snd = np.asarray(b.sender if sender is None else sender, np.uint32)
    misc = bal_corpus.encrypt(rng, 3)
    addr_s, addr_r, rvk, g_epoch, nonce = (misc[32 * i:32 * i + 32] for i in range(5))
    passing = rng.random(n_tx) >= fail_frac
    passing[list(fail_at)] = False
    pts = b.tx_points
    txs = [zk.ConfidentialTx(int(snd[k]), int(b.recipient[k]), addr_s, addr_r, *[pts[128 * k + 32 * i:128 * k + 32 * i + 32] for i in range(4)],
                             rvk, g_epoch, nonce) for k in range(n_tx)]
    out = state_call(b.balances, b.pendings, b.flags, snd, b.recipient, pts, passing.astype(np.uint8).tobytes())
    bs, st = out[0], out[2]
    passing &= np.frombuffer(st, np.uint8) != zk.BLOCK_BAD_POINT
    rows = b"".join(zk.confidential_points(t.address_sender, t.address_recipient, t.amount_sender, t.amount_recipient, t.randomness,
                                           t.fee_sender, bs[64 * k:64 * k + 64], t.rvk, t.g_epoch, t.nonce) for k, t in enumerate(txs))
    intended = [1 if p else (zk.VERDICT_INPUT_REJECTED if s == zk.BLOCK_BAD_POINT else 0) for p, s in zip(passing, st)]
    return ConfBlock((b.balances, b.pendings, b.flags), txs, key.proofs(rows, passing), intended, rows)


class AssetBlock:
    def __init__(self, state, txs, proofs, intended, next_asset_id, new_slot_flags):
        self.state, self.txs, self.proofs, self.intended = state, txs, proofs, intended
        self.next_asset_id, self.new_slot_flags = next_asset_id, new_slot_flags

    def args(self):
        return self.state, self.txs, self.proofs, self.next_asset_id, self.new_slot_flags

    def slots(self, verdicts):
        kinds = [t.kind for t in self.txs]
        fixed = [v if k != zk.ASSET_TRANSFER else 0 for k, v in zip(kinds, verdicts)]
        slots = list(self.state[0])
        table, ids, slot_a, slot_b = zk._asset_slots("corpus", slots, *self.state[1:], self.txs, fixed, self.next_asset_id,
                                                     self.new_slot_flags)
        return slots, table, slot_a, slot_b

    def oracle(self, verdicts, state_call=_oracle_assets):
        """the C oracle's zk_assets_block outputs for the final verdicts"""
        _, table, slot_a, slot_b = self.slots(verdicts)
        return state_call(*table, bytes(t.kind for t in self.txs), slot_a, slot_b, b"".join(t.points() for t in self.txs),
                          bytes(int(v == 1) for v in verdicts))


def assets(key: ForgeKey, n_keys: int, n_tx: int, seed: int, fail_frac=0.0, fixed_fail_frac=0.0, issue_frac=0.05,
           destroy_frac=0.02, skew=1.0, state_call=_oracle_assets) -> AssetBlock:
    """asset 3 held by n_keys keys (bal_corpus's tables), then n_tx calls: transfers of asset 3 between the keys (a skewed
    choice of sender), issues of new assets to them and destroys of their asset-3 slots.  fail_frac of the transfers and
    fixed_fail_frac of the issues and destroys fail.  state_call: as for confidential, with zk.assets_block's arguments."""
    rng = np.random.default_rng(seed)
    table = bal_corpus.make(n_keys, n_tx, seed + 1, zero_frac=0.0, self_frac=0.0)
    misc = bal_corpus.encrypt(rng, n_keys // 2 + 4)
    keys = [misc[32 * i:32 * i + 32] for i in range(2 * (n_keys // 2 + 4))][:n_keys]
    assert len(set(keys)) == n_keys
    rvk, g_epoch, nonce, fee = (misc[-32 * (i + 1):len(misc) - 32 * i] for i in range(4))
    ct = misc[:64]
    w = 1.0 / np.arange(1, n_keys + 1) ** skew
    pts = table.tx_points
    txs, passing = [], []
    for k in range(n_tx):
        u = rng.random()
        row = [pts[128 * k + 32 * i:128 * k + 32 * i + 32] for i in range(4)]
        if u < issue_frac:
            txs.append(zk.IssueTx(keys[int(rng.integers(0, n_keys))], row[0], fee, ct, row[3], rvk, g_epoch, nonce))
            passing.append(rng.random() >= fixed_fail_frac)
        elif u < issue_frac + destroy_frac:
            txs.append(zk.DestroyTx(keys[int(rng.integers(0, n_keys))], 3, row[0], row[2], ct, row[3], rvk, g_epoch, nonce))
            passing.append(rng.random() >= fixed_fail_frac)
        else:
            s = int(rng.choice(n_keys, p=w / w.sum()))
            r = int(rng.integers(0, n_keys))
            txs.append(zk.AssetTransferTx(3, keys[s], keys[r], *row, rvk, g_epoch, nonce))
            passing.append(rng.random() >= fail_frac)
    state = ([(3, key_) for key_ in keys], table.balances, table.pendings, table.flags)
    blk = AssetBlock(state, txs, [], None, 10, zk.ACCOUNT_DUE)
    intended = [1 if p else 0 for p in passing]
    out = blk.oracle(intended, state_call)
    bs = out[0]
    rows = b"".join(t.verify_points(bs[64 * k:64 * k + 64]) if t.kind == zk.ASSET_TRANSFER else t.verify_points() for k, t in enumerate(txs))
    blk.proofs, blk.intended, blk.rows = key.proofs(rows, passing), intended, rows
    return blk
