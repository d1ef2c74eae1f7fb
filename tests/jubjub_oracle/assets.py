"""TEST INFRASTRUCTURE (oracle): the extrinsic loop of modules/encrypted-assets, literally, on pyref.py and elgamal.py
(through balances.py's byte-level ciphertext operations).

Storage is keyed by slot, one slot per (AssetId, EncKey), like the module's storage maps: balance (EncryptedBalance),
pending (PendingTransfer) and due (LastRollOver, or 0, < current_epoch, worked out by the caller).  Per extrinsic:
  confidential_transfer (lib.rs:86-164)  rollover(a); rollover(b) (lib.rs:266-306); balance_sender = balance(a) or
                                         Ciphertext::zero(); verdict; sub_enc_balance(a); add_pending_transfer(b);
                                         balance_after = balance(a) or Ciphertext::zero()
  issue (lib.rs:32-83)                   no rollover; verdict; balance(a) = from_left_right(total, randomness); the event
                                         (and TotalSupply) holds the same ciphertext
  destroy (lib.rs:167-215)               no rollover; verdict; take balance(a) and pending(a); the event reports them
                                         (Ciphertext::default(), empty, for an absent one)

What zk_assets_block adds around the loop, and the statuses it reports:
  3  an unknown kind, or a slot out of range (slot_b for transfers only): the transaction touches nothing
  2  a point the call reads fails Point::read + as_prime_order (a transfer's four; an issue's total and randomness)
  1  the verdict is false
  0  applied
A slot named by a valid transaction whose stored balance or pending does not read raises BadAccount at its first touch."""
from __future__ import annotations

from . import balances as bal
from .balances import APPLIED, BAD_INDEX, BAD_POINT, BALANCE, DUE, NOT_APPLIED, PENDING, ZERO, BadAccount  # noqa: F401

TRANSFER, ISSUE, DESTROY = 0, 1, 2


def _point_ok(enc: bytes) -> bool:
    return bal._point_ok(enc)


def apply_block(n_slots: int, balance: dict, pending: dict, due: set, txs, verdict):
    """txs: (kind, slot_a, slot_b, p0, p1, p2, p3) with 32-byte points laid out as zk_assets_block's tx_points; verdict(k,
    balance_sender or None) -> bool.  Returns (balance_sender, balance_after, events, status, final State): balance_after
    and events are None where the call writes nothing; an event is (ciphertext bytes or None, ciphertext bytes or None)."""
    st = bal.State(balance, pending, due)
    out_bs, out_ba, out_ev, out_st = [], [], [], []

    def done(bs, ba, ev, status):
        out_bs.append(bs); out_ba.append(ba); out_ev.append(ev); out_st.append(status)

    for k, (kind, a, b, p0, p1, p2, p3) in enumerate(txs):
        if kind not in (TRANSFER, ISSUE, DESTROY) or not 0 <= a < n_slots or (kind == TRANSFER and not 0 <= b < n_slots):
            done(ZERO if kind == TRANSFER else bytes(64), None, None, BAD_INDEX)
            continue
        if kind == TRANSFER:
            amount_s, amount_r, fee_s, rnd = p0, p1, p2, p3
            st.touch(a); st.touch(b)
            st.rollover(a)
            st.rollover(b)
            bs = st.balance.get(a, ZERO)
            if not all(_point_ok(p) for p in (amount_s, amount_r, fee_s, rnd)):
                done(bs, None, None, BAD_POINT)
                continue
            if not verdict(k, bs):
                done(bs, None, None, NOT_APPLIED)
                continue
            # sub_enc_balance (lib.rs:309-334)
            amount_plus_fee = bal.ct_add(bal.from_left_right(amount_s, rnd), bal.from_left_right(fee_s, rnd))
            if a in st.balance:
                st.balance[a] = bal.ct_sub(st.balance[a], amount_plus_fee)
            # add_pending_transfer (lib.rs:337-358)
            enc_amount_r = bal.from_left_right(amount_r, rnd)
            st.pending[b] = bal.ct_add(st.pending[b], enc_amount_r) if b in st.pending else enc_amount_r
            done(bs, st.balance.get(a, ZERO), None, APPLIED)
        elif kind == ISSUE:
            total, rnd = p0, p3
            st.touch(a)
            if not (_point_ok(total) and _point_ok(rnd)):
                done(bytes(64), None, None, BAD_POINT)
                continue
            if not verdict(k, None):
                done(bytes(64), None, None, NOT_APPLIED)
                continue
            total_ct = bal.from_left_right(total, rnd)
            st.balance[a] = total_ct
            done(bytes(64), None, (total_ct, None), APPLIED)
        else:
            st.touch(a)
            if not verdict(k, None):
                done(bytes(64), None, None, NOT_APPLIED)
                continue
            done(bytes(64), None, (st.balance.pop(a, None), st.pending.pop(a, None)), APPLIED)
    return out_bs, out_ba, out_ev, out_st, st


def to_arrays(balances: bytes, pendings: bytes, flags, st: bal.State):
    """the final storage in the ABI's layout: slots no valid transaction names copied through, a named slot's absent
    ciphertexts zero, its flags' bits 0-2 replaced (bit 2: still due)"""
    nb, npd, nf = bytearray(balances), bytearray(pendings), bytearray(flags)
    for a in st.seen:
        nb[64 * a:64 * a + 64] = st.balance.get(a, bytes(64))
        npd[64 * a:64 * a + 64] = st.pending.get(a, bytes(64))
        nf[a] = ((flags[a] & ~7) | (BALANCE if a in st.balance else 0) | (PENDING if a in st.pending else 0) |
                 (DUE if a in st.due else 0))
    return bytes(nb), bytes(npd), bytes(nf)


def run_abi(balances: bytes, pendings: bytes, flags, kind, slot_a, slot_b, tx_points: bytes, applied):
    """zk_assets_block's outputs by the loop, with the mask as the verdict: (balance_sender, balance_after, event_ct,
    event_flags, status, new_balances, new_pendings, new_flags); the entries the call does not write are zero."""
    n = len(kind)
    txs = [(int(kind[k]), int(slot_a[k]), int(slot_b[k])) + tuple(tx_points[128 * k + 32 * i:128 * k + 32 * i + 32] for i in range(4))
           for k in range(n)]
    b, p, due = bal.from_arrays(balances, pendings, flags)
    bs, ba, ev, status, st = apply_block(len(flags), b, p, due, txs, lambda k, _: applied[k] == 1)
    after, evct, evf = bytearray(64 * n), bytearray(128 * n), bytearray(n)
    for k in range(n):
        if ba[k] is not None:
            after[64 * k:64 * k + 64] = ba[k]
        if ev[k] is not None:
            for w, c in enumerate(ev[k]):
                if c is not None:
                    evct[128 * k + 64 * w:128 * k + 64 * w + 64] = c
                    evf[k] |= 1 << w
    return (b"".join(bs), bytes(after), bytes(evct), bytes(evf), bytes(status)) + to_arrays(balances, pendings, flags, st)
