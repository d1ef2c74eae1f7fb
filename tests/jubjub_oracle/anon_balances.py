"""TEST INFRASTRUCTURE (oracle): the anonymous_transfer loop of modules/anonymous-balances, literally, on balances.py,
elgamal.py and pyref.py.

Storage is balances.State: three dicts keyed by account index (EncryptedBalance, PendingTransfer, and due = LastRollOver <
current_epoch, worked out by the caller).  Per transaction (lib.rs:23-82):
  rollover(e) for each of the 12 enc_keys         lib.rs:169-206, at most once per block per account (due is cleared); it
                                                  stands whatever happens to the transaction afterwards
  acc[i] = balance(e_i) or Ciphertext::zero()     what verify_anonymous_proof reads (zk-system/src/lib.rs:118-165)
  verdict                                         verdict(k, acc) -> bool (the proof check)
  add_pending_transfer(e_i, left_i, right)        lib.rs:209-232, for every member in ring order (a member listed twice
                                                  receives both additions)

What zk_balances_anonymous_block adds around the loop, and the statuses it reports:
  3  a member index out of range: the transaction touches nothing (its acc and verifier rows are zero bytes)
  2  a left or right point fails Point::read + as_prime_order: not applied (the verifier rejects the same point)
  1  the verdict is false (the mask byte is not 1)
  0  applied
A touched account whose stored ciphertext does not read raises balances.BadAccount at its first touch."""
from __future__ import annotations

from . import balances as bal

RING = 12
N_POINTS = 4 * RING + 4
APPLIED, NOT_APPLIED, BAD_POINT, BAD_INDEX = bal.APPLIED, bal.NOT_APPLIED, bal.BAD_POINT, bal.BAD_INDEX
ZERO = bal.ZERO


def apply_block(n_accounts: int, balance: dict, pending: dict, due: set, txs, verdict):
    """txs: (members, lefts, right) with 12 account indices and 32-byte points; verdict(k, acc) -> bool.  Returns (acc per
    transaction (12 ciphertexts, None for an index out of range), status, final State)."""
    st = bal.State(balance, pending, due)
    out_acc, out_st = [], []
    for k, (members, lefts, right) in enumerate(txs):
        if not all(0 <= m < n_accounts for m in members):
            out_acc.append(None); out_st.append(BAD_INDEX)
            continue
        for e in members:
            st.touch(e)
            st.rollover(e)
        acc = [st.balance.get(e, ZERO) for e in members]
        out_acc.append(acc)
        if not all(bal._point_ok(p) for p in list(lefts) + [right]):
            out_st.append(BAD_POINT)
            continue
        if not verdict(k, acc):
            out_st.append(NOT_APPLIED)
            continue
        for e, c in zip(members, lefts):
            enc_amount = bal.from_left_right(c, right)
            st.pending[e] = bal.ct_add(st.pending[e], enc_amount) if e in st.pending else enc_amount
        out_st.append(APPLIED)
    return out_acc, out_st, st


def verifier_points(keys: bytes, members, lefts, acc, right: bytes, rvk: bytes, g_epoch: bytes, nonce: bytes) -> bytes:
    """verify_anonymous_proof's pushes: enc_keys, left_ciphertexts, acc left points, acc right points, right_ciphertext,
    rvk, g_epoch, nonce"""
    return b"".join([keys[32 * m:32 * m + 32] for m in members] + list(lefts) + [c[:32] for c in acc] + [c[32:] for c in acc] +
                    [right, rvk, g_epoch, nonce])


def txs_of(members, tx_points: bytes):
    n = len(tx_points) // (32 * (RING + 1))
    rows = [[int(m) for m in members[RING * k:RING * k + RING]] for k in range(n)]
    return [(rows[k], [tx_points[32 * ((RING + 1) * k + i):32 * ((RING + 1) * k + i) + 32] for i in range(RING)],
             tx_points[32 * ((RING + 1) * k + RING):32 * ((RING + 1) * k + RING) + 32]) for k in range(n)]


def run_abi(keys: bytes, balances: bytes, pendings: bytes, flags, members, tx_points: bytes, tx_extra: bytes, g_epoch: bytes, applied):
    """zk_balances_anonymous_block's outputs by the loop: (enc_balances, verify_points, status, new_balances, new_pendings,
    new_flags), with applied[k] == 1 as the verdict."""
    members = [int(m) for m in members]
    txs = txs_of(members, tx_points)
    b, p, due = bal.from_arrays(balances, pendings, flags)
    accs, status, st = apply_block(len(flags), b, p, due, txs, lambda k, _: applied[k] == 1)
    eb, vp = [], []
    for k, ((mem, lefts, right), acc) in enumerate(zip(txs, accs)):
        if acc is None:
            eb.append(bytes(64 * RING)); vp.append(bytes(32 * N_POINTS))
            continue
        eb.append(b"".join(acc))
        vp.append(verifier_points(keys, mem, lefts, acc, right, tx_extra[64 * k:64 * k + 32], g_epoch, tx_extra[64 * k + 32:64 * k + 64]))
    return (b"".join(eb), b"".join(vp), bytes(status)) + bal.to_arrays(balances, pendings, flags, st)
