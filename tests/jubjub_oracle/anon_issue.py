"""TEST INFRASTRUCTURE (oracle): both calls of modules/anonymous-balances, anonymous_transfer and issue, literally and in
block order, on balances.py and anon_balances.py.

Storage is balances.State as in anon_balances.py.  Per transaction:
  anonymous_transfer (lib.rs:23-82)             as anon_balances.apply_block
  issue (lib.rs:87-134)                         verdict(k, None) (the proof check reads only the extrinsic's fields),
                                                then EncryptedBalance(issuer) = from_left_right(total, randomness): no
                                                rollover, the pending and the due bit stay; the Issued event carries it

What zk_anonymous_calls_block adds around the loop, and the statuses it reports for an issue:
  3  the issuer out of range, or a kind other than 0 and 1 (the transaction touches nothing; its rows are zero bytes)
  2  total or randomness fails Point::read + as_prime_order (the verifier rejects the same point)
  1  the verdict is false
  0  applied
An account a transfer touches must have stored ciphertexts that read, checked against what was stored before the block
(an issue before its first touch does not excuse it): balances.BadAccount at its first touch."""
from __future__ import annotations

from . import anon_balances as ab
from . import balances as bal

TRANSFER, ISSUE = 0, 1
RING = ab.RING
ZERO = bal.ZERO


def apply_block(n_accounts: int, balance: dict, pending: dict, due: set, txs, verdict):
    """txs: (kind, members, lefts, right) with 12 account indices and 32-byte points; an issue's issuer is members[0], its
    total lefts[0] and its randomness right.  verdict(k, acc) -> bool, acc None for an issue.  Returns (acc per transaction
    (12 ciphertexts, None for an issue or an index out of range), issued (the Issued ciphertext of an applied issue, else
    None), status, final State)."""
    st = bal.State(balance, pending, due)
    unreadable = {a for store in (balance, pending) for a, c in store.items() if not bal.eg.read(c)[0]}
    out_acc, out_issued, out_st = [], [], []
    for k, (kind, members, lefts, right) in enumerate(txs):
        out_acc.append(None); out_issued.append(None)
        if kind == ISSUE:
            issuer, total = members[0], lefts[0]
            if not 0 <= issuer < n_accounts:
                out_st.append(ab.BAD_INDEX)
            elif not (bal._point_ok(total) and bal._point_ok(right)):
                out_st.append(ab.BAD_POINT)
            elif not verdict(k, None):
                out_st.append(ab.NOT_APPLIED)
            else:
                ct = bal.from_left_right(total, right)
                st.balance[issuer] = ct
                out_issued[k] = ct
                out_st.append(ab.APPLIED)
            continue
        if kind != TRANSFER or not all(0 <= m < n_accounts for m in members):
            out_st.append(ab.BAD_INDEX)
            continue
        for e in members:
            if e not in st.seen:
                st.seen.add(e)
                if e in unreadable:
                    raise bal.BadAccount(e)
            st.rollover(e)
        acc = [st.balance.get(e, ZERO) for e in members]
        out_acc[k] = acc
        if not all(bal._point_ok(p) for p in list(lefts) + [right]):
            out_st.append(ab.BAD_POINT)
            continue
        if not verdict(k, acc):
            out_st.append(ab.NOT_APPLIED)
            continue
        for e, c in zip(members, lefts):
            enc_amount = bal.from_left_right(c, right)
            st.pending[e] = bal.ct_add(st.pending[e], enc_amount) if e in st.pending else enc_amount
        out_st.append(ab.APPLIED)
    return out_acc, out_issued, out_st, st


def txs_of(kind, members, tx_points: bytes):
    return [(int(kd),) + t for kd, t in zip(bytes(kind), ab.txs_of(members, tx_points))]


def to_arrays(balances: bytes, pendings: bytes, flags, st: bal.State, issuers):
    """balances.to_arrays, and an account of issuers (applied issues) no transfer touched: the issued balance, its pending
    bytes and its other flags kept"""
    nb, npd, nf = (bytearray(x) for x in bal.to_arrays(balances, pendings, flags, st))
    for a in set(issuers) - st.seen:
        nb[64 * a:64 * a + 64] = st.balance[a]
        nf[a] |= bal.BALANCE
    return bytes(nb), bytes(npd), bytes(nf)


def run_abi(keys: bytes, balances: bytes, pendings: bytes, flags, kind, members, tx_points: bytes, tx_extra: bytes, g_epoch: bytes,
            applied, issued_in: bytes | None = None):
    """zk_anonymous_calls_block's outputs by the loop: (enc_balances, verify_points, issued, status, new_balances,
    new_pendings, new_flags), with applied[k] == 1 as the verdict; issued starts as issued_in (zero bytes)."""
    members = [int(m) for m in members]
    txs = txs_of(kind, members, tx_points)
    b, p, due = bal.from_arrays(balances, pendings, flags)
    accs, issued, status, st = apply_block(len(flags), b, p, due, txs, lambda k, _: applied[k] == 1)
    eb, vp = [], []
    for k, ((_, mem, lefts, right), acc) in enumerate(zip(txs, accs)):
        if acc is None:
            eb.append(bytes(64 * RING)); vp.append(bytes(32 * ab.N_POINTS))
            continue
        eb.append(b"".join(acc))
        vp.append(ab.verifier_points(keys, mem, lefts, acc, right, tx_extra[64 * k:64 * k + 32], g_epoch, tx_extra[64 * k + 32:64 * k + 64]))
    out_issued = bytearray(issued_in if issued_in is not None else bytes(64 * len(txs)))
    for k, c in enumerate(issued):
        if c is not None:
            out_issued[64 * k:64 * k + 64] = c
    issuers = [txs[k][1][0] for k, c in enumerate(issued) if c is not None]
    return (b"".join(eb), b"".join(vp), bytes(out_issued), bytes(status)) + to_arrays(balances, pendings, flags, st, issuers)
