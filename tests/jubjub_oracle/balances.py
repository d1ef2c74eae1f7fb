"""TEST INFRASTRUCTURE (oracle): the confidential-transfer loop of modules/encrypted-balances, literally, on pyref.py and
elgamal.py.

Storage is three dicts keyed by account index, like the module's storage maps: balance (EncryptedBalance), pending
(PendingTransfer) and due (LastRollOver < current_epoch, worked out by the caller).  Every ciphertext operation works on
bytes the way core/primitives/src/ciphertext.rs:81-100 does: read both operands (Point::read + as_prime_order), operate,
write.  Per transaction (lib.rs:25-96):
  rollover(sender); rollover(recipient)          lib.rs:133-172, at most once per block per account (due is cleared)
  balance_sender = balance or Ciphertext::zero() what verify_confidential_proof reads
  verdict                                        verdict(k, balance_sender) -> bool (the proof check)
  sub_enc_balance; add_pending_transfer          lib.rs:174-222
  balance_after = balance or Ciphertext::zero()  the ConfidentialTransfer event

What zk_balances_confidential_block adds around the loop, and the statuses it reports:
  3  sender or recipient out of range: the transaction touches nothing (balance_sender = Ciphertext::zero())
  2  a transaction point fails Point::read + as_prime_order: not applied (the verifier rejects the same point)
  1  the verdict is false
  0  applied
A touched account whose stored balance or pending ciphertext does not read raises BadAccount at its first touch (the
reference would fail each transaction that touches it instead)."""
from __future__ import annotations

from . import elgamal as eg
from . import pyref as jj

APPLIED, NOT_APPLIED, BAD_POINT, BAD_INDEX = 0, 1, 2, 3
BALANCE, PENDING, DUE = 1, 2, 4
ZERO = eg.write(eg.ZERO)


class BadAccount(Exception):
    def __init__(self, account: int):
        super().__init__("account %d: a stored ciphertext fails Ciphertext::read" % account)
        self.account = account


def _read(b: bytes):
    ok, ct = eg.read(b)
    if not ok:
        raise ValueError("Ciphertext::read")
    return ct


def ct_add(a: bytes, b: bytes) -> bytes:
    """Ciphertext::add on bytes"""
    return eg.write(eg.add(_read(a), _read(b)))


def ct_sub(a: bytes, b: bytes) -> bytes:
    return eg.write(eg.sub(_read(a), _read(b)))


def from_left_right(left: bytes, right: bytes) -> bytes:
    """Ciphertext::from_left_right: both halves read (the LeftCiphertext / RightCiphertext conversions)"""
    return eg.write(_read(left + right))


def _point_ok(enc: bytes) -> bool:
    return jj.into_xy(enc)[0] == jj.OK


class State:
    def __init__(self, balance: dict, pending: dict, due: set):
        self.balance, self.pending, self.due = dict(balance), dict(pending), set(due)
        self.seen = set()

    def touch(self, a: int):
        """the deviation: a touched account's stored ciphertexts must read"""
        if a in self.seen:
            return
        self.seen.add(a)
        for store in (self.balance, self.pending):
            if a in store and not eg.read(store[a])[0]:
                raise BadAccount(a)

    def rollover(self, a: int):
        if a in self.due:
            pend = self.pending.get(a, ZERO)
            self.balance[a] = ct_add(self.balance[a], pend) if a in self.balance else pend
            self.pending.pop(a, None)
            self.due.discard(a)


def apply_block(n_accounts: int, balance: dict, pending: dict, due: set, txs, verdict):
    """txs: (sender, recipient, amount_sender, amount_recipient, fee_sender, randomness) with 32-byte points; verdict(k,
    balance_sender) -> bool.  Returns (balance_sender, balance_after (None unless applied), status, final State)."""
    st = State(balance, pending, due)
    out_bs, out_ba, out_st = [], [], []
    for k, (s, r, amount_s, amount_r, fee_s, rnd) in enumerate(txs):
        if not (0 <= s < n_accounts and 0 <= r < n_accounts):
            out_bs.append(ZERO); out_ba.append(None); out_st.append(BAD_INDEX)
            continue
        st.touch(s); st.touch(r)
        st.rollover(s)
        st.rollover(r)
        bs = st.balance.get(s, ZERO)
        out_bs.append(bs)
        if not all(_point_ok(p) for p in (amount_s, amount_r, fee_s, rnd)):
            out_ba.append(None); out_st.append(BAD_POINT)
            continue
        if not verdict(k, bs):
            out_ba.append(None); out_st.append(NOT_APPLIED)
            continue
        # sub_enc_balance (lib.rs:174-196)
        enc_amount = from_left_right(amount_s, rnd)
        enc_fee = from_left_right(fee_s, rnd)
        amount_plus_fee = ct_add(enc_amount, enc_fee)
        if s in st.balance:
            st.balance[s] = ct_sub(st.balance[s], amount_plus_fee)
        # add_pending_transfer (lib.rs:198-222)
        enc_amount_r = from_left_right(amount_r, rnd)
        st.pending[r] = ct_add(st.pending[r], enc_amount_r) if r in st.pending else enc_amount_r
        out_ba.append(st.balance.get(s, ZERO)); out_st.append(APPLIED)
    return out_bs, out_ba, out_st, st


def from_arrays(balances: bytes, pendings: bytes, flags):
    """the ABI's account arrays as the oracle's storage"""
    n = len(flags)
    bal = {a: balances[64 * a:64 * a + 64] for a in range(n) if flags[a] & BALANCE}
    pend = {a: pendings[64 * a:64 * a + 64] for a in range(n) if flags[a] & PENDING}
    return bal, pend, {a for a in range(n) if flags[a] & DUE}


def to_arrays(balances: bytes, pendings: bytes, flags, st: State):
    """the final storage in the ABI's layout: untouched accounts copied through, a touched account's absent ciphertexts
    zero, its flags' bits 0-2 replaced"""
    nb, npd, nf = bytearray(balances), bytearray(pendings), bytearray(flags)
    for a in st.seen:
        nb[64 * a:64 * a + 64] = st.balance.get(a, bytes(64))
        npd[64 * a:64 * a + 64] = st.pending.get(a, bytes(64))
        nf[a] = (flags[a] & ~7) | (BALANCE if a in st.balance else 0) | (PENDING if a in st.pending else 0)
    return bytes(nb), bytes(npd), bytes(nf)


def run_abi(balances: bytes, pendings: bytes, flags, sender, recipient, tx_points: bytes, applied, balance_after_in: bytes | None = None):
    """zk_balances_confidential_block's outputs by the loop: (balance_sender, balance_after, status, new_balances,
    new_pendings, new_flags), with the mask as the verdict.  balance_after starts as balance_after_in (zero bytes)."""
    n = len(sender)
    txs = [(int(sender[k]), int(recipient[k])) + tuple(tx_points[128 * k + 32 * i:128 * k + 32 * i + 32] for i in range(4))
           for k in range(n)]
    bal, pend, due = from_arrays(balances, pendings, flags)
    bs, ba, status, st = apply_block(len(flags), bal, pend, due, txs, lambda k, _: bool(applied[k]))
    after = bytearray(balance_after_in if balance_after_in is not None else bytes(64 * n))
    for k, b in enumerate(ba):
        if b is not None:
            after[64 * k:64 * k + 64] = b
    return (b"".join(bs), bytes(after), bytes(status)) + to_arrays(balances, pendings, flags, st)
