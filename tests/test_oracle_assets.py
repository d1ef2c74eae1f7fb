"""CPU checks of the encrypted-asset oracles: the C loop (assets_oracle.c) against the Python restatement of the module's
loop (assets.py) on random blocks of mixed kinds, and each rule of the module on hand-made blocks."""
import pytest

from tests.jubjub_oracle import assets as asr
from tests.jubjub_oracle import assets_coracle as ac
from tests.jubjub_oracle import assets_corpus
from tests.jubjub_oracle import bal_corpus
from tests.jubjub_oracle import balances as bal

T, I, D = asr.TRANSFER, asr.ISSUE, asr.DESTROY
B, P, DUE = bal.BALANCE, bal.PENDING, bal.DUE


@pytest.mark.parametrize("seed, n_slots, n_tx", [(1, 5, 12), (2, 3, 16), (3, 9, 12)])
def test_c_oracle_equals_python_oracle(seed, n_slots, n_tx):
    b = assets_corpus.make(n_slots, n_tx, seed, issue_frac=0.2, destroy_frac=0.15, bad_points=3, bad_index=True, zero_frac=0.3)
    bad, got = ac.block(*b.args())
    assert bad is None
    want = asr.run_abi(*b.args())
    assert got == want
    assert set(want[4]) == {0, 1, 2, 3}
    assert {0, 1, 2} <= set(b.kind)


class _Hand:
    """a block over the stored ciphertexts of a corpus table; rows (kind, slot_a, slot_b) take the valid points of a
    transfer corpus (an issue reads the first and the last as total and randomness)"""

    def __init__(self, flags, rows, applied=None, seed=7, tx_points=None):
        t = bal_corpus.make(len(flags), max(len(rows), 1), seed, zero_frac=0.0)
        self.balances, self.pendings, self.flags = t.balances, t.pendings, bytes(flags)
        self.kind = bytes(r[0] for r in rows)
        self.slot_a, self.slot_b = [r[1] for r in rows], [r[2] for r in rows]
        self.tx_points = tx_points if tx_points is not None else t.tx_points[:128 * len(rows)]
        self.applied = bytes(applied) if applied is not None else b"\x01" * len(rows)

    def args(self):
        return (self.balances, self.pendings, self.flags, self.kind, self.slot_a, self.slot_b, self.tx_points, self.applied)

    def run(self):
        want = asr.run_abi(*self.args())
        assert ac.block(*self.args()) == (None, want)
        return want

    def pt(self, k, i):
        return self.tx_points[128 * k + 32 * i:128 * k + 32 * i + 32]

    def ct(self, which, s):
        return (self.balances if which == B else self.pendings)[64 * s:64 * s + 64]


def _row(b, k, n=64):
    return b[n * k:n * k + n]


def test_issue_then_transfer_rolls_over_total_plus_pending():
    h = _Hand([B | P | DUE, 0], [(I, 0, 0), (T, 0, 1)])
    bs, ba, ev, evf, st, nb, npd, nf = h.run()
    total = bal.from_left_right(h.pt(0, 0), h.pt(0, 3))
    assert st == bytes(2) and _row(ev, 0, 128) == total + bytes(64) and evf[0] == 1
    assert _row(bs, 1) == bal.ct_add(total, h.ct(P, 0))                  # the stored balance is gone, the pending rolled in
    assert nf[0] == B and _row(npd, 0) == bytes(64)


def test_destroy_then_transfer_touch_gives_a_present_zero():
    h = _Hand([B | P | DUE, 0], [(D, 0, 0), (T, 0, 1)], applied=[1, 0])
    bs, ba, ev, evf, st, nb, npd, nf = h.run()
    assert st == bytes([0, 1])
    assert _row(ev, 0, 128) == h.ct(B, 0) + h.ct(P, 0) and evf[0] == 3
    assert _row(bs, 1) == bal.ZERO and _row(nb, 0) == bal.ZERO and nf[0] == B and _row(npd, 0) == bytes(64)


def test_rollover_then_destroy_then_send():
    h = _Hand([B | P | DUE, 0], [(T, 0, 1), (D, 0, 0), (T, 0, 1)])
    bs, ba, ev, evf, st, nb, npd, nf = h.run()
    rolled = bal.ct_add(h.ct(B, 0), h.ct(P, 0))
    assert _row(bs, 0) == rolled and st == bytes(3)
    assert _row(ev, 1, 128) == _row(ba, 0) + bytes(64) and evf[1] == 1      # the balance after the first send; no pending
    assert _row(bs, 2) == bal.ZERO and _row(ba, 2) == bal.ZERO              # absent: the verifier reads zero ...
    assert nf[0] == 0 and _row(nb, 0) == bytes(64)                          # ... and it stays absent


def test_destroy_twice_takes_nothing_the_second_time():
    h = _Hand([B | P, 0], [(D, 0, 0), (D, 0, 0)])
    bs, ba, ev, evf, st, nb, npd, nf = h.run()
    assert evf == bytes([3, 0]) and _row(ev, 1, 128) == bytes(128) and bs == bytes(128)
    assert nf[0] == 0 and _row(nb, 0) == _row(npd, 0) == bytes(64)


def test_issue_keeps_the_pending_transfer():
    h = _Hand([P, 0], [(I, 0, 0)])
    bs, ba, ev, evf, st, nb, npd, nf = h.run()
    assert nf[0] == B | P and _row(npd, 0) == h.ct(P, 0) and _row(nb, 0) == bal.from_left_right(h.pt(0, 0), h.pt(0, 3))


def test_calls_not_applied_change_nothing_and_keep_due():
    h = _Hand([B | P | DUE | 0x40, 0], [(I, 0, 0), (D, 0, 0), (I, 0, 1)], applied=[0, 2, 4])
    bs, ba, ev, evf, st, nb, npd, nf = h.run()
    assert st == bytes([1, 1, 1]) and ev == bytes(3 * 128) and evf == bytes(3)
    assert (nb, npd, nf) == (h.balances, h.pendings, h.flags)


def test_transfers_only_equal_the_confidential_loop():
    """a self-transfer of a due slot, then a random transfer block: the same bytes as modules/encrypted-balances' loop"""
    h = _Hand([B | P | DUE, P | DUE, 0], [(T, 0, 0), (T, 1, 1), (T, 2, 0)], applied=[1, 1, 0])
    got = h.run()
    conf = bal.run_abi(h.balances, h.pendings, h.flags, h.slot_a, h.slot_b, h.tx_points, h.applied)
    assert (got[0], got[1], got[4]) + got[5:] == conf[:3] + conf[3:]
    assert _row(got[0], 0) == bal.ct_add(h.ct(B, 0), h.ct(P, 0))
    b = assets_corpus.make(6, 16, 11, issue_frac=0.0, destroy_frac=0.0, bad_points=3, bad_index=False)
    b.applied = bytes(int(v == 1) for v in b.applied)                     # the confidential call applies any nonzero mask
    got = asr.run_abi(*b.args())
    conf = bal.run_abi(*b.transfers())
    assert (got[0], got[1], got[4]) + got[5:] == conf


def test_issue_with_a_rejected_point():
    for i in (0, 3):
        h = _Hand([B, 0], [(I, 0, 0)])
        pts = bytearray(h.tx_points)
        pts[32 * i:32 * i + 32] = bal_corpus.bad_curve()
        pts[32:96] = bal_corpus.BAD_FIELD * 2                             # ignored
        h.tx_points = bytes(pts)
        bs, ba, ev, evf, st, nb, npd, nf = h.run()
        assert st == bytes([2]) and (nb, nf) == (h.balances, h.flags)
    h = _Hand([B, 0], [(I, 0, 0)])
    pts = bytearray(h.tx_points)
    pts[32:96] = bal_corpus.BAD_FIELD * 2
    h.tx_points = bytes(pts)
    assert h.run()[4] == bytes([0])


def test_invalid_slot_or_kind_touches_nothing():
    h = _Hand([B | P | DUE, DUE], [(T, 0, 2), (I, 5, 0), (D, 2, 0), (3, 0, 0), (T, 1, 0xFFFFFFFF)])
    bs, ba, ev, evf, st, nb, npd, nf = h.run()
    assert st == bytes([3] * 5)
    assert _row(bs, 0) == _row(bs, 4) == bal.ZERO and bs[64:256] == bytes(192)
    assert (nb, npd, nf) == (h.balances, h.pendings, h.flags)


def test_bad_slot_is_reported():
    h = _Hand([B, B, 0], [(T, 0, 1), (I, 2, 0)])
    balances = bytearray(h.balances)
    balances[64 * 2:64 * 2 + 32] = bal_corpus.BAD_FIELD
    h.balances, h.flags = bytes(balances), bytes([B, B, B])
    with pytest.raises(bal.BadAccount) as e:
        asr.run_abi(*h.args())
    assert e.value.account == 2 and ac.block(*h.args())[0] == 2
    h.slot_a[1] = 1                                                       # not named: copied through
    want = h.run()
    assert want[5][128:192] == bytes(balances[128:192])
