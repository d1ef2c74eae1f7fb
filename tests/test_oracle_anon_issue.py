"""CPU checks of the oracles of both anonymous-balances calls: the C loop (anon_issue_oracle.c) against the Python
restatement of the module's loop (anon_issue.py) on small mixed blocks with every status, and each rule of issue on
hand-made blocks: an issue before the first touch (due and not due), after it, two issues to one account, a failed issue,
an account only issues name, and statuses 2 and 3 of an issue."""
import numpy as np
import pytest

from tests.jubjub_oracle import anon_corpus
from tests.jubjub_oracle import anon_issue as ai
from tests.jubjub_oracle import anon_issue_coracle as aic
from tests.jubjub_oracle import anon_issue_corpus
from tests.jubjub_oracle import bal_corpus
from tests.jubjub_oracle import balances as bal

DUE_FULL = bal.BALANCE | bal.PENDING | bal.DUE


@pytest.mark.parametrize("seed, n_acct, n_tx", [(71, 8, 12), (72, 20, 10)])
def test_c_oracle_equals_python_oracle(seed, n_acct, n_tx):
    b = anon_issue_corpus.make(n_acct, n_tx, seed, issue_frac=0.35, bad_issue_points=2, bad_kind=True, bad_points=1, bad_index=True,
                               dup_frac=0.5, mask_p=(0.2, 0.6, 0.0, 0.0, 0.2))
    bad, got = aic.block(*b.args())
    assert bad is None
    assert got == ai.run_abi(*b.args())
    assert set(got[3]) == {0, 1, 2, 3}


def _block(kinds, rings, flags, applied, n_acct=13):
    """transactions of the given kinds; an issue's issuer is its ring's first member"""
    b = anon_corpus.make(n_acct, len(kinds), 81, dup_frac=0.0)
    members = np.array(rings, np.uint32).reshape(-1)
    args = (b.keys, b.balances, b.pendings, bytes(flags) + b.flags[len(flags):], bytes(kinds), members, b.tx_points, b.tx_extra,
            b.g_epoch, bytes(applied))
    got = ai.run_abi(*args)
    assert aic.block(*args) == (None, got)
    return got, b


def _issued(b, k):
    t = b.tx_points
    return bal.from_left_right(t[416 * k:416 * k + 32], t[416 * k + 384:416 * k + 416])


RING = list(range(12))


@pytest.mark.parametrize("due", [False, True])
def test_issue_before_first_touch(due):
    f0 = DUE_FULL if due else bal.BALANCE | bal.PENDING
    got, b = _block([1, 0], [[0] * 12, RING], [f0], [1, 1])
    iss = _issued(b, 0)
    rolled = bal.ct_add(iss, b.pendings[:64]) if due else iss
    assert got[2][:64] == iss and got[3] == bytes([0, 0])
    assert got[0][768:768 + 64] == rolled                            # the transfer reads the issued balance, rolled over
    assert got[4][:64] == rolled
    assert got[6][0] & 7 == (bal.BALANCE | bal.PENDING)              # the transfer's own addition is pending


def test_issue_after_first_touch():
    got, b = _block([0, 1, 0], [RING, [0] * 12, RING], [DUE_FULL], [1, 1, 0])
    rolled = bal.ct_add(b.balances[:64], b.pendings[:64])
    iss = _issued(b, 1)
    assert got[0][:64] == rolled and got[0][768 * 2:768 * 2 + 64] == iss
    assert got[4][:64] == iss and got[6][0] & 7 == bal.BALANCE | bal.PENDING


def test_two_issues_to_one_account():
    got, b = _block([1, 0, 1, 1, 0], [[0] * 12, RING, [0] * 12, [0] * 12, RING], [bal.BALANCE], [1, 0, 1, 1, 0])
    assert got[0][768:768 + 64] == _issued(b, 0)
    assert got[0][768 * 4:768 * 4 + 64] == _issued(b, 3)             # the later of the two
    assert got[4][:64] == _issued(b, 3) and got[2][128:256] == _issued(b, 2) + _issued(b, 3)


def test_failed_issue_changes_nothing():
    got, b = _block([1, 0], [[0] * 12, RING], [bal.BALANCE], [0, 1])
    assert got[3] == bytes([1, 0]) and got[2] == bytes(128)
    assert got[0][768:768 + 64] == b.balances[:64]


def test_issue_only_account_keeps_due_bit_and_pending():
    got, b = _block([1, 0], [[12] * 12, RING], [], [1, 1])
    flags12 = b.flags[12]
    assert got[4][64 * 12:] == _issued(b, 0) and got[5][64 * 12:] == b.pendings[64 * 12:]
    assert got[6][12] == flags12 | bal.BALANCE


def test_issue_statuses():
    b = anon_corpus.make(13, 3, 81, dup_frac=0.0)
    t = bytearray(b.tx_points)
    t[384:416] = bal_corpus.bad_curve()                              # issue 0: randomness rejected
    t[416 + 32:416 + 64] = bal_corpus.BAD_FIELD                      # issue 1: an ignored slot, applied
    members = np.array([[0] * 12, [1] + [99] * 11, [13] * 12], np.uint32).reshape(-1)
    args = (b.keys, b.balances, b.pendings, b.flags, bytes([1, 1, 1]), members, bytes(t), b.tx_extra, b.g_epoch, b"\x01" * 3)
    got = ai.run_abi(*args)
    assert aic.block(*args) == (None, got)
    assert got[3] == bytes([2, 0, 3])
    assert got[0] == bytes(768 * 3) and got[1] == bytes(1664 * 3)
    assert aic.block(*args[:4] + (bytes([1, 2, 1]),) + args[5:])[1][3] == bytes([2, 3, 3])
