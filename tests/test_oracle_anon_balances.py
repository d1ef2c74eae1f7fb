"""CPU checks of the anonymous-transfer oracles: the C loop (anon_balances_oracle.c) against the Python restatement of the
module's loop (anon_balances.py) on small blocks with every status and every mask value, and the module's rules on
hand-made blocks: the rollover happens before the proof check and stands when the transaction is rejected, and a member
listed twice is rolled over once and receives both additions."""
import numpy as np
import pytest

from tests.jubjub_oracle import anon_balances as ab
from tests.jubjub_oracle import anon_coracle as aco
from tests.jubjub_oracle import anon_corpus
from tests.jubjub_oracle import balances as bal


@pytest.mark.parametrize("seed, n_acct, n_tx", [(1, 5, 6), (1, 20, 5)])
def test_c_oracle_equals_python_oracle(seed, n_acct, n_tx):
    b = anon_corpus.make(n_acct, n_tx, seed, bad_points=1, bad_index=True, dup_frac=0.5, mask_p=(0.2, 0.6, 0.0, 0.0, 0.2))
    bad, got = aco.block(*b.args())
    assert bad is None
    assert got == ab.run_abi(*b.args())
    assert set(got[2]) == {0, 1, 2, 3}


def _ring_block(applied: bytes, members, flags):
    b = anon_corpus.make(3, 1, 41, dup_frac=0.0)
    return (b.keys, b.balances, b.pendings, bytes(flags), np.array(members, np.uint32), b.tx_points, b.tx_extra, b.g_epoch, applied), b


def test_rejected_transaction_still_rolls_over():
    """account 0 is due with a balance and a pending: a transaction that fails its check still rolls it over"""
    flags = [bal.BALANCE | bal.PENDING | bal.DUE, bal.PENDING, 0]
    members = [0] * 6 + [1] * 3 + [2] * 3
    for mask in (b"\x00", b"\x04"):
        args, b = _ring_block(mask, members, flags)
        got = ab.run_abi(*args)
        assert aco.block(*args) == (None, got)
        assert got[2] == bytes([bal.NOT_APPLIED])
        rolled = bal.ct_add(b.balances[:64], b.pendings[:64])
        assert got[0][:64] == rolled and got[3][:64] == rolled            # the verifier reads the rolled balance; it stays
        assert got[5] == bytes([bal.BALANCE, bal.PENDING, 0])             # pending of 0 moved over, not due any more
        assert got[4][:64] == bytes(64) and got[4][64:128] == b.pendings[64:128]
        assert got[0][64 * 6:64 * 7] == bal.ZERO                          # account 1: no balance, not due: zero
        # the verifier's inputs: keys, lefts, acc left halves, acc right halves, right, rvk, g_epoch, nonce
        vp = got[1]
        assert vp[:32] == b.keys[:32] and vp[32 * 12:32 * 13] == b.tx_points[:32]
        assert vp[32 * 24:32 * 25] == rolled[:32] and vp[32 * 36:32 * 37] == rolled[32:]
        assert vp[32 * 48:] == b.tx_points[32 * 12:32 * 13] + b.tx_extra[:32] + b.g_epoch + b.tx_extra[32:64]


def test_member_listed_twice_gets_both_additions():
    flags = [bal.BALANCE | bal.DUE, 0, bal.PENDING]
    members = [1, 1] + [0] * 5 + [2] * 5
    args, b = _ring_block(b"\x01", members, flags)
    got = ab.run_abi(*args)
    assert aco.block(*args) == (None, got)
    assert got[2] == bytes([bal.APPLIED])
    t = b.tx_points
    right = t[32 * 12:32 * 13]
    want1 = bal.ct_add(bal.from_left_right(t[0:32], right), bal.from_left_right(t[32:64], right))
    assert got[4][64:128] == want1 and got[5][1] == bal.PENDING
    want2 = b.pendings[128:192]
    for i in range(7, 12):
        want2 = bal.ct_add(want2, bal.from_left_right(t[32 * i:32 * i + 32], right))
    assert got[4][128:192] == want2
