"""CPU checks of the balance-update oracles: the C loop (balances_oracle.c) against the Python restatement of the module's
loop (balances.py) on small blocks with every status, self-transfers, rollover rules and absent ciphertexts, and the rules
themselves on hand-made blocks."""
import pytest

from tests.jubjub_oracle import bal_coracle as bc
from tests.jubjub_oracle import bal_corpus
from tests.jubjub_oracle import balances as bal
from tests.jubjub_oracle import elgamal as eg


@pytest.mark.parametrize("seed, n_acct, n_tx", [(1, 5, 12), (2, 3, 20), (3, 9, 16)])
def test_c_oracle_equals_python_oracle(seed, n_acct, n_tx):
    b = bal_corpus.make(n_acct, n_tx, seed, bad_points=3, bad_index=True, zero_frac=0.3)
    bad, got = bc.block(*b.args())
    assert bad is None
    want = bal.run_abi(*b.args())
    assert got == want
    assert set(want[2]) == {0, 1, 2, 3}


def test_rules_by_hand():
    """one due account with a balance and a pending, one with neither; a self-transfer; an absent balance stays absent"""
    b = bal_corpus.make(3, 4, 7, zero_frac=0.0, self_frac=0.0)
    flags = bytes([bal.BALANCE | bal.PENDING | bal.DUE, bal.DUE, 0])
    sender, recipient = [0, 1, 2, 0], [1, 1, 0, 2]
    args = (b.balances, b.pendings, flags, sender, recipient, b.tx_points, b"\x01" * 4)
    bs, ba, st, nb, npd, nf = bal.run_abi(*args)
    assert bc.block(*args) == (None, (bs, ba, st, nb, npd, nf))
    assert st == bytes(4)
    rolled0 = bal.ct_add(b.balances[:64], b.pendings[:64])
    assert bs[:64] == rolled0                                  # rollover at the first touch
    assert bs[64:128] == bal.ZERO == eg.write(eg.ZERO)         # due with nothing: balance = zero + zero, present
    assert bs[128:192] == bal.ZERO                             # absent and not due: the verifier reads zero
    assert nf[2] & bal.BALANCE == 0 and nb[128:192] == bytes(64)   # ... and it stays absent after a send
    assert nf == bytes([bal.BALANCE | bal.PENDING, bal.BALANCE | bal.PENDING, bal.PENDING])
    # the last transaction of sender 0 sees its first one subtracted
    t = b.tx_points
    apf0 = bal.ct_add(bal.from_left_right(t[0:32], t[96:128]), bal.from_left_right(t[64:96], t[96:128]))
    assert bs[192:256] == ba[:64] == bal.ct_sub(rolled0, apf0)


def test_bad_account_is_reported():
    b = bal_corpus.make(4, 6, 9)
    balances = bytearray(b.balances)
    balances[64 * 2:64 * 2 + 32] = bal_corpus.BAD_FIELD
    flags = bytearray(b.flags)
    flags[2] |= bal.BALANCE
    args = (bytes(balances), b.pendings, bytes(flags), [0, 1, 2], [1, 0, 3], b.tx_points[:3 * 128], b"\x01" * 3)
    with pytest.raises(bal.BadAccount) as e:
        bal.run_abi(*args)
    assert e.value.account == 2
    assert bc.block(*args)[0] == 2
    # untouched: copied through
    args = (bytes(balances), b.pendings, bytes(flags), [0, 1], [1, 0], b.tx_points[:2 * 128], b"\x01" * 2)
    want = bal.run_abi(*args)
    assert bc.block(*args) == (None, want) and want[3][128:192] == bytes(balances[128:192])
