"""CPU checks of the public-input layout helpers: they must put the points in the order modules/zk-system's
PublicInputBuilder pushes them (lib.rs:69-100 for a confidential transfer, lib.rs:128-153 for an anonymous one)."""
import pytest

from zero_chain_b200 import groth16 as zk


def _pt(tag: int) -> bytes:
    return bytes([tag]) * 32


def test_confidential_points_order():
    got = zk.confidential_points(address_sender=_pt(1), address_recipient=_pt(2), amount_sender=_pt(3), amount_recipient=_pt(4),
                                 randomness=_pt(5), fee_sender=_pt(6), balance_sender=_pt(7) + _pt(8), rvk=_pt(9),
                                 g_epoch=_pt(10), nonce=_pt(11))
    assert len(got) == 32 * zk.CONFIDENTIAL_POINTS == 352
    assert [got[32 * i] for i in range(11)] == list(range(1, 12))    # randomness before fee_sender; balance left, then right
    with pytest.raises(AssertionError):
        zk.confidential_points(*([_pt(1)] * 6), _pt(7), *([_pt(1)] * 3))   # a Ciphertext is 64 bytes


def test_anonymous_points_order():
    n = zk.ANONIMITY_SIZE
    keys = [_pt(i) for i in range(n)]
    lefts = [_pt(20 + i) for i in range(n)]
    bals = [_pt(40 + i) + _pt(60 + i) for i in range(n)]
    got = zk.anonymous_points(keys, lefts, bals, _pt(100), _pt(101), _pt(102), _pt(103))
    assert len(got) == 32 * zk.ANONYMOUS_POINTS == 32 * 52
    want = list(range(n)) + [20 + i for i in range(n)] + [40 + i for i in range(n)] + [60 + i for i in range(n)] + [100, 101, 102, 103]
    assert [got[32 * i] for i in range(52)] == want
