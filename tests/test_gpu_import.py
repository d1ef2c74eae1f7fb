"""GPU tests of the block imports with their rounds on the device, zk_import_confidential_block / zk_import_assets_block and
their _device forms (groth16.confidential_import / assets_import), against the Python drivers import_confidential_block /
import_assets_block and the C oracles (balances_oracle.c, assets_oracle.c).

Proofs are forged from a toy key's trapdoor (tests/import_corpus.py): a passing transfer's proof is valid only against the
balance that excludes its chain's earlier failures, so every failure costs a round.  Covered: a random block of thousands
of transfers with failures and rejected points; 1, 2 and 5 failures in one chain, in the middle and at its end; a chain
longer than a thread block; an empty block; an all-failing block; an asset block whose issues and destroys fail; an
undecodable touched account; an index out of range; and the device forms against the host forms."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import import_corpus as ic
from tests.jubjub_oracle import bal_corpus
from zero_chain_b200 import _lib
from zero_chain_b200 import groth16 as zk

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def key(ctx):
    k = ic.ForgeKey(5)
    k.pvk = zk.PreparedVerifyingKey.prepare(ctx, k.params_bytes)
    yield k
    k.pvk.free()


def _conf_state(ctx):
    return lambda *a: zk.confidential_block(ctx, *a)


def _assets_state(ctx):
    return lambda *a: zk.assets_block(ctx, *a)


def check_confidential(ctx, key, blk, rounds=None):
    """the new call against the driver, the intended verdicts and the C oracle; returns the rounds"""
    got = zk.confidential_import(ctx, key.pvk, blk.accounts, blk.txs, blk.proofs)
    want = zk.import_confidential_block(ctx, key.pvk, blk.accounts, blk.txs, blk.proofs)
    assert got == want
    verdicts, (nb, npd, nf), after, r = got
    assert verdicts == blk.intended
    o = blk.oracle(verdicts)
    assert (o[0], o[2], o[3], o[4]) == (after, nb, npd, nf)
    if rounds is not None:
        assert r == rounds
    return r


def test_random_block_equals_driver_and_oracle(ctx, key):
    blk = ic.confidential(key, 200, 3000, 31, fail_frac=0.03, skew=1.2, bad_points=6, state_call=_conf_state(ctx))
    assert zk.VERDICT_INPUT_REJECTED in blk.intended and 0 in blk.intended
    assert check_confidential(ctx, key, blk) > 2


@pytest.mark.parametrize("fails, rounds", [((), 1), ((3,), 2), ((3, 7), 3), ((1, 2, 5, 8, 10), 6), ((4, 11), 2), ((0, 11), 2)])
def test_failures_in_one_chain(ctx, key, fails, rounds):
    """sender 0 sends 12 transfers; 1 + (its failures) rounds, one fewer when the last failure is its last transfer"""
    blk = ic.confidential(key, 4, 12, 32, fail_at=fails, sender=[0] * 12, state_call=_conf_state(ctx))
    assert [k for k, v in enumerate(blk.intended) if v != 1] == list(fails)
    check_confidential(ctx, key, blk, rounds)


def test_chain_longer_than_a_thread_block(ctx, key):
    n = 1100
    blk = ic.confidential(key, 3, n, 33, fail_at=(5, 700, 1050), sender=[1] * n, state_call=_conf_state(ctx))
    check_confidential(ctx, key, blk, 4)


def test_empty_block(ctx, key):
    b = bal_corpus.make(30, 0, 34)
    accounts = (b.balances, b.pendings, b.flags)
    assert zk.confidential_import(ctx, key.pvk, accounts, [], []) == ([], accounts, b"", 0) == \
        zk.import_confidential_block(ctx, key.pvk, accounts, [], [])


def test_all_failing_block(ctx, key):
    blk = ic.confidential(key, 5, 60, 35, fail_frac=1.0, skew=0.0, state_call=_conf_state(ctx))
    assert set(blk.intended) == {0}
    longest = np.bincount([t.sender for t in blk.txs]).max()
    check_confidential(ctx, key, blk, longest)


def test_undecodable_touched_account(ctx, key):
    blk = ic.confidential(key, 20, 40, 36, fail_frac=0.1, state_call=_conf_state(ctx))
    bal_b, flags = bytearray(blk.accounts[0]), bytearray(blk.accounts[2])
    a = blk.txs[3].recipient
    bal_b[64 * a + 32:64 * a + 64] = bal_corpus.bad_order(bytes(bal_b[64 * a + 32:64 * a + 64]))
    flags[a] |= zk.ACCOUNT_BALANCE
    accounts = (bytes(bal_b), blk.accounts[1], bytes(flags))
    for fn in (zk.confidential_import, zk.import_confidential_block):
        with pytest.raises(zk.SynthesisError) as e:
            fn(ctx, key.pvk, accounts, blk.txs, blk.proofs)
        assert e.value.code == -7 and "account %d" % a in str(e.value)
    assert zk.confidential_import(ctx, key.pvk, blk.accounts, blk.txs, blk.proofs)[0] == blk.intended    # the context recovers


def test_index_out_of_range(ctx, key):
    blk = ic.confidential(key, 10, 20, 37, state_call=_conf_state(ctx))
    blk.txs[13].recipient = 10
    blk.txs[17].sender = 99
    with pytest.raises(ValueError):
        zk.import_confidential_block(ctx, key.pvk, blk.accounts, blk.txs, blk.proofs)
    with pytest.raises(ValueError) as e:
        zk.confidential_import(ctx, key.pvk, blk.accounts, blk.txs, blk.proofs)
    assert "transaction 13" in str(e.value)
    # the C call itself: ZK_ERR_INVALID naming the transaction
    L = _lib.lib()
    n = len(blk.txs)
    u8 = lambda b: np.frombuffer(bytes(b), np.uint8)
    out = [np.zeros(64 * n, np.uint8) for _ in range(6)]
    rounds = C.c_uint(7)
    rc = L.zk_import_confidential_block(ctx._h, key.pvk._h, 10, zk._p(u8(blk.accounts[0])), zk._p(u8(blk.accounts[1])),
                                        zk._p(u8(blk.accounts[2])), n, zk._p(np.array([t.sender for t in blk.txs], np.uint32)),
                                        zk._p(np.array([t.recipient for t in blk.txs], np.uint32)),
                                        zk._p(u8(zk._confidential_rows(blk.txs))), zk._p(u8(b"".join(blk.proofs))),
                                        *[zk._p(o) for o in out], C.byref(rounds))
    assert rc == -2 and b"transaction 13" in L.zk_last_error() and rounds.value == 0
    # an asset block: a transfer's slot past the table
    ab = ic.assets(key, 6, 30, 38, state_call=_assets_state(ctx))
    t = next(k for k, x in enumerate(ab.txs) if x.kind == zk.ASSET_TRANSFER)
    slots, table, slot_a, slot_b = ab.slots(ab.intended)
    slot_b[t] = len(slots) + 3
    args = _asset_arrays(ab, table, slot_a, slot_b)
    outs = _asset_outputs(len(ab.txs), len(slots))
    rc = L.zk_import_assets_block(ctx._h, key.pvk._h, len(slots), *[zk._p(a) for a in args[:3]], len(ab.txs), *[zk._p(a) for a in args[3:]],
                                  *[zk._p(o) for o in outs], C.byref(rounds))
    assert rc == -2 and ("transaction %d" % t).encode() in L.zk_last_error()


# ---- encrypted assets ---------------------------------------------------------------------------------------------------
def _asset_arrays(ab, table, slot_a, slot_b):
    """the host arrays of zk_import_assets_block: balances, pendings, flags, kind, slot_a, slot_b, tx_points, rows, proofs,
    fixed verdicts"""
    u8 = lambda b: np.frombuffer(bytes(b), np.uint8).copy() if len(b) else np.zeros(1, np.uint8)
    rows = b"".join(x.verify_points(bytes(64)) if x.kind == zk.ASSET_TRANSFER else bytes(352) for x in ab.txs)
    fixed = bytes(v if x.kind != zk.ASSET_TRANSFER else 0 for x, v in zip(ab.txs, ab.intended))
    return [u8(table[0]), u8(table[1]), u8(table[2]), u8(bytes(x.kind for x in ab.txs)), np.asarray(slot_a, np.uint32),
            np.asarray(slot_b, np.uint32), u8(b"".join(x.points() for x in ab.txs)), u8(rows), u8(b"".join(ab.proofs)), u8(fixed)]


def _asset_outputs(n, n_slots):
    z = lambda m: np.zeros(max(m, 1), np.uint8)
    return [z(n), z(64 * n), z(128 * n), z(n), z(n), z(64 * n_slots), z(64 * n_slots), z(n_slots)]


def check_assets(ctx, key, ab, rounds=None):
    got = zk.assets_import(ctx, key.pvk, *ab.args())
    want = zk.import_assets_block(ctx, key.pvk, *ab.args())
    assert got == want
    verdicts, ids, events, (slots, nb, npd, nf), r = got
    assert verdicts == ab.intended
    out = ab.oracle(verdicts)
    assert (nb, npd, nf) == out[5:]
    st = out[4]
    for k, t in enumerate(ab.txs):
        if st[k] != zk.BLOCK_APPLIED:
            assert events[k] is None
        elif t.kind == zk.ASSET_TRANSFER:
            assert events[k] == out[1][64 * k:64 * k + 64]
    if rounds is not None:
        assert r == rounds
    return r


def test_asset_block_equals_driver_and_oracle(ctx, key):
    ab = ic.assets(key, 100, 1500, 41, fail_frac=0.03, fixed_fail_frac=0.2, skew=1.1, state_call=_assets_state(ctx))
    kinds = {t.kind for t in ab.txs}
    assert kinds == {zk.ASSET_TRANSFER, zk.ASSET_ISSUE, zk.ASSET_DESTROY}
    assert check_assets(ctx, key, ab) > 1


def test_asset_block_whose_issues_and_destroys_fail(ctx, key):
    ab = ic.assets(key, 8, 120, 42, fixed_fail_frac=1.0, issue_frac=0.2, destroy_frac=0.2, state_call=_assets_state(ctx))
    assert all(v == 0 for t, v in zip(ab.txs, ab.intended) if t.kind != zk.ASSET_TRANSFER)
    check_assets(ctx, key, ab, 1)
    empty = ic.AssetBlock(ab.state, [], [], [], 10, zk.ACCOUNT_DUE)
    assert check_assets(ctx, key, empty, 0) == 0


# ---- the device forms ---------------------------------------------------------------------------------------------------
def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).cuda()


def test_device_forms_equal_host_forms(ctx, key):
    blk = ic.confidential(key, 50, 400, 43, fail_frac=0.05, skew=1.3, state_call=_conf_state(ctx))
    n, na = len(blk.txs), len(blk.accounts[2])
    u8 = lambda b: np.frombuffer(bytes(b), np.uint8)
    ins = [_dev(u8(blk.accounts[0])), _dev(u8(blk.accounts[1])), _dev(u8(blk.accounts[2])),
           _dev(np.array([t.sender for t in blk.txs], np.uint32)), _dev(np.array([t.recipient for t in blk.txs], np.uint32)),
           _dev(u8(zk._confidential_rows(blk.txs))), _dev(u8(b"".join(blk.proofs)))]
    outs = [torch.full((m,), 0xAB, dtype=torch.uint8, device="cuda") for m in (n, 64 * n, n, 64 * na, 64 * na, na)]
    torch.cuda.synchronize()
    p = [t.data_ptr() for t in ins]
    r = zk.confidential_import_device(ctx, key.pvk, na, p[0], p[1], p[2], n, *p[3:], *[t.data_ptr() for t in outs])
    got = [t.cpu().numpy().tobytes() for t in outs]
    verdicts, (nb, npd, nf), after, rounds = zk.confidential_import(ctx, key.pvk, blk.accounts, blk.txs, blk.proofs)
    assert r == rounds > 1
    assert got[0] == bytes(verdicts) and got[1] == after and got[3:] == [nb, npd, nf]
    assert got[2] == blk.oracle(verdicts)[1]

    ab = ic.assets(key, 40, 400, 44, fail_frac=0.05, fixed_fail_frac=0.2, skew=1.3, state_call=_assets_state(ctx))
    slots, table, slot_a, slot_b = ab.slots(ab.intended)
    args = _asset_arrays(ab, table, slot_a, slot_b)
    n, ns = len(ab.txs), len(slots)
    hout = _asset_outputs(n, ns)
    hr = C.c_uint(0)
    L = _lib.lib()
    assert L.zk_import_assets_block(ctx._h, key.pvk._h, ns, *[zk._p(a) for a in args[:3]], n, *[zk._p(a) for a in args[3:]],
                                    *[zk._p(o) for o in hout], C.byref(hr)) == 0
    dins = [_dev(a) for a in args]
    douts = [torch.full((o.size,), 0xAB, dtype=torch.uint8, device="cuda") for o in hout]
    torch.cuda.synchronize()
    p = [t.data_ptr() for t in dins]
    dr = zk.assets_import_device(ctx, key.pvk, ns, p[0], p[1], p[2], n, *p[3:], *[t.data_ptr() for t in douts])
    assert dr == hr.value > 1
    assert [t.cpu().numpy().tobytes() for t in douts] == [o.tobytes() for o in hout]
    # and the host form through the wrapper equals the driver's
    assert list(hout[0][:n]) == ab.intended


def test_fixed_verdicts_are_taken_as_they_are(ctx, key):
    """Any byte but 1 fails an issue or destroy, 0xFF (the rounds' undecided marker) included, and comes back unchanged in
    verdicts; the _device form may use one buffer for fixed_verdicts and verdicts."""
    ab = ic.assets(key, 30, 300, 45, fail_frac=0.05, fixed_fail_frac=0.4, issue_frac=0.15, destroy_frac=0.1, skew=1.3,
                   state_call=_assets_state(ctx))
    slots, table, slot_a, slot_b = ab.slots(ab.intended)
    args = _asset_arrays(ab, table, slot_a, slot_b)
    n, ns = len(ab.txs), len(slots)
    L = _lib.lib()

    def host(fixed):
        out, r = _asset_outputs(n, ns), C.c_uint(0)
        assert L.zk_import_assets_block(ctx._h, key.pvk._h, ns, *[zk._p(a) for a in args[:3]], n, *[zk._p(a) for a in args[3:9]],
                                        zk._p(fixed), *[zk._p(o) for o in out], C.byref(r)) == 0
        return [o.tobytes() for o in out], r.value
    want, rounds = host(args[9])
    failing = [k for k, t in enumerate(ab.txs) if t.kind != zk.ASSET_TRANSFER and ab.intended[k] != 1]
    assert len(failing) > 10 and rounds > 1
    odd = args[9].copy()
    odd[failing] = [(0xFF, 0x80, 3)[i % 3] for i in range(len(failing))]
    got, r = host(odd)
    v = bytearray(want[0])
    for k in failing:
        v[k] = odd[k]
    assert r == rounds and got[0] == bytes(v) and got[1:] == want[1:]
    # the device form, verdicts written over the fixed verdicts
    dins = [_dev(a) for a in args[:9]] + [_dev(odd)]
    douts = [torch.full((len(o),), 0xAB, dtype=torch.uint8, device="cuda") for o in want[1:]]
    torch.cuda.synchronize()
    p = [t.data_ptr() for t in dins]
    dr = zk.assets_import_device(ctx, key.pvk, ns, p[0], p[1], p[2], n, *p[3:], p[9], *[t.data_ptr() for t in douts])
    assert dr == rounds
    assert dins[9].cpu().numpy().tobytes() == got[0] and [t.cpu().numpy().tobytes() for t in douts] == got[1:]
