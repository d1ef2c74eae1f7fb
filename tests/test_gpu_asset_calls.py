"""GPU tests of zk_import_asset_calls and its _device form (groth16.asset_calls_import / asset_calls_import_device): a
block of encrypted-asset calls from the slot table and the extrinsic fields, with the issue and destroy verification,
the asset numbering, the slot resolution and the transfer rounds on the device.  Every output is checked against the
Python driver import_assets_block, against assets_import (the transfer rounds in one call, the rest on the host) and
against the C oracle (assets_oracle.c): verdicts, asset ids, events, the grown table and the rounds.

Proofs are forged from a toy key's trapdoor (tests/import_corpus.py).  Covered: corpus blocks with failures in all three
kinds; transfers of assets issued earlier in the block and of assets never issued, with more new slots than one thread
block; a block of only issues and destroys; empty blocks; a table of more than 2^16 slots; the device form against the
host form; and every error the call returns."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import import_anon_corpus as iac
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


def _state(ctx):
    return lambda *a: zk.assets_block(ctx, *a)


def reforge(ctx, key, ab):
    """the rows and proofs of ab's transactions for its intended verdicts, after its transactions or table changed"""
    bs = ab.oracle(ab.intended, _state(ctx))[0]
    ab.rows = b"".join(t.verify_points(bs[64 * k:64 * k + 64]) if t.kind == zk.ASSET_TRANSFER else t.verify_points()
                       for k, t in enumerate(ab.txs))
    ab.proofs = key.proofs(ab.rows, [v == 1 for v in ab.intended])
    return ab


def check(ctx, key, ab, rounds=None):
    """the new call against import_assets_block, assets_import and the C oracle; returns its result"""
    got = zk.asset_calls_import(ctx, key.pvk, *ab.args())
    assert got == zk.import_assets_block(ctx, key.pvk, *ab.args())
    assert got == zk.assets_import(ctx, key.pvk, *ab.args())
    verdicts, ids, events, (slots, nb, npd, nf), r = got
    assert verdicts == ab.intended
    want_slots, _, _, _ = ab.slots(verdicts)
    assert slots == want_slots
    out = ab.oracle(verdicts)
    assert (nb, npd, nf) == out[5:]
    for k, t in enumerate(ab.txs):
        if out[4][k] != zk.BLOCK_APPLIED:
            assert events[k] is None
        elif t.kind == zk.ASSET_TRANSFER:
            assert events[k] == out[1][64 * k:64 * k + 64]
        elif t.kind == zk.ASSET_ISSUE:
            assert events[k] == out[2][128 * k:128 * k + 64] and ids[k] is not None
    if rounds is not None:
        assert r == rounds
    return got


def test_corpus_block_with_failures_in_every_kind(ctx, key):
    ab = ic.assets(key, 100, 1500, 51, fail_frac=0.03, fixed_fail_frac=0.2, skew=1.1, state_call=_state(ctx))
    for kind in (zk.ASSET_TRANSFER, zk.ASSET_ISSUE, zk.ASSET_DESTROY):
        assert {v for t, v in zip(ab.txs, ab.intended) if t.kind == kind} == {0, 1}
    assert check(ctx, key, ab)[4] > 1


def new_and_unknown_assets(ctx, key, n_keys, n_tx, seed, n_unknown):
    """ic.assets' block with transfers of the assets its issues create (from the issuer, after the issue) and n_unknown
    transfers of assets never issued, each its own id (two new slots each)"""
    ab = ic.assets(key, n_keys, n_tx, seed, fail_frac=0.02, fixed_fail_frac=0.3, issue_frac=0.1, state_call=_state(ctx))
    rng = np.random.default_rng(seed)
    ids = zk._asset_slots("t", list(ab.state[0]), *ab.state[1:], ab.txs, ab.intended, ab.next_asset_id, ab.new_slot_flags)[1]
    issued = [(k, i) for k, i in enumerate(ids) if i is not None]
    transfers = [k for k, t in enumerate(ab.txs) if t.kind == zk.ASSET_TRANSFER]
    for k in transfers:
        later = [(j, i) for j, i in issued if j < k]
        if later and rng.random() < 0.3:
            j, i = later[int(rng.integers(0, len(later)))]
            ab.txs[k].asset_id, ab.txs[k].address_sender = i, ab.txs[j].issuer
    for n, k in enumerate(rng.choice(transfers, n_unknown, replace=False)):
        ab.txs[k].asset_id = 5000 + n
    return reforge(ctx, key, ab)


def test_transfers_of_new_and_unknown_assets(ctx, key):
    ab = new_and_unknown_assets(ctx, key, 40, 1200, 52, 300)
    verdicts, ids, _, (slots, *_), _ = check(ctx, key, ab)
    issued = {i for i in ids if i is not None}
    assert any(t.kind == zk.ASSET_TRANSFER and t.asset_id in issued for t in ab.txs)
    assert len(slots) - len(ab.state[0]) > 2 * 256                 # more new slots than one thread block


def test_block_of_issues_and_destroys_only(ctx, key):
    ab = ic.assets(key, 20, 300, 53, fixed_fail_frac=0.3, issue_frac=0.6, destroy_frac=0.4, state_call=_state(ctx))
    assert {t.kind for t in ab.txs} == {zk.ASSET_ISSUE, zk.ASSET_DESTROY}
    check(ctx, key, ab, 0)


def test_empty_blocks(ctx, key):
    ab = ic.assets(key, 8, 10, 54, state_call=_state(ctx))
    check(ctx, key, ic.AssetBlock(ab.state, [], [], [], 10, zk.ACCOUNT_DUE), 0)
    nothing = ([], b"", b"", b"")
    assert zk.asset_calls_import(ctx, key.pvk, nothing, [], [], 10, 0) == ([], [], [], nothing, 0) == \
        zk.import_assets_block(ctx, key.pvk, nothing, [], [], 10, 0)


def test_table_of_more_than_2_16_slots(ctx, key):
    """70000 absent rows of other assets ahead of the corpus's table: the named rows sit past 2^16"""
    ab = ic.assets(key, 30, 400, 55, fail_frac=0.05, fixed_fail_frac=0.2, state_call=_state(ctx))
    rng = np.random.default_rng(55)
    pad = 70000
    keys = rng.integers(0, 256, (pad, 32), dtype=np.uint8)
    slots, bal, pend, fl = ab.state
    ab.state = ([(100 + r % 7, keys[r].tobytes()) for r in range(pad)] + slots, bytes(64 * pad) + bal, bytes(64 * pad) + pend,
                bytes(pad) + fl)
    reforge(ctx, key, ab)
    got = check(ctx, key, ab)
    assert len(got[3][0]) > pad + len(slots)


# ---- the C call itself --------------------------------------------------------------------------------------------------
def arrays(ab):
    """zk_import_asset_calls' host inputs: slot_ids, slot_keys, balances, pendings, flags, kind, asset_id, rows, proofs"""
    u8 = lambda b: np.frombuffer(bytes(b), np.uint8).copy() if len(b) else np.zeros(1, np.uint8)
    u32 = lambda a: np.array(list(a) or [0], np.uint32)
    slots, bal, pend, fl = ab.state
    rows = b"".join(t.verify_points(bytes(64)) if t.kind == zk.ASSET_TRANSFER else t.verify_points() for t in ab.txs)
    return [u32(a for a, _ in slots), u8(b"".join(k for _, k in slots)), u8(bal), u8(pend), u8(fl), u8(bytes(t.kind for t in ab.txs)),
            u32(t.asset_id if t.kind != zk.ASSET_ISSUE else 0 for t in ab.txs), u8(rows), u8(b"".join(ab.proofs))]


def outputs(n, ns):
    z = lambda m: np.zeros(max(m, 1), np.uint8)
    nr = ns + 2 * n
    return [z(n), z(4 * n), z(64 * n), z(128 * n), z(n), z(n), z(4 * nr), z(32 * nr), z(64 * nr), z(64 * nr), z(nr)]


def c_call(ctx, pvk, ab, ins, outs, next_id=None, n_out=None, rounds=None):
    ns, n = len(ab.state[0]), len(ab.txs)
    p = [zk._p(a) if a is not None else None for a in ins]
    o = [zk._p(a) if a is not None else None for a in outs]
    return _lib.lib().zk_import_asset_calls(ctx._h, pvk._h, ns, *p[:5], ab.next_asset_id if next_id is None else next_id,
                                            ab.new_slot_flags, n, *p[5:], *o, C.byref(n_out if n_out is not None else C.c_size_t()),
                                            C.byref(rounds if rounds is not None else C.c_uint()))


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).cuda()


def test_device_form_equals_host_form(ctx, key):
    ab = new_and_unknown_assets(ctx, key, 30, 500, 56, 40)
    ins = arrays(ab)
    n, ns = len(ab.txs), len(ab.state[0])
    hout, hn, hr = outputs(n, ns), C.c_size_t(), C.c_uint()
    assert c_call(ctx, key.pvk, ab, ins, hout, n_out=hn, rounds=hr) == 0
    dins = [_dev(a) for a in ins]
    douts = [torch.full((o.size,), 0xAB, dtype=torch.uint8, device="cuda") for o in hout]
    torch.cuda.synchronize()
    p = [t.data_ptr() for t in dins]
    dn, dr = zk.asset_calls_import_device(ctx, key.pvk, ns, *p[:5], ab.next_asset_id, ab.new_slot_flags, n, *p[5:],
                                          *[t.data_ptr() for t in douts])
    m = hn.value
    assert (dn, dr) == (m, hr.value) and dr > 1 and m > ns
    per_row = [None] * 6 + [4, 32, 64, 64, 1]
    got = [t.cpu().numpy() for t in douts]
    for i, (g, h) in enumerate(zip(got, hout)):
        size = per_row[i] * m if per_row[i] else h.size
        assert g[:size].tobytes() == h[:size].tobytes(), i
    verdicts, ids, _, (slots, nb, npd, nf), rounds = zk.asset_calls_import(ctx, key.pvk, *ab.args())
    assert bytes(verdicts) == hout[0][:n].tobytes() and rounds == dr
    assert [i or 0 for i in ids] == list(hout[1][:4 * n].view(np.uint32))
    assert hout[8][:64 * m].tobytes() == nb and [a for a, _ in slots] == list(hout[6][:4 * m].view(np.uint32))


def test_errors(ctx, key):
    ab = ic.assets(key, 12, 80, 57, fixed_fail_frac=0.2, issue_frac=0.2, state_call=_state(ctx))
    n, ns = len(ab.txs), len(ab.state[0])
    L = _lib.lib()
    # an unknown kind, named
    ins = arrays(ab)
    ins[5][[17, 40]] = [3, 200]
    assert c_call(ctx, key.pvk, ab, ins, outputs(n, ns)) == -2 and b"transaction 17" in L.zk_last_error()
    # an asset id past 2^32 - 1: m passing issues fit below it, one more does not
    passing = [k for k, t in enumerate(ab.txs) if t.kind == zk.ASSET_ISSUE and ab.intended[k] == 1]
    m = len(passing)
    assert m > 2
    ab.next_asset_id = 2**32 - m
    got = check(ctx, key, ab)
    assert got[1][passing[-1]] == 2**32 - 1
    ab.next_asset_id = 2**32 - m + 1
    for fn in (zk.asset_calls_import, zk.import_assets_block):
        with pytest.raises(ValueError):
            fn(ctx, key.pvk, *ab.args())
    assert c_call(ctx, key.pvk, ab, arrays(ab), outputs(n, ns)) == -2
    assert ("transaction %d" % passing[-1]).encode() in L.zk_last_error()
    ab.next_asset_id = 10
    # a repeated (asset id, key) in the table, the lowest repeating row named
    slots = list(ab.state[0])
    dup = ic.AssetBlock((slots[:9] + [slots[4]] + slots[9:],) + tuple(x[:64 * 9] + x[64 * 4:64 * 5] + x[64 * 9:] if i < 2 else
                                                                    x[:9] + x[4:5] + x[9:] for i, x in enumerate(ab.state[1:])),
                        ab.txs, ab.proofs, ab.intended, 10, ab.new_slot_flags)
    with pytest.raises(ValueError) as e:
        zk.asset_calls_import(ctx, key.pvk, *dup.args())
    assert "slot row 9" in str(e.value)
    # NULL arguments
    for i in (0, 1, 5, 6, 7, 8):
        ins = arrays(ab)
        ins[i] = None
        assert c_call(ctx, key.pvk, ab, ins, outputs(n, ns)) == -2 and b"NULL" in L.zk_last_error(), i
    outs = outputs(n, ns)
    outs[7] = None
    assert c_call(ctx, key.pvk, ab, arrays(ab), outs) == -2
    assert L.zk_import_asset_calls(ctx._h, key.pvk._h, 0, *[None] * 5, 10, 0, 0, *[None] * 15, None, None) == -2
    # a key of 52 points
    anon = iac.ForgeKey(zk.ANONYMOUS_POINTS, 71)
    apvk = zk.PreparedVerifyingKey.prepare(ctx, anon.params_bytes)
    assert c_call(ctx, apvk, ab, arrays(ab), outputs(n, ns)) == -9
    empty = ic.AssetBlock(([], b"", b"", b""), [], [], [], 10, 0)
    assert c_call(ctx, apvk, empty, arrays(empty), outputs(0, 0)) == -9
    apvk.free()
    # an undecodable stored ciphertext of a named slot
    t = next(k for k, x in enumerate(ab.txs) if x.kind == zk.ASSET_TRANSFER)
    r = ab.state[0].index((ab.txs[t].asset_id, ab.txs[t].address_recipient))
    bal, fl = bytearray(ab.state[1]), bytearray(ab.state[3])
    bal[64 * r + 32:64 * r + 64] = bal_corpus.bad_order(bytes(bal[64 * r + 32:64 * r + 64]))
    fl[r] |= zk.ACCOUNT_BALANCE
    bad = ic.AssetBlock((ab.state[0], bytes(bal), ab.state[2], bytes(fl)), ab.txs, ab.proofs, ab.intended, 10, ab.new_slot_flags)
    with pytest.raises(zk.SynthesisError) as e:
        zk.asset_calls_import(ctx, key.pvk, *bad.args())
    assert e.value.code == -7 and " %d: a stored ciphertext" % r in str(e.value)
    assert zk.asset_calls_import(ctx, key.pvk, *ab.args())[0] == ab.intended      # the context recovers
