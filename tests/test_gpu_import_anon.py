"""GPU tests of zk_import_anonymous_block and its _device form (groth16.anonymous_import / anonymous_import_device) against
the Python driver import_anonymous_calls_block, the intended verdicts and the C oracle (anon_issue_coracle.block).

Proofs are forged from toy keys' trapdoors at 23 and 105 public inputs (tests/import_anon_corpus.py).  Covered: a random
block of about 3000 transactions with a tenth issues, failures of each kind and rejected points; a failing issue followed
by transfers whose rings hold its issuer; one account in rings over many thread blocks; transfer-only blocks with a NULL
kind and with all-zero kinds; issue-only blocks; empty blocks; every ZK_ERR_INVALID case, a key of the wrong shape and an
undecodable touched account; and the device form against the host form, byte for byte."""
import numpy as np
import pytest
import torch

from tests import import_anon_corpus as iac
from tests.jubjub_oracle import bal_corpus
from zero_chain_b200 import _lib
from zero_chain_b200 import groth16 as zk

pytestmark = pytest.mark.gpu
SCAN_TILE = 128 * 8                       # elements per thread block of the state pass's scan (balances.cu)


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def keys(ctx):
    anon, conf = iac.ForgeKey(zk.ANONYMOUS_POINTS, 71), iac.ForgeKey(zk.CONFIDENTIAL_POINTS, 171)
    anon.pvk = zk.PreparedVerifyingKey.prepare(ctx, anon.params_bytes)
    conf.pvk = zk.PreparedVerifyingKey.prepare(ctx, conf.params_bytes)
    yield anon, conf
    anon.pvk.free()
    conf.pvk.free()


@pytest.fixture(scope="module")
def big(keys):
    return iac.block(*keys, 300, 3000, 91, issue_frac=0.1, fail_frac=0.03, skew=1.2, bad_points=30, bad_issue_points=12, free=20)


def check(ctx, keys, blk, conf=True):
    """the new call against the driver, the intended verdicts and the C oracle; returns the final statuses"""
    anon, cf = keys
    cpvk = cf.pvk if conf else None
    got = zk.anonymous_import(ctx, anon.pvk, cpvk, *blk.args())
    want = zk.import_anonymous_calls_block(ctx, anon.pvk, cpvk, *blk.args())
    assert got == want
    verdicts, state, enc_balances, issued = got
    assert verdicts == blk.intended
    o = blk.oracle(verdicts)
    assert enc_balances == o[0] and state == o[4:]
    st = o[3]
    assert issued == [o[2][64 * k:64 * k + 64] if t.kind == zk.ANON_ISSUE and st[k] == zk.BLOCK_APPLIED else None
                      for k, t in enumerate(blk.txs)]
    return st


def test_random_block_equals_driver_and_oracle(ctx, keys, big):
    kind = np.array([t.kind for t in big.txs])
    v = np.array(big.intended)
    for kd in (zk.ANON_ISSUE, zk.ANON_TRANSFER):
        assert {0, 1, zk.VERDICT_INPUT_REJECTED} <= set(v[kind == kd].tolist())
    assert (kind == zk.ANON_ISSUE).sum() > 250
    st = np.frombuffer(check(ctx, keys, big), np.uint8)
    assert set(st[v == zk.VERDICT_INPUT_REJECTED].tolist()) == {zk.BLOCK_BAD_POINT}


def test_failing_issue_then_transfers_over_its_issuer(ctx, keys):
    """transaction 0 issues to account 0 and fails; account 0 sits in most of the later rings, whose proofs read its balance
    without the issue and pass.  A later passing issue to account 0 moves the balance the transfers after it read."""
    blk = iac.block(*keys, 8, 40, 92, issues=(0, 20), issuer={0: 0, 20: 0}, fail_at=(0,), skew=4.0)
    rings = [k for k, t in enumerate(blk.txs) if t.kind == zk.ANON_TRANSFER and 0 in t.members]
    assert len(rings) > 20 and blk.intended[0] == 0 and blk.intended[20] == 1
    assert all(blk.intended[k] in (1, zk.VERDICT_INPUT_REJECTED) for k in rings)
    check(ctx, keys, blk)
    # the same transfers' proofs do not pass when the failed issue counts as applied
    wrong = blk.oracle([1] + blk.intended[1:])[0]
    assert wrong != blk.oracle(blk.intended)[0]


def test_one_account_in_rings_over_many_thread_blocks(ctx, keys):
    blk = iac.block(*keys, 6, 1500, 93, issue_frac=0.03, fail_frac=0.02, free=1, skew=5.0)
    members = np.array([t.members for t in blk.txs if t.kind == zk.ANON_TRANSFER]).reshape(-1)
    assert np.bincount(members).max() > 3 * SCAN_TILE
    check(ctx, keys, blk)


def _host(ctx, anon_pvk, conf_pvk, blk, kind=True, fields=True, n_acct=None, **over):
    """the C host form on blk's arrays; kind / fields False pass NULL.  Returns (rc, outputs as bytes)"""
    kd, members, tx_points, tx_extra, issue_fields = blk.arrays()
    keys_, bal, pend, fl = blk.accounts
    n, na = len(blk.txs), len(fl) if n_acct is None else n_acct
    kd = over.get("kind_bytes", kd)
    members = over.get("members", members)
    u8 = lambda b: np.frombuffer(bytes(b), np.uint8).copy() if len(b) else np.zeros(1, np.uint8)
    z = lambda m: np.full(max(m, 1), 0xAB, np.uint8)
    outs = [z(n), z(768 * n), z(64 * n), z(n), z(64 * na), z(64 * na), z(na)]
    rc = _lib.lib().zk_import_anonymous_block(
        ctx._h, anon_pvk._h, conf_pvk._h if conf_pvk else None, na, zk._p(u8(keys_)), zk._p(u8(bal)), zk._p(u8(pend)), zk._p(u8(fl)), n,
        zk._p(u8(kd)) if kind else None, zk._p(np.asarray(members, np.uint32) if n else np.zeros(1, np.uint32)), zk._p(u8(tx_points)),
        zk._p(u8(tx_extra)), zk._p(u8(issue_fields)) if fields else None, zk._p(u8(blk.g_epoch)),
        zk._p(u8(b"".join(blk.proofs))), *[zk._p(o) for o in outs])
    sizes = [n, 768 * n, 64 * n, n, 64 * na, 64 * na, na]
    return rc, [o[:s].tobytes() for o, s in zip(outs, sizes)]


def test_transfer_only_blocks(ctx, keys):
    anon, conf = keys
    blk = iac.block(anon, conf, 100, 600, 94, issue_frac=0.0, fail_frac=0.05, bad_points=6)
    assert all(t.kind == zk.ANON_TRANSFER for t in blk.txs) and 0 in blk.intended
    check(ctx, keys, blk)
    check(ctx, keys, blk, conf=False)                       # no confidential key needed
    want = zk.import_anonymous_block(ctx, anon.pvk, *blk.args())
    assert zk.anonymous_import(ctx, anon.pvk, None, *blk.args())[:3] == want
    # kind NULL, and issue_fields NULL, through the C call: the same bytes as all-zero kinds
    rc0, zero = _host(ctx, anon.pvk, None, blk)
    rc1, null = _host(ctx, anon.pvk, None, blk, kind=False, fields=False)
    assert rc0 == rc1 == 0 and zero == null
    assert list(zero[0]) == want[0] and zero[1] == want[2] and tuple(zero[4:]) == want[1] and zero[2] == bytes(64 * len(blk.txs))


def test_issue_only_blocks(ctx, keys):
    blk = iac.block(*keys, 40, 200, 95, issue_frac=1.0, fail_frac=0.2, bad_issue_points=6, free=5)
    assert all(t.kind == zk.ANON_ISSUE for t in blk.txs)
    st = check(ctx, keys, blk)
    assert set(st) == {zk.BLOCK_APPLIED, zk.BLOCK_NOT_APPLIED, zk.BLOCK_BAD_POINT}


def test_empty_blocks(ctx, keys):
    anon, conf = keys
    b = bal_corpus.make(30, 0, 96)
    accounts = (bytes(32 * 30), b.balances, b.pendings, b.flags)
    g = bytes(32)
    want = ([], (b.balances, b.pendings, b.flags), b"", [])
    assert zk.anonymous_import(ctx, anon.pvk, conf.pvk, accounts, [], g, []) == want == \
        zk.import_anonymous_calls_block(ctx, anon.pvk, conf.pvk, accounts, [], g, [])
    assert zk.anonymous_import(ctx, anon.pvk, None, (b"", b"", b"", b""), [], g, []) == ([], (b"", b"", b""), b"", [])


def test_errors(ctx, keys):
    anon, conf = keys
    blk = iac.block(anon, conf, 20, 40, 97, issue_frac=0.2)
    L = _lib.lib()
    iss = [k for k, t in enumerate(blk.txs) if t.kind == zk.ANON_ISSUE]
    tr = [k for k, t in enumerate(blk.txs) if t.kind == zk.ANON_TRANSFER]
    assert len(iss) > 3 and len(tr) > 20
    kd, members, _, _, _ = blk.arrays()

    def invalid(at, **over):
        rc, _ = _host(ctx, anon.pvk, over.pop("conf_pvk", conf.pvk), blk, **over)
        assert rc == -2 and ("transaction %d:" % at).encode() in L.zk_last_error(), L.zk_last_error()
    # an unknown kind; a transfer member out of range; an issuer out of range (an issue's other members are ignored)
    invalid(tr[5], kind_bytes=bytes(2 if k == tr[5] else x for k, x in enumerate(kd)))
    m = members.copy(); m[12 * tr[4] + 11] = 20
    invalid(tr[4], members=m)
    m = members.copy(); m[12 * iss[2]] = 25; m[12 * iss[1] + 3] = 0xFFFFFFFF
    invalid(iss[2], members=m)
    # an issue without the confidential key or without issue_fields
    invalid(iss[0], conf_pvk=None)
    invalid(iss[0], fields=False)
    # the wrapper: the driver's ValueError, naming the transaction
    first = blk.txs[tr[6]].members[0]
    blk.txs[tr[6]].members[0] = 20
    with pytest.raises(ValueError):
        zk.import_anonymous_calls_block(ctx, anon.pvk, conf.pvk, *blk.args())
    with pytest.raises(ValueError, match="transaction %d:" % tr[6]):
        zk.anonymous_import(ctx, anon.pvk, conf.pvk, *blk.args())
    blk.txs[tr[6]].members[0] = first
    # a key of the wrong shape, before any work and even when the block does not use it
    for a, c in ((conf.pvk, conf.pvk), (anon.pvk, anon.pvk)):
        with pytest.raises(zk.SynthesisError) as e:
            zk.anonymous_import(ctx, a, c, *blk.args())
        assert e.value.code == -9
    with pytest.raises(zk.SynthesisError) as e:
        zk.anonymous_import(ctx, anon.pvk, anon.pvk, blk.accounts, [], blk.g_epoch, [])
    assert e.value.code == -9
    # an undecodable touched account
    a = blk.txs[tr[3]].members[2]
    bal_b, flags = bytearray(blk.accounts[1]), bytearray(blk.accounts[3])
    bal_b[64 * a + 32:64 * a + 64] = bal_corpus.bad_order(bytes(bal_b[64 * a + 32:64 * a + 64]))
    flags[a] |= zk.ACCOUNT_BALANCE
    bad = iac.Block((blk.accounts[0], bytes(bal_b), blk.accounts[2], bytes(flags)), blk.txs, blk.g_epoch, blk.proofs, blk.intended)
    for fn in (zk.anonymous_import, zk.import_anonymous_calls_block):
        with pytest.raises(zk.SynthesisError) as e:
            fn(ctx, anon.pvk, conf.pvk, *bad.args())
        assert e.value.code == -7 and "account %d" % a in str(e.value)
    check(ctx, keys, blk)                                   # the context recovers


def _dev(b: bytes):
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda() if b else torch.zeros(1, dtype=torch.uint8, device="cuda")


def test_device_form_equals_host_form(ctx, keys, big):
    anon, conf = keys
    kd, members, tx_points, tx_extra, fields = big.arrays()
    n, na = len(big.txs), len(big.accounts[3])
    rc, host = _host(ctx, anon.pvk, conf.pvk, big)
    assert rc == 0
    ins = [_dev(x) for x in big.accounts] + [_dev(kd), _dev(members.tobytes()), _dev(tx_points), _dev(tx_extra), _dev(fields), _dev(big.g_epoch),
                                             _dev(b"".join(big.proofs))]
    outs = [torch.full((m,), 0xAB, dtype=torch.uint8, device="cuda") for m in (n, 768 * n, 64 * n, n, 64 * na, 64 * na, na)]
    torch.cuda.synchronize()
    p = [t.data_ptr() for t in ins]
    zk.anonymous_import_device(ctx, anon.pvk, conf.pvk, na, *p[:4], n, *p[4:], *[t.data_ptr() for t in outs])
    assert [t.cpu().numpy().tobytes() for t in outs] == host
    assert list(host[0]) == big.intended
