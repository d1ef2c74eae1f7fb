"""GPU tests of zk_anonymous_calls_block(_device) and import_anonymous_calls_block: a random block of about 3000
transactions, a tenth of them issues, over a few hundred accounts (issues before, between and after an account's touches,
on accounts no ring names, failed issues, rejected points, unknown kinds, out-of-range indices) against the C oracle byte
for byte on every output; one account taking issues among thousands of rings; an all-transfer kind against
zk_balances_anonymous_block; n_tx = 0; the argument errors; the device form against the host form; and a block imported
end to end with toy keys of both proof shapes on the reference's literal g_epoch and EncKey."""
import numpy as np
import pytest
import torch

from oracle import coracle as co
from tests.jubjub_oracle import anon_corpus
from tests.jubjub_oracle import anon_issue_coracle as aic
from tests.jubjub_oracle import anon_issue_corpus
from tests.jubjub_oracle import balances as bal
from tests.jubjub_oracle import pyref as jj
from zero_chain_b200 import _lib
from zero_chain_b200 import groth16 as zk
from zero_chain_b200 import synthetic as sy

pytestmark = pytest.mark.gpu
SCAN_TILE = 128 * 8                       # elements per thread block of the scan's first level (balances.cu)
# modules/anonymous-balances/src/lib.rs:453 (the g_epoch of block height one) and :336 (Bob's EncKey)
G_EPOCH_1 = bytes.fromhex("0953f47325251a2f479c25527df6d977925bebafde84423b20ae6c903411665a")
BOB = bytes.fromhex("45e66da531088b55dcb3b273ca825454d79d2d1d5c4fa2ba4a12c1fa1ccd6389")
NAMES = ["enc_balances", "verify_points", "issued", "status", "balances", "pendings", "flags"]


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def block():
    return anon_issue_corpus.make(300, 3000, 91, issue_frac=0.1, free=20, skew=1.2, bad_points=30, bad_index=True, bad_issue_points=12,
                                  bad_kind=True)


def _rows(b: bytes, size: int):
    return [b[size * i:size * i + size] for i in range(len(b) // size)]


def test_mixed_block_equals_c_oracle(ctx, block):
    kind = np.frombuffer(block.kind, np.uint8)
    assert (kind == 1).sum() > 250 and {2, 255} <= set(kind.tolist())
    got = zk.anonymous_calls_block(ctx, *block.args())
    bad, want = aic.block(*block.args())
    assert bad is None
    st = np.frombuffer(want[3], np.uint8)
    assert set(st[kind == 1].tolist()) == {0, 1, 2, 3} and set(st[kind == 0].tolist()) == {0, 1, 2, 3}
    for g, w, name in zip(got, want, NAMES):
        assert g == w, name
    # issue-only accounts got their issued balance with the due bit kept
    issued_free = {int(block.members[12 * k]) for k in np.flatnonzero((kind == 1) & (st == 0)).tolist()} & set(range(280, 300))
    assert issued_free and all(got[6][a] & 1 and got[6][a] >> 2 == block.flags[a] >> 2 for a in issued_free)


def test_issues_among_thousands_of_rings(ctx):
    """account 0 is in most of 4000 rings and takes a few dozen issues among them"""
    b = anon_issue_corpus.make(6, 4000, 92, issue_frac=0.03, free=1, skew=5.0, bad_points=4, mask_p=(0.0, 1.0, 0.0, 0.0, 0.0))
    kind = np.frombuffer(b.kind, np.uint8)
    assert np.bincount(b.members[b.members < 6]).max() > 3 * SCAN_TILE
    assert (b.members.reshape(-1, 12)[kind == 1, 0] == 0).sum() > 20
    assert zk.anonymous_calls_block(ctx, *b.args()) == aic.block(*b.args())[1]


def test_all_transfers_equal_anonymous_block(ctx):
    b = anon_corpus.make(300, 3000, 51, skew=1.2, bad_points=30, bad_index=True)
    want = zk.anonymous_block(ctx, *b.args())
    args = b.args()[:4] + (bytes(b.n_tx),) + b.args()[4:]
    got = zk.anonymous_calls_block(ctx, *args)
    assert got[:2] + got[3:] == want and got[2] == bytes(64 * b.n_tx)
    # the device form runs the issue passes on an all-zero kind: same bytes
    bufs = _device_buffers(*args)
    _device_call(ctx, bufs)
    ctx.sync()
    assert _device_outputs(bufs) == got


def test_no_transactions(ctx):
    b = anon_issue_corpus.make(40, 0, 93)
    assert zk.anonymous_calls_block(ctx, *b.args()) == (b"", b"", b"", b"", b.balances, b.pendings, b.flags)


def test_argument_errors(ctx):
    L = _lib.lib()
    one = [b"\0"] * 4
    # n_tx > 0 with a NULL kind, or a NULL issued
    assert L.zk_anonymous_calls_block(ctx._h, 0, *([None] * 4), 1, None, *([b"\0"] * 7), None, b"\0", None, None, None) == -2
    assert L.zk_anonymous_calls_block(ctx._h, 0, *([None] * 4), 1, *([b"\0"] * 8), None, b"\0", None, None, None) == -2
    assert L.zk_anonymous_calls_block(ctx._h, 1, None, None, None, None, 0, *([None] * 13)) == -2
    assert L.zk_anonymous_calls_block(ctx._h, (1 << 22) + 1, *one, 0, *([None] * 10), *([b"\0"] * 3)) == -2
    assert L.zk_anonymous_calls_block(ctx._h, 0, *([None] * 4), (1 << 18) + 1, *([b"\0"] * 10), None, None, None) == -2
    assert L.zk_anonymous_calls_block_device(ctx._h, 0, *([None] * 4), 1, None, *([b"\0"] * 9), None, None, None) == -2


def _dev(b: bytes):
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda() if b else torch.zeros(1, dtype=torch.uint8, device="cuda")


def _device_buffers(keys, balances, pendings, flags, kind, members, tx_points, tx_extra, g_epoch, applied):
    n_acct = len(flags)
    mem = np.asarray(members).astype(np.int64).astype(np.uint32).reshape(-1)
    n_tx = len(mem) // 12
    ins = [_dev(keys), _dev(balances), _dev(pendings), _dev(flags), _dev(kind), torch.from_numpy(mem.view(np.int32)).cuda(),
           _dev(tx_points), _dev(tx_extra), _dev(g_epoch), _dev(applied)]
    z = lambda n: torch.full((max(n, 1),), 0xAB, dtype=torch.uint8, device="cuda")
    outs = [z(768 * n_tx), z(1664 * n_tx), torch.zeros(max(64 * n_tx, 1), dtype=torch.uint8, device="cuda"), z(n_tx), z(64 * n_acct),
            z(64 * n_acct), z(n_acct)]
    torch.cuda.synchronize()
    return n_acct, n_tx, ins, outs


def _device_call(ctx, bufs):
    n_acct, n_tx, ins, outs = bufs
    p = [t.data_ptr() for t in ins]
    zk.anonymous_calls_block_device(ctx, n_acct, p[0], p[1], p[2], p[3], n_tx, *p[4:], *[t.data_ptr() for t in outs])


def _device_outputs(bufs):
    n_acct, n_tx = bufs[0], bufs[1]
    sizes = [768 * n_tx, 1664 * n_tx, 64 * n_tx, n_tx, 64 * n_acct, 64 * n_acct, n_acct]
    return tuple(t.cpu().numpy().tobytes()[:s] for t, s in zip(bufs[3], sizes))


def test_device_form_equals_host_form(ctx, block):
    bufs = _device_buffers(*block.args())
    _device_call(ctx, bufs)
    ctx.sync()
    assert _device_outputs(bufs) == zk.anonymous_calls_block(ctx, *block.args())


# ---- end to end ---------------------------------------------------------------------------------------------------------
class _Key:
    """A toy CRS whose public inputs are the coordinates of n_points Jubjub points (11: the confidential proof's shape, which
    issue is checked with; 52: the anonymous transfer's), and proofs for chosen points."""

    def __init__(self, ctx, n_points, seed):
        self.r1cs = sy.make_r1cs(60 + 2 * n_points, 2 * n_points + 1, 50, 40, 33, seed=seed)
        crs = sy.make_toy_crs(self.r1cs, co.g1_fixed_base, co.g2_fixed_base, seed=seed + 1)
        self.params = zk.Parameters.read(ctx, crs.params_bytes, checked=True)
        self.pvk = zk.PreparedVerifyingKey.prepare(ctx, crs.params_bytes)

    def prove(self, encodings: bytes, seed: int) -> bytes:
        inputs = [c for i in range(len(encodings) // 32) for c in jj.read(encodings[32 * i:32 * i + 32])[1]]
        z = sy.make_witness(self.r1cs, seed, inputs=inputs)
        a, b, c = sy.evaluate(self.r1cs, z)
        n_in = self.r1cs.n_inputs
        pa = zk.ProvingAssignment(co.ints_to_limbs(a, 4), co.ints_to_limbs(b, 4), co.ints_to_limbs(c, 4),
                                  co.ints_to_limbs(z[:n_in], 4), co.ints_to_limbs(z[n_in:], 4), *sy.densities(self.r1cs))
        return zk.create_proof(pa, self.params, 1000 + seed, 2000 + seed)

    def free(self):
        self.pvk.free(); self.params.free()


def test_import_block_end_to_end(ctx):
    """Six transactions over 14 accounts, Bob's EncKey as account 0 (due, with a balance and a pending) and block one's
    g_epoch: 0 an issue to account 0; 1 a ring with account 0 proven on the balance the issue left (passes); 2 the same
    ring proven on account 0's balance without the issue (fails); 3 an issue to account 5 whose proof is for another total
    (fails and changes nothing); 4 an issue to account 13, which no ring names; 5 a ring with account 5 proven on its
    stored balance (passes).  Verdicts [1, 1, 0, 0, 1, 1]; verdicts, issued and the final state as the C oracle's."""
    conf, anon = _Key(ctx, zk.CONFIDENTIAL_POINTS, 171), _Key(ctx, zk.ANONYMOUS_POINTS, 71)
    try:
        b = anon_corpus.make(14, 6, 172, dup_frac=0.0, mask_p=(0.0, 1.0, 0.0, 0.0, 0.0))
        keys = BOB + b.keys[32:]
        flags = bytes([bal.BALANCE | bal.PENDING | bal.DUE, bal.PENDING | bal.DUE]) + b.flags[2:]
        ring = list(range(12))
        pts = _rows(b.tx_points, 32)
        extra = _rows(b.tx_extra, 32)

        def issue(k, issuer):
            return zk.AnonIssueTx(issuer, pts[13 * k], extra[2 * k], b.balances[64 * k:64 * k + 64], pts[13 * k + 12], extra[2 * k + 1],
                                  extra[(2 * k + 5) % 12])

        def transfer(k):
            return zk.AnonymousTx(ring, pts[13 * k:13 * k + 12], pts[13 * k + 12], extra[2 * k], extra[2 * k + 1])
        txs = [issue(0, 0), transfer(1), transfer(2), issue(3, 5), issue(4, 13), transfer(5)]
        kind = bytes(t.kind for t in txs)
        members = np.array([t.members for t in txs], np.uint32).reshape(-1)
        tx_points = b"".join(t.points() for t in txs)
        tx_extra = b"".join(t.rvk + t.nonce for t in txs)

        def oracle(applied):
            return aic.block(keys, b.balances, b.pendings, flags, kind, members, tx_points, tx_extra, G_EPOCH_1, bytes(applied))
        reads = _rows(oracle([1, 0, 0, 0, 1, 0])[1][0], 768)        # the issues that pass applied
        before = _rows(oracle([0] * 6)[1][0], 768)                  # no issue applied
        assert reads[1] != before[1]

        def tpts(k, acc):
            t = txs[k]
            return zk.anonymous_points([keys[32 * a:32 * a + 32] for a in t.members], t.left_ciphertexts, _rows(acc, 64),
                                       t.right_ciphertext, t.rvk, G_EPOCH_1, t.nonce)
        other = issue(3, 5)
        other.total = pts[1]
        proofs = [conf.prove(txs[0].verify_points(keys, G_EPOCH_1), 80), anon.prove(tpts(1, reads[1]), 81),
                  anon.prove(tpts(2, before[2]), 82), conf.prove(other.verify_points(keys, G_EPOCH_1), 83),
                  conf.prove(txs[4].verify_points(keys, G_EPOCH_1), 84), anon.prove(tpts(5, reads[5]), 85)]
        accounts = (keys, b.balances, b.pendings, flags)
        verdicts, state, enc_balances, issued = zk.import_anonymous_calls_block(ctx, anon.pvk, conf.pvk, accounts, txs, G_EPOCH_1, proofs)
        assert verdicts == [1, 1, 0, 0, 1, 1]
        bad, want = oracle([1 if v == 1 else 0 for v in verdicts])
        assert bad is None and want[3] == bytes([0, 0, 1, 1, 0, 0])
        assert enc_balances == want[0] and state == want[4:]
        assert issued == [want[2][:64], None, None, None, want[2][256:320], None]
        assert state[0][64 * 13:64 * 14] == issued[4] and state[2][13] == flags[13] | bal.BALANCE
        # transfers only: import_anonymous_block's result
        tr = [txs[1], txs[2], txs[5]]
        got = zk.import_anonymous_calls_block(ctx, anon.pvk, conf.pvk, accounts, tr, G_EPOCH_1, [proofs[1], proofs[2], proofs[5]])
        assert got[:3] == zk.import_anonymous_block(ctx, anon.pvk, accounts, tr, G_EPOCH_1, [proofs[1], proofs[2], proofs[5]])
        assert got[3] == [None] * 3
        with pytest.raises(ValueError):
            zk.import_anonymous_calls_block(ctx, anon.pvk, conf.pvk, accounts, [issue(0, 14)], G_EPOCH_1, proofs[:1])
    finally:
        conf.free(); anon.free()
