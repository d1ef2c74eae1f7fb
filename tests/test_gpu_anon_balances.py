"""GPU tests of zk_balances_anonymous_block(_device) and import_anonymous_block: a random block of thousands of ring
transfers over a few hundred accounts with a skewed member choice (members listed twice, due and non-due accounts, absent
balances and pendings, every mask value, every point-rejection class, out-of-range indices) against the C oracle byte
for byte; one account named by thousands of transactions; n_tx = 0; a malformed stored ciphertext, touched and
untouched; the argument errors; the device form against the host form; and a block imported end to end with proofs of a
toy key of the anonymous shape, on the reference's literal g_epoch and EncKey."""
import numpy as np
import pytest
import torch

from oracle import coracle as co
from tests.jubjub_oracle import anon_balances as ab
from tests.jubjub_oracle import anon_coracle as aco
from tests.jubjub_oracle import anon_corpus
from tests.jubjub_oracle import bal_corpus
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


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def block():
    return anon_corpus.make(300, 3000, 51, skew=1.2, bad_points=30, bad_index=True)


def _rows(b: bytes, size: int):
    return [b[size * i:size * i + size] for i in range(len(b) // size)]


def test_random_block_equals_c_oracle(ctx, block):
    flags = np.frombuffer(block.flags, np.uint8)
    assert {f & 7 for f in flags} == set(range(8))                          # every presence / due combination
    m = block.members.reshape(-1, 12)
    assert sum(len(set(r)) < 12 for r in m.tolist()) > 300                  # members listed twice
    assert set(block.applied) == {0, 1, 2, 3, 4}
    got = zk.anonymous_block(ctx, *block.args())
    bad, want = aco.block(*block.args())
    assert bad is None
    assert set(want[2]) == {0, 1, 2, 3}
    for g, w, name in zip(got, want, ["enc_balances", "verify_points", "status", "balances", "pendings", "flags"]):
        assert g == w, name
    # the verifier's rows are anonymous_points of the oracle's acc
    st = want[2]
    for k in [k for k in range(block.n_tx) if st[k] != 3][:200]:
        mem = m[k].tolist()
        pts = _rows(block.tx_points[416 * k:416 * k + 416], 32)
        assert got[1][1664 * k:1664 * k + 1664] == zk.anonymous_points(
            [block.keys[32 * a:32 * a + 32] for a in mem], pts[:12], _rows(want[0][768 * k:768 * k + 768], 64), pts[12],
            block.tx_extra[64 * k:64 * k + 32], block.g_epoch, block.tx_extra[64 * k + 32:64 * k + 64])


def test_account_in_thousands_of_rings(ctx):
    b = anon_corpus.make(4, 3000, 52, skew=5.0, bad_points=4, mask_p=(0.0, 1.0, 0.0, 0.0, 0.0))
    assert np.bincount(b.members).max() > 3 * SCAN_TILE
    assert zk.anonymous_block(ctx, *b.args()) == aco.block(*b.args())[1]


def test_no_transactions(ctx):
    b = anon_corpus.make(40, 0, 53)
    assert zk.anonymous_block(ctx, *b.args()) == (b"", b"", b"", b.balances, b.pendings, b.flags)


def test_malformed_account(ctx):
    b = anon_corpus.make(20, 30, 54)
    bal_b = bytearray(b.balances)
    bal_b[64 * 7 + 32:64 * 7 + 64] = bal_corpus.bad_order(bal_b[64 * 7 + 32:64 * 7 + 64])
    flags = bytearray(b.flags)
    flags[7] |= bal.BALANCE
    mem = b.members.copy()
    mem[mem == 7] = 8
    args = (b.keys, bytes(bal_b), b.pendings, bytes(flags), mem, b.tx_points, b.tx_extra, b.g_epoch, b.applied)
    got = zk.anonymous_block(ctx, *args)                                    # untouched: copied through
    assert got == aco.block(*args)[1] and got[3][64 * 7:64 * 8] == bytes(bal_b[64 * 7:64 * 8])
    mem7 = mem.copy()
    mem7[12 * 5 + 3] = 7                                                    # touched
    args7 = args[:4] + (mem7,) + args[5:]
    with pytest.raises(zk.SynthesisError) as e:                          # IoError(GroupDecodingError)
        zk.anonymous_block(ctx, *args7)
    assert e.value.code == -7 and "account 7" in str(e.value)
    assert aco.block(*args7)[0] == 7
    # the device form is asynchronous: the next synchronisation reports it, once
    bufs = _device_buffers(*args7)
    _device_call(ctx, bufs)
    with pytest.raises(zk.SynthesisError) as e:
        ctx.sync()
    assert e.value.code == -7 and "account 7" in str(e.value)
    ctx.sync()
    assert zk.anonymous_block(ctx, *args) == got                             # the context works after the error


def test_argument_errors(ctx):
    L = _lib.lib()
    z = [None] * 11
    assert L.zk_balances_anonymous_block(ctx._h, 1, None, None, None, None, 0, *z) == -2
    one = [b"\0"] * 4
    assert L.zk_balances_anonymous_block(ctx._h, 0, None, None, None, None, 1, *one, b"\0", b"\0", None, b"\0", None, None, None) == -2
    assert L.zk_balances_anonymous_block(ctx._h, (1 << 22) + 1, *one, 0, *([None] * 8), *([b"\0"] * 3)) == -2
    assert L.zk_balances_anonymous_block(ctx._h, 0, *([None] * 4), (1 << 18) + 1, *([b"\0"] * 8), None, None, None) == -2
    assert L.zk_balances_anonymous_block_device(ctx._h, 1, None, None, None, None, 0, *z) == -2


def _dev(b: bytes):
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda() if b else torch.zeros(1, dtype=torch.uint8, device="cuda")


def _device_buffers(keys, balances, pendings, flags, members, tx_points, tx_extra, g_epoch, applied):
    n_acct = len(flags)
    mem = np.asarray(members).astype(np.int64).astype(np.uint32).reshape(-1)
    n_tx = len(mem) // 12
    ins = [_dev(keys), _dev(balances), _dev(pendings), _dev(flags), torch.from_numpy(mem.view(np.int32)).cuda(), _dev(tx_points),
           _dev(tx_extra), _dev(g_epoch), _dev(applied)]
    z = lambda n: torch.full((max(n, 1),), 0xAB, dtype=torch.uint8, device="cuda")
    outs = [z(768 * n_tx), z(1664 * n_tx), z(n_tx), z(64 * n_acct), z(64 * n_acct), z(n_acct)]
    torch.cuda.synchronize()
    return n_acct, n_tx, ins, outs


def _device_call(ctx, bufs):
    n_acct, n_tx, ins, outs = bufs
    p = [t.data_ptr() for t in ins]
    zk.anonymous_block_device(ctx, n_acct, p[0], p[1], p[2], p[3], n_tx, *p[4:], *[t.data_ptr() for t in outs])


def test_device_form_equals_host_form(ctx, block):
    bufs = _device_buffers(*block.args())
    _device_call(ctx, bufs)
    ctx.sync()
    sizes = [768 * block.n_tx, 1664 * block.n_tx, block.n_tx, len(block.balances), len(block.pendings), len(block.flags)]
    got = tuple(t.cpu().numpy().tobytes()[:s] for t, s in zip(bufs[3], sizes))
    assert got == zk.anonymous_block(ctx, *block.args())


def test_ring_of_other_length_is_rejected():
    pt = bal_corpus.BAD_FIELD
    with pytest.raises(ValueError):
        zk.AnonymousTx(list(range(11)), [pt] * 11, pt, pt, pt)
    with pytest.raises(ValueError):
        zk.AnonymousTx(list(range(12)), [pt] * 13, pt, pt, pt)


# ---- end to end ---------------------------------------------------------------------------------------------------------
class _Key:
    """A toy CRS whose public inputs are the coordinates of 52 Jubjub points (the anonymous transfer's shape: 105 ic
    points), and proofs for chosen points."""

    def __init__(self, ctx, seed):
        n_points = zk.ANONYMOUS_POINTS
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
    """Four rings over 14 accounts, Bob's EncKey as account 0 and block one's g_epoch: transactions 0 and 2 proven on the
    balances they read, 1 with account 0's balance before its rollover in place of its first member's, 3 on another
    transaction's balances.  The verdicts come from
    the pairing check ([1, 0, 1, 0]); the final state is the module's loop with those verdicts."""
    assert jj.into_xy(G_EPOCH_1)[0] == jj.OK and jj.into_xy(BOB)[0] == jj.OK
    key = _Key(ctx, 71)
    try:
        b = anon_corpus.make(14, 4, 72, dup_frac=0.0, mask_p=(0.0, 1.0, 0.0, 0.0, 0.0))
        keys = BOB + b.keys[32:]
        flags = bytes([bal.BALANCE | bal.PENDING | bal.DUE, bal.PENDING | bal.DUE]) + b.flags[2:]
        rings = [[0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11], [1, 0, 12, 13, 2, 3, 4, 5, 6, 7, 8, 9],
                 [13, 12, 11, 10, 9, 8, 7, 6, 5, 4, 3, 0], [0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10]]
        txs = [zk.AnonymousTx(rings[k], _rows(b.tx_points[416 * k:416 * k + 384], 32), b.tx_points[416 * k + 384:416 * k + 416],
                              b.tx_extra[64 * k:64 * k + 32], b.tx_extra[64 * k + 32:64 * k + 64]) for k in range(4)]
        members = np.array(rings, np.uint32).reshape(-1)
        args = (keys, b.balances, b.pendings, flags, members, b.tx_points, b.tx_extra, G_EPOCH_1, bytes(4))
        reads = _rows(aco.block(*args)[1][0], 768)                   # what each transaction's proof is checked against

        def pts(k, acc_bytes):
            t = txs[k]
            return zk.anonymous_points([keys[32 * a:32 * a + 32] for a in t.members], t.left_ciphertexts, _rows(acc_bytes, 64),
                                       t.right_ciphertext, t.rvk, G_EPOCH_1, t.nonce)
        stale = b.balances[:64] + reads[1][64:]                      # account 0 before its rollover
        assumed = [reads[0], stale, reads[2], reads[0]]
        proofs = [key.prove(pts(k, assumed[k]), 80 + k) for k in range(4)]
        accounts = (keys, b.balances, b.pendings, flags)
        verdicts, state, enc_balances = zk.import_anonymous_block(ctx, key.pvk, accounts, txs, G_EPOCH_1, proofs)
        assert verdicts == [1, 0, 1, 0]
        assert enc_balances == b"".join(reads)
        # the module's loop, with the verdicts taken from the pairing check of each proof against what it reads
        def verdict(k, acc):
            return zk.verify_proofs_with_points(key.pvk, proofs[k], pts(k, b"".join(acc)), zk.ANONYMOUS_POINTS) == [1]
        bal_d, pend_d, due = bal.from_arrays(b.balances, b.pendings, flags)
        accs, st, final = ab.apply_block(14, bal_d, pend_d, due, ab.txs_of(members, b.tx_points), verdict)
        assert st == [0, 1, 0, 1]
        assert [b"".join(a) for a in accs] == reads
        assert state == bal.to_arrays(b.balances, b.pendings, flags, final)
        with pytest.raises(ValueError):
            bad = zk.AnonymousTx([14] + rings[0][1:], txs[0].left_ciphertexts, txs[0].right_ciphertext, txs[0].rvk, txs[0].nonce)
            zk.import_anonymous_block(ctx, key.pvk, accounts, [bad], G_EPOCH_1, proofs[:1])
    finally:
        key.free()
