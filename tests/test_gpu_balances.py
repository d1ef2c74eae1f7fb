"""GPU tests of zk_balances_confidential_block(_device) and import_confidential_block: a random block of thousands of
transfers over a few hundred accounts with a skewed sender choice (self-transfers, due and non-due accounts, absent
balances and pendings, zeros in the mask, every point-rejection class, out-of-range indices) against the C oracle byte
for byte; one sender's chain longer than a scan tile; n_tx = 0; a malformed stored ciphertext, touched and untouched; the
device form against the host form; and a block imported end to end with proofs of a toy key of the confidential shape."""
import numpy as np
import pytest
import torch

from oracle import coracle as co
from tests.jubjub_oracle import bal_coracle as bc
from tests.jubjub_oracle import bal_corpus
from tests.jubjub_oracle import balances as bal
from tests.jubjub_oracle import pyref as jj
from zero_chain_b200 import _lib
from zero_chain_b200 import groth16 as zk
from zero_chain_b200 import synthetic as sy

pytestmark = pytest.mark.gpu
SCAN_TILE = 128 * 8                       # elements per thread block of the scan's first level (balances.cu)


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def block():
    return bal_corpus.make(300, 6000, 21, skew=1.2, bad_points=30, bad_index=True, self_frac=0.05)


def test_constants():
    assert (zk.ACCOUNT_BALANCE, zk.ACCOUNT_PENDING, zk.ACCOUNT_DUE) == (bal.BALANCE, bal.PENDING, bal.DUE)
    assert (zk.BLOCK_APPLIED, zk.BLOCK_NOT_APPLIED, zk.BLOCK_BAD_POINT, zk.BLOCK_BAD_INDEX) == \
        (bal.APPLIED, bal.NOT_APPLIED, bal.BAD_POINT, bal.BAD_INDEX)


def test_random_block_equals_c_oracle(ctx, block):
    flags = np.frombuffer(block.flags, np.uint8)
    assert {f & 7 for f in flags} == set(range(8))                          # every presence / due combination
    assert (block.sender == block.recipient).sum() > 100
    assert np.bincount(block.sender[block.sender < 300]).max() > 500         # long chains
    got = zk.confidential_block(ctx, *block.args())
    bad, want = bc.block(*block.args())
    assert bad is None
    assert set(want[2]) == {0, 1, 2, 3}
    for g, w, name in zip(got, want, ["balance_sender", "balance_after", "status", "balances", "pendings", "flags"]):
        assert g == w, name


def test_chain_longer_than_a_scan_tile(ctx):
    b = bal_corpus.make(5, 5000, 22, skew=5.0, bad_points=4)
    assert np.bincount(b.sender).max() > 3 * SCAN_TILE
    assert zk.confidential_block(ctx, *b.args()) == bc.block(*b.args())[1]


def test_no_transactions(ctx):
    b = bal_corpus.make(40, 0, 23)
    assert zk.confidential_block(ctx, *b.args()) == (b"", b"", b"", b.balances, b.pendings, b.flags)


def test_malformed_account(ctx):
    b = bal_corpus.make(20, 30, 24)
    bal_b = bytearray(b.balances)
    bal_b[64 * 7 + 32:64 * 7 + 64] = bal_corpus.bad_order(bal_b[64 * 7 + 32:64 * 7 + 64])
    flags = bytearray(b.flags)
    flags[7] |= bal.BALANCE
    s, r = b.sender.copy(), b.recipient.copy()
    s[s == 7] = 8
    r[r == 7] = 8
    args = (bytes(bal_b), b.pendings, bytes(flags), s, r, b.tx_points, b.applied)
    got = zk.confidential_block(ctx, *args)                                  # untouched: copied through
    assert got == bc.block(*args)[1] and got[3][64 * 7:64 * 8] == bytes(bal_b[64 * 7:64 * 8])
    r7 = r.copy()
    r7[5] = 7                                                                # touched
    with pytest.raises(zk.SynthesisError) as e:                          # IoError(GroupDecodingError)
        zk.confidential_block(ctx, bytes(bal_b), b.pendings, bytes(flags), s, r7, b.tx_points, b.applied)
    assert e.value.code == -7 and "account 7" in str(e.value)
    assert bc.block(bytes(bal_b), b.pendings, bytes(flags), s, r7, b.tx_points, b.applied)[0] == 7
    # the device form is asynchronous: the next synchronisation reports it, once
    bufs = _device_buffers(bytes(bal_b), b.pendings, bytes(flags), s, r7, b.tx_points, b.applied)
    _device_call(ctx, bufs)
    with pytest.raises(zk.SynthesisError) as e:
        ctx.sync()
    assert e.value.code == -7 and "account 7" in str(e.value)
    ctx.sync()
    # the context works after the error
    assert zk.confidential_block(ctx, *args) == got


def test_argument_errors(ctx):
    L = _lib.lib()
    assert L.zk_balances_confidential_block(ctx._h, 1, None, None, None, 0, None, None, None, None, None, None, None, None, None, None) == -2
    assert L.zk_balances_confidential_block(ctx._h, (1 << 22) + 1, *([b"\0"] * 3), 0, *([None] * 7), *([b"\0"] * 3)) == -2


def _dev(b: bytes):
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda() if b else torch.zeros(1, dtype=torch.uint8, device="cuda")


def _device_buffers(balances, pendings, flags, sender, recipient, tx_points, applied):
    """torch buffers of the inputs, and outputs with balance_after preset to 0xAB"""
    n_acct, n_tx = len(flags), len(sender)
    idx = lambda v: torch.from_numpy(np.asarray(v).astype(np.int64).astype(np.uint32).view(np.int32)).cuda()
    ins = [_dev(balances), _dev(pendings), _dev(flags), idx(sender), idx(recipient), _dev(tx_points), _dev(applied)]
    outs = [torch.zeros(64 * n_tx, dtype=torch.uint8, device="cuda"), torch.full((64 * n_tx,), 0xAB, dtype=torch.uint8, device="cuda"),
            torch.zeros(n_tx, dtype=torch.uint8, device="cuda"), torch.zeros(64 * n_acct, dtype=torch.uint8, device="cuda"),
            torch.zeros(64 * n_acct, dtype=torch.uint8, device="cuda"), torch.zeros(n_acct, dtype=torch.uint8, device="cuda")]
    torch.cuda.synchronize()
    return n_acct, n_tx, ins, outs


def _device_call(ctx, bufs):
    n_acct, n_tx, ins, outs = bufs
    p = [t.data_ptr() for t in ins]
    zk.confidential_block_device(ctx, n_acct, p[0], p[1], p[2], n_tx, *p[3:], *[t.data_ptr() for t in outs])


def test_device_form_equals_host_form(ctx, block):
    bufs = _device_buffers(*block.args())
    _device_call(ctx, bufs)
    ctx.sync()
    got = [t.cpu().numpy().tobytes() for t in bufs[3]]
    want = zk.confidential_block(ctx, *block.args())
    st = np.frombuffer(want[2], np.uint8)
    after = np.frombuffer(got[1], np.uint8).reshape(-1, 64)
    assert (after[st != 0] == 0xAB).all()                                   # written for applied transactions only
    ba = np.frombuffer(want[1], np.uint8).reshape(-1, 64)
    assert np.array_equal(after[st == 0], ba[st == 0])
    assert [got[0]] + got[2:] == [want[0]] + list(want[2:])


# ---- end to end ---------------------------------------------------------------------------------------------------------
class _Key:
    """A toy CRS whose public inputs are the coordinates of 11 Jubjub points (the confidential transfer's shape), and
    proofs for chosen points."""

    def __init__(self, ctx, seed):
        n_points = zk.CONFIDENTIAL_POINTS
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
    """Sender 0 sends four transfers to 1: t1 valid, t2 with a bad proof, t3 proven against the balance without t2, t4
    against the balance with t2.  The verdicts come from the pairing check: [1, 0, 1, 0], in two rounds."""
    key = _Key(ctx, 61)
    try:
        b = bal_corpus.make(3, 4, 62, zero_frac=0.0, self_frac=0.0)
        flags = bytes([bal.BALANCE | bal.PENDING | bal.DUE, bal.PENDING, 0])
        misc = bal_corpus.encrypt(np.random.default_rng(63), 3)             # addresses, rvk, g_epoch, nonce: valid points
        addr_a, addr_b, rvk, g_epoch, nonce = misc[0:32], misc[32:64], misc[64:96], misc[96:128], misc[128:160]
        txs = [zk.ConfidentialTx(0, 1, addr_a, addr_b, *[b.tx_points[128 * k + 32 * i:128 * k + 32 * i + 32] for i in range(4)],
                                 rvk, g_epoch, nonce) for k in range(4)]
        # the sender's balance as each proof assumes it
        rolled = bal.ct_add(b.balances[:64], b.pendings[:64])
        apf = [bal.ct_add(bal.from_left_right(t.amount_sender, t.randomness), bal.from_left_right(t.fee_sender, t.randomness)) for t in txs]
        without_t2 = bal.ct_sub(rolled, apf[0])
        with_t2 = bal.ct_sub(without_t2, apf[1])
        assumed = [rolled, None, without_t2, with_t2]

        def pts(t, bs):
            return zk.confidential_points(t.address_sender, t.address_recipient, t.amount_sender, t.amount_recipient, t.randomness,
                                          t.fee_sender, bs, t.rvk, t.g_epoch, t.nonce)
        proofs = [key.prove(pts(txs[k], assumed[k]), 70 + k) if assumed[k] else key.prove(pts(txs[1], rolled), 71) for k in range(4)]
        accounts = (b.balances, b.pendings, flags)
        verdicts, state, after, rounds = zk.import_confidential_block(ctx, key.pvk, accounts, txs, proofs)
        assert verdicts == [1, 0, 1, 0]
        assert rounds == 2 <= 1 + 2                                         # two failures in the one chain
        # the module's loop, with the verdicts taken from the pairing check of each proof against what it reads
        def verdict(k, bs):
            return zk.verify_proofs_with_points(key.pvk, proofs[k], pts(txs[k], bs), zk.CONFIDENTIAL_POINTS) == [1]
        tx_tuples = [(t.sender, t.recipient, t.amount_sender, t.amount_recipient, t.fee_sender, t.randomness) for t in txs]
        bal_d, pend_d, due = bal.from_arrays(b.balances, b.pendings, flags)
        bs, ba, st, final = bal.apply_block(3, bal_d, pend_d, due, tx_tuples, verdict)
        assert st == [0, 1, 0, 1]
        assert state == bal.to_arrays(b.balances, b.pendings, flags, final)
        assert after[:64] == ba[0] and after[128:192] == ba[2] and after[64:128] == after[192:] == bytes(64)
        # a block without failures takes one round
        v1, _, _, r1 = zk.import_confidential_block(ctx, key.pvk, accounts, txs[:1], proofs[:1])
        assert v1 == [1] and r1 == 1
    finally:
        key.free()
