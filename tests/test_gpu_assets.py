"""GPU tests of zk_assets_block(_device) and import_assets_block: a random block of thousands of mixed transfers, issues
and destroys over a few hundred slots against the C oracle byte for byte, across every output; one slot's chain longer
than three scan tiles with restarts inside it; n_tx = 0; a malformed stored ciphertext, named and not; argument errors;
the device form against the host form; a transfers-only block against zk_balances_confidential_block; and a block
imported end to end with proofs of a toy key of the confidential shape."""
import numpy as np
import pytest
import torch

from oracle import coracle as co
from tests.jubjub_oracle import assets as asr
from tests.jubjub_oracle import assets_coracle as ac
from tests.jubjub_oracle import assets_corpus
from tests.jubjub_oracle import bal_corpus
from tests.jubjub_oracle import balances as bal
from tests.jubjub_oracle import pyref as jj
from zero_chain_b200 import _lib
from zero_chain_b200 import groth16 as zk
from zero_chain_b200 import synthetic as sy

pytestmark = pytest.mark.gpu
SCAN_TILE = 128 * 8                       # elements per thread block of the scan's first level (balances.cu)
NAMES = ["balance_sender", "balance_after", "event_ct", "event_flags", "status", "balances", "pendings", "flags"]


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def block():
    return assets_corpus.make(300, 4000, 41, skew=1.2, issue_frac=0.1, destroy_frac=0.05, bad_points=30, bad_index=True)


def test_constants():
    assert (zk.ASSET_TRANSFER, zk.ASSET_ISSUE, zk.ASSET_DESTROY) == (asr.TRANSFER, asr.ISSUE, asr.DESTROY)


def test_random_block_equals_c_oracle(ctx, block):
    flags = np.frombuffer(block.flags, np.uint8)
    assert {f & 7 for f in flags} == set(range(8))
    got = zk.assets_block(ctx, *block.args())
    bad, want = ac.block(*block.args())
    assert bad is None
    assert set(want[4]) == {0, 1, 2, 3} and set(want[3]) == {0, 1, 2, 3}
    for g, w, name in zip(got, want, NAMES):
        assert g == w, name


def test_chain_longer_than_three_scan_tiles(ctx):
    b = assets_corpus.make(5, 5000, 42, skew=5.0, issue_frac=0.02, destroy_frac=0.01, bad_points=4)
    kinds = np.frombuffer(b.kind, np.uint8)
    assert np.bincount(b.slot_a).max() > 3 * SCAN_TILE
    assert ((kinds != 0) & (b.slot_a == 0)).sum() > 50                     # restarts inside the long chain
    assert zk.assets_block(ctx, *b.args()) == ac.block(*b.args())[1]


def test_no_transactions(ctx):
    b = assets_corpus.make(40, 0, 43)
    assert zk.assets_block(ctx, *b.args()) == (b"", b"", b"", b"", b"", b.balances, b.pendings, b.flags)


def test_malformed_slot(ctx):
    b = assets_corpus.make(20, 30, 44)
    bal_b = bytearray(b.balances)
    bal_b[64 * 7 + 32:64 * 7 + 64] = bal_corpus.bad_order(bal_b[64 * 7 + 32:64 * 7 + 64])
    flags = bytearray(b.flags)
    flags[7] |= bal.BALANCE
    sa, sb = b.slot_a.copy(), b.slot_b.copy()
    kinds = np.frombuffer(b.kind, np.uint8)
    sa[sa == 7] = 8
    sb[(sb == 7) & (kinds == 0)] = 8
    args = (bytes(bal_b), b.pendings, bytes(flags), b.kind, sa, sb, b.tx_points, b.applied)
    got = zk.assets_block(ctx, *args)                                      # not named: copied through
    assert got == ac.block(*args)[1] and got[5][64 * 7:64 * 8] == bytes(bal_b[64 * 7:64 * 8])
    kd = bytearray(b.kind)
    sa7 = sa.copy()
    kd[5], sa7[5] = zk.ASSET_DESTROY, 7                                    # named by a destroy
    args7 = (bytes(bal_b), b.pendings, bytes(flags), bytes(kd), sa7, sb, b.tx_points, b.applied)
    with pytest.raises(zk.SynthesisError) as e:
        zk.assets_block(ctx, *args7)
    assert e.value.code == -7 and "7" in str(e.value)
    assert ac.block(*args7)[0] == 7
    bufs = _device_buffers(*args7)
    _device_call(ctx, bufs)
    with pytest.raises(zk.SynthesisError) as e:
        ctx.sync()
    assert e.value.code == -7
    ctx.sync()
    assert zk.assets_block(ctx, *args) == got                              # the context works after the error


def test_argument_errors(ctx):
    L = _lib.lib()
    assert L.zk_assets_block(ctx._h, 1, None, None, None, 0, *([None] * 13)) == -2
    assert L.zk_assets_block(ctx._h, 0, None, None, None, (1 << 20) + 1, *([b"\0"] * 13)) == -2
    assert L.zk_assets_block(ctx._h, (1 << 22) + 1, *([b"\0"] * 3), 0, *([None] * 10), *([b"\0"] * 3)) == -2


def _dev(b: bytes):
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda() if b else torch.zeros(1, dtype=torch.uint8, device="cuda")


def _device_buffers(balances, pendings, flags, kind, slot_a, slot_b, tx_points, applied):
    """torch buffers of the inputs, and outputs with balance_after, event_ct and event_flags preset to 0xAB"""
    n, n_tx = len(flags), len(kind)
    idx = lambda v: torch.from_numpy(np.asarray(v).astype(np.int64).astype(np.uint32).view(np.int32)).cuda()
    ins = [_dev(balances), _dev(pendings), _dev(flags), _dev(bytes(kind)), idx(slot_a), idx(slot_b), _dev(tx_points), _dev(applied)]
    z = lambda m, v=0: torch.full((max(m, 1),), v, dtype=torch.uint8, device="cuda")
    outs = [z(64 * n_tx), z(64 * n_tx, 0xAB), z(128 * n_tx, 0xAB), z(n_tx, 0xAB), z(n_tx), z(64 * n), z(64 * n), z(n)]
    torch.cuda.synchronize()
    return n, n_tx, ins, outs


def _device_call(ctx, bufs):
    n, n_tx, ins, outs = bufs
    p = [t.data_ptr() for t in ins]
    zk.assets_block_device(ctx, n, p[0], p[1], p[2], n_tx, *p[3:], *[t.data_ptr() for t in outs])


def test_device_form_equals_host_form(ctx, block):
    bufs = _device_buffers(*block.args())
    _device_call(ctx, bufs)
    ctx.sync()
    n_tx = block.n_tx
    got = [t.cpu().numpy().tobytes() for t in bufs[3]]
    got[:5] = [g[:m * n_tx] for g, m in zip(got[:5], (64, 64, 128, 1, 1))]
    want = zk.assets_block(ctx, *block.args())
    st, kinds = np.frombuffer(want[4], np.uint8), np.frombuffer(block.kind, np.uint8)
    wrote_after = (st == 0) & (kinds == 0)
    wrote_event = (st == 0) & (kinds != 0)
    for g, w, m, wrote in ((got[1], want[1], 64, wrote_after), (got[2], want[2], 128, wrote_event), (got[3], want[3], 1, wrote_event)):
        g, w = np.frombuffer(g, np.uint8).reshape(-1, m), np.frombuffer(w, np.uint8).reshape(-1, m)
        assert (g[~wrote] == 0xAB).all() and np.array_equal(g[wrote], w[wrote])
    assert [got[0]] + got[4:] == [want[0]] + list(want[4:])


def test_transfers_only_equal_the_confidential_call(ctx):
    b = assets_corpus.make(200, 3000, 45, skew=1.1, issue_frac=0.0, destroy_frac=0.0, bad_points=20)
    b.applied = bytes(int(v == 1) for v in b.applied)                     # the confidential call applies any nonzero mask
    got = zk.assets_block(ctx, *b.args())
    conf = zk.confidential_block(ctx, *b.transfers())
    assert (got[0], got[1], got[4]) + got[5:] == conf


# ---- end to end ---------------------------------------------------------------------------------------------------------
class _Key:
    """A toy CRS whose public inputs are the coordinates of 11 Jubjub points (the confidential proof's shape), and proofs
    for chosen points."""

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
    """Genesis holds asset 0 for alice (balance, pending, due).  t0 issues asset 5 to alice; t1 is an issue with a bad
    proof, so t2's asset is 6, not 7; t3 sends asset 5 from alice to bob (its new slot rolls over the issued total); t4
    sends asset 0 with a bad proof; t5 destroys alice's asset 0 in the middle of that chain; t6 sends asset 0 again, against
    the absent balance.  The verdicts come from the pairing check: [1, 0, 1, 1, 0, 1, 1], in two rounds."""
    key = _Key(ctx, 81)
    try:
        rng = np.random.default_rng(82)
        misc = bal_corpus.encrypt(rng, 6)
        alice, bob, rvk, g_epoch, nonce, fee = (misc[32 * i:32 * i + 32] for i in range(6))
        dummy_ct = misc[64:128]
        table = bal_corpus.make(1, 3, 83, zero_frac=0.0, self_frac=0.0)
        tp = table.tx_points
        row = lambda k: [tp[128 * k + 32 * i:128 * k + 32 * i + 32] for i in range(4)]
        issued = bal_corpus.encrypt(rng, 2)
        txs = [zk.IssueTx(alice, issued[:32], fee, dummy_ct, issued[32:64], rvk, g_epoch, nonce),
               zk.IssueTx(bob, issued[64:96], fee, dummy_ct, issued[96:128], rvk, g_epoch, nonce),
               zk.IssueTx(bob, issued[64:96], fee, dummy_ct, issued[96:128], rvk, g_epoch, nonce),
               zk.AssetTransferTx(5, alice, bob, *row(0), rvk, g_epoch, nonce),
               zk.AssetTransferTx(0, alice, bob, *row(1), rvk, g_epoch, nonce),
               zk.DestroyTx(alice, 0, tp[:32], tp[64:96], dummy_ct, tp[96:128], rvk, g_epoch, nonce),
               zk.AssetTransferTx(0, alice, bob, *row(2), rvk, g_epoch, nonce)]
        total5 = bal.from_left_right(issued[:32], issued[32:64])
        rolled0 = bal.ct_add(table.balances[:64], table.pendings[:64])
        stale = table.balances[:64]                                         # t4 is proven against the balance before rollover
        proofs = [key.prove(txs[0].verify_points(), 90),
                  key.prove(txs[0].verify_points(), 91),                   # a valid proof of another statement
                  key.prove(txs[2].verify_points(), 93),
                  key.prove(txs[3].verify_points(total5), 94),
                  key.prove(txs[4].verify_points(stale), 95),
                  key.prove(txs[5].verify_points(), 96),
                  key.prove(txs[6].verify_points(bal.ZERO), 97)]
        flags0 = bal.BALANCE | bal.PENDING | bal.DUE
        state = ([(0, alice)], table.balances[:64], table.pendings[:64], bytes([flags0]))
        verdicts, ids, events, (slots, nb, npd, nf), rounds = zk.import_assets_block(ctx, key.pvk, state, txs, proofs, 5, bal.DUE)
        assert verdicts == [1, 0, 1, 1, 0, 1, 1]
        assert ids == [5, None, 6, None, None, None, None]
        assert rounds == 2
        assert slots == [(0, alice), (5, alice), (6, bob), (5, bob), (0, bob)]
        assert events[0] == total5 and events[1] is None and events[4] is None
        assert events[5] == (rolled0, b"")                                 # the failed t4 still rolled alice's asset 0 over
        # the module's loop over the same slots, with the verdicts taken from the pairing check
        index = {s: i for i, s in enumerate(slots)}
        n = len(slots)
        none = 0xFFFFFFFF
        rows = [(1, index[(5, alice)], none), (1, none, none), (1, index[(6, bob)], none), (0, index[(5, alice)], index[(5, bob)]),
                (0, index[(0, alice)], index[(0, bob)]), (2, index[(0, alice)], none), (0, index[(0, alice)], index[(0, bob)])]
        oracle_txs = [r + tuple(t.points()[32 * i:32 * i + 32] for i in range(4)) for r, t in zip(rows, txs)]

        def verdict(k, bs):
            pts = txs[k].verify_points(bs) if bs is not None else txs[k].verify_points()
            return zk.verify_proofs_with_points(key.pvk, proofs[k], pts, zk.CONFIDENTIAL_POINTS) == [1]
        balances = table.balances[:64] + bytes(64 * (n - 1))
        pendings = table.pendings[:64] + bytes(64 * (n - 1))
        flags = bytes([flags0] + [bal.DUE] * (n - 1))
        b_d, p_d, due = bal.from_arrays(balances, pendings, flags)
        bs, ba, ev, st, final = asr.apply_block(n, b_d, p_d, due, oracle_txs, verdict)
        assert st == [0, 3, 0, 0, 1, 0, 0]
        assert (nb, npd, nf) == asr.to_arrays(balances, pendings, flags, final)
        assert events[3] == ba[3] and events[6] == ba[6] and ev[5] == (rolled0, None)
        assert bs[6] == bal.ZERO
    finally:
        key.free()
