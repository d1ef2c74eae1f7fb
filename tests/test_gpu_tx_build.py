"""GPU tests of the transaction-building calls (zk_keys_from_seed_batch, zk_g_epoch_batch, zk_confidential_fields_batch,
zk_redjubjub_sign_batch) and their _device forms: every output byte-equal to the Python oracle on random and edge rows;
the reference's literals (tests/golden/tx_build.json); round trips through the existing calls — signatures made with rsk
verify under rvk one by one and in a batch, the derived dk decrypts the ciphertexts, and a block built entirely from the
new calls imports through confidential_import and block_import with every verdict 1 and the C oracle's final state; and
the argument errors."""
import json
import os

import numpy as np
import pytest

from tests import import_corpus as ic
from tests.jubjub_oracle import bal_coracle as bc
from tests.jubjub_oracle import bal_corpus
from tests.jubjub_oracle import pyref as jj
from tests.jubjub_oracle import redjubjub as rj
from tests.jubjub_oracle import tx_build as tb
from zero_chain_b200 import _lib
from zero_chain_b200 import groth16 as zk

pytestmark = pytest.mark.gpu
GOLD = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tx_build.json")))
SIGN_LENGTHS = [0, 1, 47, 48, 49, 127, 128, 129, 300]


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


def _t(b: bytes):
    import torch
    return torch.from_numpy(np.frombuffer(b if b else b"\0", np.uint8).copy()).cuda()


def _z(n: int):
    import torch
    return torch.full((max(n, 1),), 0xEE, dtype=torch.uint8, device="cuda")


def _u(v, dtype):
    import torch
    return torch.from_numpy(np.ascontiguousarray(v, dtype).view(np.int64 if dtype == np.uint64 else np.int32).copy()).cuda()


def _rows(t, size, n):
    b = t.cpu().numpy().tobytes()
    return [b[size * i:size * (i + 1)] for i in range(n)]


def _fields_row(f):
    return b"".join(f[k] for k in zk.CONFIDENTIAL_FIELDS)


# ---- parity with the oracle --------------------------------------------------------------------------------------------
def test_keys_match_oracle_both_forms(ctx):
    seeds = [b"", b"a", b"Alice" + b" " * 27, bytes(range(127)), bytes(128), bytes(range(129)) + b"x" * 300] + \
            [b"account %d" % i for i in range(40)]
    n = len(seeds)
    sks, dks, eks = zk.keys_from_seed(ctx, seeds)
    for i, s in enumerate(seeds):
        assert (sks[i], dks[i], eks[i]) == tb.keys(s), s
    pad = 5                                                  # the device form's offsets start past the buffer's head
    ds, doff = _t(b"\xa5" * pad + b"".join(seeds)), _u(zk.message_offsets(seeds) + np.uint64(pad), np.uint64)
    out = [_z(32 * n) for _ in range(3)]
    zk.keys_from_seed_device(ctx, n, ds.data_ptr(), doff.data_ptr(), *(o.data_ptr() for o in out))
    ctx.sync()
    assert [_rows(o, 32, n) for o in out] == [sks, dks, eks]


def test_g_epochs_match_oracle_both_forms(ctx):
    epochs = list(range(65)) + [2 ** 31, 2 ** 32 - 1]
    want = [tb.g_epoch(e) for e in epochs]
    assert zk.g_epoch(ctx, epochs) == [w[0] for w in want]
    tags = [w[1] for w in want]
    assert max(tags) >= 4 and tags[2] == 7 and 0 in tags     # the retry loop runs, and some epochs take the first tag
    out = _z(32 * len(epochs))
    dep = _u(epochs, np.uint32)
    zk.g_epoch_device(ctx, len(epochs), dep.data_ptr(), out.data_ptr())
    ctx.sync()
    assert _rows(out, 32, len(epochs)) == [w[0] for w in want]


def _fields_device(ctx, rows, g):
    sks, eks, amounts, fees, rs, alphas = zip(*rows)
    n = len(rows)
    sc = lambda v: b"".join(x.to_bytes(32, "little") for x in v)
    ins = [_t(sc(sks)), _t(b"".join(eks)), _u(amounts, np.uint32), _u(fees, np.uint32), _t(sc(rs)), _t(sc(alphas)), _t(g)]
    out = [_z(288 * n), _z(32 * n), _z(32 * n), _z(n)]
    zk.confidential_fields_device(ctx, n, *(x.data_ptr() for x in ins + out))
    ctx.sync()
    return _rows(out[0], 288, n), _rows(out[1], 32, n), _rows(out[2], 32, n), [int(v) for v in out[3].cpu().numpy()[:n]]


def test_confidential_fields_match_oracle_both_forms(ctx):
    rows = tb.edge_rows() + tb.random_rows(24, seed=21)
    g = tb.g_epoch(9)[0]
    want = [tb.confidential_fields(*r, g) for r in rows]
    fields, rsks, dks, st = zk.confidential_fields(ctx, *zip(*rows), g)
    assert [(_fields_row(f), a, b, s) for f, a, b, s in zip(fields, rsks, dks, st)] == want
    assert sorted(set(st)) == [0, 1, 2, 3]
    assert fields[1]["randomness"] == jj.encode(jj.IDENTITY)              # r = 0
    assert fields[2]["rvk"] == jj.encode(jj.IDENTITY) and rsks[2] == bytes(32)   # alpha = r_J - sk
    assert list(zip(*_fields_device(ctx, rows, g))) == want


def test_sign_matches_oracle_both_forms(ctx):
    rng = np.random.default_rng(31)
    sks = [0, 1, rj.R_J - 1] + [int.from_bytes(rng.bytes(64), "little") % rj.R_J for _ in range(len(SIGN_LENGTHS) * 3 - 3)]
    msgs = [rng.bytes(SIGN_LENGTHS[i % len(SIGN_LENGTHS)]) for i in range(len(sks))]
    ts = [rng.bytes(80) for _ in sks]
    sigs = zk.redjubjub_sign(ctx, sks, msgs, ts)
    assert sigs == [rj.sign(s, m, t) for s, m, t in zip(sks, msgs, ts)]
    n, pad = len(sks), 3
    dmsg, doff = _t(b"\x5a" * pad + b"".join(msgs)), _u(zk.message_offsets(msgs) + np.uint64(pad), np.uint64)
    dsk, dts, out = _t(b"".join(rj.scalar_bytes(s) for s in sks)), _t(b"".join(ts)), _z(64 * n)   # kept alive across the call
    zk.redjubjub_sign_device(ctx, n, dsk.data_ptr(), dts.data_ptr(), dmsg.data_ptr(), doff.data_ptr(), out.data_ptr())
    ctx.sync()
    assert _rows(out, 64, n) == sigs


# ---- the reference's literals ------------------------------------------------------------------------------------------
def test_known_answers(ctx):
    sks, dks, eks = zk.keys_from_seed(ctx, [GOLD["alice_seed"].encode()])
    assert eks[0].hex() == GOLD["alice_encryption_key"]["value"]
    g = zk.g_epoch(ctx, [0, 1])
    assert g[0].hex() == GOLD["g_epoch_0"]["value"] and g[1].hex() == GOLD["g_epoch_1"]["value"]
    ek_bob = zk.keys_from_seed(ctx, [b"Bob" + b" " * 29])[2]
    fields = zk.confidential_fields(ctx, [sks[0]], ek_bob, [10], [1], [5], [7], g[0])[0][0]
    assert fields["nonce"].hex() == GOLD["alice_nonce"]["value"]
    ct = bytes.fromhex(GOLD["enc10_by_alice"]["value"]) + bytes.fromhex(GOLD["randomness"]["value"])
    assert zk.elgamal_decrypt(ctx, dks, [ct]) == ([zk.ELGAMAL_OK], [10])


# ---- round trips through the existing calls ----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def batch(ctx):
    """600 transfers between 16 derived accounts"""
    rng = np.random.default_rng(41)
    seeds = [b"wallet %d" % i for i in range(16)]
    sks, dks, eks = zk.keys_from_seed(ctx, seeds)
    n = 600
    snd, rcp = rng.integers(0, 16, n), rng.integers(0, 16, n)
    fs = lambda: int.from_bytes(rng.bytes(64), "little") % rj.R_J
    amounts, fees = [int(v) for v in rng.integers(0, 10 ** 6, n)], [int(v) for v in rng.integers(0, 10 ** 6, n)]
    rs, alphas = [fs() for _ in range(n)], [fs() for _ in range(n)]
    g = zk.g_epoch(ctx, [3])[0]
    fields, rsks, fdks, st = zk.confidential_fields(ctx, [sks[s] for s in snd], [eks[r] for r in rcp], amounts, fees, rs, alphas, g)
    assert st == [0] * n and fdks == [dks[s] for s in snd]
    return dict(sks=sks, dks=dks, eks=eks, snd=snd, rcp=rcp, amounts=amounts, fees=fees, fields=fields, rsks=rsks, g=g)


def test_signatures_by_rsk_verify_under_rvk(ctx, batch):
    n = len(batch["rsks"])
    msgs = [b"extrinsic %d" % i + bytes(i % 130) for i in range(n)]
    ts = [os.urandom(80) for _ in range(n)]
    sigs = zk.redjubjub_sign(ctx, batch["rsks"], msgs, ts)
    rvks = [f["rvk"] for f in batch["fields"]]
    assert zk.redjubjub_verify(ctx, rvks, sigs, msgs) == [zk.REDJUBJUB_OK] * n
    assert zk.redjubjub_batch_verify(ctx, rvks, sigs, msgs) == (zk.REDJUBJUB_OK, None)
    bad = list(msgs)
    bad[17] = bytes([bad[17][0] ^ 1]) + bad[17][1:]
    verdicts = zk.redjubjub_verify(ctx, rvks, sigs, bad)
    assert verdicts[17] == zk.REDJUBJUB_BAD_EQUATION and verdicts.count(zk.REDJUBJUB_OK) == n - 1
    assert zk.redjubjub_batch_verify(ctx, rvks, sigs, bad)[0] == zk.REDJUBJUB_BAD_EQUATION


def test_derived_keys_decrypt_the_ciphertexts(ctx, batch):
    f, dks = batch["fields"], batch["dks"]
    sender = zk.elgamal_decrypt(ctx, [dks[s] for s in batch["snd"]], [x["amount_sender"] + x["randomness"] for x in f])
    recipient = zk.elgamal_decrypt(ctx, [dks[r] for r in batch["rcp"]], [x["amount_recipient"] + x["randomness"] for x in f])
    fee = zk.elgamal_decrypt(ctx, [dks[s] for s in batch["snd"]], [x["fee_sender"] + x["randomness"] for x in f])
    n = len(f)
    assert sender == recipient == ([zk.ELGAMAL_OK] * n, batch["amounts"])
    assert fee == ([zk.ELGAMAL_OK] * n, batch["fees"])


def test_built_block_imports(ctx, batch):
    key = ic.ForgeKey(5)
    pvk = zk.PreparedVerifyingKey.prepare(ctx, key.params_bytes)
    try:
        n = 120
        state = bal_corpus.make(16, n, 43, zero_frac=0.0)
        accounts = (state.balances, state.pendings, state.flags)
        snd, rcp = batch["snd"][:n], batch["rcp"][:n]
        txs = [zk.ConfidentialTx(int(s), int(r), **f) for s, r, f in zip(snd, rcp, batch["fields"][:n])]
        pts = b"".join(t.points() for t in txs)
        bad, out = bc.block(*accounts, snd.astype(np.uint32), rcp.astype(np.uint32), pts, b"\x01" * n)
        assert bad is None
        bs = out[0]
        rows = b"".join(zk.confidential_points(t.address_sender, t.address_recipient, t.amount_sender, t.amount_recipient, t.randomness,
                                               t.fee_sender, bs[64 * k:64 * k + 64], t.rvk, t.g_epoch, t.nonce) for k, t in enumerate(txs))
        proofs = key.proofs(rows, [True] * n)
        got = zk.confidential_import(ctx, pvk, accounts, txs, proofs)
        assert got[0] == [1] * n
        assert got[2] == out[1] and got[1] == tuple(out[3:])
        msgs = [b"confidential_transfer %d" % i for i in range(n)]
        sigs = zk.redjubjub_sign(ctx, batch["rsks"][:n], msgs, [bytes([i % 256]) * 80 for i in range(n)])
        block = zk.block_import(ctx, pvk, None, ([t.rvk for t in txs], sigs, msgs, None), confidential=(accounts, txs, proofs))
        assert block.confidential == got
    finally:
        pvk.free()


# ---- errors ------------------------------------------------------------------------------------------------------------
def test_errors(ctx):
    g = zk.g_epoch(ctx, [0])[0]
    ek = zk.keys_from_seed(ctx, [b"x"])[2][0]
    row = lambda sk=1, r=2, al=3: zk.confidential_fields(ctx, [5, sk], [ek, ek], [1, 1], [1, 1], [5, r], [5, al], g)
    for kw, what in ((dict(sk=rj.R_J), "sks"), (dict(r=rj.R_J), "rs"), (dict(al=2 ** 256 - 1), "alphas")):
        with pytest.raises(zk.SynthesisError, match=r"%s\[1\]" % what) as e:
            row(**kw)
        assert e.value.code == -8
    for bad_g, _ in tb.bad_recipient_keys():
        with pytest.raises(zk.SynthesisError, match="g_epoch") as e:
            zk.confidential_fields(ctx, [1], [ek], [1], [1], [2], [3], bad_g)
        assert e.value.code == -7
    with pytest.raises(zk.SynthesisError, match=r"sks\[0\]") as e:
        zk.redjubjub_sign(ctx, [rj.R_J], [b"m"], [bytes(80)])
    assert e.value.code == -8
    L = _lib.lib()
    sk, t, m = np.zeros(64, np.uint8), np.zeros(160, np.uint8), np.zeros(4, np.uint8)
    off = np.array([0, 3, 2], np.uint64)
    sigs = np.zeros(128, np.uint8)
    assert L.zk_redjubjub_sign_batch(ctx._h, 2, sk.ctypes.data, t.ctypes.data, m.ctypes.data, off.ctypes.data, sigs.ctypes.data) == -2
    assert L.zk_keys_from_seed_batch(ctx._h, 2, m.ctypes.data, off.ctypes.data, sigs.ctypes.data, sigs.ctypes.data, sigs.ctypes.data) == -2
    assert L.zk_g_epoch_batch(ctx._h, 1, None, sigs.ctypes.data) == -2
    assert zk.confidential_fields(ctx, [], [], [], [], [], [], g) == ([], [], [], [])
    assert zk.redjubjub_sign(ctx, [], [], []) == [] and zk.g_epoch(ctx, []) == [] and zk.keys_from_seed(ctx, []) == ([], [], [])
    # the device form reports a non-canonical scalar at the next sync, and the context stays usable
    import torch
    bufs = [_t(b"\xff" * 32), _t(ek), _u([1], np.uint32), _u([1], np.uint32), _t(bytes(32)), _t(bytes(32)), _t(g), _z(288), _z(32), _z(32), _z(1)]
    zk.confidential_fields_device(ctx, 1, *(x.data_ptr() for x in bufs))
    with pytest.raises((zk.SynthesisError, _lib.ZkError)) as e:
        ctx.sync()
    assert e.value.code == -8
    torch.cuda.synchronize()
    assert zk.g_epoch(ctx, [0]) == [g]
