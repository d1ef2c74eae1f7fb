"""GPU tests of zk_anonymous_fields_batch and its _device form: every output byte-equal to the Python oracle on edge and
random rows, and to the C oracle on a few thousand random rows; a key table much larger than the rings, with failing keys
no ring names; oracle-free round trips — the recipient's ciphertext decrypts to the amount and each decoy's to 0 under
keys from zk_keys_from_seed_batch, and signatures made with rsk verify under rvk; a block of anonymous transfers built
with the call imports through anonymous_import and block_import with every verdict 1, the C oracle's final state, and
balances that decrypt to start - sent + received; and the argument errors."""
import numpy as np
import pytest

from tests import import_anon_corpus as iac
from tests.jubjub_oracle import anon_build as ab
from tests.jubjub_oracle import anon_build_coracle as abc
from tests.jubjub_oracle import anon_coracle as aco
from tests.jubjub_oracle import pyref as jj
from tests.jubjub_oracle import redjubjub as rj
from tests.jubjub_oracle import tx_build as tb
from tests.jubjub_oracle import tx_coracle as tc
from zero_chain_b200 import _lib
from zero_chain_b200 import groth16 as zk

pytestmark = pytest.mark.gpu
sc = lambda v: b"".join(x.to_bytes(32, "little") for x in v)


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


def _u32(v):
    import torch
    return torch.from_numpy(np.ascontiguousarray(np.asarray(v, np.int64).reshape(-1).astype(np.uint32)).view(np.int32).copy()).cuda()


def _rows(t, size, n):
    b = t.cpu().numpy().tobytes()
    return [b[size * i:size * (i + 1)] for i in range(n)]


def _flat(f):
    return b"".join(f["enc_keys"]) + b"".join(f["left_ciphertexts"]) + f["right_ciphertext"] + f["rvk"] + f["nonce"]


def _host(ctx, table, rows, g):
    sks, rings, s, t, amounts, rs, alphas = zip(*rows)
    fields, rsks, dks, st = zk.anonymous_fields(ctx, table, sks, rings, list(zip(s, t)), amounts, rs, alphas, g)
    return [(_flat(f), a, b, c) for f, a, b, c in zip(fields, rsks, dks, st)]


def _device(ctx, table, rows, g):
    sks, rings, s, t, amounts, rs, alphas = zip(*rows)
    n = len(rows)
    ky = _t(b"".join(table)) if table else None
    ins = [_t(sc(sks)), _u32(rings), _t(bytes(np.array(list(zip(s, t)), np.uint8).reshape(-1))), _u32(amounts), _t(sc(rs)), _t(sc(alphas)),
           _t(g)]
    out = [_z(864 * n), _z(32 * n), _z(32 * n), _z(n)]
    zk.anonymous_fields_device(ctx, len(table), ky.data_ptr() if ky is not None else 0, n, *(x.data_ptr() for x in ins + out))
    ctx.sync()
    return list(zip(_rows(out[0], 864, n), _rows(out[1], 32, n), _rows(out[2], 32, n), [int(v) for v in out[3].cpu().numpy()[:n]]))


def _c(table, rows, g):
    sks, rings, s, t, amounts, rs, alphas = zip(*rows)
    return abc.anonymous_fields(b"".join(table), sc(sks), rings, list(zip(s, t)), amounts, sc(rs), sc(alphas), g)


# ---- parity with the oracles -------------------------------------------------------------------------------------------
def test_edge_rows_match_oracle_both_forms(ctx):
    table = ab.key_table()
    rows = ab.edge_rows()
    g = tb.g_epoch(9)[0]
    want = [ab.anonymous_fields(table, *r, g) for r in rows]
    got = _host(ctx, table, rows, g)
    assert got == want
    assert {w[3] for w in want} == {0, 1, 2, 3, zk.ANON_BAD_INDEX, zk.ANON_BAD_POSITIONS}
    ident = jj.encode(jj.IDENTITY)
    assert got[5][0][768:800] == ident                                         # r = 0: right_ciphertext is O
    assert got[8][0][800:832] == ident and got[8][1] == bytes(32)             # alpha = r_J - sk: rvk is O
    assert _device(ctx, table, rows, g) == want


def test_random_rows_match_oracles_both_forms(ctx):
    table = [tb.keys(b"random table %d" % i)[2] for i in range(64)]
    g = tb.g_epoch(2)[0]
    few = ab.random_rows(16, 64, seed=5)
    assert _host(ctx, table, few, g) == [ab.anonymous_fields(table, *r, g) for r in few]
    many = ab.random_rows(3000, 64, seed=6)                              # several grid strides of the left pass
    want = _c(table, many, g)
    assert _host(ctx, table, many, g) == want
    assert _device(ctx, table, many, g) == want


def test_large_table_with_unnamed_failing_keys(ctx):
    """20000 keys, every 7th one failing EncryptionKey::read; the rings name 300 good ones.  The rows equal those built
    over a table of just the named keys."""
    bad = [k for k, _ in tb.bad_recipient_keys()]
    good = tc.keys([b"big %d" % i for i in range(300)])[2]
    n_keys = 20000
    table, named = [], []                                   # named[i]: the first table slot holding good[i]
    for k in range(n_keys):
        if k % 7 == 3:
            table.append(bad[k % 4])
        else:
            j = k - k // 7 - (k % 7 > 3)                     # good keys before slot k
            if j < 300:
                named.append(k)
            table.append(good[j % 300])
    rows = ab.random_rows(500, 300, seed=8)
    g = tb.g_epoch(4)[0]
    big_rows = [(sk, [named[m] for m in ring], s, t, a, r, al) for sk, ring, s, t, a, r, al in rows]
    want = _c(good, rows, g)
    assert all(w[3] == 0 for w in want)
    assert _host(ctx, table, big_rows, g) == want
    assert _device(ctx, table, big_rows, g) == want


def test_no_keys(ctx):
    g = tb.g_epoch(0)[0]
    rows = [(5, list(range(11)), 0, 1, 1, 2, 3), (6, [0] * 11, 3, 3, 1, 2, 3)]
    want = [(bytes(864), bytes(32), bytes(32), zk.ANON_BAD_INDEX), (bytes(864), bytes(32), bytes(32), zk.ANON_BAD_POSITIONS)]
    assert _host(ctx, [], rows, g) == want == _device(ctx, [], rows, g)


# ---- round trips through the existing calls ----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def wallets(ctx):
    seeds = [b"anon wallet %d" % i for i in range(48)]
    return zk.keys_from_seed(ctx, seeds)


def _draw(rng, n_acct, n):
    """n transfers over n_acct accounts: (sender, ring as MultiEncKeys indices, s, t, members in ring order)"""
    out = []
    for _ in range(n):
        acc = [int(v) for v in rng.choice(n_acct, 12, replace=False)]
        sender, ring = acc[0], acc[1:]
        s, t = (int(v) for v in rng.choice(12, 2, replace=False))
        members = [None] * 12
        members[s], members[t] = sender, ring[0]
        it = iter(ring[1:])
        members = [m if m is not None else next(it) for m in members]
        out.append((sender, ring, s, t, members))
    return out


def test_ciphertexts_decrypt_and_signatures_verify(ctx, wallets):
    sks, dks, eks = wallets
    rng = np.random.default_rng(17)
    n = 400
    draws = _draw(rng, len(eks), n)
    fs = lambda: int.from_bytes(rng.bytes(64), "little") % rj.R_J
    amounts = [int(v) for v in rng.integers(0, 10 ** 6, n)]
    g = zk.g_epoch(ctx, [5])[0]
    fields, rsks, fdks, st = zk.anonymous_fields(ctx, eks, [sks[d[0]] for d in draws], [d[1] for d in draws], [(d[2], d[3]) for d in draws],
                                                 amounts, [fs() for _ in range(n)], [fs() for _ in range(n)], g)
    assert st == [0] * n and fdks == [dks[d[0]] for d in draws]
    cts, keys, want = [], [], []
    for (sender, ring, s, t, members), f, a in zip(draws, fields, amounts):
        assert f["enc_keys"] == [eks[m] for m in members]
        for p, m in enumerate(members):
            if p != s:
                cts.append(f["left_ciphertexts"][p] + f["right_ciphertext"])
                keys.append(dks[m])
                want.append(a if p == t else 0)
    assert zk.elgamal_decrypt(ctx, keys, cts) == ([zk.ELGAMAL_OK] * len(want), want)
    msgs = [b"anonymous_transfer %d" % i for i in range(n)]
    sigs = zk.redjubjub_sign(ctx, rsks, msgs, [rng.bytes(80) for _ in range(n)])
    rvks = [f["rvk"] for f in fields]
    assert zk.redjubjub_verify(ctx, rvks, sigs, msgs) == [zk.REDJUBJUB_OK] * n
    assert zk.redjubjub_batch_verify(ctx, rvks, sigs, msgs) == (zk.REDJUBJUB_OK, None)


def test_built_block_imports(ctx, wallets):
    """accounts with balances encrypt(start) under their own keys; a few hundred anonymous transfers built with the new call;
    proofs forged over the points the module reads.  Every verdict is 1, the state is the C oracle's, and every account's
    balance plus pending decrypts to start - sent + received."""
    sks, dks, eks = wallets
    n_acct, n = len(eks), 300
    rng = np.random.default_rng(23)
    start = [10000 + 37 * a for a in range(n_acct)]
    g = zk.g_epoch(ctx, [7])[0]
    fs = lambda: int.from_bytes(rng.bytes(64), "little") % rj.R_J
    bf, _, _, bst = zk.confidential_fields(ctx, sks, eks, start, [0] * n_acct, [fs() for _ in range(n_acct)], [fs() for _ in range(n_acct)], g)
    assert bst == [0] * n_acct
    balances = b"".join(f["amount_sender"] + f["randomness"] for f in bf)    # encrypt(start) under the account's own key
    assert zk.elgamal_decrypt(ctx, dks, balances) == ([zk.ELGAMAL_OK] * n_acct, start)
    accounts = (b"".join(eks), balances, bytes(64 * n_acct), bytes([zk.ACCOUNT_BALANCE]) * n_acct)
    draws = _draw(rng, n_acct, n)
    amounts = [int(v) for v in rng.integers(1, 60, n)]
    fields, rsks, _, st = zk.anonymous_fields(ctx, eks, [sks[d[0]] for d in draws], [d[1] for d in draws], [(d[2], d[3]) for d in draws],
                                              amounts, [fs() for _ in range(n)], [fs() for _ in range(n)], g)
    assert st == [0] * n
    txs = [zk.AnonymousTx(d[4], f["left_ciphertexts"], f["right_ciphertext"], f["rvk"], f["nonce"]) for d, f in zip(draws, fields)]
    members = np.array([t.members for t in txs], np.uint32).reshape(-1)
    bad, out = aco.block(*accounts, members, b"".join(t.points() for t in txs), b"".join(t.rvk + t.nonce for t in txs), g, b"\x01" * n)
    assert bad is None and out[2] == bytes(n)                                  # every transaction applied
    eb = out[0]
    rows = b"".join(zk.anonymous_points(f["enc_keys"], f["left_ciphertexts"], [eb[768 * k + 64 * m:768 * k + 64 * m + 64] for m in range(12)],
                                        f["right_ciphertext"], f["rvk"], g, f["nonce"]) for k, f in enumerate(fields))
    assert rows == out[1]                                                      # the built enc_keys are the ring's table keys
    key = iac.ForgeKey(zk.ANONYMOUS_POINTS, 29)
    pvk = zk.PreparedVerifyingKey.prepare(ctx, key.params_bytes)
    try:
        proofs = key.proofs(rows, [True] * n)
        got = zk.anonymous_import(ctx, pvk, None, accounts, txs, g, proofs)
        assert got[0] == [1] * n
        assert got[1] == tuple(out[3:]) and got[2] == eb
        msgs = [b"anonymous_transfer %d" % i for i in range(n)]
        sigs = zk.redjubjub_sign(ctx, rsks, msgs, [bytes([i % 256]) * 80 for i in range(n)])
        block = zk.block_import(ctx, None, pvk, ([t.rvk for t in txs], sigs, msgs, None), anonymous=(accounts, txs, g, proofs))
        assert block.anonymous == got
    finally:
        pvk.free()
    nb, npd, nf = got[1]
    want = list(start)
    for (sender, ring, _, _, _), a in zip(draws, amounts):
        want[sender] -= a
        want[ring[0]] += a
    touched = [a for a in range(n_acct) if nf[a] & zk.ACCOUNT_PENDING]
    untouched = [a for a in range(n_acct) if not nf[a] & zk.ACCOUNT_PENDING]
    assert len(touched) > n_acct // 2
    dec = zk.elgamal_decrypt(ctx, [dks[a] for a in touched], [nb[64 * a:64 * a + 64] for a in touched],
                             [npd[64 * a:64 * a + 64] for a in touched])
    assert dec == ([zk.ELGAMAL_OK] * len(touched), [want[a] for a in touched])
    for a in untouched:
        assert want[a] == start[a] and nb[64 * a:64 * a + 64] == balances[64 * a:64 * a + 64]


# ---- errors ------------------------------------------------------------------------------------------------------------
def test_errors(ctx, wallets):
    import torch
    _, _, eks = wallets
    g = zk.g_epoch(ctx, [0])[0]
    ring = list(range(11))
    row = lambda sk=1, r=2, al=3: zk.anonymous_fields(ctx, eks, [5, sk], [ring, ring], [(0, 1), (0, 1)], [1, 1], [5, r], [5, al], g)
    for kw, what in ((dict(sk=rj.R_J), "sks"), (dict(r=rj.R_J), "rs"), (dict(al=2 ** 256 - 1), "alphas")):
        with pytest.raises(zk.SynthesisError, match=r"%s\[1\]" % what) as e:
            row(**kw)
        assert e.value.code == -8
    for bad_g, _ in tb.bad_recipient_keys():
        with pytest.raises(zk.SynthesisError, match="g_epoch") as e:
            zk.anonymous_fields(ctx, eks, [1], [ring], [(0, 1)], [1], [2], [3], bad_g)
        assert e.value.code == -7
    assert zk.anonymous_fields(ctx, eks, [], [], [], [], [], [], g) == ([], [], [], [])
    L = _lib.lib()
    b = np.zeros(2048, np.uint8)
    p = b.ctypes.data
    assert L.zk_anonymous_fields_batch(ctx._h, 1, None, 1, *([p] * 11)) == -2                 # keys NULL with n_keys > 0
    assert L.zk_anonymous_fields_batch(ctx._h, 0, None, 1, p, None, *([p] * 9)) == -2         # rings NULL
    assert L.zk_anonymous_fields_batch(ctx._h, 0, None, 0, *([None] * 11)) == 0                # an empty call
    assert L.zk_anonymous_fields_batch(ctx._h, 1, p, (1 << 22) + 1, *([p] * 11)) == -2       # too many rows
    assert L.zk_anonymous_fields_batch_device(ctx._h, (1 << 24) + 1, p, 1, *([p] * 11)) == -2  # too many keys
    assert L.zk_anonymous_fields_batch_device(ctx._h, 1, None, 1, *([p] * 11)) == -2
    assert L.zk_anonymous_fields_batch_device(ctx._h, 0, None, 0, *([None] * 11)) == 0
    # the device form reports a non-canonical scalar or a bad g_epoch at the next sync, and the context stays usable
    good = [(5, ring, 0, 1, 7, 8, 9)]
    for sk, gb, code in ((rj.R_J, g, -8), (5, tb.bad_recipient_keys()[1][0], -7)):
        ky = _t(b"".join(eks))
        bufs = [_t(sc([sk])), _u32([ring]), _t(bytes([0, 1])), _u32([7]), _t(sc([8])), _t(sc([9])), _t(gb), _z(864), _z(32), _z(32), _z(1)]
        zk.anonymous_fields_device(ctx, len(eks), ky.data_ptr(), 1, *(x.data_ptr() for x in bufs))
        with pytest.raises((zk.SynthesisError, _lib.ZkError)) as e:
            ctx.sync()
        assert e.value.code == code
        torch.cuda.synchronize()
        assert _device(ctx, eks, good, g) == _host(ctx, eks, good, g) == [ab.anonymous_fields(eks, *good[0], g)]
