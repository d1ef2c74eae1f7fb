"""GPU tests of zk_elgamal_decrypt_batch(_device):
  every table entry (i P_G decrypts to i for all i < 10^6, -i P_G and 10^6 P_G do not), with the encodings from the C
  oracle's successive additions; a mixed corpus of > 4096 ciphertexts with every status, pending given as NULL, as
  Ciphertext::zero() and as a real ciphertext, a sample confirmed by the C oracle's walk; the reference's transaction
  literals and genesis balances; the device entry point on torch buffers; argument errors; a batch longer than one grid;
  and contexts shared with the signature and proof verifiers, and two contexts with a table each."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from oracle import coracle as co
from tests.jubjub_oracle import eg_coracle as ec
from tests.jubjub_oracle import eg_corpus
from tests.jubjub_oracle import elgamal as eg
from tests.jubjub_oracle import pyref as jj
from tests.jubjub_oracle import redjubjub as rj
from tests.jubjub_oracle import rj_corpus
from zero_chain_b200 import _lib
from zero_chain_b200 import groth16 as zk
from zero_chain_b200 import synthetic as sy

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "elgamal.json")))
POINTS = {e["name"]: bytes.fromhex(e["hex"]) for e in json.load(open(os.path.join(HERE, "golden", "jubjub_points.json")))["transaction_points"]}
BLOCKS_PER_SM, THREADS = 8, 128            # the decryption kernel's grid cap (elgamal.cu)
IDENTITY = jj.encode(jj.IDENTITY)


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def corpus():
    entries = eg_corpus.random_entries(4096, seed=41) + eg_corpus.special_entries(42)
    return entries, eg_corpus.columns(entries)


def test_constants():
    assert zk.ELGAMAL_BOUND == GOLD["bound"]["value"] == eg.BOUND
    assert zk.ELGAMAL_ZERO == eg.write(eg.ZERO) == IDENTITY * 2
    assert (zk.ELGAMAL_OK, zk.ELGAMAL_NOT_FOUND, zk.ELGAMAL_BAD_KEY, zk.ELGAMAL_BAD_BALANCE, zk.ELGAMAL_BAD_PENDING) == \
        (eg.OK, eg.NOT_FOUND, eg.BAD_KEY, eg.BAD_BALANCE, eg.BAD_PENDING)


def test_every_table_entry(ctx):
    n = zk.ELGAMAL_BOUND
    table = ec.multiples(n + 1)
    assert bytes(table[0]) == IDENTITY and bytes(table[1]) == jj.encode(rj.P_G)
    rng = np.random.default_rng(11)
    dk = (int.from_bytes(rng.bytes(32), "little") % jj.R_J).to_bytes(32, "little")
    right = np.frombuffer(IDENTITY, np.uint8)
    cts = np.concatenate([table, np.broadcast_to(right, table.shape)], axis=1)        # (i P_G, O)
    st, val = zk.elgamal_decrypt(ctx, dk * (n + 1), cts.tobytes())
    assert st[:n] == [zk.ELGAMAL_OK] * n and val[:n] == list(range(n))
    assert (st[n], val[n]) == (zk.ELGAMAL_NOT_FOUND, 0)
    neg = cts[1:n].copy()
    neg[:, 31] ^= 0x80                                                                 # (-i P_G, O)
    st, val = zk.elgamal_decrypt(ctx, dk * (n - 1), neg.tobytes())
    assert st == [zk.ELGAMAL_NOT_FOUND] * (n - 1) and not any(val)


def test_mixed_corpus(ctx, corpus):
    entries, (dks, cts, pds, want_null, want_pend) = corpus
    assert len(entries) > 4096 and set(want_pend[0]) == {0, 1, 2, 3, 4} and set(want_null[0]) == {0, 1, 2, 3}
    assert zk.elgamal_decrypt(ctx, dks, cts) == want_null
    assert zk.elgamal_decrypt(ctx, dks, cts, [zk.ELGAMAL_ZERO] * len(entries)) == want_null
    assert zk.elgamal_decrypt(ctx, dks, cts, pds) == want_pend
    # the C oracle's walk on a sample, with and without the pending transfers
    rng = np.random.default_rng(5)
    sample = sorted(set(rng.choice(len(entries) - 40, 40, replace=False).tolist()) | set(range(len(entries) - 40, len(entries))))
    sub = [entries[i] for i in sample]
    s_dks, s_cts, s_pds, s_null, s_pend = eg_corpus.columns(sub)
    for pend, want in ((None, s_null), (s_pds, s_pend)):
        st, val = ec.decrypt(s_dks, s_cts, pend)
        assert ([int(x) for x in st], [int(x) for x in val]) == want
    # every status: the Python oracle's stage agrees on the special cases
    for e in entries[-40:]:
        st, _ = eg.stage(e[0], e[1], e[2])
        assert st == (e[4][0] if e[4][0] >= 2 else eg.OK)


def _alice_bob():
    alice = eg.account_keys(json.load(open(os.path.join(HERE, "golden", "redjubjub.json")))["alice_seed"]["text"].encode())
    bob = eg.account_keys(GOLD["bob_seed"]["text"].encode())
    return {"alice": alice, "bob": bob}


def test_reference_literals_and_genesis(ctx):
    keys = _alice_bob()
    assert jj.encode(keys["alice"][1]) == POINTS["pkd_addr_alice"] and jj.encode(keys["bob"][1]) == POINTS["pkd_addr_bob"]
    lit = GOLD["literal_decryptions"]
    dks = [eg.key_bytes(keys[d["key"]][0]) for d in lit]
    cts = [POINTS[d["left"]] + POINTS[d["right"]] for d in lit]
    want = ([zk.ELGAMAL_OK if d["value"] is not None else zk.ELGAMAL_NOT_FOUND for d in lit], [d["value"] or 0 for d in lit])
    assert want == ([0, 0, 0, 1], [10, 1, 10, 0])
    assert zk.elgamal_decrypt(ctx, dks, cts) == want
    st, val = ec.decrypt(b"".join(dks), b"".join(cts))
    assert ([int(x) for x in st], [int(x) for x in val]) == want
    # the genesis balances: randomness Fs::one(), so (amount P_G + ek, P_G); one with the module test's balance pending
    dk, ek = keys["alice"]
    gen = [eg.write(eg.encrypt(g["value"], 1, ek)) for g in GOLD["genesis"]]
    assert zk.elgamal_decrypt(ctx, [eg.key_bytes(dk)] * 2, gen) == ([0, 0], [10_000, 100])
    assert zk.elgamal_decrypt(ctx, [eg.key_bytes(dk)], gen[:1], gen[1:]) == ([0], [10_100])
    assert zk.elgamal_decrypt(ctx, [eg.key_bytes(keys["bob"][0])], gen[:1]) == ([1], [0])


def _device(ctx, dks, cts, pds):
    import torch
    n = len(dks) // 32
    t = lambda b: torch.from_numpy(np.frombuffer(b, np.uint8).copy()).cuda()
    d_dk, d_ct = t(dks), t(cts)
    d_pd = t(pds) if pds is not None else None
    d_val = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    d_st = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    zk.elgamal_decrypt_device(ctx, n, d_dk.data_ptr(), d_ct.data_ptr(), d_pd.data_ptr() if d_pd is not None else 0, d_val.data_ptr(),
                              d_st.data_ptr())
    ctx.sync()
    return [int(s) for s in d_st.cpu().numpy()], [int(v) for v in d_val.cpu().numpy().view(np.uint32)]


def test_device_entry_point(ctx, corpus):
    _, (dks, cts, pds, want_null, want_pend) = corpus
    assert _device(ctx, dks, cts, None) == want_null
    assert _device(ctx, dks, cts, pds) == want_pend


def test_argument_errors(ctx, corpus):
    _, (dks, cts, pds, want_null, want_pend) = corpus
    L = _lib.lib()
    assert zk.elgamal_decrypt(ctx, [], []) == ([], [])
    assert L.zk_elgamal_decrypt_batch(ctx._h, 0, None, None, None, None, None) == 0
    assert L.zk_elgamal_decrypt_batch_device(ctx._h, 0, None, None, None, None, None) == 0
    buf = np.frombuffer(dks[:64] + cts[:128] + pds[:128], np.uint8)
    p = buf.ctypes.data
    val, st = np.zeros(2, np.uint32), np.zeros(2, np.uint8)
    args = [p, p + 64, p + 192, val.ctypes.data, st.ctypes.data]
    assert L.zk_elgamal_decrypt_batch(None, 2, *args) == -2
    assert L.zk_elgamal_decrypt_batch_device(None, 2, *args) == -2
    for k in (0, 1, 3, 4):
        a = [C.c_void_p(x) for x in args]
        a[k] = None
        assert L.zk_elgamal_decrypt_batch(ctx._h, 2, *a) == -2
        assert L.zk_elgamal_decrypt_batch_device(ctx._h, 2, *a) == -2
        assert "NULL" in L.zk_last_error().decode()
    # pending NULL is accepted, and the context is still usable
    assert L.zk_elgamal_decrypt_batch(ctx._h, 2, p, p + 64, None, val.ctypes.data, st.ctypes.data) == 0
    assert ([int(x) for x in st], [int(x) for x in val]) == (want_null[0][:2], want_null[1][:2])
    assert L.zk_elgamal_decrypt_batch(ctx._h, 2, *args) == 0
    assert ([int(x) for x in st], [int(x) for x in val]) == (want_pend[0][:2], want_pend[1][:2])


def test_batch_longer_than_one_grid(ctx, corpus):
    import torch
    entries, (dks, cts, pds, _, want_pend) = corpus
    grid = torch.cuda.get_device_properties(0).multi_processor_count * BLOCKS_PER_SM * THREADS
    reps = grid // len(entries) + 2
    assert len(entries) * reps > grid
    st, val = zk.elgamal_decrypt(ctx, dks * reps, cts * reps, pds * reps)
    assert (st, val) == (want_pend[0] * reps, want_pend[1] * reps)


def test_shared_contexts(ctx, corpus):
    """One context interleaves decryption with zk_redjubjub_verify_batch and zk_groth16_verify_points_batch, and every verdict
    is unchanged; two more contexts each build and use their own table."""
    _, (dks, cts, pds, want_null, want_pend) = corpus
    rj_entries, _ = rj_corpus.mixed(64, seed=12)
    vks, sigs, msgs = rj_corpus.columns(rj_entries)
    rj_want = [rj_corpus.python_verdict(e) for e in rj_entries[:16]]
    n_pts = zk.CONFIDENTIAL_POINTS
    r1cs = sy.make_r1cs(60 + 2 * n_pts, 2 * n_pts + 1, 50, 40, 33, seed=81)
    crs = sy.make_toy_crs(r1cs, co.g1_fixed_base, co.g2_fixed_base, seed=82)
    params = zk.Parameters.read(ctx, crs.params_bytes, checked=True)
    pvk = zk.PreparedVerifyingKey.prepare(ctx, crs.params_bytes)
    rng = np.random.default_rng(13)
    pts = [jj.prime_order_point(int.from_bytes(rng.bytes(32), "little")) for _ in range(n_pts)]
    z = sy.make_witness(r1cs, 1, inputs=[c for p in pts for c in p])
    a, b, c = sy.evaluate(r1cs, z)
    pa = zk.ProvingAssignment(co.ints_to_limbs(a, 4), co.ints_to_limbs(b, 4), co.ints_to_limbs(c, 4),
                              co.ints_to_limbs(z[:r1cs.n_inputs], 4), co.ints_to_limbs(z[r1cs.n_inputs:], 4), *sy.densities(r1cs))
    proof = zk.create_proof(pa, params, 5, 6)
    params.free()
    points = b"".join(jj.encode(p) for p in pts)
    tx_points = points + b"".join(jj.encode(p) for p in pts[::-1]) + points
    for _ in range(2):
        assert zk.verify_proofs_with_points(pvk, proof * 3, tx_points, n_pts) == [1, 0, 1]
        assert zk.elgamal_decrypt(ctx, dks, cts, pds) == want_pend
        assert zk.redjubjub_verify(ctx, vks, sigs, msgs)[:16] == rj_want
        assert zk.elgamal_decrypt(ctx, dks, cts) == want_null
    pvk.free()
    c1, c2 = zk.Context(0), zk.Context(0)
    assert zk.elgamal_decrypt(c1, dks, cts, pds) == want_pend
    assert zk.elgamal_decrypt(c2, dks, cts) == want_null
    c1.close()
    assert zk.elgamal_decrypt(c2, dks, cts, pds) == want_pend
    c2.close()
    assert zk.elgamal_decrypt(ctx, dks, cts) == want_null
