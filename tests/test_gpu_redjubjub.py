"""GPU tests of zk_redjubjub_verify_batch(_device):
  verdicts equal the C oracle's on >= 4096 signatures mixing every class (a subset against the Python oracle too), messages
  of 0..300+ bytes at unaligned offsets; signatures over the reference's messages from keys derived from the Alice seed; the
  device entry point on torch buffers; the empty batch, NULL and inconsistent arguments; a batch longer than one grid; and a
  context shared with zk_groth16_verify_points_batch."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from oracle import coracle as co
from tests.jubjub_oracle import rj_coracle as cj
from tests.jubjub_oracle import pyref as jj
from tests.jubjub_oracle import redjubjub as rj
from tests.jubjub_oracle import rj_corpus
from zero_chain_b200 import _lib
from zero_chain_b200 import groth16 as zk
from zero_chain_b200 import synthetic as sy

pytestmark = pytest.mark.gpu
GOLD = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "redjubjub.json")))
BLOCKS_PER_SM, THREADS = 8, 128            # the verifier's grid cap (redjubjub.cu)


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def corpus():
    lengths = rj_corpus.EDGE_LENGTHS + [301, 400, 513, 1000]
    entries, n_special = rj_corpus.mixed(4096, seed=29, lengths=lengths)
    vks, sigs, msgs = rj_corpus.columns(entries)
    want = [int(v) for v in cj.redjubjub_verify(vks, sigs, msgs)]
    return entries, vks, sigs, msgs, want


def _device(ctx, vks, sigs, msgs, pad=3):
    """Device buffers from torch; every message starts `pad` bytes further into the buffer, so offsets are unaligned."""
    import torch
    n = len(msgs)
    mb = b"\xa5" * pad + b"".join(msgs)
    off = zk.message_offsets(msgs) + np.uint64(pad)
    t = lambda b: torch.from_numpy(np.frombuffer(b, np.uint8).copy()).cuda()
    dvk, dsg, dmsg = t(vks), t(sigs), t(mb)
    doff = torch.from_numpy(off.view(np.int64).copy()).cuda()
    dv = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    zk.redjubjub_verify_device(ctx, n, dvk.data_ptr(), dsg.data_ptr(), dmsg.data_ptr(), doff.data_ptr(), dv.data_ptr())
    ctx.sync()
    return [int(v) for v in dv.cpu().numpy()]


def test_verdicts_match_oracles(ctx, corpus):
    entries, vks, sigs, msgs, want = corpus
    assert len(entries) >= 4096 and set(want) == {0, 1, 2, 3, 4}
    assert all(w == e[3] for w, e in zip(want, entries) if e[3] is not None)
    assert max(len(m) for m in msgs) > 256
    special = [i for i, e in enumerate(entries) if e[3] != rj.OK][:40] + list(range(24))
    assert [rj_corpus.python_verdict(entries[i]) for i in special] == [want[i] for i in special]
    assert zk.redjubjub_verify(ctx, vks, sigs, msgs) == want
    # one message buffer with the messages at odd offsets, through the host form's base offset
    assert _device(ctx, vks, sigs, msgs) == want


def test_reference_messages_with_alice_keys(ctx):
    seed = GOLD["alice_seed"]["text"].encode()
    m1, m2 = [m["text"].encode() for m in GOLD["messages"]]
    sk = rj.spending_key(seed)
    vk = rj.public_key(sk)
    rng = np.random.default_rng(3)
    alpha = int.from_bytes(rng.bytes(32), "little") % rj.R_J
    rsk, rvk = (sk + alpha) % rj.R_J, rj.randomize_public_key(vk, alpha)
    s1, s2 = rj.sign(sk, m1, rng.bytes(80)), rj.sign(sk, m2, rng.bytes(80))
    r1 = rj.sign(rsk, m1, rng.bytes(80))
    _, a = jj.read(vk)
    torsion_vk = jj.encode(jj.add(a, jj.torsion_point(8)))
    vks = [vk, vk, vk, vk, rvk, rvk, torsion_vk, torsion_vk]
    sigs = [s1, s2, s2, s1, r1, s1, s1, s2]
    msgs = [m1, m2, m1, m2, m1, m1, m1, m1]
    want = [1, 1, 0, 0, 1, 0, 1, 0]
    assert [rj.verify(k, m, s) for k, s, m in zip(vks, sigs, msgs)] == want
    assert zk.redjubjub_verify(ctx, vks, sigs, msgs) == want
    assert _device(ctx, b"".join(vks), b"".join(sigs), msgs, pad=1) == want


def test_edge_cases(ctx, corpus):
    _, vks, sigs, msgs, want = corpus
    assert zk.redjubjub_verify(ctx, [], [], []) == []
    L = _lib.lib()
    v = np.zeros(2, np.uint8)
    off = np.array([0, 7, 16], np.uint64)
    buf = np.frombuffer(vks[:64] + sigs[:128] + b"Foo barSpam eggs", np.uint8)
    p = buf.ctypes.data
    assert L.zk_redjubjub_verify_batch(ctx._h, 0, None, None, None, None, None) == 0
    assert L.zk_redjubjub_verify_batch_device(ctx._h, 0, None, None, None, None, None) == 0
    assert L.zk_redjubjub_verify_batch(None, 2, p, p + 64, p + 192, off.ctypes.data, v.ctypes.data) == -2
    for k in range(5):
        args = [C.c_void_p(p), C.c_void_p(p + 64), C.c_void_p(p + 192), C.c_void_p(off.ctypes.data), C.c_void_p(v.ctypes.data)]
        args[k] = None
        assert L.zk_redjubjub_verify_batch(ctx._h, 2, *args) == -2
        assert L.zk_redjubjub_verify_batch_device(ctx._h, 2, *args) == -2
    bad = np.array([0, 9, 7], np.uint64)                        # decreasing: the second message would end before it starts
    assert L.zk_redjubjub_verify_batch(ctx._h, 2, p, p + 64, p + 192, bad.ctypes.data, v.ctypes.data) == -2
    assert "msg_off" in L.zk_last_error().decode()
    # the context is still usable, and messages that start past zero in the host buffer are read from their offset
    shifted = np.array([3, 10, 19], np.uint64)
    buf2 = np.frombuffer(b"xyz" + b"Foo barSpam eggs", np.uint8)
    L.zk_redjubjub_verify_batch(ctx._h, 2, p, p + 64, buf2.ctypes.data, shifted.ctypes.data, v.ctypes.data)
    assert list(v) == zk.redjubjub_verify(ctx, vks[:64], sigs[:128], [b"Foo bar", b"Spam eggs"])


def test_batch_longer_than_one_grid(ctx, corpus):
    import torch
    _, vks, sigs, msgs, want = corpus
    grid = torch.cuda.get_device_properties(0).multi_processor_count * BLOCKS_PER_SM * THREADS
    n0 = len(msgs)
    reps = grid // n0 + 2
    n = n0 * reps
    assert n > grid
    got = zk.redjubjub_verify(ctx, vks * reps, sigs * reps, msgs * reps)
    assert got == want * reps


def test_shared_context_with_proof_verifier(ctx, corpus):
    """zk_groth16_verify_points_batch right before and after on the same context: both keep their verdicts; the transaction's
    signer is its rvk point."""
    _, vks, sigs, msgs, want = corpus
    n_pts = zk.CONFIDENTIAL_POINTS
    r1cs = sy.make_r1cs(60 + 2 * n_pts, 2 * n_pts + 1, 50, 40, 33, seed=71)
    crs = sy.make_toy_crs(r1cs, co.g1_fixed_base, co.g2_fixed_base, seed=72)
    params = zk.Parameters.read(ctx, crs.params_bytes, checked=True)
    pvk = zk.PreparedVerifyingKey.prepare(ctx, crs.params_bytes)
    rng = np.random.default_rng(9)
    sk = int.from_bytes(rng.bytes(32), "little") % rj.R_J
    rvk = rj.public_key(sk)
    _, rvk_pt = jj.read(rvk)
    pts = [jj.prime_order_point(int.from_bytes(rng.bytes(32), "little")) for _ in range(n_pts)]
    pts[8] = rvk_pt                                               # rvk's slot in verify_confidential_proof's push order
    z = sy.make_witness(r1cs, 1, inputs=[c for p in pts for c in p])
    a, b, c = sy.evaluate(r1cs, z)
    pa = zk.ProvingAssignment(co.ints_to_limbs(a, 4), co.ints_to_limbs(b, 4), co.ints_to_limbs(c, 4),
                              co.ints_to_limbs(z[:r1cs.n_inputs], 4), co.ints_to_limbs(z[r1cs.n_inputs:], 4), *sy.densities(r1cs))
    proof = zk.create_proof(pa, params, 5, 6)
    params.free()
    points = b"".join(jj.encode(p) for p in pts)
    other = b"".join(jj.encode(p) for p in pts[::-1])
    proofs, tx_points = proof * 3, points + other + points
    tx_sig = rj.sign(sk, b"transfer payload digest.........", rng.bytes(80))
    assert zk.verify_proofs_with_points(pvk, proofs, tx_points, n_pts) == [1, 0, 1]
    assert zk.redjubjub_verify(ctx, vks, sigs, msgs) == want
    assert zk.redjubjub_verify(ctx, [points[256:288]], [tx_sig], [b"transfer payload digest........."]) == [1]
    assert zk.verify_proofs_with_points(pvk, proofs, tx_points, n_pts) == [1, 0, 1]
    assert zk.redjubjub_verify(ctx, vks, sigs, msgs) == want
    pvk.free()
