"""GPU tests of zk_redjubjub_batch_verify(_device) and redjubjub_verify_batched: the verdict and first_bad equal the C
oracle's batch_verify on valid-only batches from a 4096+ corpus and on batches with one defect of each class (the code
and index also equal the per-signature kernel's first rejection); the Alice keys with the reference's messages; messages at
unaligned offsets through torch buffers; n = 0, n = 1, a batch longer than one grid; z errors; and a context that still
gives unchanged results from zk_redjubjub_verify_batch and zk_groth16_verify_points_batch."""
import json
import os

import numpy as np
import pytest

from oracle import coracle as co
from tests.jubjub_oracle import pyref as jj
from tests.jubjub_oracle import redjubjub as rj
from tests.jubjub_oracle import rjb_coracle as cjb
from tests.jubjub_oracle import rj_coracle as cj
from tests.jubjub_oracle import rj_corpus
from zero_chain_b200 import _lib
from zero_chain_b200 import groth16 as zk
from zero_chain_b200 import synthetic as sy

pytestmark = pytest.mark.gpu
GOLD = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "redjubjub.json")))
BLOCKS_PER_SM, THREADS = 8, 128            # the per-entry kernel's grid cap (jubjub_msm.cu)


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def corpus():
    lengths = rj_corpus.EDGE_LENGTHS + [301, 400, 513, 1000]
    entries, _ = rj_corpus.mixed(4096, seed=31, lengths=lengths)
    vks, sigs, msgs = rj_corpus.columns(entries)
    want = [int(v) for v in cj.redjubjub_verify(vks, sigs, msgs)]
    return entries, want


def _zs(n, seed):
    rng = np.random.default_rng(seed)
    return b"".join((int.from_bytes(rng.bytes(64), "little") % rj.R_J).to_bytes(32, "little") for _ in range(n))


def _check(ctx, entries, seed):
    """device verdict == C oracle verdict; returns it"""
    vks, sigs, msgs = rj_corpus.columns(entries)
    zs = _zs(len(entries), seed)
    want = cjb.redjubjub_batch_verify(vks, sigs, msgs, zs)
    assert zk.redjubjub_batch_verify(ctx, vks, sigs, msgs, zs) == want
    return want


def _device(ctx, vks, sigs, msgs, zs, pad=3):
    import torch
    n = len(msgs)
    mb = b"\x5a" * pad + b"".join(msgs)
    off = zk.message_offsets(msgs) + np.uint64(pad)
    t = lambda b: torch.from_numpy(np.frombuffer(b if b else b"\0", np.uint8).copy()).cuda()
    dvk, dsg, dmsg, dz = t(vks), t(sigs), t(mb), t(zs)
    doff = torch.from_numpy(off.view(np.int64).copy()).cuda()
    dv = torch.full((1,), 0xEE, dtype=torch.uint8, device="cuda")
    dfb = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    zk.redjubjub_batch_verify_device(ctx, n, dvk.data_ptr(), dsg.data_ptr(), dmsg.data_ptr(), doff.data_ptr(), dz.data_ptr(),
                                     dv.data_ptr(), dfb.data_ptr())
    ctx.sync()
    return int(dv.cpu()[0]), int(dfb.cpu()[0])


def test_valid_batches(ctx, corpus):
    entries, want = corpus
    valid = [e for e, w in zip(entries, want) if w == rj.OK]
    assert len(valid) >= 4096
    assert _check(ctx, valid, 1) == (rj.OK, None)
    for k in range(0, len(valid), 1000):
        assert _check(ctx, valid[k:k + 1000], 2 + k) == (rj.OK, None)


def test_one_defect_of_each_class(ctx, corpus):
    entries, want = corpus
    valid = [e for e, w in zip(entries, want) if w == rj.OK]
    seen = set()
    for j, (e, w) in enumerate(zip(entries, want)):
        if w == rj.OK or (w in seen and j % 7):
            continue
        seen.add(w)
        pos = j % 300
        batch = valid[:pos] + [e] + valid[pos:300]
        got = _check(ctx, batch, 100 + j)
        if w in (rj.BAD_VK, rj.BAD_R, rj.BAD_S):
            assert got == (w, pos)
            per = zk.redjubjub_verify(ctx, *rj_corpus.columns(batch))
            assert next(v for v in per if v != rj.OK) == w
        else:
            assert got == (rj.BAD_EQUATION, None)
    assert seen == {0, 2, 3, 4}
    # two rejected entries: the lower index decides, whatever the codes
    bad_s = next(e for e, w in zip(entries, want) if w == rj.BAD_S)
    bad_vk = next(e for e, w in zip(entries, want) if w == rj.BAD_VK)
    assert _check(ctx, valid[:10] + [bad_s] + valid[10:20] + [bad_vk], 7) == (rj.BAD_S, 10)


def test_reference_messages_with_alice_keys(ctx):
    seed = GOLD["alice_seed"]["text"].encode()
    m1, m2 = [m["text"].encode() for m in GOLD["messages"]]
    sk = rj.spending_key(seed)
    vk = rj.public_key(sk)
    rng = np.random.default_rng(3)
    s1, s2 = rj.sign(sk, m1, rng.bytes(80)), rj.sign(sk, m2, rng.bytes(80))
    _, a = jj.read(vk)
    torsion_vk = jj.encode(jj.add(a, jj.torsion_point(8)))
    good = ([vk, vk, torsion_vk], [s1, s2, s1], [m1, m2, m1])
    zs = _zs(3, 4)
    assert zk.redjubjub_batch_verify(ctx, *good, zs) == (1, None) == cjb.redjubjub_batch_verify(*map(b"".join, good[:2]), good[2], zs)
    swapped = ([vk, vk], [s2, s2], [m1, m2])
    assert zk.redjubjub_batch_verify(ctx, *swapped, zs[:64]) == (0, None)
    assert _device(ctx, b"".join(good[0]), b"".join(good[1]), good[2], zs, pad=1) == (1, 3)
    assert _device(ctx, b"".join(swapped[0]), b"".join(swapped[1]), swapped[2], zs[:64], pad=5) == (0, 2)


def test_device_form_and_edges(ctx, corpus):
    entries, want = corpus
    valid = [e for e, w in zip(entries, want) if w == rj.OK][:500]
    bad_r = next(e for e, w in zip(entries, want) if w == rj.BAD_R)
    batch = valid[:123] + [bad_r] + valid[123:]
    vks, sigs, msgs = rj_corpus.columns(batch)
    zs = _zs(len(batch), 9)
    assert _device(ctx, vks, sigs, msgs, zs) == (rj.BAD_R, 123)
    vks, sigs, msgs = rj_corpus.columns(valid)
    assert _device(ctx, vks, sigs, msgs, _zs(500, 10)) == (1, 500)
    # z_i >= r_J: the host form refuses the call, the device form rejects the entry with code 5
    zbad = _zs(500, 11)
    zbad = zbad[:32 * 77] + rj.R_J.to_bytes(32, "little") + zbad[32 * 78:]
    with pytest.raises(zk.SynthesisError) as e:
        zk.redjubjub_batch_verify(ctx, vks, sigs, msgs, zbad)
    assert e.value.code == -8
    assert _device(ctx, vks, sigs, msgs, zbad) == (zk.REDJUBJUB_BAD_Z, 77)
    # n = 1, n = 0
    one = valid[:1]
    assert _check(ctx, one, 12) == (1, None)
    assert _check(ctx, [(one[0][0], one[0][1], one[0][2] + b"!", 0)], 13) == (0, None)
    assert zk.redjubjub_batch_verify(ctx, [], [], [], b"") == (1, None)
    assert _device(ctx, b"", b"", [], b"", pad=0) == (1, 0)
    L = _lib.lib()
    assert L.zk_redjubjub_batch_verify(ctx._h, 0, None, None, None, None, None, None, None) == -2     # no verdict pointer
    v = np.zeros(1, np.uint8)
    assert L.zk_redjubjub_batch_verify(ctx._h, 0, None, None, None, None, None, v.ctypes.data, None) == 0 and v[0] == 1
    buf = np.frombuffer(vks[:64] + sigs[:128] + zs[:64] + b"Foo barSpam eggs", np.uint8)
    p = buf.ctypes.data
    off = np.array([0, 7, 16], np.uint64)
    for k in range(5):
        args = [p, p + 64, p + 256, off.ctypes.data, p + 192]
        args[k] = None
        assert L.zk_redjubjub_batch_verify(ctx._h, 2, *args, v.ctypes.data, None) == -2
        assert L.zk_redjubjub_batch_verify_device(ctx._h, 2, *args, v.ctypes.data, None) == -2
    bad = np.array([0, 9, 7], np.uint64)
    assert L.zk_redjubjub_batch_verify(ctx._h, 2, p, p + 64, p + 256, bad.ctypes.data, p + 192, v.ctypes.data, None) == -2
    assert "msg_off" in L.zk_last_error().decode()


def test_batch_longer_than_one_grid(ctx, corpus):
    import torch
    entries, want = corpus
    valid = [e for e, w in zip(entries, want) if w == rj.OK]
    grid = torch.cuda.get_device_properties(0).multi_processor_count * BLOCKS_PER_SM * THREADS
    reps = grid // len(valid) + 2
    batch = valid * reps
    assert len(batch) > grid
    assert _check(ctx, batch, 14) == (1, None)
    bad_s = next(e for e, w in zip(entries, want) if w == rj.BAD_S)
    batch[grid + 5] = bad_s                                         # an entry the grid-stride loop reaches on its second pass
    assert _check(ctx, batch, 15) == (rj.BAD_S, grid + 5)
    batch[grid + 5] = (valid[0][0], valid[1][1], valid[0][2], 0)
    assert _check(ctx, batch, 16) == (rj.BAD_EQUATION, None)


def test_zero_randomizer_lets_a_forgery_pass(ctx, corpus):
    """The equation is exactly the reference's: with z_i = 0 entry i drops out, so a bad signature there passes."""
    entries, want = corpus
    valid = [e for e, w in zip(entries, want) if w == rj.OK][:50]
    batch = valid[:20] + [(valid[0][0], valid[1][1], valid[0][2], 0)] + valid[20:]
    vks, sigs, msgs = rj_corpus.columns(batch)
    zs = _zs(len(batch), 17)
    assert zk.redjubjub_batch_verify(ctx, vks, sigs, msgs, zs)[0] == 0
    z0 = zs[:32 * 20] + bytes(32) + zs[32 * 21:]
    assert zk.redjubjub_batch_verify(ctx, vks, sigs, msgs, z0) == (1, None) == cjb.redjubjub_batch_verify(vks, sigs, msgs, z0)


def test_verify_batched_matches_per_signature(ctx, corpus):
    entries, want = corpus
    valid = [e for e, w in zip(entries, want) if w == rj.OK]
    for batch in (entries, valid, valid[:1], entries[:700]):
        vks, sigs, msgs = rj_corpus.columns(batch)
        per = zk.redjubjub_verify(ctx, vks, sigs, msgs)
        assert zk.redjubjub_verify_batched(ctx, vks, sigs, msgs, _zs(len(batch), 18)) == per
        assert zk.redjubjub_verify_batched(ctx, vks, sigs, msgs) == per


def test_shared_context_with_proof_verifier(ctx, corpus):
    entries, want = corpus
    vks, sigs, msgs = rj_corpus.columns(entries)
    n_pts = zk.CONFIDENTIAL_POINTS
    r1cs = sy.make_r1cs(60 + 2 * n_pts, 2 * n_pts + 1, 50, 40, 33, seed=71)
    crs = sy.make_toy_crs(r1cs, co.g1_fixed_base, co.g2_fixed_base, seed=72)
    params = zk.Parameters.read(ctx, crs.params_bytes, checked=True)
    pvk = zk.PreparedVerifyingKey.prepare(ctx, crs.params_bytes)
    rng = np.random.default_rng(9)
    pts = [jj.prime_order_point(int.from_bytes(rng.bytes(32), "little")) for _ in range(n_pts)]
    z = sy.make_witness(r1cs, 1, inputs=[c for p in pts for c in p])
    a, b, c = sy.evaluate(r1cs, z)
    pa = zk.ProvingAssignment(co.ints_to_limbs(a, 4), co.ints_to_limbs(b, 4), co.ints_to_limbs(c, 4),
                              co.ints_to_limbs(z[:r1cs.n_inputs], 4), co.ints_to_limbs(z[r1cs.n_inputs:], 4), *sy.densities(r1cs))
    proof = zk.create_proof(pa, params, 5, 6)
    params.free()
    points = b"".join(jj.encode(p) for p in pts)
    other = b"".join(jj.encode(p) for p in pts[::-1])
    proofs, tx_points = proof * 3, points + other + points
    assert zk.verify_proofs_with_points(pvk, proofs, tx_points, n_pts) == [1, 0, 1]
    assert zk.redjubjub_verify(ctx, vks, sigs, msgs) == want
    assert _check(ctx, entries, 19)[0] in (rj.BAD_VK, rj.BAD_R, rj.BAD_S)
    assert zk.jubjub_msm(ctx, [jj.encode(rj.P_G)], [5]) == rj.public_key(5)
    assert zk.verify_proofs_with_points(pvk, proofs, tx_points, n_pts) == [1, 0, 1]
    assert zk.redjubjub_verify(ctx, vks, sigs, msgs) == want
    pvk.free()
