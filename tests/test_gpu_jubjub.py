"""GPU tests of the Jubjub public-input path:
  zk_jubjub_into_xy                       vs the Python oracle on mixed encodings and on the reference's literals
  zk_groth16_verify_points_batch(_device) vs verify_proofs on the host-decoded inputs, on toy keys shaped like the confidential
                                          (11 points, 22 inputs) and anonymous (52 points, 104 inputs) circuits, with proofs from
                                          the GPU prover: valid, swapped point, every rejection class in several slots, bad proof
                                          encodings, MalformedVerifyingKey, and a batch longer than one verifier slice"""
import json
import os

import numpy as np
import pytest

from oracle import coracle as co
from tests.jubjub_oracle import pyref as jj
from zero_chain_b200 import groth16 as zk
from zero_chain_b200 import synthetic as sy

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
VERIFY_CHUNK = 1 << 18          # transactions per slice of the verifier (pairing.cu)


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


def _limbs_to_int(a):
    return sum(int(v) << (64 * k) for k, v in enumerate(a))


def _device_decoded(ctx, encs):
    xy, st = zk.jubjub_into_xy(ctx, b"".join(encs))
    return [(int(st[i]), _limbs_to_int(xy[i, 0]), _limbs_to_int(xy[i, 1])) for i in range(len(encs))]


def _points(rng, n):
    return [jj.prime_order_point(int.from_bytes(rng.bytes(32), "little")) for _ in range(n)]


def _off_curve():
    y = 2
    while jj.point_for_y(y) is not None:
        y += 1
    return y.to_bytes(32, "little")


def test_into_xy_matches_oracle(ctx):
    rng = np.random.default_rng(21)
    encs = [rng.bytes(32) for _ in range(2797)]
    encs += [jj.encode(p) for p in _points(rng, 1000)]
    encs += [(jj.R + int(rng.integers(0, 1 << 60))).to_bytes(32, "little") for _ in range(200)]
    base = _points(rng, 4)
    encs += [jj.encode(jj.add(base[i % 4], jj.torsion_point((2, 4, 8)[i % 3]))) for i in range(96)]
    encs += [bytes([1]) + bytes(31), bytes([1]) + bytes(30) + b"\x80", jj.encode((0, jj.R - 1))]
    rng.shuffle(encs)
    assert len(encs) >= 4096
    want = [jj.into_xy(e) for e in encs]
    assert set(w[0] for w in want) == {0, 1, 2, 3}
    assert _device_decoded(ctx, encs) == want
    # the reference's literals (tests/golden/jubjub_points.json)
    g = json.load(open(os.path.join(GOLD, "jubjub_points.json")))
    lits = [bytes.fromhex(e["hex"]) for e in g["transaction_points"] + g["read_vectors"]]
    got = _device_decoded(ctx, lits)
    assert got == [jj.into_xy(e) for e in lits]
    assert [s for s, _, _ in got] == [0] * 9 + [3, 3]
    assert zk.jubjub_into_xy(ctx, b"")[0].shape == (0, 2, 4)


class _Key:
    """A toy CRS whose public inputs are the coordinates of n_points Jubjub points, and proofs for chosen points."""

    def __init__(self, ctx, n_points, seed):
        self.n_points = n_points
        self.r1cs = sy.make_r1cs(60 + 2 * n_points, 2 * n_points + 1, 50, 40, 33, seed=seed)
        crs = sy.make_toy_crs(self.r1cs, co.g1_fixed_base, co.g2_fixed_base, seed=seed + 1)
        self.params = zk.Parameters.read(ctx, crs.params_bytes, checked=True)
        self.pvk = zk.PreparedVerifyingKey.prepare(ctx, crs.params_bytes)
        assert self.pvk.num_inputs == 2 * n_points

    def prove(self, pts, seed):
        inputs = [c for p in pts for c in p]
        z = sy.make_witness(self.r1cs, seed, inputs=inputs)
        a, b, c = sy.evaluate(self.r1cs, z)
        n_in = self.r1cs.n_inputs
        pa = zk.ProvingAssignment(co.ints_to_limbs(a, 4), co.ints_to_limbs(b, 4), co.ints_to_limbs(c, 4),
                                  co.ints_to_limbs(z[:n_in], 4), co.ints_to_limbs(z[n_in:], 4), *sy.densities(self.r1cs))
        return zk.create_proof(pa, self.params, 1000 + seed, 2000 + seed)

    def free(self):
        self.pvk.free(); self.params.free()


def _host_verdicts(key, proofs, encs_per_tx):
    """The reference's order: decode every point (a rejection ends the call), then Proof::read + verify_proof."""
    out = [None] * len(encs_per_tx)
    rows, idx = [], []
    for t, encs in enumerate(encs_per_tx):
        dec = [jj.into_xy(e) for e in encs]
        if any(s for s, _, _ in dec):
            out[t] = zk.VERDICT_INPUT_REJECTED
        else:
            rows.append([c for _, x, y in dec for c in (x, y)]); idx.append(t)
    if idx:
        got = zk.verify_proofs(key.pvk, b"".join(proofs[t] for t in idx), rows)
        for t, v in zip(idx, got):
            out[t] = v
    return out


def _device(ctx, key, proofs, points):
    import torch
    n = len(proofs) // 192
    dp = torch.from_numpy(np.frombuffer(proofs, np.uint8).copy()).cuda()
    dpt = torch.from_numpy(np.frombuffer(points, np.uint8).copy()).cuda()
    dv = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    zk.verify_proofs_with_points_device(key.pvk, n, dp.data_ptr(), dpt.data_ptr(), key.n_points, dv.data_ptr())
    ctx.sync()
    return [int(v) for v in dv.cpu().numpy()]


def test_confidential_shape_verdicts(ctx):
    key = _Key(ctx, zk.CONFIDENTIAL_POINTS, seed=41)
    rng = np.random.default_rng(5)
    txs = [_points(rng, 11) for _ in range(4)]
    proofs = [key.prove(p, s + 1) for s, p in enumerate(txs)]
    encs = [[jj.encode(p) for p in pts] for pts in txs]
    bad_field = (jj.R + 3).to_bytes(32, "little")
    bad_curve = _off_curve()
    bad_order = jj.encode(jj.add(txs[0][0], jj.torsion_point(8)))
    good = proofs[0]
    flag_cleared = bytes([good[0] & 0x7F]) + good[1:]                      # Proof::read -> InvalidData
    a_infinity = bytes([0xC0]) + bytes(47) + good[48:]                     # Proof::read -> PointInfinity
    cases = [(proofs[t], encs[t], 1) for t in range(4)]
    swapped = list(encs[1]); swapped[4] = encs[2][7]
    cases.append((proofs[1], swapped, 0))                                 # another valid point in one slot
    cases.append((proofs[2], encs[3], 0))                                 # another transaction's points
    for bad in (bad_field, bad_curve, bad_order):
        for slot in (0, 5, 6, 7, 10):                                     # 6 / 7: the two halves of balance_sender
            e = list(encs[0]); e[slot] = bad
            cases.append((proofs[0], e, zk.VERDICT_INPUT_REJECTED))
    for bad in (bad_field, bad_order):
        e = list(encs[0]); e[3] = bad
        cases.append((flag_cleared, e, zk.VERDICT_INPUT_REJECTED))         # the inputs are built before Proof::read
        cases.append((a_infinity, e, zk.VERDICT_INPUT_REJECTED))
    cases.append((flag_cleared, encs[0], zk.VERDICT_INVALID_DATA))
    cases.append((a_infinity, encs[0], zk.VERDICT_POINT_INFINITY))
    proofs_b = b"".join(c[0] for c in cases)
    points_b = b"".join(b"".join(c[1]) for c in cases)
    want = [c[2] for c in cases]
    assert _host_verdicts(key, [c[0] for c in cases], [c[1] for c in cases]) == want
    assert zk.verify_proofs_with_points(key.pvk, proofs_b, points_b, 11) == want
    assert _device(ctx, key, proofs_b, points_b) == want
    # the lane-parallel and the thread-per-proof pairing kernels see the same decoded inputs
    ctx.set_opt(zk.Context.OPT_VERIFY_LANES, 0)
    try:
        assert zk.verify_proofs_with_points(key.pvk, proofs_b, points_b, 11) == want
    finally:
        ctx.set_opt(zk.Context.OPT_VERIFY_LANES, 1)
    # the layout helper in the reference's push order gives back the points of a valid transaction
    p = encs[0]
    cp = zk.confidential_points(p[0], p[1], p[2], p[3], p[4], p[5], p[6] + p[7], p[8], p[9], p[10])
    assert cp == b"".join(p) and zk.verify_proofs_with_points(key.pvk, proofs[0], cp, 11) == [1]
    # MalformedVerifyingKey: 2 * n_points + 1 != ic.len()
    with pytest.raises(zk.SynthesisError) as e:
        zk.verify_proofs_with_points(key.pvk, proofs[0], b"".join(encs[0][:10]), 10)
    assert e.value.code == -9
    assert zk.verify_proofs_with_points(key.pvk, b"", b"", 11) == []
    key.free()


def test_anonymous_shape(ctx):
    key = _Key(ctx, zk.ANONYMOUS_POINTS, seed=53)
    rng = np.random.default_rng(8)
    pts = _points(rng, 52)
    e = [jj.encode(p) for p in pts]
    layout = zk.anonymous_points(e[0:12], e[12:24], [e[24 + i] + e[36 + i] for i in range(12)], e[48], e[49], e[50], e[51])
    assert layout == b"".join(e)
    proof = key.prove(pts, 3)
    other = key.prove(_points(rng, 52), 4)
    rejected = list(e); rejected[40] = jj.encode(jj.add(pts[40], jj.torsion_point(4)))
    swapped = list(e); swapped[51] = e[50]
    proofs = [proof, other, proof, proof]
    points = [e, e, rejected, swapped]
    want = [1, 0, zk.VERDICT_INPUT_REJECTED, 0]
    assert _host_verdicts(key, proofs, points) == want
    pb, ptb = b"".join(proofs), b"".join(b"".join(p) for p in points)
    assert zk.verify_proofs_with_points(key.pvk, pb, ptb, 52) == want
    assert _device(ctx, key, pb, ptb) == want
    key.free()


def test_batch_longer_than_one_slice(ctx):
    """VERIFY_CHUNK + 3 transactions: the second slice must read its points at offset VERIFY_CHUNK * n_points."""
    key = _Key(ctx, zk.CONFIDENTIAL_POINTS, seed=61)
    rng = np.random.default_rng(13)
    txs = [_points(rng, 11) for _ in range(3)]
    proofs = [key.prove(p, s + 1) for s, p in enumerate(txs)]
    encs = [b"".join(jj.encode(p) for p in pts) for pts in txs]
    bad = list(jj.encode(p) for p in txs[1]); bad[9] = _off_curve()
    pattern = [(proofs[0], encs[0], 1), (proofs[1], encs[1], 1), (proofs[2], encs[2], 1), (proofs[1], encs[2], 0),
               (proofs[1], b"".join(bad), zk.VERDICT_INPUT_REJECTED), (proofs[2], encs[2], 1), (proofs[0], encs[1], 0)]
    n = VERIFY_CHUNK + 3
    reps = (n + len(pattern) - 1) // len(pattern)
    seq = (pattern * reps)[:n]
    pb = b"".join(c[0] for c in seq)
    ptb = b"".join(c[1] for c in seq)
    want = [c[2] for c in seq]
    assert zk.verify_proofs_with_points(key.pvk, pb, ptb, 11) == want
    assert _device(ctx, key, pb, ptb) == want
    key.free()
