"""The batched Groth16 verifier on its exceptional branches, with proofs forged from the toy key's trapdoor
(tests/verify_forge.py) so that every branch is met with an expected verdict of 1, not only of 0:
  k_ic_table / k_ic_partial   every reachable row d * 2^(8w) * ic_j of the window table, one forged proof per row
  k_ic_sum                    a term equal to the running sum, a term that cancels it, entry from the point at infinity,
                              skipped zero terms, a final sum equal to the point at infinity (the Miller kernels must then
                              drop the (acc, -gamma) pair), for keys of 3 and of 22 public inputs
  zk_pvk_load                 prepared keys whose -gamma / -delta carry the infinity flag, and the load rejections beside them
  k_miller_lanes / k_verify_final_lanes   batch sizes across the group, warp and block boundaries with every kind of proof
                              in the shadowed slot n - 1; nothing is written beyond verdicts[n - 1]
  zk_pairing_batch            the point at infinity on either side and on both
Every expected verdict comes from the trapdoor algebra or from the C oracle, never from the device."""
import numpy as np
import pytest

from oracle import coracle as co
from oracle import pyref as pr
from tests import verify_forge as vf
from zero_chain_b200 import groth16 as zk

pytestmark = pytest.mark.gpu
A_S, B_S = vf.A_S, vf.B_S
INF1 = bytes([0xC0]) + bytes(47)


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


class _Key(vf.ToyKey):
    """the toy key, also prepared on the device"""

    def __init__(self, ctx, n_inputs=4, seed=3):
        super().__init__(n_inputs, seed)
        self.pvk = zk.PreparedVerifyingKey.prepare(ctx, self.crs.params_bytes)
        assert self.pvk.num_inputs == self.n and self.pvk.write() == self.opvk.write()


@pytest.fixture(scope="module")
def key(ctx):
    k = _Key(ctx)
    yield k
    k.pvk.free()


def _verdicts(pvk, proofs, rows):
    return zk.verify_proofs(pvk, b"".join(proofs), [list(r) for r in rows])


def _on_both_paths(ctx, pvk, proofs, rows):
    """verdicts of the lane-parallel kernels and of the thread-per-proof kernels"""
    out = [_verdicts(pvk, proofs, rows)]
    ctx.set_opt(zk.Context.OPT_VERIFY_LANES, 0)
    try:
        out.append(_verdicts(pvk, proofs, rows))
    finally:
        ctx.set_opt(zk.Context.OPT_VERIFY_LANES, 1)
    return out


def _mismatches(tags, got, want, limit=8):
    return [(t, g, w) for t, g, w in zip(tags, got, want) if g != w][:limit]


def test_every_row_of_the_window_table(ctx, key):
    """One forged proof per reachable (input, window, digit), each accepted; every 8th of them also against the row with the
    digit's low bit flipped (digit 1 becomes the skipped zero digit), each rejected.  A failure names the table rows."""
    rows, cells = [], []
    for j in (1, 2, 3):
        for row, cell in vf.table_sweep(key.k, j):
            rows.append(row); cells.append(cell)
    assert len(rows) == 3 * (31 * 255 + 0x73 + 2)
    proofs = vf.proofs_for(key.crs, rows, A_S, B_S)
    t_rows, t_proofs, t_cells = [], [], []
    for i in range(0, len(rows), 8):
        j, w, d = cells[i]
        r2 = list(rows[i]); r2[j - 1] = r2[j - 1] ^ (1 << (8 * w)) if w >= 0 else r2[j - 1] - 1
        t_rows.append(r2); t_proofs.append(proofs[i]); t_cells.append((j, w, d, "digit ^ 1"))
    got = _verdicts(key.pvk, proofs + t_proofs, rows + t_rows)
    want = [1] * len(rows) + [0] * len(t_rows)
    assert _mismatches(cells + t_cells, got, want) == []
    pick = list(range(0, len(rows), 64))
    assert key.oracle([proofs[i] for i in pick], [rows[i] for i in pick]) == [1] * len(pick)


def _named_batch(key, rows):
    proofs = vf.proofs_for(key.crs, [row for row, _ in rows], A_S, B_S)
    batch_p, batch_r, want, tags = [], [], [], []
    for (row, name), proof in zip(rows, proofs):
        steps, final_inf = vf.sum_steps(key.k, row)
        want_steps, want_inf = vf.expected_reach(name, key.n)
        assert final_inf == want_inf and all(steps[j] == b for j, b in want_steps), (name, steps)
        batch_p.append(proof); batch_r.append(row); want.append(1); tags.append(name)
        for what, p2, r2 in vf.tamperings(key.crs, row, A_S, B_S):
            batch_p.append(p2 or proof); batch_r.append(r2 or row); want.append(0); tags.append(name + " " + what)
    return batch_p, batch_r, want, tags


def test_degenerate_public_input_sums(ctx, key):
    """Each named row reaches its branch of the sum (asserted on the model first) and its forged proof is accepted; one
    input + 1, C + G and the neighbouring row's proof are rejected.  Both Miller paths, and the key re-loaded from its image."""
    batch_p, batch_r, want, tags = _named_batch(key, vf.named_rows(key.k, pr.SplitMix64(77)))
    for got in _on_both_paths(ctx, key.pvk, batch_p, batch_r):
        assert _mismatches(tags, got, want) == []
    assert key.oracle(batch_p, batch_r) == want
    k2 = zk.PreparedVerifyingKey.read(ctx, key.pvk.write())
    try:
        assert _mismatches(tags, _verdicts(k2, batch_p, batch_r), want) == []
    finally:
        k2.free()


def test_one_doubling_among_generic_sums_in_a_warp(ctx, key):
    """Regression: one proof whose sum takes XYZZ::add's doubling branch between proofs on the generic branch, so that the
    32 threads of a k_ic_sum warp diverge there.  The doubling used to be a call made by part of the warp, and it overwrote
    a uniform register the other lanes' loads still used: the launch ended in "an illegal instruction was encountered"."""
    rng = pr.SplitMix64(88)
    for place in (0, 13, 31, 40):
        rows = [[rng.fr() for _ in range(3)] for _ in range(64)]
        rows[place] = vf.sum_doubling(key.k, rng, 2)[0]
        steps = [vf.sum_steps(key.k, r)[0] for r in rows]
        assert steps[place][1] == vf.DOUBLE and all(s == [vf.GENERIC] * 3 for i, s in enumerate(steps) if i != place)
        proofs = vf.proofs_for(key.crs, rows, A_S, B_S)
        assert _verdicts(key.pvk, proofs, rows) == [1] * 64, place


def test_infinity_sum_at_every_place_of_a_batch(ctx, key):
    """Proofs whose public-input sum is the point at infinity among ordinary ones (alternating true and false): first, last, a
    whole warp of five, every other slot.  The skip of the (acc, -gamma) pair is per proof and leaks to no neighbour."""
    rng = pr.SplitMix64(23)
    n = 23
    rows = [[rng.fr() for _ in range(3)] for _ in range(n)]
    cs = [vf.forge(key.crs, row, A_S, B_S, k=key.k)[2] + (i & 1) for i, row in enumerate(rows)]      # odd slots: C + G, false
    ordinary = vf.proofs_from_c(A_S, B_S, cs)
    inf_rows = [vf.total_infinity(key.k, rng, p)[0] for p in (None, "cancel", "zeros", None, None)]
    assert all(vf.sum_steps(key.k, r)[1] for r in inf_rows)
    inf_proofs = vf.proofs_for(key.crs, inf_rows, A_S, B_S)
    for name, places in (("first", [0]), ("last", [n - 1]), ("first and last", [0, n - 1]), ("warp 1", [5, 6, 7, 8, 9]),
                         ("odd slots", list(range(1, n, 2))), ("even slots", list(range(0, n, 2))), ("all", list(range(n)))):
        p, r, want = list(ordinary), list(rows), [1 - (i & 1) for i in range(n)]
        for t, i in enumerate(places):
            p[i], r[i], want[i] = inf_proofs[t % 5], inf_rows[t % 5], 1
        for got in _on_both_paths(ctx, key.pvk, p, r):
            assert got == want, name
    # a false proof with an infinity sum stays false: the ordinary slots' proofs against the infinity rows
    assert _verdicts(key.pvk, ordinary[:5], inf_rows) == [0] * 5


def test_key_of_22_public_inputs(ctx):
    """The confidential transfer's shape: the sum has 22 terms.  Cancellation at the first, a middle and the last input,
    doubling at the first, a middle and the last, the all-zero row, and sums equal to the point at infinity."""
    key = _Key(ctx, n_inputs=23, seed=41)
    try:
        rng = pr.SplitMix64(9)
        rows = [vf.mid_sum_infinity(key.k, rng, j) for j in (1, 11, 22)] + [vf.sum_doubling(key.k, rng, j) for j in (1, 12, 22)]
        rows += [vf.total_infinity(key.k, rng, p) for p in (None, "cancel", "zeros")] + [([0] * 22, "zero_terms/all")]
        batch_p, batch_r, want, tags = _named_batch(key, rows)
        for got in _on_both_paths(ctx, key.pvk, batch_p, batch_r):
            assert _mismatches(tags, got, want) == []
        assert key.oracle(batch_p, batch_r) == want
    finally:
        key.pvk.free()


@pytest.mark.parametrize("gamma,delta", [(True, False), (False, True), (True, True)])
def test_keys_with_the_infinity_flag(ctx, key, gamma, delta):
    """A PreparedVerifyingKey whose -gamma (-delta, both) is the prepared point at infinity (no coefficients, flag set; what
    the reference's G2Prepared::read accepts is stated in tests/test_oracle_verify_edges.py): it loads, writes back its
    image, and drops that pairing, so it accepts exactly the proofs forged without the term."""
    img = vf.flag_image(key.pvk.write(), gamma, delta)
    flagged = zk.PreparedVerifyingKey.read(ctx, img)
    oflag = co.PreparedVerifyingKey.read(img)
    try:
        assert flagged.num_inputs == 3 and flagged.write() == img == oflag.write()
        proofs, rows, want, tags = vf.flag_key_batch(key.crs, A_S, B_S, gamma, delta)
        good = proofs[0]
        proofs += [bytes([good[0] & 0x7F]) + good[1:], good[:144] + INF1]      # Proof::read: InvalidData, PointInfinity
        rows += [rows[0], rows[0]]; want += [2, 3]; tags += ["A without the compression flag", "C = O"]
        assert key.oracle(proofs, rows, oflag) == want
        for got in _on_both_paths(ctx, flagged, proofs, rows):
            assert _mismatches(tags, got, want) == []
    finally:
        flagged.free()


def test_flag_image_load_rejections(ctx, key):
    image = key.pvk.write()
    (g0, g1), (d0, d1) = vf.g2_prepared_spans(image)

    def code(buf):
        with pytest.raises(zk.SynthesisError) as e:
            zk.PreparedVerifyingKey.read(ctx, bytes(buf))
        return e.value.code

    for end in (g1, d1):
        bad = bytearray(image); bad[end - 1] = 2                                # a flag byte that is neither 0 nor 1
        assert code(bad) == -7
    # flag 0 with 67 coefficients: the Miller loop would run out of lines
    short = image[:g0] + (67).to_bytes(4, "big") + image[g0 + 4:g1 - 1 - 288] + b"\x00" + image[g1:]
    assert code(short) == -6
    short = image[:d0] + (0).to_bytes(4, "big") + b"\x00" + image[d1:]          # ... and with none
    assert code(short) == -6
    assert code(image[:d0 + 4 + 288 * 3]) == -6                                 # truncated inside the second table
    assert code(image[:d0 + 2]) == -6                                           # ... and inside its count
    # flag 1 keeps whatever coefficients it came with: loads, the image is kept, the pair is dropped
    kept = bytearray(image); kept[g1 - 1] = 1
    k2 = zk.PreparedVerifyingKey.read(ctx, bytes(kept))
    try:
        assert k2.write() == bytes(kept)
        proofs, rows, want, tags = vf.flag_key_batch(key.crs, A_S, B_S, True, False)
        assert _mismatches(tags, _verdicts(k2, proofs, rows), want) == []
    finally:
        k2.free()


LAST = ["valid", "false", "invalid_data", "point_infinity", "sum_is_infinity"]


@pytest.mark.parametrize("lanes", [1, 0])
def test_lane_groups_at_every_batch_boundary(ctx, key, lanes):
    """n across the boundaries of a group of five proofs (one warp) and of twenty (one block): the lanes and groups past the
    batch shadow proof n - 1, so that slot holds, in turn, a true proof, a false one, both Proof::read rejections and a true
    proof whose public-input sum is the point at infinity; the others alternate true and false.  Verdicts are the closed-form list and nothing is
    written beyond verdicts[n - 1]."""
    import torch
    assert vf.PROOFS_PER_BLOCK == 20
    sizes = list(range(1, 13)) + [19, 20, 21, 40, 41]
    rng = pr.SplitMix64(61)
    top = max(sizes)
    rows = [[rng.fr() for _ in range(3)] for _ in range(top)]
    cs = [vf.forge(key.crs, row, A_S, B_S, k=key.k)[2] for row in rows]
    valid = vf.proofs_from_c(A_S, B_S, cs)
    false = vf.proofs_from_c(A_S, B_S, [c + 1 for c in cs])
    inf_row = vf.total_infinity(key.k, rng)[0]
    inf_proof = vf.proofs_for(key.crs, [inf_row], A_S, B_S)[0]
    ctx.set_opt(zk.Context.OPT_VERIFY_LANES, lanes)
    bad = []
    try:
        for n in sizes:
            for last in LAST:
                p = [valid[i] if i % 2 == 0 else false[i] for i in range(n)]
                r = [list(x) for x in rows[:n]]
                want = [1 - (i & 1) for i in range(n)]
                e = n - 1
                if last == "valid":
                    p[e], want[e] = valid[e], 1
                elif last == "false":
                    p[e], want[e] = false[e], 0
                elif last == "invalid_data":
                    p[e], want[e] = bytes([valid[e][0] & 0x7F]) + valid[e][1:], 2
                elif last == "point_infinity":
                    p[e], want[e] = valid[e][:144] + INF1, 3                    # Proof::read: C = O
                else:
                    p[e], r[e], want[e] = inf_proof, inf_row, 1                 # a true proof whose public-input sum is O
                dp = torch.from_numpy(np.frombuffer(b"".join(p), np.uint8).copy()).cuda()
                di = torch.from_numpy(co.ints_to_limbs([x for row in r for x in row], 4).view(np.int64)).cuda()
                dv = torch.full((n + 64,), 0xEE, dtype=torch.uint8, device="cuda")
                torch.cuda.synchronize()
                zk.verify_proofs_device(key.pvk, n, dp.data_ptr(), di.data_ptr(), 3, dv.data_ptr())
                ctx.sync()
                out = dv.cpu().numpy()
                if [int(v) for v in out[:n]] != want or not (out[n:] == 0xEE).all():
                    bad.append((n, last, [int(v) for v in out[:n]], [int(v) for v in out[n:n + 24]]))
    finally:
        ctx.set_opt(zk.Context.OPT_VERIFY_LANES, 1)
    assert bad[:4] == []


def test_pairing_with_the_point_at_infinity_on_either_side(ctx):
    """Engine::pairing drops a pair with a zero side: (P, O), (O, Q) and (O, O) give Fq12::one(), between ordinary pairs whose
    results are the oracle's, in a batch of more than one 64-thread block."""
    n = vf.PAIRING_BLOCK + 10
    rng = pr.SplitMix64(47)
    sa = co.ints_to_limbs([rng.fr() or 1 for _ in range(n)], 4)
    sb = co.ints_to_limbs([rng.fr() or 1 for _ in range(n)], 4)
    e1, e2 = co.g1_fixed_base(sa, enc=True), co.g2_fixed_base(sb, enc=True)
    o1, o2 = pr.g1_uncompressed(pr.INF), pr.g2_uncompressed(pr.INF)
    g1 = [o1 if i % 4 in (2, 3) else e1[96 * i:96 * i + 96] for i in range(n)]
    g2 = [o2 if i % 4 in (1, 3) else e2[192 * i:192 * i + 192] for i in range(n)]
    assert {i % 4 for i in range(vf.PAIRING_BLOCK, n)} == {0, 1, 2, 3}          # every kind in the second block too
    got = zk.pairing(ctx, b"".join(g1), b"".join(g2))
    one = pr.f12_to_tower_bytes(pr.F12_ONE)
    for i in range(n):
        want = one if i % 4 else co.pairing(g1[i], g2[i])
        assert got[576 * i:576 * i + 576] == want, i
        assert i % 4 or want != one
    assert co.pairing(e1[:96], o2) == co.pairing(o1, e2[:192]) == co.pairing(o1, o2) == one
