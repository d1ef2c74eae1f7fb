"""The forged-proof corpus (tests/verify_forge.py) through the two host oracles, before any GPU is involved: every named
degenerate public-input row is accepted by the big-integer Python verifier and by the C verifier and rejected after each
tampering, a thinned sweep of the window-table rows is accepted by the C verifier, prepared keys that carry the infinity
flag load, write back and verify in both, and the reach model and its copies of the kernels' constants are checked
against the CUDA sources.  CPU only."""
import os
import re

import pytest

from oracle import coracle as co
from oracle import pyref as pr
from tests import verify_forge as vf
from zero_chain_b200 import synthetic as sy

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "zero_chain_b200", "csrc")
A_S, B_S = vf.A_S, vf.B_S


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _const(text, name):
    m = re.search(r"\b%s\s*=\s*([^,;]+)[,;]" % name, text)
    assert m, name
    expr = re.sub(r"\b(0x[0-9a-fA-F]+|\d+)[uUlL]+\b", r"\1", m.group(1).strip()).replace("(size_t)", "")
    return eval(expr, {"__builtins__": {}}, {})


# ---- the model's constants and branch conditions against the sources ---------------------------------------------------
@pytest.mark.parametrize("source,name,copy", [
    ("pairing.cu", "IC_WIN", vf.IC_WIN),
    ("pairing.cu", "IC_DIG", vf.IC_DIG),
    ("pairing.cu", "PT", vf.PAIRING_BLOCK),
    ("pairing.cu", "VERIFY_CHUNK", vf.VERIFY_CHUNK),
    ("pairing.cuh", "N_COEFFS", vf.N_COEFFS),
    ("pairing_lanes.cuh", "GROUPS_PER_WARP", vf.GROUPS_PER_WARP),
])
def test_constant_matches_source(source, name, copy):
    assert _const(_src(source), name) == copy


def test_lane_block_geometry():
    blocks = set(re.findall(r"k_(?:miller|verify_final)_lanes<<<g, (\d+),", _src("pairing_lanes.cu")))
    assert blocks == {str(vf.LANES_BLOCK)} and vf.PROOFS_PER_BLOCK == vf.LANES_BLOCK // 32 * vf.GROUPS_PER_WARP == 20
    assert 6 * vf.GROUPS_PER_WARP == 30              # lanes 30 and 31 of a warp carry no proof of their own


# ---- the toy key --------------------------------------------------------------------------------------------------------
class _Key(vf.ToyKey):
    def __init__(self):
        super().__init__()
        self.vk = pr.vk_read(self.crs.params_bytes)

    def c_verdicts(self, proofs, rows, opvk=None):
        return self.oracle(proofs, rows, opvk)


@pytest.fixture(scope="module")
def key():
    return _Key()


def test_ic_scalars_are_the_discrete_logs_of_ic(key):
    want = b"".join(pr.g1_uncompressed(p) for p in key.vk["ic"])
    assert co.g1_fixed_base(co.ints_to_limbs(key.k, 4), enc=True) == want
    assert all(key.k)


# ---- the reach model ------------------------------------------------------------------------------------------------------
def test_sum_steps_on_hand_made_sums():
    k = [5, 1, 2, 3]                                  # ic_0 = 5 G, ic_1 = G, ic_2 = 2 G, ic_3 = 3 G
    assert vf.sum_steps(k, [1, 1, 1]) == ([vf.GENERIC] * 3, False)
    assert vf.sum_steps(k, [5, 1, 1]) == ([vf.DOUBLE, vf.GENERIC, vf.GENERIC], False)        # 5 + 5
    assert vf.sum_steps(k, [1, 3, 4]) == ([vf.GENERIC, vf.DOUBLE, vf.DOUBLE], False)         # 6 + 6, 12 + 12
    assert vf.sum_steps(k, [vf.R - 5, 4, 1]) == ([vf.CANCEL, vf.ENTER, vf.GENERIC], False)   # 5 - 5, O + 8, 8 + 3
    assert vf.sum_steps(k, [vf.R - 5, 0, 0]) == ([vf.CANCEL, vf.SKIP, vf.SKIP], True)
    assert vf.sum_steps(k, [0, 0, 0]) == ([vf.SKIP] * 3, False)
    assert vf.sum_steps(k, [1, 0, vf.R - 2]) == ([vf.GENERIC, vf.SKIP, vf.CANCEL], True)     # 6 - 6
    assert vf.public_sum(k, [1, 1, 1]) == 11
    with pytest.raises(AssertionError):
        vf.sum_steps([5, 0, 2], [1, 1])


@pytest.mark.parametrize("n_inputs", [4, 23])
def test_named_rows_reach_their_branches(n_inputs):
    """Each builder's row takes the branch it is named after, under the keys the GPU tests use (3 and 22 public inputs)."""
    k = vf.ToyKey(n_inputs, seed=3 if n_inputs == 4 else 41).k
    n = n_inputs - 1
    rows = vf.named_rows(k, pr.SplitMix64(77))
    rows += [vf.mid_sum_infinity(k, pr.SplitMix64(5), j) for j in sorted({n // 2, n} - {1, 2})]
    names = [name for _, name in rows]
    assert len(set(names)) == len(names)
    for row, name in rows:
        assert len(row) == n and all(0 <= x < vf.R for x in row)
        steps, final_inf = vf.sum_steps(k, row)
        want_steps, want_inf = vf.expected_reach(name, n)
        assert final_inf == want_inf, name
        for j, branch in want_steps:
            assert steps[j] == branch, (name, j, steps)
    # the window rows: the chosen bytes are zero and nothing else about the row is degenerate
    win = {name: row for row, name in rows if name.startswith("zero_terms/windows")}
    assert vf.window_digits(win["zero_terms/windows0"][0])[0] == 0
    assert vf.window_digits(win["zero_terms/windows0"][1])[31] == 0
    assert [d for d in vf.window_digits(win["zero_terms/windows0"][2])] == [0, 0xA5] * 15 + [0, 0]


def test_table_sweep_covers_every_reachable_row():
    k = [3, 5, 7, 11]
    for j in (1, 2, 3):
        sweep = vf.table_sweep(k, j)
        cells = {(w, d) for _, (_, w, d) in sweep if w >= 0}
        want = {(w, d) for w in range(32) for d in range(1, 256) if (d << (8 * w)) < vf.R}
        assert cells == want and len(want) == 31 * 255 + 0x73
        for row, (jj, w, d) in sweep:
            assert jj == j and row[j - 1] < vf.R and all(x == 7 for i, x in enumerate(row) if i != j - 1)
            if w >= 0:
                dig = vf.window_digits(row[j - 1])
                assert dig[w] == d and sum(1 for x in dig if x) == 1
        extra = [row[j - 1] for row, (_, w, _) in sweep if w < 0]
        assert extra[0] == vf.R - 1 and vf.window_digits(extra[1]) == [0xFF] * 31 + [0x72]


# ---- the degenerate rows through both oracles -------------------------------------------------------------------------------
def _py_verifier(key, gamma=True, delta=True):
    vk = key.vk
    ab = pr.pairing_reference(vk["alpha_g1"], vk["beta_g2"])
    gam = pr.g2_prepare(pr.ec_neg(pr.FQ2, vk["gamma_g2"])) if gamma else []
    dlt = pr.g2_prepare(pr.ec_neg(pr.FQ2, vk["delta_g2"])) if delta else []
    return lambda proof, row: int(pr.verify_prepared(ab, gam, dlt, vk["ic"], pr.proof_read(proof), row))


def test_degenerate_rows_are_accepted_and_tamperings_rejected_by_both_oracles(key):
    """The forged proof of every named row verifies in the C oracle, and is rejected after one input + 1, C + G, and when it
    is the proof of the neighbouring row; the big-integer verifier (about a second per proof) agrees.  A sum equal to the
    point at infinity must be accepted by both: Engine::miller_loop drops a pair with a zero side."""
    rows = vf.named_rows(key.k, pr.SplitMix64(77))
    proofs = vf.proofs_for(key.crs, [row for row, _ in rows], A_S, B_S)
    batch_p, batch_r, want, tags = [], [], [], []
    for (row, name), proof in zip(rows, proofs):
        batch_p.append(proof); batch_r.append(row); want.append(1); tags.append(name)
        for what, p2, r2 in vf.tamperings(key.crs, row, A_S, B_S):
            batch_p.append(p2 or proof); batch_r.append(r2 or row); want.append(0); tags.append(name + " " + what)
    got = key.c_verdicts(batch_p, batch_r)
    assert [t for t, g, w in zip(tags, got, want) if g != w] == []
    # big-integer verifier: every accepted proof; all three tamperings of the O-sum row, one (rotating) of every other row
    py = _py_verifier(key)
    kinds = ["input+1", "C+G", "neighbour"]
    for i, (tag, p, r, w) in enumerate(zip(tags, batch_p, batch_r, want)):
        name, _, what = tag.partition(" ")
        if not what or name == "total_infinity" or what == kinds[(i // 4) % 3]:
            assert py(p, r) == w, tag


def test_thinned_table_sweep_is_accepted_by_the_c_oracle(key):
    """Every 16th (window, digit) row of each input's table, plus every digit of windows 0 and 31, r - 1 and the all-0xff
    value: forged proofs, all accepted; the same proofs against the row with the digit's low bit flipped, all rejected."""
    rows, cells = [], []
    for j in (1, 2, 3):
        for i, (row, cell) in enumerate(vf.table_sweep(key.k, j)):
            if i % 16 == 0 or cell[1] in (0, 31, -1):
                rows.append(row); cells.append(cell)
    proofs = vf.proofs_for(key.crs, rows, A_S, B_S)
    got = key.c_verdicts(proofs, rows)
    assert [c for c, g in zip(cells, got) if g != 1] == []
    flipped = []
    for row, (j, w, d) in zip(rows[::8], cells[::8]):
        r2 = list(row)
        r2[j - 1] = r2[j - 1] ^ (1 << (8 * w)) if w >= 0 else r2[j - 1] - 1
        flipped.append(r2)
    assert key.c_verdicts(proofs[::8], flipped) == [0] * len(flipped)


# ---- prepared keys that carry the infinity flag -------------------------------------------------------------------------------
@pytest.mark.parametrize("gamma,delta", [(True, False), (False, True), (True, True)])
def test_infinity_flag_keys_in_both_oracles(key, gamma, delta):
    """G2Prepared::read (core/pairing/src/bls12_381/ec.rs:1652-1684) takes a u32 count, that many coefficient triples
    (Fq2::read: each Fq must be canonical, else the read fails) and a flag byte that must be 0 or 1; it keeps both, whatever
    the count, and G2Prepared::write gives the same bytes back.  G2Prepared::from_affine of the point at infinity is count 0
    with the flag set, and Engine::miller_loop drops a pair whose G2Prepared has the flag set.  So a PreparedVerifyingKey
    with such a -gamma (-delta) loads, writes back byte for byte, and verifies exactly the proofs with
    e(A, B) = e(alpha, beta) e(C, delta)  (resp. e(alpha, beta) e(acc, gamma)): with -gamma dropped the verdict no longer
    depends on the public inputs."""
    image = pr.pvk_write(key.vk)
    assert co.PreparedVerifyingKey.read(image).write() == image == key.opvk.write()
    img = vf.flag_image(image, gamma, delta)
    assert len(img) == len(image) - 288 * vf.N_COEFFS * (int(gamma) + int(delta))
    flagged = co.PreparedVerifyingKey.read(img)
    assert flagged.write() == img
    proofs, rows, want, tags = vf.flag_key_batch(key.crs, A_S, B_S, gamma, delta)
    # the matching proof of three rows (a random one, one whose sum is O, all zero), the first of them against the other two
    # rows, then the three ordinary proofs: with only -gamma dropped the ordinary proof of the O-sum row still holds
    assert want == [1, 1, 1, int(gamma), int(gamma), 0, int(gamma and not delta), 0]
    got = key.c_verdicts(proofs, rows, flagged)
    assert [t for t, g, w in zip(tags, got, want) if g != w] == []
    py = _py_verifier(key, gamma=not gamma, delta=not delta)
    for i in (0, 3, 5):
        assert py(proofs[i], rows[i]) == want[i], tags[i]
    # under the ordinary key the matching proof of the random row is false
    assert key.c_verdicts(proofs[:1], rows[:1]) == [0]


def test_flag_image_load_rejections_in_the_c_oracle(key):
    image = pr.pvk_write(key.vk)
    (g0, g1), (d0, d1) = vf.g2_prepared_spans(image)
    assert (g1 - g0, d1 - d0) == (4 + 288 * vf.N_COEFFS + 1,) * 2
    bad = bytearray(image); bad[g1 - 1] = 2                         # flag byte 2
    with pytest.raises(ValueError):
        co.PreparedVerifyingKey.read(bytes(bad))
    with pytest.raises(ValueError):
        co.PreparedVerifyingKey.read(image[:d0 + 4 + 288 * 3])      # truncated inside the second table
    bad = bytearray(image); bad[g0 + 4:g0 + 52] = b"\xff" * 48      # a coefficient >= q
    with pytest.raises(ValueError):
        co.PreparedVerifyingKey.read(bytes(bad))


def test_flag_set_on_a_full_coefficient_table(key):
    """G2Prepared::read keeps the coefficients of a record whose flag is set, and write gives them back; the pair is dropped
    all the same.  (The C oracle used to write such a record back as count 0.)"""
    image = pr.pvk_write(key.vk)
    (g0, g1), _ = vf.g2_prepared_spans(image)
    kept = bytearray(image); kept[g1 - 1] = 1
    k2 = co.PreparedVerifyingKey.read(bytes(kept))
    assert k2.write() == bytes(kept)
    proofs, rows, want, tags = vf.flag_key_batch(key.crs, A_S, B_S, True, False)
    assert key.c_verdicts(proofs, rows, k2) == want
