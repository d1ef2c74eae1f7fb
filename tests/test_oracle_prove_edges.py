"""The prover's forged-witness corpus (tests/prove_forge.py) through the host oracles, before any GPU is involved: every
named blinding case reaches the branch it is named after, the C oracle's create_proof returns the closed-form bytes for it,
non-degenerate proofs verify under the C verifier and proofs with a point at infinity get the PointInfinity verdict; the
hand-written circuits have the density corners they are named after; the model's copies of the kernels' constants are
read back out of the CUDA sources.  CPU only."""
import os
import re

import pytest

from oracle import coracle as co
from tests import prove_forge as pf
from zero_chain_b200 import synthetic as sy

R = pf.R
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "zero_chain_b200", "csrc")


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _const(text, name):
    m = re.search(r"\b%s\s*=\s*([^,;]+)[,;]" % name, text)
    assert m, name
    expr = re.sub(r"\b(0x[0-9a-fA-F]+|\d+)[uUlL]+\b", r"\1", m.group(1).strip()).replace("(size_t)", "")
    return eval(expr, {"__builtins__": {}}, {})


# ---- the model's constants against the sources ------------------------------------------------------------------------------
@pytest.mark.parametrize("source,name,copy", [
    ("groth16.cu", "PROVE_CHUNK", pf.PROVE_CHUNK),
    ("groth16.cu", "SCALE_T", pf.SCALE_T),
    ("ntt.cu", "MAX_TILE_LOG", pf.MAX_TILE_LOG),
])
def test_constant_matches_source(source, name, copy):
    assert _const(_src(source), name) == copy


def test_finish_block_and_glv_clamp_match_source():
    g = _src("groth16.cu")
    assert re.search(r"k_finish_proofs<<<\(unsigned\)\(\(batch \+ %d\) / %d\), %d," % (pf.FINISH_BLOCK - 1, pf.FINISH_BLOCK, 3 * pf.FINISH_BLOCK), g)
    assert "(size_t)blockIdx.x * %d + (threadIdx.x & %d)" % (pf.FINISH_BLOCK, pf.FINISH_BLOCK - 1) in g
    assert re.search(r"if \(glv && top > %d\) top = %d;" % (pf.GLV_TOP, pf.GLV_TOP), g)
    assert "zkglv::split_u2(k, kk[0], kk[1])" in g
    words = re.search(r"#define ZK_GLV_U2_INIT \{([^}]*)\}", _src("glv_split.cuh")).group(1)
    assert tuple(int(w.strip().rstrip("u"), 16) for w in words.split(",")) == pf.U2_WORDS


# ---- the GLV split model ------------------------------------------------------------------------------------------------------
def test_glv_edges_split_where_the_issue_says():
    s = {name: pf.glv_split(k) for name, k in pf.GLV_EDGES.items()}
    assert s["r-1"] == (0, pf.U2 - 1) and s["r-2"] == (pf.U2 - 1, pf.U2 - 2)
    assert s["u2-1"] == (pf.U2 - 1, 0) and s["u2"] == (0, 1) and s["u2+1"] == (1, 1) and s["2u2"] == (0, 2)
    assert s["2^127"] == (1 << 127, 0)                                   # u^2 > 2^127: no quotient yet
    assert s["2^128"] == ((1 << 128) - pf.U2, 1) and s["2^128+u2"] == ((1 << 128) - pf.U2, 2)
    for name, k in pf.GLV_EDGES.items():
        k0, k1 = s[name]
        assert 0 <= k < 1 << 255 and k0 < pf.U2 < 1 << 128 and k1 < 1 << 128 and k1 * pf.U2 + k0 == k
    # the chain reaches bit 127 exactly where k1 or k0 has it; r - 1 and r - 2 are such scalars
    assert pf.chain_bits(R - 1, True) == pf.chain_bits(R - 2, True) == pf.GLV_TOP
    assert max(pf.chain_bits(k, True) for k in pf.GLV_EDGES.values()) == pf.GLV_TOP
    assert pf.chain_bits(1 << 254, False) == 254 and pf.chain_bits(0, True) == -1


# ---- the toy key and its witness ------------------------------------------------------------------------------------------------
TINY = dict(n_constraints=60, n_inputs=4, n_aux=50, a_aux_density=40, b_density=33)


class Tiny:
    def __init__(self, seed=3):
        self.r1cs = sy.make_r1cs(seed=seed, **TINY)
        self.crs = sy.make_toy_crs(self.r1cs, co.g1_fixed_base, co.g2_fixed_base, seed=seed + 1)
        self.oparams = co.Params(self.crs.params_bytes, checked=False)
        self.opvk = co.PreparedVerifyingKey.prepare(self.crs.params_bytes)

    def prove(self, z, r, s):
        return self.oparams.prove(*pf.assignment(self.r1cs, z), r, s)

    def verdicts(self, proofs, zs):
        n = self.r1cs.n_inputs
        return self.opvk.verify_batch(b"".join(proofs), co.ints_to_limbs([x for z in zs for x in z[1:n]], 4), n - 1)


@pytest.fixture(scope="module")
def tiny():
    return Tiny()


def test_model_matches_expected_proof_scalars(tiny):
    z = sy.make_witness(tiny.r1cs, 1)
    w = pf.witness_scalars(tiny.crs, z)
    for r, s in ((0x1234, 0x5678), (R - 1, R - 2), (0, 0)):
        iv = pf.intermediates(tiny.crs, w, r, s)
        assert (iv["A"], iv["B"], iv["C"]) == sy.expected_proof_scalars(tiny.crs, z, r, s)
        assert pf.finish_steps(iv) == [pf.GENERIC] * 3 or (r, s) == (0, 0)


@pytest.mark.parametrize("case", pf.BLINDING_CASES)
def test_named_case_reaches_its_branch_and_the_oracle_agrees(tiny, case):
    """The solved (r, s) makes the relation hold, the model names the branch, the C oracle's create_proof returns the
    closed-form bytes, and the C verifier says 1, or 3 when a proof point is the point at infinity."""
    z = sy.make_witness(tiny.r1cs, 2)
    w = pf.witness_scalars(tiny.crs, z)
    r, s = pf.solve(tiny.crs, w, case)
    iv = pf.intermediates(tiny.crs, w, r, s)
    inf, steps = pf.expected_reach(case)
    assert pf.infinities(iv) == inf
    got_steps = pf.finish_steps(iv)
    for j, branch in steps:
        assert got_steps[j] == branch, (case, got_steps)
    if case == "T0+T1+H'=L":
        assert iv["C"] == 2 * iv["L"] % R
    want = pf.proofs_from_scalars([(iv["A"], iv["B"], iv["C"])])[0]
    assert tiny.prove(z, r, s) == want
    assert tiny.verdicts([want], [z]) == [3 if inf else 1]


def test_zero_witness_gives_l_at_infinity(tiny):
    z = pf.zero_witness(tiny.r1cs)
    assert pf.check_witness(tiny.r1cs, z)
    w = pf.witness_scalars(tiny.crs, z)
    assert w["laux"] == 0
    iv = pf.intermediates(tiny.crs, w, 0x77, 0x99)
    assert iv["L"] == 0 and pf.finish_steps(iv)[2] == pf.SKIP
    want = pf.closed_form(tiny.crs, z, 0x77, 0x99)
    assert tiny.prove(z, 0x77, 0x99) == want and tiny.verdicts([want], [z]) == [1]


def test_glv_blindings_through_the_oracle(tiny):
    z = sy.make_witness(tiny.r1cs, 4)
    cases = pf.glv_blindings()
    want = [pf.closed_form(tiny.crs, z, r, s) for _, r, s in cases]
    got = [tiny.prove(z, r, s) for _, r, s in cases]
    assert [n for (n, _, _), g, w in zip(cases, got, want) if g != w] == []
    assert tiny.verdicts(want, [z] * len(want)) == [1] * len(want)


# ---- circuits -----------------------------------------------------------------------------------------------------------
CIRCUITS = {
    "m2": pf.circuit_m2,
    "no_aux_in_a": pf.circuit_no_aux_in_a,
    "no_input_in_b": pf.circuit_no_input_in_b,
    "no_aux_in_b": pf.circuit_no_aux_in_b,
    "all_aux_in_ab": pf.circuit_all_aux_in_ab,
    "pow2": lambda: pf.circuit_pow2(6),
    "pow2+1": lambda: pf.circuit_pow2(6, above=True),
    "witness_corners": pf.circuit_witness_corners,
    "dense": lambda: pf.circuit_dense(16),
}


@pytest.mark.parametrize("name", sorted(CIRCUITS))
def test_circuit_corners(name):
    """each circuit has the corner it is named after, its witness satisfies it, and the C oracle proves it to the closed
    form and verifies the proof"""
    r1cs = CIRCUITS[name]()
    a_aux, b_in, b_aux = sy.densities(r1cs)
    n_rows = r1cs.n_constraints + r1cs.n_inputs
    log_m = max(1, (n_rows - 1).bit_length())
    corner = {
        "m2": r1cs.n_inputs == 1 and r1cs.n_aux == 1 and log_m == 1,
        "no_aux_in_a": not a_aux.any() and b_in.any() and b_aux.any(),
        "no_input_in_b": not b_in.any() and a_aux.any() and b_aux.any(),
        "no_aux_in_b": not b_aux.any() and b_in.any() and a_aux.any(),
        "all_aux_in_ab": a_aux.all() and b_aux.all(),
        "pow2": n_rows == 64 and log_m == 6,
        "pow2+1": n_rows == 65 and log_m == 7,
        "witness_corners": any(not row for row in r1cs.A) and any(len({v for v, _ in row}) < len(row) for row in r1cs.A)
                           and any(c == R - 1 for row in r1cs.A for _, c in row)
                           and all(any(v == r1cs.n_inputs + r1cs.n_aux - 1 for row in M for v, _ in row) for M in (r1cs.A, r1cs.B, r1cs.C)),
        "dense": all(r1cs.A) and all(r1cs.B) and all(r1cs.C),
    }[name]
    assert corner
    crs = sy.make_toy_crs(r1cs, co.g1_fixed_base, co.g2_fixed_base, seed=5)
    z = pf.witness_dense(9) if name == "dense" else pf.witness_for(r1cs, 9)
    assert pf.check_witness(r1cs, z)
    op = co.Params(crs.params_bytes, checked=False)
    want = pf.closed_form(crs, z, 0x1111, 0x2222)
    assert op.prove(*pf.assignment(r1cs, z), 0x1111, 0x2222) == want
    n = r1cs.n_inputs
    verdict = co.PreparedVerifyingKey.prepare(crs.params_bytes).verify_batch(want, co.ints_to_limbs(z[1:n], 4), n - 1)
    assert verdict == [1]


def test_dense_tables_match_the_toy_crs():
    """the Lagrange-sum shortcut of the large-domain CRS gives the toy CRS's own at / bt / ct"""
    r1cs = pf.circuit_dense(29)
    crs = sy.make_toy_crs(r1cs, co.g1_fixed_base, co.g2_fixed_base, seed=6)
    lag, _ = sy._lagrange_at(crs.trapdoor["tau"], crs.log_m, 29)
    n_c = r1cs.n_constraints
    at, bt, ct = pf.dense_tables(n_c, sum(lag[:n_c]) % R, lag)
    assert (at, bt, ct) == (crs.at, crs.bt, crs.ct)


def test_empty_query_vectors_are_accepted_by_the_oracle():
    """bellman reads an empty l or b query; the device loader refuses it (DESIGN deviation 8).  The oracle, like bellman,
    reads it: a circuit without aux has an empty l vector."""
    r1cs = pf._R1(2, 0, [([(1, 1)], [(0, 1)], [(1, 1)])] * 3)
    crs = sy.make_toy_crs(r1cs, co.g1_fixed_base, co.g2_fixed_base, seed=5)
    assert co.Params(crs.params_bytes, checked=False).n_l == 0
