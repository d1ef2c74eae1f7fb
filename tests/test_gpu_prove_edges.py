"""create_proof on its exceptional branches, with witnesses and blinding scalars chosen from the toy key's trapdoor
(tests/prove_forge.py), so that every case has its expected proof bytes in closed form:
  k_finish_proofs     A, B or C at infinity, and the doubling / cancellation branch of each addition of g_c = T0 + T1 + H' + L,
                      each degenerate proof alone among honest ones at positions 0, 31, 32 and 39 of a 40-proof batch
  k_scale_points      the GLV split's edge scalars as r and as s, under a checked load, an unchecked load (254-step chain)
                      and the decoded-CRS cache
  k_gather32          circuits with no aux in A, no input in B, no aux in B, through the evaluations path and the resident
                      constraint system (zk_r1cs_load), which must give the same bytes
  PROVE_CHUNK         a batch of 257 proofs, sliced
  zk_ntt_run          domains 2^1 .. 2^23, a batch of 2 at 2^23 (three-pass schedule, once per vector)
  zk_params_load      the empty l and b query vectors it refuses
Every expected proof comes from the trapdoor algebra, and where it is cheap also from the C oracle, never from the device;
the device verifier must accept each proof, or give PointInfinity (3) where a proof point is the point at infinity."""
import numpy as np
import pytest

from oracle import coracle as co
from oracle import pyref as pr
from tests import prove_forge as pf
from zero_chain_b200 import groth16 as zk
from zero_chain_b200 import synthetic as sy

pytestmark = pytest.mark.gpu
R = pf.R
TINY = dict(n_constraints=60, n_inputs=4, n_aux=50, a_aux_density=40, b_density=33)


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


def _pa(r1cs, z):
    return zk.ProvingAssignment(*pf.assignment(r1cs, z))


def _device_verdicts(ctx, params, proofs, zs, n_in):
    pvk = zk.PreparedVerifyingKey.prepare(ctx, params.vk_bytes())
    try:
        return zk.verify_proofs(pvk, b"".join(proofs), [list(z[1:n_in]) for z in zs])
    finally:
        pvk.free()


class _Tiny:
    def __init__(self, ctx, seed=3):
        self.r1cs = sy.make_r1cs(seed=seed, **TINY)
        self.crs = sy.make_toy_crs(self.r1cs, co.g1_fixed_base, co.g2_fixed_base, seed=seed + 1)
        self.checked = zk.Parameters.read(ctx, self.crs.params_bytes, checked=True)
        self.unchecked = zk.Parameters.read(ctx, self.crs.params_bytes, checked=False)
        self.oparams = co.Params(self.crs.params_bytes, checked=False)

    def oracle(self, z, r, s):
        return self.oparams.prove(*pf.assignment(self.r1cs, z), r, s)

    def free(self):
        self.checked.free(); self.unchecked.free()


@pytest.fixture(scope="module")
def tiny(ctx):
    t = _Tiny(ctx)
    yield t
    t.free()


def _split(blob):
    return [blob[192 * i:192 * i + 192] for i in range(len(blob) // 192)]


# ---- degenerate proofs among honest ones ---------------------------------------------------------------------------------------
def test_degenerate_proofs_in_a_batch(ctx, tiny):
    """Each named case (and the all-zero witness, L = O) alone among 39 honest proofs at positions 0, 31, 32 and 39: the
    first and last lane of a k_finish_proofs block and of the next one, so one lane takes the exceptional branch while
    the other 31 take the generic one."""
    n = 40
    rng = pr.SplitMix64(808)
    hz = [sy.make_witness(tiny.r1cs, 500 + k) for k in range(n)]
    hrs = [(rng.fr(), rng.fr()) for _ in range(n)]
    honest = pf.proofs_from_scalars([sy.expected_proof_scalars(tiny.crs, z, r, s) for z, (r, s) in zip(hz, hrs)])
    hpa = [_pa(tiny.r1cs, z) for z in hz]
    dz = sy.make_witness(tiny.r1cs, 2)
    w = pf.witness_scalars(tiny.crs, dz)
    cases = [(case, dz) + pf.solve(tiny.crs, w, case) for case in pf.BLINDING_CASES]
    cases.append(("zero_witness", pf.zero_witness(tiny.r1cs), 0x77, 0x99))
    bad = []
    for case, z, r, s in cases:
        want = pf.closed_form(tiny.crs, z, r, s)
        assert tiny.oracle(z, r, s) == want, case
        inf = pf.infinities(pf.intermediates(tiny.crs, pf.witness_scalars(tiny.crs, z), r, s))
        dpa = _pa(tiny.r1cs, z)
        for pos in (0, pf.FINISH_BLOCK - 1, pf.FINISH_BLOCK, n - 1):
            for params in ((tiny.checked, tiny.unchecked) if pos == pf.FINISH_BLOCK - 1 else (tiny.checked,)):
                pas = hpa[:pos] + [dpa] + hpa[pos + 1:]
                rs = [x[0] for x in hrs[:pos]] + [r] + [x[0] for x in hrs[pos + 1:]]
                ss = [x[1] for x in hrs[:pos]] + [s] + [x[1] for x in hrs[pos + 1:]]
                got = _split(zk.create_proof_batch(pas, params, rs, ss))
                exp = honest[:pos] + [want] + honest[pos + 1:]
                bad += [(case, pos, i) for i in range(n) if got[i] != exp[i]]
        zs = hz[:1] + [z]
        v = _device_verdicts(ctx, tiny.checked, [honest[0], want], zs, tiny.r1cs.n_inputs)
        assert v == [1, 3 if inf else 1], (case, v)
    assert bad[:8] == []


# ---- the GLV split under the three loads ----------------------------------------------------------------------------------------
def test_glv_edges_under_three_loads(ctx, tiny, tmp_path):
    """The GLV edge scalars as r and as s: the checked load splits k = k1 u^2 + k0, the unchecked load runs the 254-step
    chain, the cached load splits again; all three must give the closed form and the oracle's bytes."""
    cases = pf.glv_blindings()
    z = sy.make_witness(tiny.r1cs, 4)
    pas = [_pa(tiny.r1cs, z)] * len(cases)
    rs, ss = [c[1] for c in cases], [c[2] for c in cases]
    want = pf.proofs_from_scalars([sy.expected_proof_scalars(tiny.crs, z, r, s) for r, s in zip(rs, ss)])
    cache = str(tmp_path / "tiny.zkcache")
    miss = zk.Parameters.read_cached(ctx, tiny.crs.params_bytes, cache)
    hit = zk.Parameters.read_cached(ctx, tiny.crs.params_bytes, cache)
    assert not miss.cache_hit and hit.cache_hit
    for name, params in (("checked", tiny.checked), ("unchecked", tiny.unchecked), ("cache miss", miss), ("cache hit", hit)):
        got = _split(zk.create_proof_batch(pas, params, rs, ss))
        assert [c[0] for c, g, w in zip(cases, got, want) if g != w] == [], name
    miss.free(); hit.free()
    for i in (0, 6, 7, 8, 9):                                       # u2-1 and r-1 / r-2, both ways: the oracle too
        assert tiny.oracle(z, rs[i], ss[i]) == want[i], cases[i][0]
    assert _device_verdicts(ctx, tiny.checked, want, [z] * len(want), tiny.r1cs.n_inputs) == [1] * len(want)


# ---- density and shape corners ----------------------------------------------------------------------------------------------
CIRCUITS = {
    "m2": pf.circuit_m2,
    "no_aux_in_a": pf.circuit_no_aux_in_a,
    "no_input_in_b": pf.circuit_no_input_in_b,
    "no_aux_in_b": pf.circuit_no_aux_in_b,
    "all_aux_in_ab": pf.circuit_all_aux_in_ab,
    "pow2": lambda: pf.circuit_pow2(6),
    "pow2+1": lambda: pf.circuit_pow2(6, above=True),
    "witness_corners": pf.circuit_witness_corners,
}


@pytest.mark.parametrize("name", sorted(CIRCUITS))
def test_density_corners_on_both_paths(ctx, name):
    """host evaluations (create_proof_batch) and the resident constraint system (create_proof_from_witness_batch) give the
    same bytes, equal to the closed form and the oracle, and the device verifier accepts them"""
    r1cs = CIRCUITS[name]()
    crs = sy.make_toy_crs(r1cs, co.g1_fixed_base, co.g2_fixed_base, seed=5)
    params = zk.Parameters.read(ctx, crs.params_bytes, checked=True)
    zs = [pf.witness_for(r1cs, 10 + k) for k in range(3)] + [pf.zero_witness(r1cs)]
    rs, ss = [0x1111, R - 1, 0, 0x3333], [0x2222, R - 2, 0x4444, 0]
    got = zk.create_proof_batch([_pa(r1cs, z) for z in zs], params, rs, ss)
    cs = zk.ConstraintSystem(ctx, r1cs.n_inputs, r1cs.n_aux, r1cs.A, r1cs.B, r1cs.C)
    n_in = r1cs.n_inputs
    inputs = np.stack([co.ints_to_limbs(z[:n_in], 4) for z in zs])
    aux = np.stack([co.ints_to_limbs(z[n_in:], 4) for z in zs])
    assert zk.create_proof_from_witness_batch(cs, params, len(zs), inputs, aux, co.ints_to_limbs(rs, 4), co.ints_to_limbs(ss, 4)) == got
    want = [pf.closed_form(crs, z, r, s) for z, r, s in zip(zs, rs, ss)]
    assert _split(got) == want
    op = co.Params(crs.params_bytes, checked=False)
    assert op.prove(*pf.assignment(r1cs, zs[0]), rs[0], ss[0]) == want[0]
    assert _device_verdicts(ctx, params, want, zs, n_in) == [1] * len(zs)
    cs.free(); params.free()


def test_empty_query_vectors_are_refused(ctx):
    """A circuit without aux has an empty l query, one with empty B rows an empty b query.  bellman reads both; the device
    loader refuses them with IoError (-6), "empty query vector" (DESIGN deviation 8)."""
    no_aux = pf._R1(2, 0, [([(1, 1)], [(0, 1)], [(1, 1)])] * 3)
    no_b = pf._R1(2, 2, [([(2, 1)], [], []), ([(3, 1)], [], [])])
    for r1cs in (no_aux, no_b):
        crs = sy.make_toy_crs(r1cs, co.g1_fixed_base, co.g2_fixed_base, seed=5)
        co.Params(crs.params_bytes, checked=False)                     # the oracle reads it, as bellman does
        with pytest.raises(zk.SynthesisError) as e:
            zk.Parameters.read(ctx, crs.params_bytes, checked=True)
        assert e.value.code == -6 and "empty query vector" in str(e.value)


# ---- batch slicing ----------------------------------------------------------------------------------------------------------
def test_batch_above_prove_chunk(ctx, tiny):
    """257 proofs: a full 256-proof slice and a slice of one; expected bytes in bulk from the trapdoor"""
    n = pf.PROVE_CHUNK + 1
    rng = pr.SplitMix64(257)
    zs = [sy.make_witness(tiny.r1cs, 1000 + k) for k in range(n)]
    rs = [rng.fr() for _ in range(n)]; ss = [rng.fr() for _ in range(n)]
    rs[pf.PROVE_CHUNK - 1], ss[pf.PROVE_CHUNK] = 0, 0
    want = pf.proofs_from_scalars([sy.expected_proof_scalars(tiny.crs, z, r, s) for z, r, s in zip(zs, rs, ss)])
    got = _split(zk.create_proof_batch([_pa(tiny.r1cs, z) for z in zs], tiny.checked, rs, ss))
    assert [i for i in range(n) if got[i] != want[i]] == []


# ---- the domain sweep ---------------------------------------------------------------------------------------------------------
def _mont(x):
    return x * (1 << 256) % R


def _limb_int(row):
    return sum(int(x) << (64 * i) for i, x in enumerate(row))


def _fr_powers(ctx, base, n):
    """Montgomery limbs of base^i, i < n, by doubling the table with one device product per step"""
    out = co.ints_to_limbs([_mont(1)], 4)
    while out.shape[0] < n:
        k = min(out.shape[0], n - out.shape[0])
        step = np.tile(co.ints_to_limbs([_mont(pow(base, out.shape[0], R))], 4), (k, 1))
        out = np.concatenate([out, zk.field_op(ctx, zk.FIELD_FR, zk.OP_MUL, out[:k], step)])
    return out


def _fr_sum(ctx, v):
    """the sum of Montgomery limbs, as a canonical int (pairwise device additions)"""
    while v.shape[0] > 1:
        if v.shape[0] % 2:
            v = np.concatenate([v, np.zeros((1, 4), np.uint64)])
        h = v.shape[0] // 2
        v = zk.field_op(ctx, zk.FIELD_FR, zk.OP_ADD, v[:h], v[h:])
    return pr.fr_from_mont(_limb_int(v[0]))


def _g1_uncompressed_many(ctx, pts):
    """(n, 12) Montgomery affine limbs (none at infinity) -> n * 96 bytes of the uncompressed grammar"""
    canon = zk.field_op(ctx, zk.FIELD_FQ, zk.OP_INTO_REPR, np.ascontiguousarray(pts).reshape(-1, 6))
    be = np.ascontiguousarray(canon.view(np.uint8).reshape(-1, 48)[:, ::-1])
    return be.reshape(-1, 96).tobytes()


def toy_crs_dense(ctx, r1cs, seed):
    """sy.make_toy_crs(r1cs, ...) for a circuit_dense circuit, with the domain-sized parts on the device: the Lagrange
    weights from one batched inversion of tau - w^j, the h query as scalar_mul_many of zt/delta tau^i.  Same bytes."""
    import struct
    rng = sy.SplitMix64(seed)
    tau, alpha, beta, gamma, delta = (rng.fr() or 1 for _ in range(5))
    n_c, n_in = r1cs.n_constraints, r1cs.n_inputs
    n_rows = n_c + n_in
    log_m = max(1, (n_rows - 1).bit_length())
    m = 1 << log_m
    w = pow(sy._ROOT, 1 << (32 - log_m), R)
    zt = (pow(tau, m, R) - 1) % R
    W = _fr_powers(ctx, w, n_rows)
    D = zk.field_op(ctx, zk.FIELD_FR, zk.OP_SUB, np.tile(co.ints_to_limbs([_mont(tau)], 4), (n_rows, 1)), W)
    T = zk.field_op(ctx, zk.FIELD_FR, zk.OP_MUL, W, zk.field_op(ctx, zk.FIELD_FR, zk.OP_INV, D))
    scale = zt * pow(m, -1, R) % R
    lag = {j: scale * pr.fr_from_mont(_limb_int(T[j])) % R for j in (0, n_c, n_c + 1)}
    at, bt, ct = pf.dense_tables(n_c, scale * _fr_sum(ctx, T[:n_c]) % R, lag)
    a_aux_d, b_in_d, b_aux_d = sy.densities(r1cs)
    ginv, dinv = pow(gamma, -1, R), pow(delta, -1, R)
    comb = lambda i: (beta * at[i] + alpha * bt[i] + ct[i]) % R
    ic_s = [comb(i) * ginv % R for i in range(n_in)]
    l_s = [comb(n_in + i) * dinv % R for i in range(r1cs.n_aux)]
    a_s = [at[i] for i in range(n_in)] + [at[n_in + i] for i in range(r1cs.n_aux) if a_aux_d[i]]
    b_s = [bt[i] for i in range(n_in) if b_in_d[i]] + [bt[n_in + i] for i in range(r1cs.n_aux) if b_aux_d[i]]
    hs = zk.field_op(ctx, zk.FIELD_FR, zk.OP_MUL, _fr_powers(ctx, tau, m - 1), np.tile(co.ints_to_limbs([_mont(zt * dinv)], 4), (m - 1, 1)))
    hs = zk.field_op(ctx, zk.FIELD_FR, zk.OP_INTO_REPR, hs)
    h_bytes = _g1_uncompressed_many(ctx, zk.scalar_mul_many(ctx, 1, zk.G1_GENERATOR, hs))
    small = [alpha, beta, delta] + ic_s + l_s + a_s + b_s
    e1 = [sy.g1_limbs_to_uncompressed(p) for p in co.g1_fixed_base(co.ints_to_limbs(small, 4))]
    e2 = [sy.g2_limbs_to_uncompressed(p) for p in co.g2_fixed_base(co.ints_to_limbs([beta, gamma, delta] + b_s, 4))]
    out = bytearray(e1[0] + e1[1] + e2[0] + e2[1] + e1[2] + e2[2])
    off = 3
    out += struct.pack(">I", n_in) + b"".join(e1[off:off + n_in]); off += n_in
    out += struct.pack(">I", m - 1) + h_bytes
    for n in (len(l_s), len(a_s), len(b_s)):
        out += struct.pack(">I", n) + b"".join(e1[off:off + n]); off += n
    out += struct.pack(">I", len(b_s)) + b"".join(e2[3:])
    td = dict(tau=tau, alpha=alpha, beta=beta, gamma=gamma, delta=delta)
    return sy.ToyCRS(bytes(out), td, at, bt, ct, zt, log_m, r1cs)


def _dense_assignment(r1cs, z):
    """pf.assignment for circuit_dense without a Python loop over the rows"""
    n_c, n_rows = r1cs.n_constraints, r1cs.n_constraints + r1cs.n_inputs
    L = lambda v: co.ints_to_limbs([v], 4)[0]
    a = np.zeros((n_rows, 4), np.uint64); b = np.zeros_like(a); c = np.zeros_like(a)
    a[:n_c] = L(z[2]); a[n_c] = L(z[0]); a[n_c + 1] = L(z[1])
    b[0] = L(1); b[1:n_c] = L(z[2])
    c[0] = L(z[2]); c[1:n_c] = L(z[3])
    return zk.ProvingAssignment(a, b, c, co.ints_to_limbs(z[:2], 4), co.ints_to_limbs(z[2:], 4), *sy.densities(r1cs))


def test_dense_crs_builder_matches_the_toy_crs(ctx):
    r1cs = pf.circuit_dense(1 << 11)
    assert toy_crs_dense(ctx, r1cs, 8).params_bytes == sy.make_toy_crs(r1cs, co.g1_fixed_base, co.g2_fixed_base, seed=8).params_bytes


@pytest.mark.parametrize("log_m", [1, 2, 3, 5, 11, 12, 13, 17, 22, 23])
def test_domain_sweep(ctx, log_m):
    """Every constraint row non-empty, so the three NTT inputs are dense on the whole domain: 2^1 (the m = 2 circuit), the
    one-tile sizes, 2^12 and 2^13 (first two-pass sizes, even and odd split), 2^17, 2^22 (largest two-pass size) and 2^23
    (three passes), with a batch of 2 at 2^23."""
    if log_m == 1:
        r1cs = pf.circuit_m2()
        zs = [pf.witness_for(r1cs, 3), pf.witness_for(r1cs, 4)]
        crs = sy.make_toy_crs(r1cs, co.g1_fixed_base, co.g2_fixed_base, seed=8)
        pas = [_pa(r1cs, z) for z in zs]
    else:
        r1cs = pf.circuit_dense(1 << log_m)
        zs = [pf.witness_dense(30), pf.witness_dense(31)]
        crs = (sy.make_toy_crs(r1cs, co.g1_fixed_base, co.g2_fixed_base, seed=8) if log_m <= 13 else toy_crs_dense(ctx, r1cs, 8))
        pas = [_dense_assignment(r1cs, z) for z in zs]
    assert crs.log_m == log_m
    params = zk.Parameters.read(ctx, crs.params_bytes, checked=log_m <= 13)
    assert params.n_h == (1 << log_m) - 1
    rs, ss = [0xABCDEF, R - 1], [R - 2, 0x123456]
    batch = 2 if log_m in (11, 23) else 1
    got = _split(zk.create_proof_batch(pas[:batch], params, rs[:batch], ss[:batch]))
    want = [pf.closed_form(crs, z, r, s) for z, r, s in zip(zs[:batch], rs, ss)]
    assert got == want
    if log_m <= 13:
        op = co.Params(crs.params_bytes, checked=False)
        assert op.prove(*pf.assignment(r1cs, zs[0]), rs[0], ss[0]) == want[0]
    assert _device_verdicts(ctx, params, want, zs[:batch], r1cs.n_inputs) == [1] * batch
    params.free()
