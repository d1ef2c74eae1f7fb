"""Synthetic workloads of the confidential_transfer shape (host-side, pure Python/numpy).

The real circuit's witness needs the Rust gadget library (sapling-crypto, un-vendored; SURVEY.md
§8c.2), so benchmarks and tests use a synthetic R1CS with the SAME shape as the reference's
`confidential_transfer` circuit (core/proofs/src/circuit/confidential_transfer.rs:383-386 and the
CRS vector lengths parsed from zface/params/conf_pk.dat):

    constraints 19 974 (+23 input rows -> domain 2^15), inputs 23, aux 19 955,
    |a query| 15 598, |b query| 12 402, |h| 32 767, |l| 19 955.

and a toy CRS with a KNOWN trapdoor (tau, alpha, beta, gamma, delta) written in the exact
`Parameters::write` grammar (SURVEY.md §3.3).  Knowing the trapdoor gives a closed-form expected
proof for any satisfying witness — an end-to-end check that shares no code with the NTT/MSM kernels.

Nothing here touches the oracle: curve points are produced by a caller-supplied generator
`gen_g1(scalars)->(n,12) uint64 limb-form` / `gen_g2(scalars)->(n,24)` (the GPU library's batched
scalar multiplication in bench.py; the oracle's in CPU-only tests).
"""
from __future__ import annotations

import struct
from dataclasses import dataclass, field

import numpy as np

R = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001
_ROOT = pow(7, (R - 1) >> 32, R)

CONF_SHAPE = dict(n_constraints=19974, n_inputs=23, n_aux=19955, a_aux_density=15575, b_density=12402)
# The reference's second circuit (SURVEY.md §8 f3): anonymous_transfer, ~50 634 constraints, 105 inputs, domain 2^16;
# CRS vector lengths parsed from zface/params/anony_pk.dat: h 65 535, l 50 429, a 39 133, b 31 257, ic 105
# (core/proofs/src/circuit/anonymous_transfer.rs:449-451, core/proofs/src/anonymous.rs:165).
ANON_SHAPE = dict(n_constraints=50634, n_inputs=105, n_aux=50429, a_aux_density=39028, b_density=31257)


class SplitMix64:
    def __init__(self, seed):
        self.s = seed & 0xFFFFFFFFFFFFFFFF

    def next(self):
        self.s = (self.s + 0x9E3779B97F4A7C15) & 0xFFFFFFFFFFFFFFFF
        z = self.s
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & 0xFFFFFFFFFFFFFFFF
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & 0xFFFFFFFFFFFFFFFF
        return z ^ (z >> 31)

    def fr(self):
        x = 0
        for i in range(5):
            x |= self.next() << (64 * i)
        return x % R

    def below(self, n):
        return self.next() % n


def ints_to_limbs(vals, n_limbs=4):
    out = np.zeros((len(vals), n_limbs), dtype=np.uint64)
    mask = 0xFFFFFFFFFFFFFFFF
    for i, v in enumerate(vals):
        for j in range(n_limbs):
            out[i, j] = (v >> (64 * j)) & mask
    return out


def random_fr_limbs(n, seed):
    """n uniform canonical Fr elements as (n,4) uint64 (vectorised; rejection by masking + fixup)."""
    rng = np.random.Generator(np.random.Philox(seed))
    a = rng.integers(0, 1 << 64, size=(n, 4), dtype=np.uint64)
    a[:, 3] &= np.uint64((1 << 62) - 1)     # < 2^254 < r : uniform on a 254-bit range (documented)
    return a


@dataclass
class R1CS:
    n_inputs: int
    n_aux: int
    A: list = field(default_factory=list)   # rows: list of (var, coeff); var < n_inputs => input, else aux
    B: list = field(default_factory=list)
    C: list = field(default_factory=list)
    n_bool: int = 0

    @property
    def n_constraints(self):
        return len(self.A)


def make_r1cs(n_constraints, n_inputs, n_aux, a_aux_density, b_density, seed=1, frac_bool=0.6):
    """Satisfiable R1CS of the requested shape.

    aux 0..n_bool-1 are booleans constrained by x*(ONE-x)=0 (the real circuit's witness is mostly
    booleans, SURVEY.md §7 'hard parts'); every other aux w is a product variable constrained by
    <A,z>*<B,z> = w with sparse A/B rows over earlier variables.  A rows only touch aux < a_aux_density
    and B rows only aux < b_density-3 (plus inputs 0..2), and every such variable is touched at least
    once, so the density popcounts equal the requested |a query| / |b query| sizes exactly.
    Rows beyond n_aux re-constrain booleans (the real circuit has 19 more constraints than aux)."""
    assert n_constraints >= n_aux and n_inputs >= 3
    rng = SplitMix64(seed)
    nb_in = 3                                    # ONE and inputs 1,2 appear in B rows
    nb_aux = b_density - nb_in
    n_bool = max(1, min(int(n_aux * frac_bool), a_aux_density, nb_aux))
    assert n_bool <= a_aux_density <= n_aux and n_bool <= nb_aux <= n_aux
    r = R1CS(n_inputs, n_aux, n_bool=n_bool)
    V = lambda aux_idx: n_inputs + aux_idx
    coeff = lambda: rng.fr() if rng.below(4) == 0 else 1 + rng.below(3)
    for x in range(n_bool):
        r.A.append([(V(x), 1)]); r.B.append([(0, 1), (V(x), R - 1)]); r.C.append([])
    for w in range(n_bool, n_aux):
        rowa = [(1 + rng.below(n_inputs - 1), 1 + rng.below(5))]          # a public input in A
        rowb = [(rng.below(nb_in), 1 + rng.below(5))]                     # ONE / input in B
        if w - 1 < a_aux_density:
            rowa.append((V(w - 1), coeff()))
        if w - 1 < nb_aux:
            rowb.append((V(w - 1), coeff()))
        for _ in range(2):
            rowa.append((V(rng.below(min(w, a_aux_density))), coeff()))
        rowb.append((V(rng.below(min(w, nb_aux))), coeff()))
        r.A.append(rowa); r.B.append(rowb); r.C.append([(V(w), 1)])
    k = 0
    while r.n_constraints < n_constraints:
        x = k % n_bool; k += 1
        r.A.append([(V(x), 1)]); r.B.append([(0, 1), (V(x), R - 1)]); r.C.append([])
    return r


def densities(r: R1CS):
    a_aux = np.zeros(r.n_aux, np.uint8); b_in = np.zeros(r.n_inputs, np.uint8); b_aux = np.zeros(r.n_aux, np.uint8)
    for row in r.A:
        for v, _ in row:
            if v >= r.n_inputs:
                a_aux[v - r.n_inputs] = 1
    for row in r.B:
        for v, _ in row:
            if v >= r.n_inputs:
                b_aux[v - r.n_inputs] = 1
            else:
                b_in[v] = 1
    return a_aux, b_in, b_aux


def make_witness(r: R1CS, seed=1, inputs=None):
    """Full assignment z = (inputs | aux) satisfying r; returns python ints.  inputs: the n_inputs - 1 public inputs after
    ONE (random when None)."""
    rng = SplitMix64(seed ^ 0xabcdef)
    z = [0] * (r.n_inputs + r.n_aux)
    z[0] = 1
    for i in range(1, r.n_inputs):
        z[i] = rng.fr()
    if inputs is not None:
        assert len(inputs) == r.n_inputs - 1
        z[1:r.n_inputs] = [int(v) % R for v in inputs]
    for x in range(r.n_bool):
        z[r.n_inputs + x] = rng.next() & 1
    dot = lambda row: sum(c * z[v] for v, c in row) % R
    for j in range(r.n_bool, r.n_aux):
        z[r.n_inputs + j] = dot(r.A[j]) * dot(r.B[j]) % R
    return z


def evaluate(r: R1CS, z):
    """Per-constraint evaluations <A_j,z>, <B_j,z>, <C_j,z> followed by the n_inputs rows
    `input_i * 0 = 0` that create_proof appends (SURVEY.md §3.2)."""
    dot = lambda row: sum(c * z[v] for v, c in row) % R
    a = [dot(x) for x in r.A] + [z[i] for i in range(r.n_inputs)]
    b = [dot(x) for x in r.B] + [0] * r.n_inputs
    c = [dot(x) for x in r.C] + [0] * r.n_inputs
    return a, b, c


def _lagrange_at(tau, log_m, count):
    m = 1 << log_m
    w = pow(_ROOT, 1 << (32 - log_m), R)
    zt = (pow(tau, m, R) - 1) % R
    minv = pow(m, -1, R)
    out, wj = [], 1
    for _ in range(count):
        out.append(zt * minv % R * wj % R * pow((tau - wj) % R, -1, R) % R)
        wj = wj * w % R
    return out, zt


@dataclass
class ToyCRS:
    params_bytes: bytes
    trapdoor: dict
    at: list
    bt: list
    ct: list
    zt: int
    log_m: int
    r1cs: R1CS


def _enc_fq(limbs6) -> bytes:
    """Montgomery limbs -> canonical 48-byte big-endian (host-side, python ints)."""
    q = 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab
    v = sum(int(x) << (64 * i) for i, x in enumerate(limbs6))
    return (v * _enc_fq.rinv % q).to_bytes(48, "big")


_enc_fq.rinv = pow(1 << 384, -1, 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab)


def g1_limbs_to_uncompressed(p) -> bytes:
    p = np.asarray(p, np.uint64).reshape(12)
    if not p.any():
        return bytes([0x40]) + bytes(95)
    return _enc_fq(p[:6]) + _enc_fq(p[6:])


def g2_limbs_to_uncompressed(p) -> bytes:
    p = np.asarray(p, np.uint64).reshape(24)
    if not p.any():
        return bytes([0x40]) + bytes(191)
    return _enc_fq(p[6:12]) + _enc_fq(p[0:6]) + _enc_fq(p[18:24]) + _enc_fq(p[12:18])


def make_toy_crs(r: R1CS, gen_g1, gen_g2, seed=7) -> ToyCRS:
    rng = SplitMix64(seed)
    tau, alpha, beta, gamma, delta = (rng.fr() or 1 for _ in range(5))
    n_rows = r.n_constraints + r.n_inputs
    log_m = max(1, (n_rows - 1).bit_length())
    m = 1 << log_m
    L, zt = _lagrange_at(tau, log_m, n_rows)
    nv = r.n_inputs + r.n_aux
    at, bt, ct = [0] * nv, [0] * nv, [0] * nv
    for j in range(r.n_constraints):
        for v, c in r.A[j]:
            at[v] = (at[v] + c * L[j]) % R
        for v, c in r.B[j]:
            bt[v] = (bt[v] + c * L[j]) % R
        for v, c in r.C[j]:
            ct[v] = (ct[v] + c * L[j]) % R
    for i in range(r.n_inputs):
        at[i] = (at[i] + L[r.n_constraints + i]) % R
    a_aux_d, b_in_d, b_aux_d = densities(r)
    ginv, dinv = pow(gamma, -1, R), pow(delta, -1, R)
    comb = lambda i: (beta * at[i] + alpha * bt[i] + ct[i]) % R
    ic_s = [comb(i) * ginv % R for i in range(r.n_inputs)]
    l_s = [comb(r.n_inputs + i) * dinv % R for i in range(r.n_aux)]
    h_s, t = [], zt * dinv % R
    for _ in range(m - 1):
        h_s.append(t); t = t * tau % R
    a_s = [at[i] for i in range(r.n_inputs)] + [at[r.n_inputs + i] for i in range(r.n_aux) if a_aux_d[i]]
    b_s = [bt[i] for i in range(r.n_inputs) if b_in_d[i]] + [bt[r.n_inputs + i] for i in range(r.n_aux) if b_aux_d[i]]
    g1_s = [alpha, beta, delta] + ic_s + h_s + l_s + a_s + b_s
    g2_s = [beta, gamma, delta] + b_s
    P1 = gen_g1(ints_to_limbs(g1_s))
    P2 = gen_g2(ints_to_limbs(g2_s))
    e1 = [g1_limbs_to_uncompressed(p) for p in P1]
    e2 = [g2_limbs_to_uncompressed(p) for p in P2]
    out = bytearray()
    out += e1[0] + e1[1] + e2[0] + e2[1] + e1[2] + e2[2]
    off = 3
    for n in (len(ic_s), len(h_s), len(l_s), len(a_s), len(b_s)):
        out += struct.pack(">I", n) + b"".join(e1[off:off + n]); off += n
    out += struct.pack(">I", len(b_s)) + b"".join(e2[3:])
    td = dict(tau=tau, alpha=alpha, beta=beta, gamma=gamma, delta=delta)
    return ToyCRS(bytes(out), td, at, bt, ct, zt, log_m, r)


def expected_proof_scalars(crs: ToyCRS, z, r: int, s: int):
    """Closed-form discrete logs (A, B, C) of the proof for satisfying assignment z and randomness r, s."""
    td = crs.trapdoor
    n_in = crs.r1cs.n_inputs
    za = sum(zi * a for zi, a in zip(z, crs.at)) % R
    zb = sum(zi * b for zi, b in zip(z, crs.bt)) % R
    zc = sum(zi * c for zi, c in zip(z, crs.ct)) % R
    dinv = pow(td["delta"], -1, R)
    A = (td["alpha"] + za + r * td["delta"]) % R
    B = (td["beta"] + zb + s * td["delta"]) % R
    laux = sum(z[i] * (td["beta"] * crs.at[i] + td["alpha"] * crs.bt[i] + crs.ct[i]) for i in range(n_in, len(z))) % R
    ht = (za * zb - zc) % R          # = h(tau) * t(tau) for a satisfying witness
    C = ((laux + ht) * dinv + A * s + B * r - r * s % R * td["delta"]) % R
    return A, B, C
