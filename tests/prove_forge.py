"""Forged-witness corpus of the Groth16 prover (zero_chain_b200/csrc/groth16.cu, ntt.cu).

The toy CRS (zero_chain_b200/synthetic.py) hands out its trapdoor, so for a satisfying witness z the discrete log of every
intermediate group element of create_proof is known (za, zb, zc, laux as in synthetic.expected_proof_scalars,
ht = za zb - zc = h(tau) t(tau)):

    A  = alpha + za + r delta        B (= B1 in G1, B in G2) = beta + zb + s delta
    T0 = s A      T1 = r B      H' = ht / delta - r s delta      L = laux / delta
    C  = T0 + T1 + H' + L        (k_finish_proofs: c = T0; c += T1; c += H'; c += L)

Each degenerate relation below is linear in r once s is fixed (B = O is linear in s), so the builders solve for the blinding
scalars that put one of XYZZ::add's exceptional branches, or a proof point at infinity, on a chosen step; `finish_steps`
names the branch each of the three additions of g_c takes, so a test states its branch before it runs.  The GLV scalar
set drives the split k = k1 u^2 + k0 of k_scale_points (glv_split.cuh) through its edges, and the circuit builders reach the
density corners in which the prover skips its gathers.

The constants are copies of the kernels' constants; tests/test_oracle_prove_edges.py reads each out of the CUDA sources and
fails when one moves.  Plain Python on the C oracle's fixed-base multiplication; no GPU."""
from oracle import coracle as co
from zero_chain_b200 import synthetic as sy

R = sy.R

# copies of the kernels' constants (checked against the sources by test_oracle_prove_edges.py)
PROVE_CHUNK = 256                 # groth16.cu: proofs per slice of zk_groth16_prove_batch
FINISH_BLOCK = 32                 # groth16.cu: proofs per block of k_finish_proofs (three warps, one lane per proof)
SCALE_T = 64                      # groth16.cu: threads per block of k_scale_points
GLV_TOP = 127                     # groth16.cu: highest bit of the GLV doubling chain
MAX_TILE_LOG = 11                 # ntt.cu: one shared-memory tile; two passes up to 2^22, three above
U2_WORDS = (0x00000000, 0x00000001, 0x0001A402, 0xAC45A401)      # glv_split.cuh: u^2, little-endian 32-bit words

U = 0xD201000000010000
U2 = U * U
assert U2 == sum(w << (32 * i) for i, w in enumerate(U2_WORDS)) and R == U2 * U2 - U2 + 1

# ---- the GLV split -------------------------------------------------------------------------------------------------------
GLV_EDGES = {
    "u2-1": U2 - 1, "u2": U2, "u2+1": U2 + 1,
    "r-1": R - 1,                 # k0 = 0, k1 = u^2 - 1 (bit 127 set)
    "r-2": R - 2,                 # k0 = u^2 - 1, k1 = u^2 - 2
    "2^127": 1 << 127, "2^128": 1 << 128, "2^254": 1 << 254,
    "(r-1)/2": (R - 1) // 2, "2u2": 2 * U2, "2^128+u2": (1 << 128) + U2, "r-u2": R - U2,
}


def glv_split(k):
    """(k0, k1) with k = k1 u^2 + k0, k0 < u^2: what split_u2 must return"""
    k1, k0 = divmod(k, U2)
    return k0, k1


def chain_bits(k, glv):
    """the highest bit index of the doubling chain that k_scale_points needs for k (-1 for k = 0)"""
    if not glv:
        return k.bit_length() - 1
    k0, k1 = glv_split(k)
    return max(k0.bit_length(), k1.bit_length()) - 1


# ---- the intermediates of create_proof -------------------------------------------------------------------------------------
def _inv(x):
    x %= R
    assert x, "the relation does not determine the scalar: zero denominator"
    return pow(x, -1, R)


def witness_scalars(crs, z):
    """za, zb, zc, laux and ht of a full assignment z (ONE | inputs | aux)"""
    td, n_in = crs.trapdoor, crs.r1cs.n_inputs
    za = sum(zi * a for zi, a in zip(z, crs.at)) % R
    zb = sum(zi * b for zi, b in zip(z, crs.bt)) % R
    zc = sum(zi * c for zi, c in zip(z, crs.ct)) % R
    laux = sum(z[i] * (td["beta"] * crs.at[i] + td["alpha"] * crs.bt[i] + crs.ct[i]) for i in range(n_in, len(z))) % R
    return dict(za=za, zb=zb, zc=zc, laux=laux, ht=(za * zb - zc) % R)


def intermediates(crs, w, r, s):
    """discrete logs of A, B, T0, T1, H', L, C for witness scalars w (witness_scalars) and blinding r, s"""
    td = crs.trapdoor
    d, dinv = td["delta"], _inv(td["delta"])
    A = (td["alpha"] + w["za"] + r * d) % R
    B = (td["beta"] + w["zb"] + s * d) % R
    T0, T1 = s * A % R, r * B % R
    H = (w["ht"] * dinv - r * s % R * d) % R
    L = w["laux"] * dinv % R
    return dict(A=A, B=B, T0=T0, T1=T1, H=H, L=L, C=(T0 + T1 + H + L) % R)


SKIP, ENTER, DOUBLE, CANCEL, GENERIC = "skip", "enter", "double", "cancel", "generic"


def _step(acc, t):
    if t == 0:
        return SKIP
    if acc == 0:
        return ENTER
    if t == acc:
        return DOUBLE
    if (t + acc) % R == 0:
        return CANCEL
    return GENERIC


def finish_steps(iv):
    """the branch of XYZZ::add that each addition of g_c = T0 + T1 + H' + L takes in k_finish_proofs"""
    acc, steps = iv["T0"], []
    for t in (iv["T1"], iv["H"], iv["L"]):
        steps.append(_step(acc, t))
        acc = (acc + t) % R
    return steps


def infinities(iv):
    """which proof points are the point at infinity"""
    return tuple(k for k in ("A", "B", "C") if iv[k] == 0)


# ---- blinding scalars that reach a named branch ------------------------------------------------------------------------------
def _ab0(crs, w):
    td = crs.trapdoor
    return (td["alpha"] + w["za"]) % R, (td["beta"] + w["zb"]) % R


def solve(crs, w, case, s=0x5EED5):
    """(r, s) for a named case.  Every relation except B = O is linear in r for the given s; the model asserts that its
    coefficient is non-zero.  Returns the scalars reduced mod r."""
    td = crs.trapdoor
    d, dinv = td["delta"], _inv(td["delta"])
    a0, b0 = _ab0(crs, w)
    ht, laux = w["ht"], w["laux"]
    s %= R
    if case in ("B=O", "A=O,B=O"):
        s = -b0 * dinv % R
    if case in ("A=O", "A=O,B=O"):
        return -a0 * dinv % R, s
    if case == "B=O":
        return 0xB10B, s
    if case == "T0=T1":                       # s a0 = r b0  (the r s delta of A s and B r cancel)
        return s * a0 * _inv(b0) % R, s
    if case == "T0=-T1":                      # s a0 + r (b0 + 2 s delta) = 0
        return -s * a0 * _inv(b0 + 2 * s * d) % R, s
    if case == "T0+T1=H'":                    # s a0 + r (b0 + 2 s delta) = ht/delta - r s delta
        return (ht * dinv - s * a0) * _inv(b0 + 3 * s * d) % R, s
    if case == "T0+T1=-H'":
        return (-ht * dinv - s * a0) * _inv(b0 + s * d) % R, s
    if case == "T0+T1+H'=L":                  # s a0 + r (b0 + s delta) + ht/delta = laux/delta: C = 2L
        return ((laux - ht) * dinv - s * a0) * _inv(b0 + s * d) % R, s
    if case == "T0+T1+H'=-L":                 # C = O
        return (-(laux + ht) * dinv - s * a0) * _inv(b0 + s * d) % R, s
    if case == "H'=O":                        # ht/delta = r s delta
        return ht * _inv(s * d * d) % R, s
    if case == "r=0":
        return 0, s
    if case == "s=0":
        return 0x7A11, 0
    raise KeyError(case)


BLINDING_CASES = ["A=O", "B=O", "A=O,B=O", "T0=T1", "T0=-T1", "T0+T1=H'", "T0+T1=-H'", "T0+T1+H'=L", "T0+T1+H'=-L", "H'=O",
                  "r=0", "s=0"]


def expected_reach(case):
    """the points at infinity and the (step, branch) pairs of finish_steps that a named case must produce.  Step 0 is
    T0 + T1, step 1 adds H', step 2 adds L."""
    if case == "A=O":                         # T0 = s O = O: the sum enters from O at T1
        return ("A",), [(0, ENTER)]
    if case == "B=O":                         # T1 = r O = O is skipped
        return ("B",), [(0, SKIP)]
    if case == "A=O,B=O":
        return ("A", "B"), [(0, SKIP), (1, ENTER)]
    if case == "T0=T1":
        return (), [(0, DOUBLE)]
    if case == "T0=-T1":
        return (), [(0, CANCEL), (1, ENTER)]
    if case == "T0+T1=H'":
        return (), [(1, DOUBLE)]
    if case == "T0+T1=-H'":
        return (), [(1, CANCEL), (2, ENTER)]
    if case == "T0+T1+H'=L":
        return (), [(2, DOUBLE)]
    if case == "T0+T1+H'=-L":
        return ("C",), [(2, CANCEL)]
    if case == "H'=O":
        return (), [(1, SKIP)]
    if case == "r=0":                         # T1 = 0 B
        return (), [(0, SKIP)]
    if case == "s=0":                         # T0 = 0 A: the sum enters from O at T1
        return (), [(0, ENTER)]
    raise KeyError(case)


def glv_blindings():
    """(name, r, s): every GLV edge as r and as s, the other scalar a plain one"""
    out = []
    for name, k in GLV_EDGES.items():
        out.append(("r=" + name, k, 0x51DE))
        out.append(("s=" + name, 0x51DE, k))
    return out


# ---- witnesses and circuits --------------------------------------------------------------------------------------------------
def zero_witness(r1cs):
    """z = e_0: ONE and nothing else.  It satisfies every make_r1cs circuit (each product row has a zero factor) and the
    builders below, and gives L = O."""
    return [1] + [0] * (r1cs.n_inputs + r1cs.n_aux - 1)


def check_witness(r1cs, z):
    dot = lambda row: sum(c * z[v] for v, c in row) % R
    return all(dot(a) * dot(b) % R == dot(c) for a, b, c in zip(r1cs.A, r1cs.B, r1cs.C))


def _R1(n_in, n_aux, rows, n_bool=0):
    r = sy.R1CS(n_in, n_aux, n_bool=n_bool)
    for a, b, c in rows:
        r.A.append(list(a)); r.B.append(list(b)); r.C.append(list(c))
    return r


def circuit_m2():
    """one constraint x * ONE = x: ONE is the only input, one aux; n_c + n_in = 2, the smallest domain (2^1)"""
    return _R1(1, 1, [([(1, 1)], [(0, 1)], [(1, 1)])])


def circuit_no_aux_in_a(n_aux=6):
    """A rows hold inputs only: c_j ONE * (x_j + input1) = c_j x_j + c_j input1.  The A-query gather is skipped."""
    V = lambda j: 2 + j
    return _R1(2, n_aux, [([(0, 3 + j)], [(V(j), 1), (1, 1)], [(V(j), 3 + j), (1, 3 + j)]) for j in range(n_aux)])


def circuit_no_input_in_b(n_aux=6):
    """B rows hold aux only: x_1 = input1 x_0, then x_{j+1} = x_j^2.  The B-input gather is skipped."""
    V = lambda j: 2 + j
    rows = [([(1, 1)], [(V(0), 1)], [(V(1), 1)])]
    rows += [([(V(j), 1)], [(V(j), 1)], [(V(j + 1), 1)]) for j in range(1, n_aux - 1)]
    return _R1(2, n_aux, rows)


def circuit_no_aux_in_b(n_aux=6):
    """B rows hold inputs only: x_j * (input1 + 2 ONE) = y_j, the y_j only in C.  The B-aux gather is skipped."""
    V = lambda j: 2 + j
    half = n_aux // 2
    return _R1(2, n_aux, [([(V(j), 1)], [(1, 1), (0, 2)], [(V(half + j), 1)]) for j in range(half)])


def circuit_all_aux_in_ab(n_aux=7, n_rows=None):
    """x (ONE - x) = 0 for every aux (booleans, as in make_r1cs): every aux is in A and in B.  n_rows: repeat the boolean
    rows up to that many constraints, to pin n_c + n_in on a power of two or one above it."""
    V = lambda j: 2 + j
    n_rows = n_rows or n_aux
    rows = [([(V(j % n_aux), 1)], [(0, 1), (V(j % n_aux), R - 1)], []) for j in range(n_rows)]
    return _R1(2, n_aux, rows, n_bool=n_aux)


def circuit_pow2(log_m, above=False):
    """booleans with n_c + n_in = 2^log_m exactly, or 2^log_m + 1 (the next domain)"""
    n_rows = (1 << log_m) + (1 if above else 0) - 2
    return circuit_all_aux_in_ab(n_aux=min(7, n_rows), n_rows=n_rows)


def circuit_witness_corners(n_aux=6):
    """what zk_r1cs_load must take as it is: rows with no terms at all (0 * 0 = 0), a column repeated within a row, the
    coefficient r - 1, and the last variable index (the last aux) in every matrix."""
    V = lambda j: 2 + j
    last = V(n_aux - 1)
    rows = [
        ([], [], []),                                                                # empty row
        ([(V(0), 1), (V(0), 2)], [(0, 1)], [(V(0), 3)]),                             # 3 x0 = 3 x0, column repeated in A
        ([(V(1), R - 1)], [(V(1), 1), (0, 0)], [(V(2), R - 1)]),                     # -(x1 x1) = -x2, coefficient r - 1, zero coeff
        ([(V(2), 1)], [(1, 1), (1, 1)], [(V(3), 1)]),                                # x2 * 2 in1 = x3, input repeated in B
        ([(V(3), 1)], [(last, 1)], [(V(4), 1)]),                                     # x3 x_last = x4
        ([(last, 1)], [(0, 1)], [(last, 1)]),                                        # last variable in A, B (via row 4) and C
        ([], [(V(0), 1)], []),                                                       # empty A: 0 * x0 = 0
    ]
    return _R1(2, n_aux, rows)


def witness_for(r1cs, seed=1):
    """a satisfying assignment of the hand-written circuits above: the free variables random, the rest propagated"""
    rng = sy.SplitMix64(seed ^ 0x5A5A)
    nv = r1cs.n_inputs + r1cs.n_aux
    z = [1] + [rng.fr() for _ in range(nv - 1)]
    if r1cs.n_bool:
        for j in range(r1cs.n_aux):
            z[r1cs.n_inputs + j] = rng.next() & 1
    dot = lambda row: sum(c * z[v] for v, c in row) % R
    for _ in range(len(r1cs.A) + 1):          # propagate: a C row with one term defines its variable
        for a, b, c in zip(r1cs.A, r1cs.B, r1cs.C):
            if len(c) == 1 and c[0][0] >= r1cs.n_inputs:
                v, k = c[0]
                z[v] = dot(a) * dot(b) * _inv(k) % R
    assert check_witness(r1cs, z)
    return z


def circuit_dense(n_rows):
    """n_rows = n_c + 2 constraint rows (two inputs), none empty, so A, B and C are dense on the domain:
    row 0: x * ONE = x, rows 1..: x * x = y.  The CRS needs only the Lagrange sum over the rows (toy_crs_dense)."""
    n_c = n_rows - 2
    assert n_c >= 2
    rows = [([(2, 1)], [(0, 1)], [(2, 1)])] + [([(2, 1)], [(2, 1)], [(3, 1)])] * (n_c - 1)
    return _R1(2, 2, rows)


def witness_dense(seed):
    x = sy.SplitMix64(seed).fr()
    return [1, sy.SplitMix64(seed + 1).fr(), x, x * x % R]


def dense_tables(n_c, lag_sum, lag):
    """at, bt, ct of circuit_dense from S = sum_{j < n_c} L_j(tau) and L_j(tau) for j in (0, n_c, n_c + 1)"""
    at = [lag[n_c], lag[n_c + 1], lag_sum, 0]
    bt = [lag[0], 0, (lag_sum - lag[0]) % R, 0]
    ct = [0, 0, lag[0], (lag_sum - lag[0]) % R]
    return at, bt, ct


# ---- evaluations, densities and expected bytes -----------------------------------------------------------------------------
def assignment(r1cs, z):
    """the ProvingAssignment arrays (evaluations, inputs, aux, densities) of z, as C-oracle limbs"""
    a, b, c = sy.evaluate(r1cs, z)
    dens = sy.densities(r1cs)
    n_in = r1cs.n_inputs
    return (co.ints_to_limbs(a, 4), co.ints_to_limbs(b, 4), co.ints_to_limbs(c, 4),
            co.ints_to_limbs(z[:n_in], 4), co.ints_to_limbs(z[n_in:], 4)) + tuple(dens)


def proofs_from_scalars(triples):
    """Proof::write bytes of (A, B, C) discrete logs, many at once through the C oracle's fixed-base multiplication"""
    if not triples:
        return []
    g1 = co.g1_fixed_base(co.ints_to_limbs([x % R for t in triples for x in (t[0], t[2])], 4))
    g2 = co.g2_fixed_base(co.ints_to_limbs([t[1] % R for t in triples], 4))
    out = []
    for i in range(len(triples)):
        out.append(co.g1_encode(g1[2 * i], True) + co.g2_encode(g2[i], True) + co.g1_encode(g1[2 * i + 1], True))
    return out


def closed_form(crs, z, r, s):
    """the proof bytes create_proof must return, from the trapdoor alone"""
    iv = intermediates(crs, witness_scalars(crs, z), r, s)
    return proofs_from_scalars([(iv["A"], iv["B"], iv["C"])])[0]
