"""Forged-proof corpus of the batched Groth16 verifier (zero_chain_b200/csrc/pairing.cu, pairing_lanes.cu).

A toy CRS (zero_chain_b200/synthetic.py) hands out its trapdoor, so the discrete log k_j of every ic_j is known and a proof
that verifies can be written down for ANY public inputs, without a witness:

    e(A, B) = e(alpha, beta) e(acc, gamma) e(C, delta),   acc = ic_0 + sum_j x_j ic_j = s G1,   s = k_0 + sum_j x_j k_j
    A = a G1, B = b G2, C = c G1   verifies   <=>   a b = alpha beta + s gamma + c delta   (mod r)

That turns the verifier's exceptional branches into expected verdicts of 1: the builders below solve for public inputs
that make a term of the public-input sum equal the running sum (XYZZ::add's doubling branch), cancel it (the point at
infinity in the middle of the sum, then the entry from infinity), make the whole sum the point at infinity (the Miller
loop must skip the (acc, -gamma) pair), or fetch one chosen row of the per-key window table d * 2^(8w) * ic_j.  A small
model of the sum (`sum_steps`) names the branch each row reaches, so a test states its branch before it runs and a change
of the toy key's seed cannot move a case off its branch unnoticed.

The constants are copies of the kernels' constants; tests/test_oracle_verify_edges.py reads each out of the CUDA sources
and fails when one moves.  Plain Python on the C oracle's fixed-base multiplication and point encoders; no GPU."""
from oracle import coracle as co
from zero_chain_b200 import synthetic as sy

R = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001

# copies of the kernels' constants (checked against the sources by test_oracle_verify_edges.py)
IC_WIN = 32                       # pairing.cu: 8-bit windows of a public input
IC_DIG = 255                      # pairing.cu: table rows per window, d = 1..255
PAIRING_BLOCK = 64                # pairing.cu: PT, threads per block of the thread-per-item kernels
VERIFY_CHUNK = 1 << 18            # pairing.cu: proofs per slice of zk_groth16_verify_batch
GROUPS_PER_WARP = 5               # pairing_lanes.cuh: proofs per warp of the lane kernels (lanes 30, 31 shadow group 4)
LANES_BLOCK = 128                 # pairing_lanes.cu: threads per block of k_miller_lanes / k_verify_final_lanes
PROOFS_PER_BLOCK = LANES_BLOCK // 32 * GROUPS_PER_WARP
N_COEFFS = 68                     # pairing.cuh: line coefficients of one G2Prepared


A_S, B_S = 0x1234567, 0x89ABCDE          # a, b of the forged proofs: A and B are shared by a whole corpus, only C varies


class ToyKey:
    """A toy CRS of n_inputs - 1 public inputs with the discrete logs of its ic, prepared in the C oracle."""

    def __init__(self, n_inputs=4, seed=3):
        self.r1cs = sy.make_r1cs(n_constraints=56 + n_inputs, n_inputs=n_inputs, n_aux=50, a_aux_density=40, b_density=33, seed=seed)
        self.crs = sy.make_toy_crs(self.r1cs, co.g1_fixed_base, co.g2_fixed_base, seed=seed + 1)
        self.k = ic_scalars(self.crs)
        self.n = n_inputs - 1
        self.opvk = co.PreparedVerifyingKey.prepare(self.crs.params_bytes)

    def oracle(self, proofs, rows, opvk=None):
        """the C oracle's verdicts"""
        return (opvk or self.opvk).verify_batch(b"".join(proofs), co.ints_to_limbs([x for row in rows for x in row], 4), self.n)


def _inv(x):
    return pow(x % R, -1, R)


def ic_scalars(crs) -> list:
    """k_i with ic_i = k_i G1: (beta at_i + alpha bt_i + ct_i) / gamma for the ONE wire and every public input."""
    td = crs.trapdoor
    ginv = _inv(td["gamma"])
    return [(td["beta"] * crs.at[i] + td["alpha"] * crs.bt[i] + crs.ct[i]) * ginv % R for i in range(crs.r1cs.n_inputs)]


def public_sum(k, row) -> int:
    """s with ic_0 + sum_j row[j] ic_{j+1} = s G1"""
    assert len(row) + 1 == len(k)
    return (k[0] + sum(x * kj for x, kj in zip(row, k[1:]))) % R


def forge(crs, row, a, b, skip_gamma=False, skip_delta=False, c=1, k=None):
    """Scalars (a, b, c) of a proof A = a G1, B = b G2, C = c G1 that verifies for the public inputs `row`.
    skip_gamma / skip_delta: for a key whose prepared -gamma / -delta carries the infinity flag, so that the verifier drops
    that pairing.  With delta dropped C is free (the caller's c is kept) and b is solved for instead of c.
    k: ic_scalars(crs), when the caller already has them."""
    td = crs.trapdoor
    rhs = td["alpha"] * td["beta"] % R
    if not skip_gamma:
        rhs = (rhs + public_sum(k or ic_scalars(crs), row) * td["gamma"]) % R
    if skip_delta:
        assert a % R and rhs and c % R
        return a, rhs * _inv(a) % R, c
    c = (a * b - rhs) * _inv(td["delta"]) % R
    assert a % R and b % R and c, "pick other a, b: the proof would hold a point at infinity"
    return a, b, c


def holds(crs, row, a, b, c, skip_gamma=False, skip_delta=False) -> int:
    """The verdict the pairing equation gives the proof (a G1, b G2, c G1) for `row`, from the trapdoor alone: the pairing
    is non-degenerate, so the equation holds in GT exactly when it holds for the discrete logs."""
    td = crs.trapdoor
    rhs = td["alpha"] * td["beta"]
    if not skip_gamma:
        rhs += public_sum(ic_scalars(crs), row) * td["gamma"]
    if not skip_delta:
        rhs += c * td["delta"]
    return int((a * b - rhs) % R == 0)


# ---- the reach model of k_ic_sum ---------------------------------------------------------------------------------------
SKIP, ENTER, DOUBLE, CANCEL, GENERIC = "skip", "enter", "double", "cancel", "generic"


def sum_steps(k, row):
    """Branch of XYZZ::add that each step `acc += x_j ic_j` of k_ic_sum takes, and whether the final sum is the point at
    infinity: SKIP (the term is O: x_j = 0), ENTER (acc is O), DOUBLE (term == acc), CANCEL (term == -acc), GENERIC."""
    assert all(kj % R for kj in k), "an ic element at infinity"
    acc, steps = k[0] % R, []
    for x, kj in zip(row, k[1:]):
        t = x * kj % R
        if t == 0:
            steps.append(SKIP)
        elif acc == 0:
            steps.append(ENTER)
        elif t == acc:
            steps.append(DOUBLE)
        elif (t + acc) % R == 0:
            steps.append(CANCEL)
        else:
            steps.append(GENERIC)
        acc = (acc + t) % R
    return steps, acc == 0


def window_digits(x) -> list:
    """the IC_WIN base-256 digits of a public input, lowest window first; k_ic_partial skips the zero ones"""
    return [(x >> (8 * w)) & 0xFF for w in range(IC_WIN)]


# ---- rows that reach a named branch ------------------------------------------------------------------------------------
def _random_row(k, rng):
    return [rng.fr() or 1 for _ in k[1:]]


def mid_sum_infinity(k, rng, j=1):
    """Input j (1-based, as ic_j) cancels the running sum: acc is O after step j and step j + 1 enters from O."""
    row = _random_row(k, rng)
    row[j - 1] = -public_sum(k[:j], row[:j - 1]) * _inv(k[j]) % R
    return row, "mid_sum_infinity@%d" % j


def sum_doubling(k, rng, j=2):
    """Input j's term equals the running sum: step j is a doubling."""
    row = _random_row(k, rng)
    row[j - 1] = public_sum(k[:j], row[:j - 1]) * _inv(k[j]) % R
    return row, "sum_doubling@%d" % j


def total_infinity(k, rng, prefix=None):
    """The whole sum is the point at infinity: the last input cancels it.  prefix = "cancel": input 1 already cancels ic_0
    and the rest sums to O again; prefix = "zeros": input 1 cancels ic_0 and every later input is zero."""
    row = _random_row(k, rng)
    if prefix is not None:
        row[0] = -k[0] * _inv(k[1]) % R
    if prefix == "zeros":
        row[1:] = [0] * (len(row) - 1)
        return row, "total_infinity/zeros"
    n = len(row)
    row[n - 1] = -public_sum(k[:n], row[:n - 1]) * _inv(k[n]) % R
    return row, "total_infinity" + ("/" + prefix if prefix else "")


def zero_terms(k, rng):
    """Rows whose terms are skipped: all inputs zero, each single input zero, and inputs with zero bytes in chosen windows
    (window 0, the top window, every other window, all but one window)."""
    n = len(k) - 1
    out = [([0] * n, "zero_terms/all")]
    for j in range(n):
        row = _random_row(k, rng)
        row[j] = 0
        out.append((row, "zero_terms/input%d" % (j + 1)))
    odd = sum(0xA5 << (8 * w) for w in range(1, IC_WIN - 1, 2))
    shapes = [(rng.fr() >> 8 << 8) or 256, rng.fr() & ((1 << 248) - 1) or 1, odd, 0x5A << (8 * 17), 1, 1 << 248]
    for i in range(0, len(shapes), n):
        row = (shapes[i:i + n] + [3] * n)[:n]
        out.append((row, "zero_terms/windows%d" % (i // n)))
    return out


def table_sweep(k, j, fixed=7):
    """Every row of input j's window table: x_j = d << (8 w) for d = 1..255, w = 0..31 below r (the top window stops at
    0x73), then r - 1 and the value with 0xff in all 31 lower windows; the other inputs are `fixed`.
    Returns [(row, (j, w, d))]; w = -1 marks the two extra values."""
    n = len(k) - 1
    out = []
    for w in range(IC_WIN):
        for d in range(1, IC_DIG + 1):
            x = d << (8 * w)
            if x < R:
                row = [fixed] * n
                row[j - 1] = x
                out.append((row, (j, w, d)))
    for i, x in enumerate((R - 1, (0x72 << 248) | ((1 << 248) - 1))):
        row = [fixed] * n
        row[j - 1] = x
        out.append((row, (j, -1, i)))
    return out


def named_rows(k, rng):
    """Every degenerate row of a key with at least three public inputs, with the steps the model must report for it."""
    n = len(k) - 1
    assert n >= 3
    rows = [mid_sum_infinity(k, rng, 1), mid_sum_infinity(k, rng, 2), sum_doubling(k, rng, 1), sum_doubling(k, rng, 2),
            sum_doubling(k, rng, n), total_infinity(k, rng), total_infinity(k, rng, "cancel"), total_infinity(k, rng, "zeros")]
    return rows + zero_terms(k, rng)


def expected_reach(name, n):
    """(index of the step, its branch) pairs and the final-sum flag that `sum_steps` must report for a named row of n inputs"""
    kind, _, arg = name.partition("@")
    if kind == "mid_sum_infinity":
        j = int(arg)
        return [(j - 1, CANCEL)] + ([(j, ENTER)] if j < n else []), j == n
    if kind == "sum_doubling":
        return [(int(arg) - 1, DOUBLE)], False
    if name == "total_infinity":
        return [(n - 1, CANCEL)], True
    if name == "total_infinity/cancel":
        return [(0, CANCEL), (1, ENTER), (n - 1, CANCEL)], True
    if name == "total_infinity/zeros":
        return [(0, CANCEL)] + [(j, SKIP) for j in range(1, n)], True
    if name == "zero_terms/all":
        return [(j, SKIP) for j in range(n)], False
    if name.startswith("zero_terms/input"):
        return [(int(name[len("zero_terms/input"):]) - 1, SKIP)], False
    return [], False


# ---- points and proof bytes --------------------------------------------------------------------------------------------
def g1_compressed(scalars) -> list:
    pts = co.g1_fixed_base(co.ints_to_limbs([s % R for s in scalars], 4))
    return [co.g1_encode(p, True) for p in pts]


def g2_compressed(scalars) -> list:
    pts = co.g2_fixed_base(co.ints_to_limbs([s % R for s in scalars], 4))
    return [co.g2_encode(p, True) for p in pts]


def proofs_from_c(a, b, cs) -> list:
    """192-byte proofs (a G1, b G2, c G1) for every c: A and B are encoded once, the C points come from one fixed-base call"""
    head = g1_compressed([a])[0] + g2_compressed([b])[0]
    return [head + c for c in g1_compressed(cs)]


def proofs_for(crs, rows, a, b, skip_gamma=False):
    """One forged proof per row, all sharing A = a G1 and B = b G2: only C varies."""
    k = ic_scalars(crs)
    return proofs_from_c(a, b, [forge(crs, row, a, b, skip_gamma=skip_gamma, k=k)[2] for row in rows])


def proof_from_scalars(a, b, c) -> bytes:
    return g1_compressed([a])[0] + g2_compressed([b])[0] + g1_compressed([c])[0]


def g2_prepared_spans(image: bytes) -> list:
    """[(start, end)] of the two G2Prepared records (u32 count | count * 288 bytes | flag byte) of a
    PreparedVerifyingKey::write image: -gamma, then -delta"""
    spans, off = [], 576
    for _ in range(2):
        cnt = int.from_bytes(image[off:off + 4], "big")
        end = off + 4 + 288 * cnt + 1
        spans.append((off, end))
        off = end
    return spans


def flag_image(image: bytes, gamma=False, delta=False) -> bytes:
    """The image with the chosen G2Prepared records replaced by the prepared point at infinity as G2Prepared::from_affine
    makes it: no coefficients, infinity flag set."""
    (g0, g1), (d0, d1) = g2_prepared_spans(image)
    inf = bytes(4) + b"\x01"
    return image[:g0] + (inf if gamma else image[g0:g1]) + (inf if delta else image[d0:d1]) + image[d1:]


def flag_key_batch(crs, a, b, gamma, delta, seed=19):
    """(proofs, rows, verdicts, tags) for a key whose -gamma / -delta carry the infinity flag.  Three rows (a random one, one
    whose sum is O, all zero): the proof forged with the dropped terms for each, the first of those proofs against the other
    two rows (accepted when -gamma is dropped: the verdict no longer depends on the inputs), then the ordinary forged
    proofs.  The verdicts are those of the equation with the flagged pairings left out."""
    from oracle.pyref import SplitMix64
    rng = SplitMix64(seed)
    k = ic_scalars(crs)
    rows = [[rng.fr() for _ in k[1:]], total_infinity(k, rng)[0], [0] * (len(k) - 1)]
    abc = [forge(crs, row, a, b, skip_gamma=gamma, skip_delta=delta, c=0x5EED) for row in rows]
    abc += [abc[0], abc[0]] + [forge(crs, row, a, b) for row in rows]
    all_rows = rows + rows[1:] + rows
    tags = ["matching/%d" % i for i in range(3)] + ["matching/0 on row %d" % i for i in (1, 2)] + ["ordinary/%d" % i for i in range(3)]
    want = [holds(crs, row, *s, skip_gamma=gamma, skip_delta=delta) for s, row in zip(abc, all_rows)]
    return [proof_from_scalars(*s) for s in abc], all_rows, want, tags


def tamperings(crs, row, a, b, **skip):
    """The three ways a forged proof for `row` must be rejected, as (proof or None, inputs or None) replacements:
    one input + 1, C + G, and the proof forged for the neighbouring row (last input + 1)."""
    j = len(row) // 2
    bumped = list(row); bumped[j] = (bumped[j] + 1) % R
    near = list(row); near[-1] = (near[-1] + 1) % R
    fa, fb, fc = forge(crs, row, a, b, **skip)
    na, nb, nc = forge(crs, near, a, b, **skip)
    return [("input+1", None, bumped), ("C+G", proof_from_scalars(fa, fb, fc + 1), None),
            ("neighbour", proof_from_scalars(na, nb, nc), None)]
