"""MSM branches that uniform random scalars never reach, driven on purpose and checked bit-exactly.

Every case first asserts, through the reach model (tests/msm_reach.py), which branch of the sort, the batched-affine (BA)
rounds or the bucket reduction it takes, then compares the device result with the C oracle's multiexp or with the closed
form (sum s_i k_i) G over bases k_i G, and, where the window is wider than 16 bits, with the same MSM at 16-bit windows:
  - the three scatter modes of k_fine_sort (a whole bin straight to HBM, staged segments, a bucket larger than the window
    as a direct segment between staged ones) and the bin totals at their boundaries, with and without BA rounds;
  - BA rounds at 17..20-bit windows over doublings, cancellations, infinity operands, one coarse bin and zero scalars;
  - the production shape (2^20 terms, 20-bit windows, library defaults) on witness-like, constant and cancelling inputs;
  - G2 through the two-level sort, with and without BA rounds, and at 2^20 terms;
  - batched domains with tables on both sides of the switch to k_rowcol_sums (8 domains);
  - the order-3 G1 points (0, +-2), whose x = 0 makes the BA passes decide from the full points."""
import numpy as np
import pytest

from oracle import coracle as co
from oracle import pyref as pr
from tests import msm_reach as mr
from zero_chain_b200 import groth16 as zk
from zero_chain_b200 import synthetic as sy

pytestmark = pytest.mark.gpu

DEFAULT = (mr.BA_MIN_ENTRIES, -1)          # library defaults: BA rounds from 2^22 entries, count from the heuristic


def BA(levels):
    return (0, levels)                     # BA rounds forced on every MSM, `levels` of them


S = mr.FINE_STAGE


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


def _set(ctx, cfg):
    ctx.set_opt(zk.Context.OPT_AFFINE_MIN_ENTRIES, cfg[0])
    ctx.set_opt(zk.Context.OPT_AFFINE_LEVELS, cfg[1])


def _gen(group):
    return zk.G1_GENERATOR if group == 1 else zk.G2_GENERATOR


def _mult_bases(ctx, group, ks):
    """bases k_i G (G1) or k_i G2 for integer multipliers k_i (repeats computed once)"""
    ks = [int(k) % pr.R for k in ks]
    uniq = sorted(set(ks))
    pts = zk.scalar_mul_many(ctx, group, _gen(group), co.ints_to_limbs(uniq, 4))
    pos = {k: i for i, k in enumerate(uniq)}
    return np.ascontiguousarray(pts[[pos[k] for k in ks]])


def _ints(scal):
    s = np.ascontiguousarray(scal, np.uint64).reshape(-1, 4).astype(object)
    return s[:, 0] + (s[:, 1] << 64) + (s[:, 2] << 128) + (s[:, 3] << 192)


def _closed_form(group, ks, scal):
    k = int((_ints(scal) * np.array([int(x) for x in ks], dtype=object)).sum()) % pr.R
    if group == 1:
        return pr.g1_uncompressed(pr.ec_mul(pr.FQ, pr.G1_GEN, k))
    return pr.g2_uncompressed(pr.ec_mul(pr.FQ2, pr.G2_GEN, k))


def _oracle(group, bases, scal):
    if group == 1:
        return co.g1_encode(co.g1_msm(bases, scal), False)
    return co.g2_encode(co.g2_msm(bases, scal), False)


def _run(ctx, group, bases, scal, c, cfgs, tables=True):
    """one MSM per option set in cfgs over the same bases; c = 0 takes the library's window"""
    b = zk.Bases(ctx, group, bases, window_bits=c, precompute=tables)
    try:
        if c:
            assert b.window_bits == c
        out = []
        for cfg in cfgs:
            _set(ctx, cfg)
            out.append(zk.multiexp(b, scal))
        return b.window_bits, out
    finally:
        _set(ctx, DEFAULT)
        b.free()


def _usable_windows(c):
    """windows a positive digit can fill without carries while the scalar stays below 2^253 < r"""
    return sum(1 for w in range(mr.windows(c)) if c * (w + 1) <= 253)


def _scalars_from_keys(keys, c, seed):
    """scalars whose non-zero window digits are exactly key + 1 for every key given (one entry each, positive digits in
    [1, 2^(c-1)] so no carry moves them), spread over the points and windows in random order"""
    keys = np.random.default_rng(seed).permutation(np.asarray(keys, np.int64))
    U = _usable_windows(c)
    n = -(-len(keys) // U)
    pad = np.full(n * U, -1, np.int64)
    pad[:len(keys)] = keys
    dig = (pad + 1).reshape(n, U)
    vals = [sum(int(d) << (c * w) for w, d in enumerate(row) if d) for row in dig]
    assert max(vals) < pr.R
    return co.ints_to_limbs(vals, 4)


def _spread(rng, lo, hi, count):
    return rng.integers(lo, hi, size=count)


def _even(lo, nb, total):
    """total entries over buckets [lo, lo + nb) as evenly as possible"""
    per = np.full(nb, total // nb, np.int64)
    per[:total % nb] += 1
    return np.repeat(np.arange(lo, lo + nb), per)


# ---- 1. the scatter modes of k_fine_sort -------------------------------------------------------------------------
def _fine_layout(kind, c):
    low = c - 10
    B, top = 1 << low, 1 << (c - 1)
    rng = np.random.default_rng(c * 7 + len(kind))
    parts = []
    if kind == "direct_segment":
        # bin 0: a bucket over the window between non-empty buckets, bin total under FINE_MAX_SEGMENTS windows
        parts += [np.full(300, 2), np.full(S + 1000, B // 2), np.full(500, B - 3), _spread(rng, 0, B, 3000)]
        parts.append(_spread(rng, B, top, 20000))
    elif kind == "two_direct_segments":
        # bin 1: two adjacent buckets over the window, one direct segment after the other
        parts += [np.full(200, B + 1), np.full(S + 1, B + 3), np.full(S + 77, B + 4), np.full(100, 2 * B - 1), _spread(rng, B, 2 * B, 1000)]
        parts.append(_spread(rng, 2 * B, top, 20000))
    else:
        # bins 2..5: totals of exactly one window, one more, FINE_MAX_SEGMENTS windows, one more; bins 6 / 7: one bucket
        # of exactly the window / one more
        for b, total in ((2, S), (3, S + 1), (4, 4 * S), (5, 4 * S + 1)):
            parts.append(_even(b * B, B, total))
        parts += [np.full(S, 6 * B + 5), np.full(S + 1, 7 * B + 9)]
        parts.append(_spread(rng, 8 * B, top, 5000))
    return np.concatenate(parts)


def _check_fine_reach(kind, r):
    modes = r.fine[0]
    if kind == "direct_segment":
        assert modes[0] == "staged+direct" and r.bins[0, 0] <= mr.FINE_MAX_SEGMENTS * S
        segs = r.segments(0, 0)
        i = [k for k, sg in enumerate(segs) if sg[2]]
        assert len(i) == 1 and 0 < i[0] < len(segs) - 1
        sz = r.sizes[0]
        for lo, hi, _ in (segs[i[0] - 1], segs[i[0] + 1]):
            assert sz[lo:hi].sum() > 0                     # non-empty staged segments before and after the direct one
    elif kind == "two_direct_segments":
        assert modes[1] == "staged+direct"
        segs = r.segments(0, 1)
        assert any(a[2] and b[2] for a, b in zip(segs, segs[1:]))
    else:
        assert list(r.bins[0, 2:8]) == [S, S + 1, 4 * S, 4 * S + 1, S, S + 1]
        assert modes[2:8] == ["staged", "staged", "staged", "direct", "staged", "staged+direct"]
        assert len(r.segments(0, 2)) == 1 and len(r.segments(0, 3)) == 2
    assert all(m == "staged" for m in modes[8:])


@pytest.mark.parametrize("c", [17, 20])
@pytest.mark.parametrize("kind", ["direct_segment", "two_direct_segments", "bin_total_boundaries"])
def test_fine_sort_modes(ctx, kind, c):
    scal = _scalars_from_keys(_fine_layout(kind, c), c, seed=c)
    n = scal.shape[0]
    r = mr.reach(scal, c)
    assert r.E < mr.BA_MIN_ENTRIES and r.levels == 0
    _check_fine_reach(kind, r)
    for lv in (1, 3):
        assert mr.reach(scal, c, ba_min_entries=0, ba_levels=lv).levels == lv
    ks = list(range(1, n + 1))
    bases = _mult_bases(ctx, 1, ks)
    want = _closed_form(1, ks, scal)
    _, got = _run(ctx, 1, bases, scal, c, [DEFAULT, BA(1), BA(3)])
    assert got == [want] * 3
    _, (g16,) = _run(ctx, 1, bases, scal, 16, [DEFAULT])
    assert g16 == want


# ---- 2. BA rounds at wide windows ---------------------------------------------------------------------------------
def _groups(rng, members):
    """terms in groups of equal scalars: members(j) -> the group's base multipliers"""
    ks, ss = [], []
    for j in range(4):
        s = int(rng.integers(1, 1 << 62)) * int(rng.integers(1, 1 << 62)) * int(rng.integers(1, 1 << 62)) % pr.R
        m = members(j)
        ks += m
        ss += [s] * len(m)
    return ks, co.ints_to_limbs(ss, 4)


def _ba_case(kind, c, n):
    """(base multipliers, scalars) of one BA case"""
    rng = np.random.default_rng(100 * len(kind) + c)
    a = [int(x) for x in rng.integers(2, 1 << 60, size=8)]
    m = n // 8
    if kind == "cancel":               # m copies each of P and -P under one scalar: O
        return _groups(rng, lambda j: [a[j]] * m + [pr.R - a[j]] * m)
    if kind == "double":               # copies of P under one scalar: every pair of every round is a doubling
        return _groups(rng, lambda j: [a[j]] * (2 * m))
    if kind == "survivor":             # cancelling copies plus one survivor per bucket
        return _groups(rng, lambda j: [a[j]] * (m - 1) + [pr.R - a[j]] * (m - 1) + [a[j + 4]])
    ks = list(range(1, n + 1))
    if kind == "one_coarse_bin":       # every digit below 2^(c-10): all entries in coarse bin 0
        low = c - 10
        vals = [sum(int(rng.integers(1, 1 << low)) << (c * w) for w in range(_usable_windows(c))) for _ in range(n)]
        return ks, co.ints_to_limbs(vals, 4)
    if kind == "zero":
        return ks, np.zeros((n, 4), np.uint64)
    scal = sy.random_fr_limbs(n, 5 + c)
    scal[:6] = co.ints_to_limbs([0, 1, pr.R - 1, 2, 1 << (c - 1), pr.R - (1 << (c - 1))], 4)
    return ks, scal


def _ba_wide(ctx, group, kind, c, n, levels):
    ks, scal = _ba_case(kind, c, n)
    r = mr.reach(scal, c)
    assert r.levels == 0 and r.reduction == "rowcol_stage1"
    for lv in levels:
        assert mr.reach(scal, c, ba_min_entries=0, ba_levels=lv).levels == lv
    top = r.sizes[0].max()
    if kind in ("cancel", "double", "survivor"):
        assert top >= 2 * (n // 8) - 2                     # one scalar's whole group in one bucket of some window
    elif kind == "one_coarse_bin":
        assert r.bins[0, 0] == r.sizes[0].sum() > 0
    elif kind == "zero":
        assert top == 0
    bases = _mult_bases(ctx, group, ks)
    want = _closed_form(group, ks, scal)
    if kind == "cancel":
        assert want == (pr.g1_uncompressed if group == 1 else pr.g2_uncompressed)(pr.INF)
    _, got = _run(ctx, group, bases, scal, c, [DEFAULT] + [BA(lv) for lv in levels])
    assert got == [want] * (1 + len(levels))
    _, (g16,) = _run(ctx, group, bases, scal, 16, [BA(levels[0])])
    assert g16 == want


BA_KINDS = ["cancel", "double", "survivor", "one_coarse_bin", "zero", "random"]


@pytest.mark.parametrize("c", [17, 18, 19, 20])
@pytest.mark.parametrize("kind", BA_KINDS)
def test_ba_rounds_wide_windows_g1(ctx, kind, c):
    _ba_wide(ctx, 1, kind, c, 4096, [1, 2, 3, 8])


@pytest.mark.parametrize("c", [17, 20])
@pytest.mark.parametrize("kind", ["cancel", "survivor", "one_coarse_bin", "random"])
def test_ba_rounds_wide_windows_g2(ctx, kind, c):
    _ba_wide(ctx, 2, kind, c, 2048, [1, 3])


# ---- 3. the production configuration: 2^20 terms, library defaults -------------------------------------------------
N20 = 1 << 20


@pytest.fixture(scope="module")
def index_bases_2_20(ctx):
    return _mult_bases(ctx, 1, range(1, N20 + 1))


def _witness_like(n, seed):
    """the shape of the prover's aux vectors: mostly 0 and 1, some below 2^16, a few full-size"""
    rng = np.random.default_rng(seed)
    scal = np.zeros((n, 4), np.uint64)
    u = rng.random(n)
    scal[:, 0] = np.where(u < 0.6, 0, np.where(u < 0.9, 1, rng.integers(2, 1 << 16, size=n))).astype(np.uint64)
    big = u >= 0.97
    scal[big] = sy.random_fr_limbs(int(big.sum()), seed + 1)
    return scal


def _production(ctx, bases, ks, scal):
    r = mr.reach(scal, 20)
    assert r.levels == 2 and r.ordered and r.reduction == "rowcol_stage1"
    want = _closed_form(1, ks, scal)
    c, (got,) = _run(ctx, 1, bases, scal, 0, [DEFAULT])
    assert c == 20
    assert got == want
    return r


@pytest.mark.parametrize("kind", ["witness", "one_scalar", "r_minus_1"])
def test_production_shape(ctx, index_bases_2_20, kind):
    n = N20
    if kind == "witness":
        scal = _witness_like(n, 11)
    else:
        s = pr.R - 1 if kind == "r_minus_1" else 0x1234_5678_9ABC_DEF0_0FED_CBA9_8765_4321 * 0x1_0000_0001 % pr.R
        scal = np.tile(co.ints_to_limbs([s], 4), (n, 1))
    ks = range(1, n + 1)
    r = _production(ctx, index_bases_2_20, ks, scal)
    heavy = r.heavy()[0]
    if kind == "witness":
        assert r.fine[0][0] == "direct" and heavy[0]       # bucket of the ones: a whole-bin HBM scatter, a warp combine
    else:
        assert heavy.sum() >= 1 and r.sizes[0].max() >= n  # each window's one bucket holds every term
        assert any(m == "direct" for m in r.fine[0])


def test_production_shape_cancellations(ctx):
    """2048 groups of 512 terms under one scalar each: 256 copies of P, 255 of -P and one Q, so that full-size buckets are
    dominated by doublings and cancellations in both BA rounds"""
    rng = np.random.default_rng(17)
    G, per = 2048, N20 // 2048
    a = [int(x) for x in rng.integers(2, 1 << 62, size=G)]
    q = [int(x) for x in rng.integers(2, 1 << 62, size=G)]
    s = sy.random_fr_limbs(G, 18)
    ks, idx = [], []
    for j in range(G):
        ks += [a[j]] * (per // 2) + [pr.R - a[j]] * (per // 2 - 1) + [q[j]]
        idx += [j] * per
    perm = rng.permutation(N20)
    ks = [ks[i] for i in perm]
    scal = np.ascontiguousarray(s[np.asarray(idx)[perm]])
    bases = _mult_bases(ctx, 1, ks)
    r = _production(ctx, bases, ks, scal)
    assert r.sizes[0].max() >= per
    _, (g16,) = _run(ctx, 1, bases, scal, 16, [DEFAULT])
    assert g16 == _closed_form(1, ks, scal)


def test_production_shape_matches_16_bit_windows(ctx, index_bases_2_20):
    scal = _witness_like(N20, 23)
    _, (a,) = _run(ctx, 1, index_bases_2_20, scal, 0, [DEFAULT])
    _, (b,) = _run(ctx, 1, index_bases_2_20, scal, 16, [DEFAULT])
    assert a == b


# ---- 4. G2 through the two-level sort -----------------------------------------------------------------------------
@pytest.mark.parametrize("c", [17, 20])
@pytest.mark.parametrize("kind", ["random", "heavy", "one_coarse_bin"])
def test_g2_wide_windows_vs_oracle(ctx, kind, c):
    n = 3000
    bases = co.g2_fixed_base(sy.random_fr_limbs(n, 300 + c))
    scal = sy.random_fr_limbs(n, 301 + c)
    scal[:3] = co.ints_to_limbs([0, 1, pr.R - 1], 4)
    if kind == "heavy":
        scal[100:1600] = 0; scal[100:1600, 0] = 3              # 1500 entries in bucket 2
    elif kind == "one_coarse_bin":
        _, scal = _ba_case("one_coarse_bin", c, n)
    r = mr.reach(scal, c)
    assert r.levels == 0 and r.reduction == "rowcol_stage1" and r.bins is not None
    if kind == "heavy":
        assert r.sizes[0, 2] >= 1500
    elif kind == "one_coarse_bin":
        assert r.bins[0, 0] == r.sizes[0].sum()
    want = _oracle(2, bases, scal)
    _, got = _run(ctx, 2, bases, scal, c, [DEFAULT, BA(2)])
    assert got == [want, want]
    _, (g16,) = _run(ctx, 2, bases, scal, 16, [DEFAULT])
    assert g16 == want


def test_g2_2_20_default_window(ctx):
    """pick_window gives 20-bit windows to a G2 MSM with tables from 2^20 terms: two-level sort and two BA rounds on Fq2
    (tables ~2.6 GB)"""
    n = N20
    ks = range(1, n + 1)
    bases = _mult_bases(ctx, 2, ks)
    scal = sy.random_fr_limbs(n, 404)
    scal[:1000] = 0; scal[:1000, 0] = 1
    r = mr.reach(scal, 20)
    assert r.levels == 2 and r.ordered and r.reduction == "rowcol_stage1"
    c, (got,) = _run(ctx, 2, bases, scal, 0, [DEFAULT])
    assert c == 20
    assert got == _closed_form(2, ks, scal)


# ---- 5. batched domains with tables ---------------------------------------------------------------------------------
def _batch_items(n, count, seed):
    scal = sy.random_fr_limbs(n * count, seed).reshape(count, n, 4)
    scal[0] = 0                                                  # an all-zero item: O
    scal[1] = 0; scal[1, :, 0] = np.arange(n) % 3 == 0           # a 0/1 item: one heavy bucket
    scal[2, :4] = co.ints_to_limbs([0, 1, pr.R - 1, 2], 4)
    return np.ascontiguousarray(scal)


@pytest.fixture(scope="module")
def g1_batch():
    n = 600
    bases = co.g1_fixed_base(sy.random_fr_limbs(n, 501))
    scal = _batch_items(n, 33, 502)
    return bases, scal, [_oracle(1, bases, s) for s in scal]


@pytest.fixture(scope="module")
def g2_batch():
    n = 300
    bases = co.g2_fixed_base(sy.random_fr_limbs(n, 601))
    scal = _batch_items(n, 9, 602)
    return bases, scal, [_oracle(2, bases, s) for s in scal]


def _batched(ctx, group, bases, scal, c):
    import torch
    batch, n = scal.shape[:2]
    d = torch.from_numpy(scal.reshape(-1, 4).view(np.int64).copy()).cuda()
    torch.cuda.synchronize()
    b = zk.Bases(ctx, group, bases, window_bits=c, precompute=True)
    try:
        assert b.window_bits == c
        out = zk.multiexp_device(b, d.data_ptr(), n, batch)
    finally:
        b.free()
    per = 96 if group == 1 else 192
    return [out[per * k:per * (k + 1)] for k in range(batch)]


def _batched_case(ctx, group, data, n_dom, c):
    bases, scal, want = data
    scal = scal[:n_dom]
    r = mr.reach(scal.reshape(-1, 4), c, batch=n_dom)
    assert r.n_dom == n_dom
    if n_dom >= 8:
        assert r.reduction == "rowcol_sums"
    else:
        assert r.reduction != "rowcol_sums"
    got = _batched(ctx, group, bases, scal, c)
    for k in range(n_dom):
        assert got[k] == want[k], k
    if c > 16:
        assert _batched(ctx, group, bases, scal, 16) == got


@pytest.mark.parametrize("c", [9, 14, 17, 20])
@pytest.mark.parametrize("n_dom", [7, 8, 9, 33])
def test_batched_domains_g1(ctx, g1_batch, n_dom, c):
    _batched_case(ctx, 1, g1_batch, n_dom, c)


@pytest.mark.parametrize("c", [8, 17])
@pytest.mark.parametrize("n_dom", [8, 9])
def test_batched_domains_g2(ctx, g2_batch, n_dom, c):
    _batched_case(ctx, 2, g2_batch, n_dom, c)


# ---- 6. G1 points of order 3 ----------------------------------------------------------------------------------------
T3 = (0, 2)                          # y^2 = x^3 + 4: (0, +-2) are on the curve, outside the prime-order subgroup, 3 (0, 2) = O


@pytest.fixture(scope="module")
def order3():
    enc = pr.g1_uncompressed(T3) + pr.g1_uncompressed(pr.ec_neg(pr.FQ, T3))
    with pytest.raises(ValueError, match="GroupDecodingError 5"):
        co.g1_decode_many(enc, checked=True)                 # not in the subgroup: a checked decode rejects them
    assert pr.ec_mul(pr.FQ, T3, 3) is pr.INF
    return co.g1_decode_many(enc, checked=False)


def _order3_case(order3, n, seed):
    """pyref points and limb-form bases mixing (0, +-2) with subgroup points; equal scalars put (0, 2) three times, and
    (0, 2) next to (0, -2), into one bucket of every window"""
    rng = np.random.default_rng(seed)
    sub_k = [int(x) for x in rng.integers(1, 1 << 62, size=8)]
    sub = [pr.ec_mul(pr.FQ, pr.G1_GEN, k) for k in sub_k]
    sub_limbs = co.g1_decode_many(b"".join(pr.g1_uncompressed(p) for p in sub), checked=False)
    t, tn = order3[0], order3[1]
    pts, limbs, vals = [], [], []

    def add(which, s):
        if which == "T":
            pts.append(T3); limbs.append(t)
        elif which == "-T":
            pts.append(pr.ec_neg(pr.FQ, T3)); limbs.append(tn)
        else:
            pts.append(sub[which]); limbs.append(sub_limbs[which])
        vals.append(s % pr.R)

    s3, s2 = int(rng.integers(1, 1 << 62)) ** 4 % pr.R, int(rng.integers(1, 1 << 62)) ** 4 % pr.R
    for _ in range(3):
        add("T", s3)                                          # (0, 2) three times: T + T (a doubling) + T = O
    add("T", s2); add("-T", s2)                               # (0, 2) + (0, -2) = O
    add("T", s2); add(0, s2); add(1, s2)                      # (0, 2) next to subgroup points in one bucket
    while len(vals) < n:
        u = rng.random()
        k = int.from_bytes(rng.bytes(32), "little") % pr.R
        add("T" if u < 0.3 else "-T" if u < 0.45 else int(rng.integers(0, 8)), k if rng.random() < 0.7 else s3)
    return pts, np.array(limbs), co.ints_to_limbs(vals, 4), vals


@pytest.mark.parametrize("n", [48, 3000])
@pytest.mark.parametrize("c,tables", [(5, True), (5, False), (8, True), (8, False), (17, True)])
def test_order3_bases(ctx, order3, n, c, tables):
    pts, bases, scal, vals = _order3_case(order3, n, 700 + n + c)
    want = _oracle(1, bases, scal)
    if n <= 64:
        assert want == pr.g1_uncompressed(pr.ec_msm(pr.FQ, pts, vals))
    for lv in (1, 2, 3):
        assert mr.reach(scal, c, tables=tables, ba_min_entries=0, ba_levels=lv).levels == lv
    assert mr.reach(scal, c, tables=tables).levels == 0
    _, got = _run(ctx, 1, bases, scal, c, [DEFAULT, BA(1), BA(2), BA(3)], tables=tables)
    assert got == [want] * 4
