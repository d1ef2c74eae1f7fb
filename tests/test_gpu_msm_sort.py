"""Shapes of the two-level bucket sort (windows above 16 bits) that the other MSM tests do not reach.

The coarse pass cuts each sort domain into tiles sized from the SM count (at least two waves of 256-thread blocks; a tile
is a multiple of 4096 entries, which the scatter groups by coarse bin in shared memory 4096 at a time), and the fine pass
reads each coarse bin with 16-byte loads.  The cases here put the entry count just below, at and just above a tile boundary, make every digit
zero, put every digit into one coarse bin or one bucket, and run batches whose domains do not start on a 16-byte boundary.
Every result is checked against the oracle or the closed form (bases (i+1) G) and must be byte-identical to the one-level
sort of the same inputs (window_bits = 16)."""
import numpy as np
import pytest

from oracle import coracle as co
from oracle import pyref as pr
from tests import msm_reach as mr
from zero_chain_b200 import groth16 as zk
from zero_chain_b200 import synthetic as sy

pytestmark = pytest.mark.gpu

CHUNK = mr.COARSE_CHUNK   # entries per chunk of the coarse scatter, and the least tile length (checked against msm.cuh)


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


def _windows(c):
    return 255 // c + 1


def _index_bases(ctx, n):
    idx = np.zeros((n, 4), np.uint64)
    idx[:, 0] = np.arange(1, n + 1, dtype=np.uint64)
    return zk.scalar_mul_many(ctx, 1, zk.G1_GENERATOR, idx)


def _ints(scal):
    s = scal.astype(object)
    return s[:, 0] + (s[:, 1] << 64) + (s[:, 2] << 128) + (s[:, 3] << 192)


def _closed_form(scal):
    """sum s_i (i+1) G, the MSM over the bases (i+1) G"""
    k = int(sum(int(v) * (i + 1) for i, v in enumerate(_ints(scal))) % pr.R)
    return pr.g1_uncompressed(pr.ec_mul(pr.FQ, pr.G1_GEN, k))


def _msm(ctx, bases, scal, c):
    b = zk.Bases(ctx, 1, bases, window_bits=c, precompute=True)
    assert b.window_bits == c
    try:
        return zk.multiexp(b, scal)
    finally:
        b.free()


@pytest.mark.parametrize("c", [17, 20])
@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_entry_count_at_tile_boundary(ctx, c, delta):
    """4096 points give W x 4096 entries: a whole number of one-chunk tiles (the least tile length, which such small MSMs
    get); one point fewer or more leaves the last tile short by W entries or starts a new tile of W entries."""
    n = CHUNK + delta
    bases = co.g1_fixed_base(sy.random_fr_limbs(n, 50 + n + c))
    scal = sy.random_fr_limbs(n, 51 + n + c)
    scal[:3] = co.ints_to_limbs([0, 1, pr.R - 1], 4)
    got = _msm(ctx, bases, scal, c)
    assert got == co.g1_encode(co.g1_msm(bases, scal), False)
    assert got == _msm(ctx, bases, scal, 16)


def test_tiles_above_the_minimum(ctx):
    """2^20 + 1 points at c = 20: tiles of several chunks (two waves of blocks over 13.6 M entries), the last tile partly
    filled."""
    n = (1 << 20) + 1
    bases = _index_bases(ctx, n)
    scal = sy.random_fr_limbs(n, 4242)
    got = _msm(ctx, bases, scal, 20)
    assert got == _closed_form(scal)
    assert got == _msm(ctx, bases, scal, 16)


@pytest.mark.parametrize("c", [17, 20])
def test_all_zero_scalars(ctx, c):
    """every digit is DIGIT_ZERO: empty coarse bins and buckets, the point at infinity"""
    n = 5000
    bases = co.g1_fixed_base(sy.random_fr_limbs(n, 60 + c))
    scal = np.zeros((n, 4), np.uint64)
    got = _msm(ctx, bases, scal, c)
    assert got == pr.g1_uncompressed(pr.INF)
    assert got == _msm(ctx, bases, scal, 16)


def _small_digit_scalars(n, c, seed, one_bucket):
    """scalars whose every c-bit window digit lies in [1, 2^(c-10)): all entries in coarse bin 0 (the high 9 bits of every
    bucket key are zero), spread over its buckets, or all in bucket 0 (every digit 1)"""
    low = c - 10
    rng = np.random.default_rng(seed)
    vals = []
    for _ in range(n):
        s = 0
        for w in range(_windows(c)):
            if c * w + low > 250:            # keep the scalar below r
                break
            s |= (1 if one_bucket else int(rng.integers(1, 1 << low))) << (c * w)
        vals.append(s)
    assert max(vals) < pr.R
    return co.ints_to_limbs(vals, 4)


@pytest.mark.parametrize("c", [17, 20])
@pytest.mark.parametrize("one_bucket", [False, True])
def test_one_coarse_bin(ctx, c, one_bucket):
    """one coarse bin holds every entry, so a single block of the fine pass sorts all of them"""
    n = 20000
    bases = _index_bases(ctx, n)
    scal = _small_digit_scalars(n, c, 70 + c, one_bucket)
    got = _msm(ctx, bases, scal, c)
    assert got == _closed_form(scal)
    assert got == _msm(ctx, bases, scal, 16)


@pytest.mark.parametrize("c", [17, 20])
def test_batch_of_domains(ctx, c):
    """a batch of 3 domains with tables; with an odd number of points the second domain's digits do not start on a
    16-byte boundary, so the coarse pass reads its head and tail one code at a time"""
    import torch
    n, batch = 1025, 3
    bases = co.g1_fixed_base(sy.random_fr_limbs(n, 80 + c))
    scal = sy.random_fr_limbs(n * batch, 81 + c).reshape(batch, n, 4)
    scal[1, :7] = 0
    d = torch.from_numpy(np.ascontiguousarray(scal).view(np.int64)).cuda()
    torch.cuda.synchronize()
    outs = {}
    for w in (c, 16):
        b = zk.Bases(ctx, 1, bases, window_bits=w, precompute=True)
        outs[w] = zk.multiexp_device(b, d.data_ptr(), n, batch)
        b.free()
    assert outs[c] == outs[16]
    for k in range(batch):
        assert outs[c][96 * k:96 * k + 96] == co.g1_encode(co.g1_msm(bases, scal[k]), False)
