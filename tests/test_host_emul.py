"""CPU check of the PRODUCT's device headers (zero_chain_b200/csrc/field.cuh, curve.cuh): the same
C++ source is compiled with ZK_HOST_EMUL (PTX carry-chain primitives replaced by an explicit carry
flag) and compared with the oracle.  This validates the limb-level algorithms (even/odd CIOS
Montgomery product, XYZZ group law and its exceptional cases) where no GPU exists; the real PTX
path is covered by the -m gpu tests."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import coracle as co
from oracle import pyref as pr

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul") / "libemul.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "zero_chain_b200", "csrc"),
                           "-o", so, os.path.join(HERE, "host_emul", "emul.cpp")])
    return C.CDLL(so)


def _call(lib, name, n, *vals):
    arrs = [np.array([(v >> (32 * i)) & 0xFFFFFFFF for i in range(n)], dtype=np.uint32) for v in vals]
    o = np.zeros(n, np.uint32)
    getattr(lib, name)(*[a.ctypes.data_as(C.c_void_p) for a in arrs], o.ctypes.data_as(C.c_void_p))
    return sum(int(x) << (32 * i) for i, x in enumerate(o))


@pytest.mark.parametrize("f,mod,n,bits", [("fq", pr.Q, 12, 384), ("fr", pr.R, 8, 256)])
def test_field_emulation(emu, f, mod, n, bits):
    rng = pr.SplitMix64(21)
    rinv = pow(1 << bits, -1, mod)
    vals = [0, 1, mod - 1, mod - 2, 2, (1 << bits) % mod, mod >> 1] + [rng.below(mod, bits // 64 + 1) for _ in range(1500)]
    for i in range(len(vals) - 1):
        a, b = vals[i], vals[i + 1]
        assert _call(emu, "emu_%s_mul" % f, n, a, b) == a * b * rinv % mod
        assert _call(emu, "emu_%s_add" % f, n, a, b) == (a + b) % mod
        assert _call(emu, "emu_%s_sub" % f, n, a, b) == (a - b) % mod
        assert _call(emu, "emu_%s_neg" % f, n, a) == (-a) % mod
        assert _call(emu, "emu_%s_from" % f, n, a) == (a << bits) % mod
        assert _call(emu, "emu_%s_to" % f, n, a) == a * rinv % mod
    for a in vals[1:40]:
        want = pow(a * rinv, -1, mod) * (1 << bits) % mod
        assert _call(emu, "emu_%s_inv" % f, n, a) == want            # binary extended Euclid (fq.rs:854-907)
    for a in vals[6:9]:
        assert _call(emu, "emu_%s_invf" % f, n, a) == pow(a * rinv, -1, mod) * (1 << bits) % mod   # Fermat cross-check
    assert _call(emu, "emu_%s_inv" % f, n, 0) == 0
    # the reference's own mul KAT (fq.rs:2564-2588 / fr.rs:1241-1259) through the emulated device code
    import json
    K = json.load(open(os.path.join(HERE, "golden", "kats.json")))
    g = [sum(int(v, 16) << (64 * i) for i, v in enumerate(x)) for x in K["tests"]["%s.rs::test_%s_mul_assign" % (f, f)]["groups"]]
    assert _call(emu, "emu_%s_mul" % f, n, g[0], g[1]) == g[2]


def _pt(lib, name, a, b, w, *extra):
    a = np.ascontiguousarray(a, np.uint64); b = np.ascontiguousarray(b, np.uint64)
    o = np.zeros(w, np.uint64)
    getattr(lib, name)(a.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), o.ctypes.data_as(C.c_void_p), *extra)
    return o


@pytest.mark.parametrize("g", [1, 2])
def test_curve_emulation(emu, g):
    w = 12 if g == 1 else 24
    fixed = co.g1_fixed_base if g == 1 else co.g2_fixed_base
    add = co.g1_add if g == 1 else co.g2_add
    mul = co.g1_mul if g == 1 else co.g2_mul
    dbl = co.g1_double if g == 1 else co.g2_double
    pts = fixed(co.ints_to_limbs([0, 1, 2, 3, 5, pr.R - 2, 123456789, pr.R - 1], 4))
    inf = pts[0]
    for a in pts:
        for b in pts:
            want = add(dbl(a), b)
            assert np.array_equal(_pt(emu, "emu_g%d_2a_plus_b" % g, a, b, w), want)
            want = add(dbl(a), add(dbl(b), b))
            assert np.array_equal(_pt(emu, "emu_g%d_2a_plus_3b" % g, a, b, w), want)
            for mixed in (0, 1):     # includes P+P, P+(-P), inf+P, P+inf
                assert np.array_equal(_pt(emu, "emu_g%d_add" % g, a, b, w, mixed), add(a, b))
    rng = pr.SplitMix64(4)
    for k in [0, 1, 2, pr.R - 1, rng.fr()]:
        kk = co.ints_to_limbs([k], 4)
        assert np.array_equal(_pt(emu, "emu_g%d_mul" % g, pts[4], kk, w), mul(pts[4], k))
    assert not np.any(_pt(emu, "emu_g%d_mul" % g, inf, co.ints_to_limbs([5], 4), w))


@pytest.mark.parametrize("g", [1, 2])
def test_batched_affine_pairs_emulation(emu, g):
    """msm_affine_core.cuh: pairwise affine additions with ONE shared inversion, incl. the exceptional pairs
    (P+P, P+(-P), infinity operand, odd leftover) — against the oracle's group law."""
    w = 12 if g == 1 else 24
    fixed = co.g1_fixed_base if g == 1 else co.g2_fixed_base
    add = co.g1_add if g == 1 else co.g2_add
    ks = [3, 5, 7, 7, 9, pr.R - 9, 0, 11, 13, 0, 0, 0, 21, 34, 55, 89, 144, 233, 377, 610, 17]      # odd count: leftover copied
    pts = np.ascontiguousarray(fixed(co.ints_to_limbs(ks, 4)))
    m = (len(ks) + 1) // 2
    out = np.zeros((m, w), np.uint64)
    getattr(emu, "emu_g%d_batch_pairs" % g)(pts.ctypes.data_as(C.c_void_p), len(ks), out.ctypes.data_as(C.c_void_p))
    for j in range(m):
        want = add(pts[2 * j], pts[2 * j + 1]) if 2 * j + 1 < len(ks) else pts[2 * j]
        assert np.array_equal(out[j], want), j


def test_separated_multiply_reduce_emulation(emu):
    """field_wide.cuh: column-wise product, dedicated squaring, shared reduction of a*b - c*d — all must equal the
    interleaved Montgomery product's values (hence the reference's)."""
    mod, n = pr.Q, 12
    rinv = pow(1 << 384, -1, mod)
    rng = pr.SplitMix64(77)
    vals = [0, 1, mod - 1, mod - 2, (1 << 384) % mod, mod >> 1] + [rng.fq() for _ in range(600)]
    for i in range(len(vals) - 3):
        a, b, c, d = vals[i], vals[i + 1], vals[i + 2], vals[i + 3]
        assert _call(emu, "emu_fq_mul_sep", n, a, b) == a * b * rinv % mod
        assert _call(emu, "emu_fq_sqr_sep", n, a) == a * a * rinv % mod
        assert _call(emu, "emu_fq_mul_sub_mul", n, a, b, c, d) == (a * b - c * d) * rinv % mod


def test_glv_split_emulation(emu):
    """glv_split.cuh: k = k1 u^2 + k0 by shift-and-subtract, as k_scale_points runs it on one thread, against divmod for the
    GLV edge scalars (tests/prove_forge.py) and 10^5 random scalars below 2^255."""
    from tests import prove_forge as pf
    rng = np.random.Generator(np.random.Philox(31))
    words = rng.integers(0, 1 << 32, size=(100000, 8), dtype=np.uint64).astype(np.uint32)
    words[:, 7] &= 0x7FFFFFFF
    words[::3, 7] &= 0x73EDA753                        # a third of them below r, like every canonical blinding scalar
    edges = list(pf.GLV_EDGES.values()) + [0, 1, pr.R - 1, (1 << 255) - 1]
    edge_words = np.array([[(k >> (32 * i)) & 0xFFFFFFFF for i in range(8)] for k in edges], np.uint32)
    k = np.ascontiguousarray(np.concatenate([edge_words, words]))
    out = np.zeros((k.shape[0], 8), np.uint32)
    emu.emu_glv_split_many(k.ctypes.data_as(C.c_void_p), C.c_size_t(k.shape[0]), out.ctypes.data_as(C.c_void_p))
    as_int = lambda row: sum(int(x) << (32 * i) for i, x in enumerate(row))
    bad = []
    for i in range(k.shape[0]):
        kk = as_int(k[i])
        if (as_int(out[i, :4]), as_int(out[i, 4:])) != pf.glv_split(kk):
            bad.append(hex(kk))
    assert bad[:5] == []
