"""TEST INFRASTRUCTURE (oracle): zface's hierarchical key derivation (zface/src/derive/mod.rs, a ZIP-32-style scheme),
restated with Python integers on pyref.py and redjubjub.py, in the byte layouts of zk_xsk_master_batch,
zk_xsk_derive_batch and zk_xpgk_derive_batch (include/zkb200.h).

  prf_expand_vec(k, ts)   BLAKE2b-512 "zech_ExpandSeed_" (k || ts...)       core/proofs/src/no_std_aliases/keys.rs:25-40
  master(seed)            I = BLAKE2b-512 "Zerochain_Master" (seed); sk = SpendingKey::from_seed(I_L), chain code I_R
  xsk derive_child(i)     I = prf_expand_vec(c, [0x11, sk, i LE]) for i >= 2^31, else [0x12, Point::write(sk P_G), i LE];
                          sk' = to_uniform(prf_expand(I_L, [0x13])) + sk, chain code I_R, depth + 1, index i, parent tag
                          = BLAKE2b-256 "ZerochainEFinger" (Point::write(sk P_G))[:4]
  xpgk derive_child(i)    an error for i >= 2^31; pgk' = to_uniform(prf_expand(I_L, [0x13])) P_G + pgk, the same header
  From<&xsk>              the header with key = sk P_G
  write / read            depth | tag | index LE | chain code | key, 73 bytes

Each step is computed the reference's way: an xsk child's pgk is sk' P_G by double-and-add, never the xpgk shortcut.
Every hash is hashlib's BLAKE2b with its own personalization."""
from __future__ import annotations

import functools
import hashlib
import struct

import numpy as np

from . import pyref as jj
from . import redjubjub as rj

MASTER_PERSONALIZATION = b"Zerochain_Master"     # zface/src/derive/constants.rs
EKFP_PERSONALIZATION = b"ZerochainEFinger"
XK = 73
HARDENED = 1 << 31
BAD_INDEX, HARDENED_INDEX, DEPTH = 4, 5, 6        # row statuses besides the zk_jubjub_into_xy codes


class NotInField(ValueError):
    """SpendingKey::read of a value >= r_J"""


def prf_expand_vec(k: bytes, ts) -> bytes:
    return hashlib.blake2b(k + b"".join(ts), digest_size=64, person=rj.EXPAND_SEED_PERSONALIZATION).digest()


def tag(pgk) -> bytes:
    """EncKeyFingerPrint::try_from(pgk).tag()"""
    return hashlib.blake2b(jj.encode(pgk), digest_size=32, person=EKFP_PERSONALIZATION).digest()[:4]


def mul(p, k: int):
    """Point::mul: MSB-first double-and-add, as pyref.mul, in extended coordinates so a row costs milliseconds"""
    R, d2 = jj.R, 2 * jj.D % jj.R

    def add(a, b):
        (x1, y1, z1, t1), (x2, y2, z2, t2) = a, b
        e, h = (y1 - x1) * (y2 - x2) % R, (y1 + x1) * (y2 + x2) % R
        c, dd = t1 * d2 * t2 % R, 2 * z1 * z2 % R
        e, f, g, h = h - e, dd - c, dd + c, h + e
        return e * f % R, g * h % R, f * g % R, e * h % R

    q = (p[0], p[1], 1, p[0] * p[1] % R)
    acc = (0, 1, 1, 0)
    for bit in bin(k)[2:] if k else "":
        acc = add(acc, acc)
        if bit == "1":
            acc = add(acc, q)
    zi = pow(acc[2], -1, R)
    return acc[0] * zi % R, acc[1] * zi % R


@functools.lru_cache(maxsize=4096)
def pgk_of(sk: int):
    """ProofGenerationKey::from_spending_key: sk P_G by double-and-add"""
    return mul(rj.P_G, sk)


def write(depth: int, ptag: bytes, index: int, chain: bytes, key: bytes) -> bytes:
    return bytes([depth]) + ptag + struct.pack("<I", index) + chain + key


def read_xsk(b: bytes):
    """ExtendedSpendingKey::read: (depth, tag, index, chain, sk); NotInField for sk >= r_J"""
    assert len(b) == XK
    sk = int.from_bytes(b[41:], "little")
    if sk >= rj.R_J:
        raise NotInField("sk >= r_J")
    return b[0], b[1:5], struct.unpack("<I", b[5:9])[0], b[9:41], sk


@functools.lru_cache(maxsize=4096)
def read_xpgk(b: bytes):
    """ExtendedProofGenerationKey::read: (status, (depth, tag, index, chain, pgk point)); status the zk_jubjub_into_xy code"""
    assert len(b) == XK
    st, x, y = jj.into_xy(b[41:])
    if st != jj.OK:
        return st, None
    return jj.OK, (b[0], b[1:5], struct.unpack("<I", b[5:9])[0], b[9:41], (x, y))


def master(seed: bytes) -> bytes:
    """ExtendedSpendingKey::master(seed), written"""
    i = hashlib.blake2b(seed, digest_size=64, person=MASTER_PERSONALIZATION).digest()
    return write(0, bytes(4), 0, i[32:], rj.scalar_bytes(rj.spending_key(i[:32])))


def xpgk_from_xsk(xsk: bytes) -> bytes:
    """From<&ExtendedSpendingKey> for ExtendedProofGenerationKey, written"""
    depth, ptag, index, chain, sk = read_xsk(xsk)
    return write(depth, ptag, index, chain, jj.encode(pgk_of(sk)))


def _tweak(i_l: bytes) -> int:
    return rj.to_uniform(prf_expand_vec(i_l, [b"\x13"]))


def xsk_derive_child(xsk: bytes, index: int) -> bytes:
    """ExtendedSpendingKey::derive_child(ChildIndex::from_index(index)), written; ValueError at depth 255"""
    depth, _, _, chain, sk = read_xsk(xsk)
    if depth == 255:
        raise ValueError("depth + 1 overflows a u8")
    pgk = pgk_of(sk)
    if index >= HARDENED:
        h = prf_expand_vec(chain, [b"\x11", rj.scalar_bytes(sk), struct.pack("<I", index)])
    else:
        h = prf_expand_vec(chain, [b"\x12", jj.encode(pgk), struct.pack("<I", index)])
    child = (_tweak(h[:32]) + sk) % rj.R_J
    return write(depth + 1, tag(pgk), index, h[32:], rj.scalar_bytes(child))


def xpgk_derive_child(xpgk: bytes, index: int):
    """ExtendedProofGenerationKey::derive_child: (status, written child); status 0, a read code, HARDENED_INDEX or DEPTH"""
    st, f = read_xpgk(xpgk)
    if st != jj.OK:
        return st, None
    depth, _, _, chain, pgk = f
    if index >= HARDENED:
        return HARDENED_INDEX, None
    if depth == 255:
        return DEPTH, None
    h = prf_expand_vec(chain, [b"\x12", jj.encode(pgk), struct.pack("<I", index)])
    child = jj.add(mul(rj.P_G, _tweak(h[:32])), pgk)
    return jj.OK, write(depth + 1, tag(pgk), index, h[32:], jj.encode(child))


def account_of_pgk(pgk_enc: bytes):
    """(dk, ek) of the account whose pgk encodes to pgk_enc: into_decryption_key(pgk) and dk P_G"""
    st, pgk = jj.read(pgk_enc)
    assert st == jj.OK
    dk = rj.decryption_key(pgk)
    return rj.scalar_bytes(dk), jj.encode(mul(rj.P_G, dk))


# ---- the rows of the C calls ------------------------------------------------------------------------------------------------
def master_row(seed: bytes):
    """(xsk, xpgk, dk, ek) of zk_xsk_master_batch"""
    xsk = master(seed)
    xpgk = xpgk_from_xsk(xsk)
    return (xsk, xpgk) + account_of_pgk(xpgk[41:])


def xsk_derive_rows(parents: list, parent_idx, child_idx) -> list:
    """[(xsk, xpgk, dk, ek, status)] of zk_xsk_derive_batch; NotInField naming the lowest bad named parent"""
    bad = sorted({p for p in parent_idx if p < len(parents) and int.from_bytes(parents[p][41:], "little") >= rj.R_J})
    if bad:
        raise NotInField("parents[%d]" % bad[0])
    out = []
    for p, i in zip(parent_idx, child_idx):
        if p >= len(parents):
            out.append((bytes(XK), bytes(XK), bytes(32), bytes(32), BAD_INDEX))
        elif parents[p][0] == 255:
            out.append((bytes(XK), bytes(XK), bytes(32), bytes(32), DEPTH))
        else:
            xsk = xsk_derive_child(parents[p], i)
            xpgk = xpgk_from_xsk(xsk)
            out.append((xsk, xpgk) + account_of_pgk(xpgk[41:]) + (0,))
    return out


def xpgk_derive_rows(parents: list, parent_idx, child_idx) -> list:
    """[(xpgk, dk, ek, status)] of zk_xpgk_derive_batch"""
    out = []
    for p, i in zip(parent_idx, child_idx):
        st, child = (BAD_INDEX, None) if p >= len(parents) else xpgk_derive_child(parents[p], i)
        out.append((child,) + account_of_pgk(child[41:]) + (0,) if st == jj.OK else (bytes(XK), bytes(32), bytes(32), st))
    return out


# ---- corpora ----------------------------------------------------------------------------------------------------------------
def bad_pgks() -> list:
    """(encoding, status) for each way ProofGenerationKey::read fails"""
    not_in_field = jj.R.to_bytes(32, "little")
    y = 2
    while jj.point_for_y(y) is not None:
        y += 1
    return [(not_in_field, jj.NOT_IN_FIELD), (y.to_bytes(32, "little"), jj.NOT_ON_CURVE), (jj.encode(jj.torsion_point(4)), jj.NOT_PRIME_ORDER)]


IDENTITY_SIGNED = (1 | (1 << 255)).to_bytes(32, "little")   # the identity written with its sign bit set: it reads as O


def edge_xsk_parents() -> list:
    """xsk parents at the edges: a master, depths 0 / 254 / 255, sk = 0 (identity pgk) and r_J - 1, all-zero and all-0xff
    chain codes"""
    m = master(b"edge master seed")
    return [m, write(254, b"\x01\x02\x03\x04", 7, b"\x5a" * 32, m[41:]), write(255, bytes(4), 0, m[9:41], m[41:]),
            write(3, bytes(4), 1, m[9:41], bytes(32)), write(0, bytes(4), 0, bytes(32), rj.scalar_bytes(rj.R_J - 1)),
            write(1, b"\xff" * 4, 2 ** 32 - 1, b"\xff" * 32, rj.scalar_bytes(12345))]


def edge_xpgk_parents() -> list:
    """xpgk parents at the edges: the xpgks of edge_xsk_parents, the identity written with its sign bit set, and one
    failing each way"""
    good = [xpgk_from_xsk(x) for x in edge_xsk_parents()]
    return good + [write(2, bytes(4), 5, good[0][9:41], IDENTITY_SIGNED)] + [write(0, bytes(4), 0, good[0][9:41], k) for k, _ in bad_pgks()]


EDGE_INDICES = [0, 1, 2 ** 31 - 1, 2 ** 31, 2 ** 32 - 1]


def edge_rows(n_parents: int):
    """(parent_idx, child_idx): every parent with every edge index, then out-of-range parents"""
    rows = [(p, i) for p in range(n_parents) for i in EDGE_INDICES]
    rows += [(n_parents, 0), (n_parents + 5, 3), (2 ** 32 - 1, 2 ** 31)]
    return [r[0] for r in rows], [r[1] for r in rows]


def random_xsk_parents(n: int, seed: int) -> list:
    rng = np.random.default_rng(seed)
    return [write(int(rng.integers(0, 256)), rng.bytes(4), int(rng.integers(0, 2 ** 32)), rng.bytes(32),
                  rj.scalar_bytes(int.from_bytes(rng.bytes(64), "little") % rj.R_J)) for _ in range(n)]


def random_rows(n: int, n_parents: int, seed: int):
    """(parent_idx, child_idx): uniform parents (a few out of range), indices half hardened"""
    rng = np.random.default_rng(seed)
    pidx = [int(v) for v in rng.integers(0, n_parents + max(1, n_parents // 16), n)]
    cidx = [int(v) for v in rng.integers(0, 2 ** 32, n, dtype=np.uint64)]
    return pidx, cidx
