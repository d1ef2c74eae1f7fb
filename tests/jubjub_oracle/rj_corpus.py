"""TEST INFRASTRUCTURE — mixed RedJubjub corpora that hit every verdict of zk_redjubjub_verify_batch.

Valid signatures are made in bulk by the C oracle (rj_coracle.redjubjub_sign); the special cases that need curve arithmetic
(torsion components, a nonce point with a torsion component) by the Python oracle.  Each entry carries the verdict the
construction intends; the tests compare it with both oracles and with the device."""
from __future__ import annotations

import numpy as np

from . import rj_coracle as cj
from . import pyref as jj
from . import redjubjub as rj

# message lengths: 0..300 in steps, the BLAKE2b block edges (96 and 224 bytes of message = 128 and 256 bytes hashed) and
# one past each
EDGE_LENGTHS = [0, 1, 7, 31, 32, 33, 63, 64, 95, 96, 97, 127, 128, 129, 200, 223, 224, 225, 255, 256, 257, 300]


def off_curve_y() -> bytes:
    y = 2
    while jj.point_for_y(y) is not None:
        y += 1
    return y.to_bytes(32, "little")


def _scalar(rng) -> int:
    return int.from_bytes(rng.bytes(32), "little") % rj.R_J


def sign_with_torsion_nonce(sk: int, msg: bytes, r: int, t8) -> bytes:
    """A signature whose nonce point is r P_G + t8: c is taken over that encoding, so [8] removes the excess and it verifies."""
    rbar = jj.encode(jj.add(jj.mul(rj.P_G, r), t8))
    s = (rj.h_star(rbar, msg) * sk + r) % rj.R_J
    return rbar + rj.scalar_bytes(s)


def mixed(n_valid: int, seed: int, lengths=None):
    """(entries, n_special): a list of (vk, sig, msg, intended verdict), n_valid valid signatures first, then the special
    cases, shuffled together."""
    rng = np.random.default_rng(seed)
    lengths = lengths or EDGE_LENGTHS
    sks = [_scalar(rng) for _ in range(n_valid)]
    msgs = [rng.bytes(lengths[i % len(lengths)]) for i in range(n_valid)]
    vks = cj.redjubjub_public_key(sks)
    sigs = cj.redjubjub_sign(sks, rng.bytes(80 * n_valid), msgs)
    vk = [vks[32 * i:32 * i + 32] for i in range(n_valid)]
    sg = [sigs[64 * i:64 * i + 64] for i in range(n_valid)]
    out = [(vk[i], sg[i], msgs[i], rj.OK) for i in range(n_valid)]
    special = []
    bad_field = [(jj.R + k).to_bytes(32, "little") for k in (0, 1, 5)] + [b"\xff" * 32]
    bad_curve = off_curve_y()
    t8, t4, t2 = jj.torsion_point(8), jj.torsion_point(4), jj.torsion_point(2)
    m = max(1, n_valid // 64)
    for j in range(m):
        i, k = j % n_valid, (j + 1) % n_valid
        special.append((vk[i], sg[i], msgs[i] + b"\x00", rj.BAD_EQUATION))                  # a wrong message
        special.append((vk[k], sg[i], msgs[i], rj.BAD_EQUATION if vk[k] != vk[i] else rj.OK))   # a wrong key
        special.append((vk[i], sg[k], msgs[i], rj.BAD_EQUATION))                           # another signature
        special.append((bad_field[j % 4], sg[i], msgs[i], rj.BAD_VK))
        special.append((bad_curve, sg[i], msgs[i], rj.BAD_VK))
        special.append((vk[i], bad_field[j % 4] + sg[i][32:], msgs[i], rj.BAD_R))
        special.append((vk[i], bad_curve + sg[i][32:], msgs[i], rj.BAD_R))
        special.append((vk[i], sg[i][:32] + rj.scalar_bytes(rj.R_J), msgs[i], rj.BAD_S))
        special.append((vk[i], sg[i][:32] + b"\xff" * 32, msgs[i], rj.BAD_S))
        special.append((bad_curve, bad_curve + b"\xff" * 32, msgs[i], rj.BAD_VK))          # the reference's order decides
        special.append((vk[i], bad_field[0] + b"\xff" * 32, msgs[i], rj.BAD_R))
        special.append((vk[i], sg[i][:32] + rj.scalar_bytes(int.from_bytes(sg[i][32:], "little") ^ 1), msgs[i], rj.BAD_EQUATION))
        special.append((rng.bytes(32), rng.bytes(32) + sg[i][32:], msgs[i], None))           # whatever the oracles say
    for j in range(min(m, 8)):                                                              # Python-oracle constructions
        i = j % n_valid
        _, a = jj.read(vk[i])
        special.append((jj.encode(jj.add(a, (t8, t4, t2)[j % 3])), sg[i], msgs[i], rj.OK))   # torsion vk: accepted
        sk = _scalar(rng)
        msg = msgs[i]
        special.append((rj.public_key(sk), sign_with_torsion_nonce(sk, msg, _scalar(rng), t8), msg, rj.OK))
    special.append((jj.encode(t8), sg[0], msgs[0], None))                                  # a key of order 8
    special.append((jj.encode(jj.IDENTITY), sg[0], msgs[0], None))
    out += special
    order = rng.permutation(len(out))
    return [out[i] for i in order], len(special)


def python_verdict(entry) -> int:
    vk, sig, msg = entry[:3]
    return rj.verify(vk, msg, sig)


def columns(entries):
    """(vks bytes, sigs bytes, msgs list) of a corpus."""
    return b"".join(e[0] for e in entries), b"".join(e[1] for e in entries), [e[2] for e in entries]
