"""TEST INFRASTRUCTURE — mixed ElGamal corpora that hit every status of zk_elgamal_decrypt_batch.

Each entry is (dk, ct, pend, want_null, want_pend): a 32-byte key, a 64-byte ciphertext, a 64-byte pending transfer
(ELGAMAL_ZERO where there is none), and the (status, value) the construction intends with pending given as NULL and as
`pend`.  The random entries are encrypted in bulk by the C oracle; the special cases (bad keys, bad encodings in every
point, the bound) are made with the Python oracle."""
from __future__ import annotations

import numpy as np

from . import eg_coracle as ec
from . import elgamal as eg
from . import pyref as jj
from . import rj_coracle as cj
from .rj_corpus import off_curve_y

ZERO_CT = eg.write(eg.ZERO)
NF = (eg.NOT_FOUND, 0)


def _scalar(rng) -> int:
    return int.from_bytes(rng.bytes(32), "little") % jj.R_J or 1


def _bad_points(good: bytes):
    """Encodings Ciphertext::read rejects: y >= r, y with no x on the curve, and a point with a torsion component."""
    _, p = jj.read(good)
    return [jj.R.to_bytes(32, "little"), off_curve_y(), jj.encode(jj.add(p, jj.torsion_point(8)))]


def random_entries(n: int, seed: int):
    rng = np.random.default_rng(seed)
    keys = [_scalar(rng) for _ in range(n)]
    eks = cj.redjubjub_public_key(keys)
    other = cj.redjubjub_public_key([_scalar(rng) for _ in range(n)])
    rows = []                       # (amount of ct, negated, amount of pend, key index of the encryption, want_null, want_pend)
    B = eg.BOUND
    for i in range(n):
        kind = i % 8
        a = int(rng.integers(0, B))
        if kind == 1:                                   # the sum reaches the bound
            b = int(rng.integers(B - a, B))
            rows.append((a, False, b, (eg.OK, a), NF))
        elif kind == 2:                                 # at or above the bound
            a = int(rng.integers(B, 1 << 32))
            rows.append((a, False, 0, NF, NF))
        elif kind == 3:                                 # neg_encrypt(a), then a pending transfer of b >= a: b - a
            a = max(a, 1)
            b = int(rng.integers(a, B))
            rows.append((a, True, b, NF, (eg.OK, b - a)))
        elif kind == 5:
            a, b = int(rng.integers(0, 100)), int(rng.integers(0, 100))
            rows.append((a, False, b, (eg.OK, a), (eg.OK, a + b)))
        else:
            b = int(rng.integers(0, B - a))
            rows.append((a, False, b, (eg.OK, a), (eg.OK, a + b)))
    rs = [_scalar(rng) for _ in range(2 * n)]
    ek_of = lambda i: (other if i % 8 == 4 else eks)[32 * i:32 * i + 32]   # kind 4: encrypted to another key
    ek_all = b"".join(ek_of(i) for i in range(n))
    plain = ec.encrypt([r[0] for r in rows], rs[:n], ek_all)
    neg = ec.encrypt([r[0] for r in rows], rs[:n], ek_all, neg=True)
    pend = ec.encrypt([r[2] for r in rows], rs[n:], ek_all)
    out = []
    for i, (a, is_neg, b, wn, wp) in enumerate(rows):
        ct = (neg if is_neg else plain)[64 * i:64 * i + 64]
        if i % 8 == 4:
            wn = wp = NF
        pd = pend[64 * i:64 * i + 64] if i % 16 != 0 else ZERO_CT      # every 16th: no pending transfer
        if pd == ZERO_CT:
            wp = wn
        out.append((keys[i].to_bytes(32, "little"), ct, pd, wn, wp))
    return out


def special_entries(seed: int):
    rng = np.random.default_rng(seed)
    dk = _scalar(rng)
    ek = jj.mul(eg.P_G, dk)
    kb = dk.to_bytes(32, "little")
    enc = lambda a: eg.write(eg.encrypt(a, _scalar(rng), ek))
    good, pd = enc(7), enc(3)
    out = [(kb, good, pd, (eg.OK, 7), (eg.OK, 10)),
           (kb, ZERO_CT, ZERO_CT, (eg.OK, 0), (eg.OK, 0)),
           (kb, enc(999_999), ZERO_CT, (eg.OK, 999_999), (eg.OK, 999_999)),
           (kb, enc(1_000_000), ZERO_CT, NF, NF),
           (kb, enc(2 ** 32 - 1), ZERO_CT, NF, NF),
           (kb, eg.write(eg.neg_encrypt(5, _scalar(rng), ek)), ZERO_CT, NF, NF),
           (kb, enc(999_999), enc(1), (eg.OK, 999_999), NF),
           (kb, enc(999_998), enc(1), (eg.OK, 999_998), (eg.OK, 999_999))]
    for bad_dk in (jj.R_J, jj.R_J + 1, 2 ** 256 - 1):
        out.append((bad_dk.to_bytes(32, "little"), good, pd, (eg.BAD_KEY, 0), (eg.BAD_KEY, 0)))
    bads = _bad_points(good[:32])
    out.append((jj.R_J.to_bytes(32, "little"), bads[0] + good[32:], bads[1] + pd[32:], (eg.BAD_KEY, 0), (eg.BAD_KEY, 0)))
    for bad in bads:
        for half in (0, 1):
            ct_bad = bad + good[32:] if half == 0 else good[:32] + bad
            pd_bad = bad + pd[32:] if half == 0 else pd[:32] + bad
            out.append((kb, ct_bad, pd, (eg.BAD_BALANCE, 0), (eg.BAD_BALANCE, 0)))
            out.append((kb, good, pd_bad, (eg.OK, 7), (eg.BAD_PENDING, 0)))
            out.append((kb, ct_bad, pd_bad, (eg.BAD_BALANCE, 0), (eg.BAD_BALANCE, 0)))
    return out


def columns(entries):
    """(dks, cts, pends) as concatenated bytes, and the wanted (statuses, values) with pending NULL and with pending."""
    dks, cts, pds = (b"".join(e[k] for e in entries) for k in range(3))
    want = lambda k: ([e[k][0] for e in entries], [e[k][1] for e in entries])
    return dks, cts, pds, want(3), want(4)
