"""TEST INFRASTRUCTURE (oracle): lifted ElGamal with the Diversifier generator, restated with Python integers on pyref.py
and redjubjub.py (P_G, key derivation).

  encrypt        (amount P_G + r ek, r P_G)                      core/crypto/src/elgamal.rs:49-67
  neg_encrypt    (-amount P_G + r ek, r P_G)                     elgamal.rs:70-85
  decrypt        V = left - dk right; the i < 1 000 000 with i P_G == V by the reference's own walk, else None
                                                                  elgamal.rs:87-110
  write / read   left | right, each Point::read + as_prime_order elgamal.rs:112-136
  add / sub      pointwise                                        elgamal.rs:138-178
  decrypt_bytes  what zface's BalanceQuery does (zface/src/utils/getter.rs:135-175): DecryptionKey::read, Ciphertext::read
                 of the balance and of the pending transfer, add, decrypt; the statuses of zk_elgamal_decrypt_batch

A ciphertext is a pair of affine points (left, right).  decrypt walks up to 10^6 affine additions: call it only where the
answer is small (stage() gives the encoding of V without the walk)."""
from __future__ import annotations

from . import pyref as jj
from . import redjubjub as rj

BOUND = 1_000_000
OK, NOT_FOUND, BAD_KEY, BAD_BALANCE, BAD_PENDING = 0, 1, 2, 3, 4
ZERO = (jj.IDENTITY, jj.IDENTITY)
P_G = rj.P_G


def encrypt(amount: int, r: int, ek) -> tuple:
    """ek: the encryption key point."""
    return jj.add(jj.mul(P_G, amount), jj.mul(ek, r)), jj.mul(P_G, r)


def neg_encrypt(amount: int, r: int, ek) -> tuple:
    return jj.add(jj.neg(jj.mul(P_G, amount)), jj.mul(ek, r)), jj.mul(P_G, r)


def add(a, b) -> tuple:
    return jj.add(a[0], b[0]), jj.add(a[1], b[1])


def sub(a, b) -> tuple:
    return jj.add(a[0], jj.neg(b[0])), jj.add(a[1], jj.neg(b[1]))


def write(ct) -> bytes:
    return jj.encode(ct[0]) + jj.encode(ct[1])


def read(b: bytes):
    """Ciphertext::read: (True, ciphertext) or (False, None)."""
    assert len(b) == 64
    pts = []
    for enc in (b[:32], b[32:]):
        st, x, y = jj.into_xy(enc)
        if st != jj.OK:
            return False, None
        pts.append((x, y))
    return True, tuple(pts)


def v_point(ct, dk: int):
    return jj.add(ct[0], jj.neg(jj.mul(ct[1], dk)))


def decrypt(ct, dk: int, bound: int = BOUND):
    """The reference's loop, literally: acc = O, compare, acc += P_G.  Returns the amount or None."""
    v = v_point(ct, dk)
    acc = jj.IDENTITY
    for i in range(bound):
        if acc == v:
            return i
        acc = jj.add(acc, P_G)
    return None


def key_bytes(dk: int) -> bytes:
    return dk.to_bytes(32, "little")


def stage(dk_b: bytes, ct_b: bytes, pend_b: bytes | None = None):
    """(status, encoding of V) without the walk: status BAD_KEY / BAD_BALANCE / BAD_PENDING (encoding None) or OK."""
    dk = int.from_bytes(dk_b, "little")
    if dk >= jj.R_J:
        return BAD_KEY, None
    ok, ct = read(ct_b)
    if not ok:
        return BAD_BALANCE, None
    if pend_b is not None:
        ok, pd = read(pend_b)
        if not ok:
            return BAD_PENDING, None
        ct = add(ct, pd)
    return OK, jj.encode(v_point(ct, dk))


def decrypt_bytes(dk_b: bytes, ct_b: bytes, pend_b: bytes | None = None, bound: int = BOUND):
    """(status, value) as zk_elgamal_decrypt_batch returns them, the walk included (small answers only)."""
    st, _ = stage(dk_b, ct_b, pend_b)
    if st != OK:
        return st, 0
    ct = read(ct_b)[1]
    if pend_b is not None:
        ct = add(ct, read(pend_b)[1])
    v = decrypt(ct, int.from_bytes(dk_b, "little"), bound)
    return (NOT_FOUND, 0) if v is None else (OK, v)


def account_keys(seed: bytes):
    """(decryption key, encryption key point) of an account seed (core/keys/src/lib.rs)."""
    dk = rj.decryption_key(rj.proof_generation_key(rj.spending_key(seed)))
    return dk, jj.mul(P_G, dk)
