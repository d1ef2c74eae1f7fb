"""TEST INFRASTRUCTURE (oracle): RedJubjub with the Diversifier generator, restated with Python integers on pyref.py.

  H*(a || b)       BLAKE2b-512, personalization "Zcash_RedJubjubH", then Fs::to_uniform: the 64 digest bytes as one
                   little-endian integer mod r_J          core/jubjub/src/redjubjub.rs:24-26, util.rs:5-11, curve/fs.rs:587-592
  P_G              find_group_hash(b"r", "Zcash_PH"): BLAKE2s-256(GH_FIRST_BLOCK || tag) read as a point, times the cofactor,
                   first tag "r" || i that gives neither an error nor the identity      curve/mod.rs:325-326, group_hash.rs
  sign             with the 80 random bytes T supplied by the caller                    redjubjub.rs:73-103
  verify           redjubjub.rs:127-155 as the runtime reaches it (core/primitives/src/signature.rs:65-82): the signer's
                   Point::read first, then R = Point::read(rbar), S = read_scalar(sbar), [8](c vk + R - S P_G) == O
  key derivation   SpendingKey::from_seed -> ProofGenerationKey -> DecryptionKey -> EncryptionKey (core/keys/src/lib.rs)

verify returns the verdict codes of zk_redjubjub_verify_batch (include/zkb200.h)."""
from __future__ import annotations

import hashlib

from . import pyref as jj

GH_FIRST_BLOCK = b"096b36a5804bfacef1691e173c366a47ff5ba84a44f26ddd7e8d9f79d5b42df0"   # core/jubjub/src/constants.rs:5-6
PH_PERSONALIZATION = b"Zcash_PH"                          # constants.rs:20
H_STAR_PERSONALIZATION = b"Zcash_RedJubjubH"              # redjubjub.rs:25
EXPAND_SEED_PERSONALIZATION = b"zech_ExpandSeed_"         # core/keys/src/lib.rs:40
BDK_PERSONALIZATION = b"zech_bdk"                         # core/keys/src/lib.rs:41
R_J = jj.R_J
BAD_EQUATION, OK, BAD_VK, BAD_R, BAD_S = 0, 1, 2, 3, 4


def to_uniform(digest: bytes) -> int:
    assert len(digest) == 64
    return int.from_bytes(digest, "little") % R_J


def h_star(a: bytes, b: bytes) -> int:
    return to_uniform(hashlib.blake2b(a + b, digest_size=64, person=H_STAR_PERSONALIZATION).digest())


def group_hash(tag: bytes, personalization: bytes):
    h = hashlib.blake2s(GH_FIRST_BLOCK + tag, digest_size=32, person=personalization).digest()
    st, p = jj.read(h)
    if st != jj.OK:
        return None
    p = jj.mul(p, jj.COFACTOR)
    return None if p == jj.IDENTITY else p


def find_group_hash(m: bytes, personalization: bytes):
    """(point, i): the first i with group_hash(m || i) defined (group_hash.rs via curve/mod.rs:find_group_hash)."""
    for i in range(256):
        p = group_hash(m + bytes([i]), personalization)
        if p is not None:
            return p, i
    raise AssertionError("no generator")


P_G, P_G_INDEX = find_group_hash(b"r", PH_PERSONALIZATION)   # FixedGenerators::Diversifier


def scalar_bytes(s: int) -> bytes:
    return s.to_bytes(32, "little")


def public_key(sk: int) -> bytes:
    """PublicKey::from_private: sk P_G, encoded."""
    return jj.encode(jj.mul(P_G, sk))


def sign(sk: int, msg: bytes, t: bytes) -> bytes:
    """PrivateKey::sign with T = t (80 bytes) in place of the RNG output: rbar || sbar."""
    assert len(t) == 80
    r = h_star(t, msg)
    rbar = jj.encode(jj.mul(P_G, r))
    s = (h_star(rbar, msg) * sk + r) % R_J
    return rbar + scalar_bytes(s)


def verify(vk: bytes, msg: bytes, sig: bytes) -> int:
    assert len(vk) == 32 and len(sig) == 64
    c = h_star(sig[:32], msg)                    # computed from the raw bytes before any check
    st, a = jj.read(vk)
    if st != jj.OK:
        return BAD_VK
    st, r = jj.read(sig[:32])
    if st != jj.OK:
        return BAD_R
    s = int.from_bytes(sig[32:], "little")
    if s >= R_J:
        return BAD_S
    p = jj.add(jj.add(jj.mul(a, c), r), jj.neg(jj.mul(P_G, s)))
    return OK if jj.mul(p, jj.COFACTOR) == jj.IDENTITY else BAD_EQUATION


def randomize_public_key(vk: bytes, alpha: int) -> bytes:
    """PublicKey::randomize: vk + alpha P_G (the rvk of a transaction; its secret is sk + alpha)."""
    st, a = jj.read(vk)
    assert st == jj.OK
    return jj.encode(jj.add(jj.mul(P_G, alpha), a))


# ---- key derivation (core/keys/src/lib.rs) -------------------------------------------------------------------------------
def spending_key(seed: bytes) -> int:
    """SpendingKey::from_seed: to_uniform(BLAKE2b-512 "zech_ExpandSeed_" (seed))."""
    return to_uniform(hashlib.blake2b(seed, digest_size=64, person=EXPAND_SEED_PERSONALIZATION).digest())


def proof_generation_key(sk: int):
    return jj.mul(P_G, sk)


def decryption_key(pgk) -> int:
    """ProofGenerationKey::into_decryption_key: BLAKE2s-256 "zech_bdk" of the encoded point, top five bits dropped."""
    h = bytearray(hashlib.blake2s(jj.encode(pgk), digest_size=32, person=BDK_PERSONALIZATION).digest())
    h[31] &= 0x07
    dk = int.from_bytes(h, "little")
    assert dk < R_J
    return dk


def encryption_key(seed: bytes) -> bytes:
    """EncryptionKey::from_seed, encoded (the account address)."""
    return jj.encode(jj.mul(P_G, decryption_key(proof_generation_key(spending_key(seed)))))
