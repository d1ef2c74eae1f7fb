"""TEST INFRASTRUCTURE (oracle): redjubjub::batch_verify with the Diversifier generator and a Jubjub multiexp, restated with
Python integers on pyref.py and redjubjub.py.

  multiexp       sum_i s_i P_i as the naive sum of pyref.mul (edwards::Point<Unknown>)
  batch_verify   core/jubjub/src/redjubjub.rs:166-204 entry by entry, with the randomizers z_i supplied by the caller in place
                 of E::Fs::rand(rng): the early `return false` on a bad rbar / sbar, per-entry mul by z, the cofactor at the end

batch_verify returns the verdict codes of zk_redjubjub_batch_verify (include/zkb200.h)."""
from __future__ import annotations

from . import pyref as jj
from . import redjubjub as rj


def multiexp(points, scalars):
    """sum_i scalars[i] points[i]: the naive sum of pyref.mul."""
    acc = jj.IDENTITY
    for p, s in zip(points, scalars):
        acc = jj.add(acc, jj.mul(p, s))
    return acc


def batch_verify(vks, sigs, msgs, zs):
    """(verdict, first_bad).  A rejected encoding ends the loop early (the reference's `return false`; a vk that fails
    PublicKey::read cannot make a BatchEntry at all) with its code (BAD_VK / BAD_R / BAD_S) and index; otherwise OK or
    BAD_EQUATION with first_bad None."""
    acc = jj.IDENTITY
    for i, (vk, sig, msg, z) in enumerate(zip(vks, sigs, msgs, zs)):
        st, a = jj.read(vk)
        if st != jj.OK:
            return rj.BAD_VK, i
        st, r = jj.read(sig[:32])
        if st != jj.OK:
            return rj.BAD_R, i
        s = int.from_bytes(sig[32:], "little")
        if s >= rj.R_J:
            return rj.BAD_S, i
        c = rj.h_star(sig[:32], msg)
        s = (-(s * z)) % rj.R_J
        acc = jj.add(acc, jj.mul(r, z))
        acc = jj.add(acc, jj.mul(a, (c * z) % rj.R_J))
        acc = jj.add(acc, jj.mul(rj.P_G, s))
    return (rj.OK if jj.mul(acc, jj.COFACTOR) == jj.IDENTITY else rj.BAD_EQUATION), None
